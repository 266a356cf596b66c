"""Device image front-end on the H100 (SURVEY.md §8f.2): the CUDA resampler behind `vr_resample_u8` against PIL itself
(bit for bit), and the encode path with device-rendered slices against the same path with PIL-rendered slices
(bit-identical embeddings)."""
import numpy as np
import pytest
import torch
from PIL import Image

from tests.helpers import synth_pages

pytestmark = pytest.mark.gpu

# (W, H, out_w, out_h, cell_w, cell_h): both passes, horizontal only, vertical only, copy, grids, tiny and wide
CASES = [(640, 480, 448, 336, 448, 336), (1700, 2200, 350, 448, 350, 448), (100, 75, 448, 336, 448, 336),
         (517, 301, 518, 301, 518, 301), (301, 517, 301, 520, 301, 520), (448, 448, 448, 448, 448, 448),
         (900, 1200, 756, 1008, 378, 504), (2000, 700, 1344, 448, 448, 448), (33, 400, 14, 434, 14, 14),
         (5000, 60, 28, 28, 28, 28), (3, 2, 6, 8, 3, 4)]


def _pil(img, ow, oh):
    return np.asarray(Image.fromarray(img).resize((ow, oh), Image.Resampling.BICUBIC))


@pytest.mark.parametrize("rgbx", [False, True])
@pytest.mark.parametrize("W,H,ow,oh,cw,ch", CASES)
def test_resampler_equals_pillow(W, H, ow, oh, cw, ch, rgbx):
    from visrag_b200.frontend import DeviceFrontEnd

    fe = DeviceFrontEnd(torch.device("cuda:0"))
    rs = np.random.RandomState(W + 3 * H)
    n = 3
    pages = rs.randint(0, 256, (n, H, W, 3), dtype=np.uint8)
    pages[1, : H // 2] = 0       # hard edges: bicubic overshoot must clip like Pillow on both sides
    pages[1, H // 2:] = 255
    gx, gy = ow // cw, oh // ch
    cells = gx * gy
    # pages land in a shuffled order with a gap slice in between, like slices of different pages sharing a group
    first = np.asarray([cells + 1, 0, 2 * cells + 2], dtype=np.int32)
    out = torch.full((3 * cells + 3, ch, cw, 3), 7, dtype=torch.uint8, device="cuda:0")
    src = pages
    if rgbx:  # Pillow's native row layout: 4 bytes per pixel, the 4th is padding (garbage here on purpose)
        src = np.concatenate([pages, rs.randint(0, 256, (n, H, W, 1), dtype=np.uint8)], axis=3)
    fe.resize_into(torch.from_numpy(src).cuda(), ow, oh, out, torch.from_numpy(first).cuda(), cw, ch)
    got = out.cpu().numpy()
    for i in range(n):
        want = _pil(pages[i], ow, oh)
        for cy in range(gy):
            for cx in range(gx):
                assert np.array_equal(got[first[i] + cy * gx + cx], want[cy * ch:(cy + 1) * ch, cx * cw:(cx + 1) * cw]), (i, cy, cx)
    untouched = sorted(set(range(3 * cells + 3)) - {int(f) + c for f in first for c in range(cells)})
    assert all((got[u] == 7).all() for u in untouched)


def test_bad_arguments_are_rejected():
    from visrag_b200 import _lib as L

    z = torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    f = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    lib = L.lib()
    # width changes but no horizontal tables
    rc = lib.vr_resample_u8(z.data_ptr(), 3, 1, 2, 2, None, None, 0, None, None, 0, 0, 2, 2, 4, None, z.data_ptr(), f.data_ptr(), 2, 4, None)
    assert rc != 0 and b"horizontal" in lib.vr_last_error()
    # output not a whole grid of cells
    rc = lib.vr_resample_u8(z.data_ptr(), 3, 1, 2, 2, None, None, 0, None, None, 0, 0, 2, 2, 2, None, z.data_ptr(), f.data_ptr(), 2, 3, None)
    assert rc != 0 and b"grid" in lib.vr_last_error()
    # only RGB / RGBX sources
    rc = lib.vr_resample_u8(z.data_ptr(), 2, 1, 2, 2, None, None, 0, None, None, 0, 0, 2, 2, 2, None, z.data_ptr(), f.data_ptr(), 2, 2, None)
    assert rc != 0 and b"src_pixel_bytes" in lib.vr_last_error()


def test_encode_with_device_frontend_is_bit_identical():
    """Mixed-resolution pages (1-7 slices, shared geometry groups, a text-only item): embeddings from device-rendered
    slices equal the embeddings from PIL-rendered slices exactly, through the engine and through the B2 wrapper loop."""
    from visrag_b200 import inference as I
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.modeling import DRModelForInference, VisRAGRetB200
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 5)
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages([(448, 448), (700, 900), (1100, 500), (224, 224), (700, 900), (1344, 1000), (640, 320)], 4)
    texts = [""] * len(pages) + ["what is on the page"]
    images = pages + [None]
    eng = VisRAGEngine(cfg, sd, device_frontend=False)
    want = eng.encode(texts, images, tok)
    eng.device_frontend = True
    got = eng.encode(texts, images, tok)
    assert torch.equal(got, want)
    # same through the pipelined loop of the B2 wrapper
    lm = VisRAGRetB200(cfg, sd, "cuda:0")
    model = DRModelForInference(lm_q=lm, pooling="wmean", normalize=True)
    data = [{"id": f"p{i}", "text": "", "image": im} for i, im in enumerate(pages)]
    kw = {"tokenizer": tok, "max_inp_length": 2048}
    lm.engine.device_frontend = False
    ref = np.concatenate([arr for _, arr in I.encode_stream(I._batches(data, 3), model, kw)])
    lm.engine.device_frontend = True
    dev = np.concatenate([arr for _, arr in I.encode_stream(I._batches(data, 3), model, kw)])
    assert np.array_equal(ref, dev) and np.array_equal(ref, want[: len(pages)].cpu().numpy())
