"""The vision path on tall and wide pages: long screenshots, infographics, banners and thin strips, whose slices are far
from the square 448 x 448 of an ordinary page (geometry pins: tests/golden/geometry_v2.npz).

  page (W x H)    thumbnail (patches)      grid cell (patches)
  1280 x 40000    84 x 2506   (6 x 179)    238 x 840   (17 x 60)
  600 x 8000      126 x 1638  (9 x 117)    364 x 546   (26 x 39)
  8000 x 600      1624 x 126  (116 x 9)    546 x 364   (39 x 26)
  3000 x 100      2436 x 84   (174 x 6)    1414 x 140  (101 x 10)
  33964 x 287     4858 x 42   (347 x 3)    1624 x 126  (116 x 9)
  30000 x 30      14000 x 14  (1000 x 1)   5670 x 28   (405 x 2)
  3000 x 1        23996 x 14  (1714 x 1)   -

Checked here: im2col bit for bit at every kernel the slice width selects (including strips wider than shared memory, which
are converted in chunks of patch columns), ViT and resampler attention at the slicer's sequence lengths against float64
bounds, the tiny vision tower and resampler against the oracle on these slices, and whole encodes of such pages."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF
from tests.helpers import cosine_rows, synth_pages

pytestmark = pytest.mark.gpu

DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "f16"]
COS_MIN = 0.9999

# the pages of the module docstring plus two ordinary ones (the end-to-end batch)
TALL_WIDE = [(1280, 10000), (1280, 40000), (600, 8000), (8000, 600), (3000, 100), (33964, 287), (30000, 30)]
ORDINARY = [(700, 900), (448, 448)]


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------- im2col


def _pixels(S, h, w, seed, offset=0):
    """uint8 [S,h,w,3] on the device whose first byte lies `offset` bytes past a 256-byte boundary; the first 256 bytes
    hold every byte value."""
    n = S * h * w * 3
    buf = torch.randint(0, 256, (n + offset,), dtype=torch.uint8, device=DEV, generator=_gen(seed))
    px = buf[offset:].view(S, h, w, 3)
    px.view(-1)[:256] = torch.arange(256, dtype=torch.uint8, device=DEV)
    assert px.is_contiguous() and px.data_ptr() % 16 == offset % 16
    return px


def _check_im2col(px, patch, ldo, dtype):
    """vr_im2col_norm_ex into a buffer pre-filled with 0xFF bytes (NaN in both types) and followed by guard rows, against
    CPU F.unfold of (u/255 - 0.5)/0.5 in fp32 rounded once to `dtype`; the pad columns must be +0 bit for bit."""
    from visrag_b200 import _lib as L
    from visrag_b200 import ops

    S, h, w, _ = px.shape
    per = (h // patch) * (w // patch)
    K = 3 * patch * patch
    guard = 3
    buf = torch.full((S * per + guard, ldo), -1, dtype=torch.int16, device=DEV).view(dtype)
    vr_dtype = L.VR_F16 if dtype == torch.float16 else L.VR_BF16
    ops._launch("im2col", 0.0, L.lib().vr_im2col_norm_ex, px.data_ptr(), S, h, w, patch, buf.data_ptr(), ldo, vr_dtype,
                L.stream_ptr())
    got = buf.cpu()
    assert (got[S * per:].view(torch.int16) == -1).all(), "im2col wrote past its output"
    got = got[:S * per]
    step = max(1, 4_000_000 // (h * w))
    for s0 in range(0, S, step):
        x = ((px[s0:s0 + step].cpu().float() / 255 - 0.5) / 0.5).permute(0, 3, 1, 2)
        want = F.unfold(x, kernel_size=patch, stride=patch).transpose(1, 2).reshape(-1, K).to(dtype)
        g = got[s0 * per:(s0 + step) * per]
        same = g[:, :K].view(torch.int16) == want.view(torch.int16)
        if not same.all():
            r, c = (~same).nonzero()[0].tolist()
            raise AssertionError(f"{tuple(px.shape)} patch={patch} ldo={ldo} {dtype}: row {s0 * per + r} column {c}: got "
                                 f"{float(g[r, c])} want {float(want[r, c])} ({int((~same).sum())} values differ)")
        assert (g[:, K:].view(torch.int16) == 0).all(), "pad columns are not +0"


# (S, h, w): the kernel that patch 14 with ldo 640 runs at this width (gw = w / 14 patches)
IM2COL_CASES = [
    (3, 448, 448),      # gw 32: 16-byte bulk copies, double buffered
    (1, 2506, 84),      # gw 6: 4-byte rows (the 1280 x 40000 thumbnail)
    (3, 28, 98),        # gw 7: 2-byte rows
    (2, 42, 1232),      # gw 88: generic (gw % 8 == 0 past the bulk kernel's shared memory)
    (2, 126, 1624),     # gw 116: generic (the 8000 x 600 thumbnail)
    (1, 84, 2436),      # gw 174: generic (the 3000 x 100 thumbnail)
    (1, 42, 4858),      # gw 347: chunked (the 33964 x 287 thumbnail)
    (2, 14, 14000),     # gw 1000: chunked (the 30000 x 30 thumbnail)
    (2, 28, 22848),     # gw 1632: chunked
    (1, 14, 23996),     # gw 1714: chunked (the 3000 x 1 page, a single slice)
]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("ldo", [640, 592])
@pytest.mark.parametrize("S,h,w", IM2COL_CASES, ids=[f"gw{c[2] // 14}" for c in IM2COL_CASES])
def test_im2col_is_bit_exact_at_every_slice_width(S, h, w, ldo, dtype):
    _check_im2col(_pixels(S, h, w, seed=h + w + ldo), 14, ldo, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("offset", [4, 2, 1])
@pytest.mark.parametrize("S,h,w", [(3, 448, 448), (1, 2506, 84), (3, 28, 98), (2, 42, 1232), (1, 42, 4858), (2, 28, 22848)],
                         ids=["gw32", "gw6", "gw7", "gw88", "gw347", "gw1632"])
def test_im2col_is_bit_exact_at_unaligned_pixels(S, h, w, offset, dtype):
    """A slice view inside a batch starts 588 * gh * gw bytes after the previous one: 4-byte but not always 16-byte
    aligned. Offsets 2 and 1 are pointers the C ABI accepts too; they take the generic kernel's narrower loads."""
    _check_im2col(_pixels(S, h, w, seed=w + offset, offset=offset), 14, 640, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("S,h,w,offset", [(300, 448, 448, 0), (300, 448, 448, 4), (300, 448, 448, 2), (200, 42, 4858, 0)],
                         ids=["bulk", "rows4", "generic", "chunked"])
def test_im2col_is_bit_exact_with_many_strips_per_cta(S, h, w, offset, dtype):
    """Far more strips (chunks) than CTAs: 300 slices of 448 x 448 are 9600 strips, so every CTA of the bulk kernel runs
    dozens of strips through both of its buffers and mbarrier phases; 200 slices 4858 wide are 1200 chunks."""
    _check_im2col(_pixels(S, h, w, seed=S + offset, offset=offset), 14, 640, dtype)


def test_im2col_other_patch_sizes_past_the_strip_buffer():
    """Patch 16 and patch 85 (the largest the offset table encodes) on strips wider than shared memory, and an ldo whose
    offset table leaves no room for a single patch (refused)."""
    from visrag_b200 import ops

    _check_im2col(_pixels(2, 32, 16 * 300, seed=16), 16, 768, torch.bfloat16)     # 16 * 4800 * 3 B per strip
    _check_im2col(_pixels(1, 85, 85 * 12, seed=85), 85, 21680, torch.float16)     # 85 * 1020 * 3 B per strip
    with pytest.raises(RuntimeError, match="leaves no shared memory"):
        ops.im2col_norm(_pixels(1, 14, 14 * 400, seed=1), 14, 102400)


# ---------------------------------------------------------------------------------------------------------- attention


@pytest.fixture(params=[0, 1], ids=["auto", "single_tile"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


def _attend_checked(name, q, k, v, dtype, *, cu_k, cu_q, max_q, **kw):
    from visrag_b200 import ops

    rows = int(cu_q[-1]) if cu_q is not None else (cu_k.numel() - 1) * max_q
    out = torch.full((rows, kw["heads"] * kw["head_dim"]), float("nan"), dtype=dtype, device=DEV)
    max_k = int((cu_k[1:] - cu_k[:-1]).max())
    ops.attention(q, k, v, batch=cu_k.numel() - 1, cu_k=cu_k, max_k=max_k, cu_q=cu_q, max_q=max_q, out=out, **kw)
    ref_fn = KF.attention_ref_f16 if dtype == torch.float16 else KB.attention_ref
    ref, e = ref_fn(q, k, v, cu_k=cu_k, cu_q=cu_q, max_q=max_q, **{n: kw[n] for n in (
        "q_col0", "k_col0", "v_col0", "head_stride", "head_dim", "heads", "causal", "scale")})
    KF.check(name, out, ref, e)


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_vit_attention_at_the_slicers_lengths(attn_variant, dtype):
    """16 heads of 72 at stride 80, non-causal, at N = 1044 (8000 x 600 thumbnail), 1053 (600 x 8000), 1074 (1280 x 40000)
    and 1710 (14 x 40000): alone, and mixed with 1024-token slices in one launch."""
    nh, hd, hs = 16, 72, 80
    for lens in ([1044], [1053], [1074], [1710], [1024, 1044], [1710, 1024], [1024, 1053, 1074, 1710, 1024]):
        T = sum(lens)
        qkv = torch.zeros(T, 3, nh, hs, device=DEV)
        qkv[..., :hd] = torch.randn(T, 3, nh, hd, device=DEV, generator=_gen(T))
        qkv = qkv.reshape(T, 3 * nh * hs).to(dtype)
        cu = _cu(lens)
        _attend_checked(f"vit lens={lens} {dtype}", qkv, qkv, qkv, dtype, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs,
                        head_stride=hs, head_dim=hd, heads=nh, cu_k=cu, cu_q=cu, max_q=max(lens), causal=False,
                        scale=hd ** -0.5)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_resampler_attention_at_the_slicers_lengths(attn_variant, dtype):
    """64 learned queries, 18 heads of 128, over 1074 and 1710 keys per slice."""
    E = 18 * 128
    for N in (1074, 1710):
        S = 2
        q = torch.zeros(128, E, device=DEV)
        q[:64] = torch.randn(64, E, device=DEV, generator=_gen(N))
        k = torch.randn(S * N, E, device=DEV, generator=_gen(N + 1)).to(dtype)
        v = torch.randn(S * N, E, device=DEV, generator=_gen(N + 2)).to(dtype)
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=DEV)
        _attend_checked(f"resampler N={N} {dtype}", q.to(dtype), k, v, dtype, q_col0=0, k_col0=0, v_col0=0, head_stride=128,
                        head_dim=128, heads=18, cu_k=cu, cu_q=None, max_q=64, causal=False, scale=128 ** -0.5)


# ------------------------------------------------------------------------------------------------- towers and end to end


@pytest.fixture(scope="module")
def tiny():
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    return cfg, random_state_dict(cfg, 4242)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_vision_tower_and_resampler_on_tall_and_wide_slices(tiny, dtype):
    """Thumbnail and first grid cell of each tall or wide page: ViT tokens after the final LayerNorm and the resampler's
    output against the oracle's fp32 towers on the same pixels (skinny grids for the position-embedding resampling and
    the resampler's 2-D sincos table: 179 x 6, 1 x 1000, 3 x 347, ...). Tolerance as for ordinary slices: 3e-2 of the
    largest reference value."""
    from PIL import Image

    from oracle import restated as O
    from visrag_b200 import host
    from visrag_b200.encoder import VisRAGEngine

    cfg, sd = tiny
    eng = VisRAGEngine(cfg, sd, dtype=dtype)

    def close(got, want, tol):
        want = torch.as_tensor(want).float()
        err = (got.float().cpu() - want).abs().max().item()
        return err <= tol * max(want.abs().max().item(), 1.0) and bool(torch.isfinite(got.float()).all())

    grids = set()
    for i, size in enumerate([(1280, 40000), (600, 8000), (8000, 600), (3000, 100), (33964, 287), (30000, 30)]):
        img = synth_pages([size], 70 + i)[0]
        for s in host.render_slices(img, host.plan_slices(*img.size, cfg))[:2]:
            gh, gw = s.shape[0] // 14, s.shape[1] // 14
            grids.add((gh, gw))
            tok = eng.vit_tokens(torch.from_numpy(s)[None].cuda())
            want = O.vit_forward(sd, cfg, O.pixel_values(Image.fromarray(s)))
            assert close(tok, want, 3e-2), (size, s.shape)
            out = torch.empty(cfg.query_num, cfg.hidden, device="cuda")
            eng.resample(tok, 1, gh, gw, out)
            assert close(out, O.resampler_forward(sd, cfg, want, gh, gw), 3e-2), (size, s.shape)
    assert {(179, 6), (1, 1000), (3, 347), (9, 116), (6, 174), (2, 405)} <= grids


@pytest.fixture(scope="module")
def batch(tiny):
    from oracle import restated as O
    from visrag_b200.tokenizer_stub import StubTokenizer

    cfg, sd = tiny
    tok = StubTokenizer(cfg.vocab)
    pages = synth_pages(TALL_WIDE + ORDINARY, 808)
    return pages, tok, O.encode(sd, cfg, tok, [""] * len(pages), pages)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_tall_and_wide_pages_end_to_end(tiny, batch, dtype):
    """One batch of the tall and wide pages (two of them wider than the device front-end takes, so PIL renders their
    slices) and two ordinary pages: every embedding within cos 0.9999 of the oracle, the same bits with the slices
    rendered by PIL on the host, and the same bits for each page encoded alone."""
    from visrag_b200 import host
    from visrag_b200.encoder import VisRAGEngine

    cfg, sd = tiny
    pages, tok, want = batch
    assert any(p.size[0] > host.MAX_DEVICE_PAGE_WIDTH for p in pages)
    assert any(p.size[0] <= host.MAX_DEVICE_PAGE_WIDTH and p.size[1] >= 10000 for p in pages)
    eng = VisRAGEngine(cfg, sd, dtype=dtype)
    got = eng.encode([""] * len(pages), pages, tok)
    c = cosine_rows(got.cpu().numpy(), want)
    print(f"{dtype}: cos >= {c.min():.7f}", flush=True)
    assert c.min() >= COS_MIN, c
    pil = VisRAGEngine(cfg, sd, dtype=dtype, device_frontend=False)
    assert torch.equal(pil.encode([""] * len(pages), pages, tok), got)
    for i, p in enumerate(pages):
        assert torch.equal(eng.encode([""], [p], tok)[0], got[i]), p.size
