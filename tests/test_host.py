"""Host-side logic (geometry, placeholders, tokenisation, packing) against the reference's golden geometry and
against the oracle restatement. CPU only."""
import numpy as np
import pytest
from PIL import Image

from oracle import restated as O
from tests.helpers import GOLDEN, synth_pages
from visrag_b200 import host
from visrag_b200.config import VisRAGConfig
from visrag_b200.tokenizer_stub import StubTokenizer

CFG = VisRAGConfig.tiny()


def _check_plans(cases):
    for W, H, sw, sh, gx, gy, pw, ph, npatch in cases:
        plan = host.plan_slices(int(W), int(H), CFG)
        assert plan.source_size == (sw, sh), (W, H)
        if gx == 0:
            assert plan.grid is None and npatch == 0
        else:
            assert plan.grid == (gx, gy) and plan.cell_size == (pw, ph) and plan.n_slices == 1 + npatch, (W, H)


def test_plan_matches_reference_golden_geometry():
    _check_plans(np.load(f"{GOLDEN}/geometry_v1.npz")["cases"])


def test_plan_matches_reference_golden_geometry_of_tall_and_wide_pages():
    """geometry_v2: long screenshots, infographics, banners and thin strips (aspect ratios up to 1:20000, sides up to 40000),
    whose thumbnails and slices reach 60004 pixels in width and 4525 patches."""
    cases = np.load(f"{GOLDEN}/geometry_v2.npz")["cases"]
    assert len(cases) == 200 and cases[:, :2].max() == 40000
    _check_plans(cases)


def test_known_geometries():
    # SURVEY.md §8c: 564x3040 page -> thumbnail 196x1036, grid [1,8], eight 546x364 slices
    p = host.plan_slices(564, 3040, CFG)
    assert p.source_size == (196, 1036) and p.grid == (1, 8) and p.cell_size == (546, 364)
    for s in (224, 448):
        p = host.plan_slices(s, s, CFG)
        assert p.source_size == (448, 448) and p.grid is None


@pytest.mark.parametrize("size", [(224, 224), (700, 900), (760, 141), (1200, 500), (449, 449),
                                  # tall and wide pages: slices down to 1 and 3 patches on one side, up to 1000 on the other
                                  (1280, 40000), (600, 8000), (8000, 600), (3000, 100), (33964, 287), (30000, 30), (3000, 1)])
def test_render_is_pixel_exact_vs_oracle(size):
    img = synth_pages([size], 3)[0]
    src, patches, grid = O.slice_image(img, 9, 448, 14)
    want = [np.asarray(src)] + [np.asarray(p) for row in patches for p in row]
    got = host.render_slices(img, host.plan_slices(*img.size, CFG))
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == np.uint8 and g.shape == w.shape and np.array_equal(g, w)


def test_tokenisation_and_packing_match_oracle():
    tok = StubTokenizer(CFG.vocab)
    imgs = synth_pages([(224, 224), (700, 900)], 5) + [None]
    texts = ["", "caption text", "Represent this query for retrieving relevant documents: hello"]
    pb = host.prepare_batch(texts, imgs, tok, CFG, 2048)
    assert pb.n_items == 3 and pb.cu_seqlens[-1] == pb.token_src.shape[0] == pb.positions.shape[0]
    slice_rows = []
    for b, (t, im) in enumerate(zip(texts, imgs)):
        content, slices = O.prepare_context(t, im, tok, CFG.query_num)
        ids, bound = O.convert_to_tensors(tok, content, 2048)
        lo, hi = pb.cu_seqlens[b], pb.cu_seqlens[b + 1]
        assert hi - lo == len(ids)
        src = pb.token_src[lo:hi]
        assert np.array_equal(pb.positions[lo:hi], np.arange(len(ids)))
        is_img = np.zeros(len(ids), bool)
        for (s, e) in bound:
            is_img[s:e] = True
        assert np.array_equal(-(src[~is_img] + 1), ids[~is_img])
        assert (src[is_img] >= 0).all()
        for n, (s, e) in enumerate(bound):
            rows = src[s:e]
            assert np.array_equal(rows - rows[0], np.arange(64)) and rows[0] % 64 == 0
            slice_rows.append((rows[0] // 64, np.asarray(slices[n])))
    # every slice index maps to the right pixels inside its geometry group
    for idx, px in slice_rows:
        key = (px.shape[0], px.shape[1])
        j = idx - pb.group_row0[key]
        assert np.array_equal(pb.groups[key][j], px)
    assert pb.n_slices == len(slice_rows) == 1 + 5  # 224^2 page: 1 slice; 700x900: thumbnail + 2x2


def test_text_only_and_errors():
    tok = StubTokenizer(CFG.vocab)
    pb = host.prepare_batch(["a", "bcd"], [None, None], tok, CFG, 3)
    assert list(pb.seq_lens) == [2, 3] and pb.n_slices == 0 and not pb.groups
    with pytest.raises(ValueError):
        host.prepare_batch([""], [Image.new("RGB", (224, 224))], tok, CFG, 40)  # span cut by truncation
    with pytest.raises(NotImplementedError):
        host.prepare_batch([["chat"]], [None], tok, CFG)


def test_graph_plan_buckets_text_batches_and_leaves_pages_alone():
    """Host side of the CUDA-graph path (encoder._graph_plan): text-only batches are padded to 16-token buckets with ONE extra
    dummy sequence (token id 0, positions 0..pad-1) so that different queries share a captured graph; batches with pages keep
    their exact arrays; oversized batches are not graphed."""
    from types import SimpleNamespace

    import numpy as np

    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import GRAPH_MAX_LM_TOKENS, GRAPH_TEXT_BUCKET, VisRAGEngine
    from visrag_b200.host import prepare_batch
    from visrag_b200.synth import synth_pages
    from visrag_b200.tokenizer_stub import StubTokenizer

    cfg = VisRAGConfig.tiny()
    tok = StubTokenizer(cfg.vocab)
    eng = SimpleNamespace(cuda_graphs=True, cfg=cfg)
    for texts in (["a"], ["hello world this is", "x"], ["q" * 31], ["q" * 14, "r" * 15, "s" * 16]):
        pb = prepare_batch(texts, [None] * len(texts), tok, cfg, 2048)
        src, pos, cu, max_len, n_out = VisRAGEngine._graph_plan(eng, pb)
        T = int(pb.cu_seqlens[-1])
        assert n_out == len(texts) and len(cu) == len(texts) + 2
        assert len(src) == len(pos) == cu[-1] and cu[-1] % GRAPH_TEXT_BUCKET == 0 and cu[-1] > T      # at least one pad token
        assert np.array_equal(src[:T], pb.token_src) and np.array_equal(pos[:T], pb.positions) and np.array_equal(cu[:-1], pb.cu_seqlens)
        pad = cu[-1] - T
        assert (src[T:] == -1).all() and np.array_equal(pos[T:], np.arange(pad))                      # token id 0, its own positions
        assert max_len % GRAPH_TEXT_BUCKET == 0 and max_len >= max(int(pb.seq_lens.max()), pad)
    pages = synth_pages([(448, 448), (300, 500)], 3)
    pb = prepare_batch(["", ""], pages, tok, cfg, 2048)
    src, pos, cu, max_len, n_out = VisRAGEngine._graph_plan(eng, pb)
    assert src is pb.token_src and cu is pb.cu_seqlens and max_len == int(pb.seq_lens.max()) and n_out == 2
    big = prepare_batch(["w" * 600] * 8, [None] * 8, tok, cfg, 2048)                                # > GRAPH_MAX_LM_TOKENS tokens
    assert int(big.cu_seqlens[-1]) > GRAPH_MAX_LM_TOKENS and VisRAGEngine._graph_plan(eng, big) is None
    assert VisRAGEngine._graph_plan(SimpleNamespace(cuda_graphs=False, cfg=cfg), pb) is None
