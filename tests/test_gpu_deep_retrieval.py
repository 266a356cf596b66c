"""Deep top-k on the GPU (DESIGN §4, "Deep top-k"): vr_select_rows against vr_topk_rows bit for bit, and score_topk at
k above 16 (the scan's radix select, and the deep route of a sampled threshold on the range filter) against the fp32
scan called directly: vr_score_exact + vr_topk_rows. Every comparison is torch.equal on scores and ids."""
import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu


def _unit(rs, n, d):
    x = rs.randn(n, d).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _rows(name, scores, k, ids=None, masks=None, id_offset=0, chunks=0):
    """One call of vr_<name> (topk_rows or select_rows) into poisoned outputs: (scores, ids) [rows, k]."""
    rows, cols = scores.shape
    out_s = torch.full((rows, k), float("nan"), device="cuda")
    out_i = torch.full((rows, k), -7, dtype=torch.int64, device="cuda")
    lib, sp = L.lib(), L.stream_ptr()
    tail = (out_s.data_ptr(), out_i.data_ptr()) + ((masks.arg(),) if masks is not None else ()) + (sp,)
    form = ("_chunked" if chunks else "") + ("_masks" if masks is not None else "")
    fn = getattr(lib, f"vr_{name}{form}")
    if chunks:
        ws_s = torch.empty((rows, chunks, k), device="cuda")
        ws_i = torch.empty((rows, chunks, k), dtype=torch.int64, device="cuda")
        L.check(fn(scores.data_ptr(), rows, cols, k, id_offset, chunks, ws_s.data_ptr(), ws_i.data_ptr(), *tail))
    else:
        L.check(fn(scores.data_ptr(), L.ptr(ids), rows, cols, k, id_offset, *tail))
    return out_s, out_i


def _same(a, b, what):
    assert torch.equal(a[1], b[1]), (what, int((a[1] != b[1]).sum()))
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)), what  # the bits, -0 and +0 apart


SPECIAL = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40, 1.0, -1.0], np.float32)


def _adversarial(rs, rows, cols):
    """Rows of every kind: random, all equal, few distinct values (ties at every boundary), special values only, and a
    mix of special values and random scores."""
    out = np.empty((rows, cols), np.float32)
    for r in range(rows):
        kind = r % 5
        if kind == 0:
            out[r] = rs.randn(cols)
        elif kind == 1:
            out[r] = 0.25
        elif kind == 2:
            out[r] = rs.randint(0, 4, cols).astype(np.float32) / 4
        elif kind == 3:
            out[r] = SPECIAL[rs.randint(0, len(SPECIAL), cols)]
        else:
            out[r] = np.where(rs.rand(cols) < 0.3, SPECIAL[rs.randint(0, len(SPECIAL), cols)], rs.randn(cols))
    return torch.from_numpy(out).cuda()


@pytest.mark.parametrize("cols", [1, 7, 100, 513, 4097, 70000])
def test_select_rows_equals_topk_rows(cols):
    rs = np.random.RandomState(cols)
    sc = _adversarial(rs, 10, cols)
    ids = torch.from_numpy(rs.randint(-3, 1 << 40, (10, cols))).cuda()          # negative ids are skipped
    m = torch.from_numpy(rs.rand(3, cols) < 0.6).cuda()
    masks = R._MaskSet(R.pack_doc_mask(m), torch.from_numpy(rs.randint(0, 3, 10).astype(np.int32)).cuda())
    one = R._MaskSet(R.pack_doc_mask(m[0]).view(1, -1), None)
    for k in [1, 16, 17, 100, 1000, 4096]:
        for what, kw in [("plain", {}), ("ids", dict(ids=ids)), ("per-row masks", dict(masks=masks)),
                         ("one mask", dict(masks=one)), ("id_offset", dict(id_offset=1 << 33))]:
            _same(_rows("select_rows", sc, k, **kw), _rows("topk_rows", sc, k, **kw), (cols, k, what))


def test_select_rows_repeated_pairs_and_duplicate_ids():
    """A repeated (score, id) pair is emitted once, as vr_topk_rows does (the list path relies on it); one id with two
    scores is two entries; +0 and -0 of one id are one pair."""
    rs = np.random.RandomState(5)
    cols = 3000
    sc = torch.from_numpy(rs.randint(0, 50, (6, cols)).astype(np.float32) / 50).cuda()
    ids = torch.from_numpy(rs.randint(0, 400, (6, cols))).cuda()
    sc[1] = 0.0
    sc[1, ::2] = -0.0
    ids[2] = torch.arange(cols).cuda() // 2                                    # every id twice, mostly two scores
    sc[3] = sc[3].round()
    ids[3] = torch.arange(cols).cuda() % 700
    for k in [17, 200, 1000, 4096]:
        _same(_rows("select_rows", sc, k, ids=ids), _rows("topk_rows", sc, k, ids=ids), k)


@pytest.mark.parametrize("cols,chunks", [(1 << 20, 256), (300000, 73), (5000, 2)])
def test_select_rows_chunked(cols, chunks):
    rs = np.random.RandomState(chunks)
    sc = _adversarial(rs, 3, cols)
    sc[0] = torch.randn(cols, device="cuda")
    m = torch.from_numpy(rs.rand(3, cols) < 0.5).cuda()
    masks = R._MaskSet(R.pack_doc_mask(m), torch.arange(3, dtype=torch.int32, device="cuda"))
    for k in [17, 100, 1000, 4096]:
        for kw in [{}, dict(masks=masks)]:
            got = _rows("select_rows", sc, k, chunks=chunks, id_offset=11, **kw)
            _same(got, _rows("topk_rows", sc, k, chunks=chunks, id_offset=11, **kw), (cols, k, bool(kw)))
            if not kw:  # and the chunked form equals the one-block form
                _same(got, _rows("select_rows", sc, k, id_offset=11), (cols, k, "one block"))


def test_select_rows_refusals():
    sc = torch.zeros((2, 10), device="cuda")
    out = torch.empty((2, 5000), device="cuda")
    oi = torch.empty((2, 5000), dtype=torch.int64, device="cuda")
    lib = L.lib()
    assert lib.vr_select_rows(sc.data_ptr(), None, 2, 10, 4097, 0, out.data_ptr(), oi.data_ptr(), None) != 0
    assert lib.vr_select_rows(sc.data_ptr(), None, 2, 10, 0, 0, out.data_ptr(), oi.data_ptr(), None) != 0
    assert lib.vr_select_rows(sc.data_ptr(), None, 2, 10, 5, 0, out.data_ptr(), oi.data_ptr() + 4, None) != 0


# ---------------------------------------------------------------------------------------------------------- score_topk
def _scan(q, idx, k, masks=None, id_offset=0):
    """The fp32 scan called directly: vr_score_exact, then vr_topk_rows(_masks) (the k-pass selection)."""
    nq = q.shape[0]
    scratch = torch.empty((nq, idx.nd), device="cuda")
    L.check(L.lib().vr_score_exact(q.data_ptr(), nq, idx.emb.data_ptr(), idx.nd, q.shape[1], scratch.data_ptr(),
                                   L.stream_ptr()))
    return _rows("topk_rows", scratch, k, masks=masks, id_offset=id_offset)


def _corpus(kind, nq=600, nd=20000, d=64, seed=0):
    rs = np.random.RandomState(seed)
    D = _unit(rs, nd, d)
    if kind == "clustered":  # 200 clusters of near-copies, and every 7th page an exact duplicate of the one before
        c = _unit(rs, 200, d)
        D = c[rs.randint(0, 200, nd)] + 0.05 * rs.randn(nd, d).astype(np.float32) / np.sqrt(d)
        D[1::7] = D[0:-1:7][: len(D[1::7])]
        D /= np.linalg.norm(D, axis=1, keepdims=True)
        Q = c[rs.randint(0, 200, nq)] + 0.1 * rs.randn(nq, d).astype(np.float32) / np.sqrt(d)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    else:
        Q = _unit(rs, nq, d)
    return torch.from_numpy(Q.astype(np.float32)).cuda(), R.build_index(D)


def _expected_path(k):
    return "deep" if R.DEEP_K_MIN < k <= R.DEEP_K_MAX else "filter+rescore"


KS = [17, 64, 100, 128, 256, 1000, 4096]


@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_score_topk_equals_the_scan(kind):
    q, idx = _corpus(kind)
    for k in KS:
        stats = {}
        got = R.score_topk(q, idx, k, id_offset=5, stats=stats)
        _same(got, _scan(q, idx, k, id_offset=5), (kind, k))
        assert stats["path"] == _expected_path(k), (k, stats)
        if stats["path"] == "deep":
            assert stats["sample_stride"] == k // 8 and stats["candidates"] >= k * (q.shape[0] - stats["fallback"])
            assert stats["fallback"] < q.shape[0] // 4, stats


def test_score_topk_masks_and_lists():
    q, idx = _corpus("random", nq=400, seed=1)
    nq, nd = q.shape[0], idx.nd
    rs = np.random.RandomState(2)
    one = torch.from_numpy(rs.rand(nd) < 0.7).cuda()
    few = torch.zeros(nd, dtype=torch.bool, device="cuda")
    few[torch.from_numpy(rs.choice(nd, 50, replace=False)).cuda()] = True      # fewer eligible pages than k
    per = torch.from_numpy(rs.rand(5, nd) < 0.5).cuda()
    of = torch.from_numpy(rs.randint(0, 5, nq)).cuda()
    for k in [100, 1000]:
        for what, m, mo in [("1-D mask", one, None), ("fewer eligible than k", few, None), ("per-query masks", per, of)]:
            stats = {}
            got = R.score_topk(q, idx, k, doc_mask=m, mask_of=mo, stats=stats)
            ms = R._check_doc_mask(m, idx, nq, mo)
            _same(got, _scan(q, idx, k, masks=ms), (what, k))
            assert stats["path"] == _expected_path(k), (what, k, stats)
        # lists: each row equals the call with a doc_mask of exactly its list's docs
        lens = rs.randint(0, 6000, 3)
        offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).cuda()
        ids = torch.from_numpy(rs.randint(0, nd, int(lens.sum()))).cuda()         # repeats count once
        lof = torch.from_numpy(rs.randint(0, 3, nq)).cuda()
        got = R.score_topk(q, idx, k, doc_lists=(offsets, ids), list_of=lof)
        lm = torch.zeros((3, nd), dtype=torch.bool, device="cuda")
        for j in range(3):
            lm[j, ids[offsets[j]:offsets[j + 1]]] = True
        _same(got, _scan(q, idx, k, masks=R._check_doc_mask(lm, idx, nq, lof)), ("lists", k))


def test_k_beyond_the_index():
    q, idx = _corpus("random", nq=16000, nd=300, d=64, seed=3)
    for k in [400, 1000]:
        stats = {}
        got = R.score_topk(q, idx, k, stats=stats)
        _same(got, _scan(q, idx, k), k)
        assert stats["path"] == "deep" and stats["fallback"] == q.shape[0]
        assert bool((got[1][:, 300:] == -1).all())


def test_misleading_sample_falls_back():
    """Only the sampled pages score high for query 0: its threshold is the sample's 16th score, fewer than k pages reach
    it, and the row reruns through the scan while the others take the range answer."""
    q, idx = _corpus("random", nq=300, seed=4)
    k = 500
    stride = k // 8
    emb = idx.emb.clone()
    near = q[0] + 0.05 * torch.randn((40, q.shape[1]), device="cuda")
    emb[:40 * stride:stride] = near / near.norm(dim=1, keepdim=True)                # 40 sampled pages near query 0
    idx = R.build_index(emb)
    stats = {}
    got = R.score_topk(q, idx, k, stats=stats)
    _same(got, _scan(q, idx, k), "misleading sample")
    assert stats["path"] == "deep" and 1 <= stats["fallback"] < 30, stats


def test_batch_invariance():
    q, idx = _corpus("clustered", nq=500, seed=6)
    for k in [64, 1000]:
        batch = R.score_topk(q, idx, k)
        for r in [0, 17, 499]:
            alone = R.score_topk(q[r:r + 1], idx, k)
            _same((batch[0][r:r + 1], batch[1][r:r + 1]), alone, (k, r))


def test_downstream_callers():
    q, idx = _corpus("clustered", nq=500, seed=7)
    ref = _scan(q, idx, 128)
    got = R.score_mmr(q, idx, 10, lambda_mult=0.5, fetch_k=128)
    _same(got, R.mmr_select(idx, ref[0], ref[1], 10, 0.5), "mmr fetch_k=128")
    for k in [100, 1000]:
        _same(R.sharded_topk(q, idx, k, 3), _scan(q, idx, k, id_offset=3), ("sharded, world 1", k))
        s, i = _scan(q, idx, k)
        half = (torch.cat([s[:, ::2], s[:, 1::2]], 1), torch.cat([i[:, ::2], i[:, 1::2]], 1))
        _same(R.merge_topk(*half, k), (s, i), ("merge_topk", k))
