"""Hybrid retrieval without a GPU: numpy restatements of the weighted-sum and reciprocal-rank fusions over the full score
matrix, the candidate-set argument (the exact fused top-k lies in the dense top-k plus the query's hits) on random and
adversarial cases, the host-side refusal of bad hit lists, and the C entry points' ctypes signatures and refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "visrag_b200.h")


def fused_sum(S, V, w):
    """fl(S + fl(w V)) elementwise, the two fp32 roundings of the definition."""
    return (S.astype(np.float32) + np.float32(w) * V.astype(np.float32)).astype(np.float32)


def order(s, elig=None):
    """Columns of s in (score desc, id asc) order, NaN and ineligible columns left out."""
    ok = ~np.isnan(s) if elig is None else (~np.isnan(s) & elig)
    cols = np.nonzero(ok)[0]
    return cols[np.lexsort((cols, -s[cols].astype(np.float64)))]


def topk(s, k, elig=None):
    o = order(s, elig)[:k]
    return s[o], o


def rrf_term(c, rank):
    return np.float32(1.0) / np.float32(c + rank)


def rrf_full(S_row, hits_row, k, window, c, elig=None):
    """Reciprocal rank fusion of one query over the full score row: dense ranks in the exact top-`window`, external
    ranks in the hits by (value desc, id asc); only pages of the union are ranked."""
    dense = order(S_row, elig)[:window]
    ids = np.array(sorted(hits_row), dtype=np.int64)
    vals = np.array([hits_row[i] for i in ids], dtype=np.float32)
    ext = ids[np.lexsort((ids, -vals.astype(np.float64)))] if len(ids) else ids
    score = {}
    for r, p in enumerate(dense):
        score[int(p)] = rrf_term(c, r + 1)
    for r, p in enumerate(ext):
        score[int(p)] = np.float32(score.get(int(p), np.float32(0)) + rrf_term(c, r + 1))
    pages = np.array(sorted(score), dtype=np.int64)
    s = np.array([score[p] for p in pages], dtype=np.float32)
    o = np.lexsort((pages, -s.astype(np.float64)))[:k]
    return s[o], pages[o]


def candidates_sum(S_row, hits_row, w, k, elig=None):
    """The library's route: dense top-k, minus the hit pages, plus every hit with its fused score, then the top-k."""
    _, dense = topk(S_row, k, elig)
    cand = {int(p): S_row[p] for p in dense if int(p) not in hits_row}
    for p, v in hits_row.items():
        cand[p] = fused_sum(np.array([S_row[p]]), np.array([v]), w)[0]
    pages = np.array(sorted(cand), dtype=np.int64)
    s = np.array([cand[p] for p in pages], dtype=np.float32)
    o = np.lexsort((pages, -s.astype(np.float64)))[:k]
    return s[o], pages[o]


def full_sum(S_row, hits_row, w, k, elig=None):
    V = np.zeros_like(S_row)
    for p, v in hits_row.items():
        V[p] = v
    return topk(fused_sum(S_row, V, w), k, elig)


def overfetch_join(S_row, hits_row, w, k, fetch):
    """The approximate recipe: search(fetch), join with the hits found there, re-sort."""
    _, dense = topk(S_row, fetch)
    cand = {int(p): fused_sum(np.array([S_row[p]]), np.array([hits_row.get(int(p), 0.0)]), w)[0] for p in dense}
    pages = np.array(sorted(cand), dtype=np.int64)
    s = np.array([cand[p] for p in pages], dtype=np.float32)
    o = np.lexsort((pages, -s.astype(np.float64)))[:k]
    return s[o], pages[o]


def _random_hits(rs, nd, n):
    ids = rs.choice(nd, size=n, replace=False)
    return {int(p): float(v) for p, v in zip(ids, rs.rand(n).astype(np.float32))}


@pytest.mark.parametrize("seed", range(20))
def test_candidate_set_holds_the_exact_fused_topk_random(seed):
    rs = np.random.RandomState(seed)
    nd, k = int(rs.randint(20, 400)), int(rs.randint(1, 30))
    S = rs.randn(nd).astype(np.float32)
    if seed % 3 == 0:
        S = np.round(S * 4) / 4  # many ties
    hits = _random_hits(rs, nd, int(rs.randint(0, min(nd, 60))))
    w = float(rs.choice([0.0, 0.1, 1.0, 3.0]))
    elig = rs.rand(nd) < 0.7 if seed % 2 else None
    hits_e = {p: v for p, v in hits.items() if elig is None or elig[p]}
    a, b = candidates_sum(S, hits_e, w, k, elig), full_sum(S, hits_e, w, k, elig)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.int32), b[0].view(np.int32))


def test_adversarial_cases():
    nd, k = 50, 5
    S = -np.arange(nd, dtype=np.float32) / 10  # page i ranks i-th by dense score
    # a listed page far below the dense top-k lifted into it
    hits = {45: 10.0}
    s, p = candidates_sum(S, hits, 1.0, k)
    assert p[0] == 45 and np.array_equal(p, full_sum(S, hits, 1.0, k)[1])
    # a page in both sets: appears once, with its fused score
    hits = {1: 0.5, 45: 10.0}
    s, p = candidates_sum(S, hits, 1.0, k)
    assert list(p) == [45, 1, 0, 2, 3] and s[1] == np.float32(np.float32(-0.1) + np.float32(0.5))
    # ties in fused scores are broken by id
    T = np.zeros(nd, dtype=np.float32)
    hits = {30: 1.0, 7: 1.0, 12: 1.0}
    s, p = candidates_sum(T, hits, 1.0, k)
    assert list(p) == [7, 12, 30, 0, 1] and np.array_equal(p, full_sum(T, hits, 1.0, k)[1])
    # empty lists and w = 0 are the dense top-k, bit for bit
    for hits, w in (({}, 1.0), ({3: 2.0, 40: 9.0}, 0.0)):
        s, p = candidates_sum(S, hits, w, k)
        d = topk(S, k)
        assert np.array_equal(p, d[1]) and np.array_equal(s.view(np.int32), d[0].view(np.int32))
    # every hit outside the scope: the scoped dense top-k
    elig = np.arange(nd) < 20
    hits_e = {p: v for p, v in {25: 5.0, 30: 5.0}.items() if elig[p]}
    assert np.array_equal(candidates_sum(S, hits_e, 1.0, k, elig)[1], topk(S, k, elig)[1])


def test_overfetch_and_join_is_not_exact():
    """The recipe the feature replaces: a page outside search(4k) that its external score lifts into the top-k is lost."""
    nd, k = 200, 5
    S = -np.arange(nd, dtype=np.float32) / 100
    hits = {150: 2.0}
    exact = full_sum(S, hits, 1.0, k)[1]
    assert exact[0] == 150
    assert 150 not in overfetch_join(S, hits, 1.0, k, 4 * k)[1]
    assert np.array_equal(candidates_sum(S, hits, 1.0, k)[1], exact)


@pytest.mark.parametrize("seed", range(10))
def test_rrf_model(seed):
    """RRF from the full row equals the union route of the library; ranks start at 1 and missing ranks add 0."""
    rs = np.random.RandomState(100 + seed)
    nd, k, window, c = 300, 10, int(rs.choice([10, 30, 100])), 60
    S = rs.randn(nd).astype(np.float32)
    hits = _random_hits(rs, nd, int(rs.randint(0, 40)))
    s, p = rrf_full(S, hits, k, window, c)
    dense = order(S)[:window]
    for sc, pg in zip(s, p):
        a = rrf_term(c, int(np.nonzero(dense == pg)[0][0]) + 1) if pg in dense else np.float32(0)
        ids = np.array(sorted(hits), dtype=np.int64)
        vals = np.array([hits[i] for i in ids], dtype=np.float32)
        ext = list(ids[np.lexsort((ids, -vals.astype(np.float64)))]) if len(ids) else []
        b = rrf_term(c, ext.index(pg) + 1) if pg in ext else np.float32(0)
        assert sc == np.float32(a + b)
    assert s[0] >= rrf_term(c, 1)


def test_document_candidates_hold_the_exact_fused_documents():
    """A document's fused score is the max of its pages' fused scores: the dense top-k documents plus the documents of
    the hits hold the exact top-k, and scoring only the listed pages of a listed document is not exact."""
    rs = np.random.RandomState(7)
    for trial in range(30):
        nd, k, G = 120, 4, 30
        groups = rs.randint(0, G, nd)
        S = rs.randn(nd).astype(np.float32)
        hits = _random_hits(rs, nd, int(rs.randint(0, 15)))
        V = np.zeros(nd, np.float32)
        for p, v in hits.items():
            V[p] = v
        F = fused_sum(S, V, 0.5)

        def doc_top(x):
            best = {}
            for p in order(x):
                best.setdefault(int(groups[p]), (x[p], int(p)))
            return sorted(best.items(), key=lambda t: (-float(t[1][0]), t[1][1]))[:k]

        exact = doc_top(F)
        dense_docs = {g for g, _ in doc_top(S)}
        cands = dense_docs | {int(groups[p]) for p in hits}
        Fc = np.where(np.isin(groups, list(cands)), F, np.nan).astype(np.float32)
        assert doc_top(Fc) == exact, trial
    # a listed document whose best page is not a hit
    groups = np.array([0, 0, 1])
    S = np.array([0.9, 0.1, 0.5], np.float32)
    F = fused_sum(S, np.array([0, 0.2, 0], np.float32), 1.0)
    assert F[0] > F[1]  # the document's fused score comes from its unlisted page 0, not from the hit (page 1)


def _cpu_hits(offsets, ids, values):
    return torch.tensor(offsets), torch.tensor(ids), torch.tensor(values, dtype=torch.float32)


def test_hits_are_refused_on_the_host():
    cpu = torch.device("cpu")
    good = ([0, 2, 3], [4, 1, 4], [0.5, 1.0, 0.0])
    h = R._check_hits(_cpu_hits(*good), 2, 10, cpu)
    assert h.width == 2 and h.offsets.tolist() == [0, 2, 3] and h.ids[:h.n].tolist() == [1, 4, 4]
    h = R._check_hits(_cpu_hits(*good), 2, 10, cpu, rank_order=True)
    assert h.ids[:h.n].tolist() == [1, 4, 4] and h.values[:h.n].tolist() == [1.0, 0.5, 0.0]
    bad = {
        "more than once": ([0, 3], [2, 5, 2], [1.0, 1.0, 0.5]),
        ">= 0": ([0, 2], [2, 5], [1.0, -0.5]),
        "finite": ([0, 2], [2, 5], [float("nan"), 1.0]),
        "finite ": ([0, 2], [2, 5], [float("inf"), 1.0]),
        "must lie in": ([0, 2], [2, 10], [1.0, 1.0]),
        "must lie in ": ([0, 2], [-1, 3], [1.0, 1.0]),
        "start at 0": ([1, 2], [2, 5], [1.0, 1.0]),
        "non-decreasing": ([0, 3, 2], [2, 5], [1.0, 1.0]),
        "end at": ([0, 1], [2, 5], [1.0, 1.0]),
    }
    for msg, hits in bad.items():
        with pytest.raises(ValueError, match=msg.strip()):
            R._check_hits(_cpu_hits(*hits), len(hits[0]) - 1, 10, cpu)
    with pytest.raises(ValueError, match="shape"):
        R._check_hits(_cpu_hits([0, 1], [2], [1.0]), 2, 10, cpu)
    with pytest.raises(ValueError, match="float32"):
        R._check_hits((torch.tensor([0, 1]), torch.tensor([2]), torch.tensor([1.0], dtype=torch.float64)), 1, 10, cpu)
    with pytest.raises(ValueError, match="triple"):
        R._check_hits((torch.tensor([0, 1]), torch.tensor([2])), 1, 10, cpu)


def test_negative_zero_is_a_zero_score():
    """-0.0 passes as a zero value and becomes +0.0, so the (row, value desc, id asc) order keeps every hit in its row."""
    cpu = torch.device("cpu")
    hits = _cpu_hits([0, 2, 4], [1, 2, 7, 8], [-0.0, 0.5, 0.3, 0.2])
    h = R._check_hits(hits, 2, 10, cpu, rank_order=True)
    assert h.offsets.tolist() == [0, 2, 4] and h.ids[:h.n].tolist() == [2, 1, 7, 8]
    assert h.values[:h.n].view(torch.int32).tolist()[1] == 0  # +0.0
    h = R._check_hits(_cpu_hits([0, 3, 3], [5, 1, 2], [-0.0, -0.0, 0.0]), 2, 10, cpu, rank_order=True)
    assert h.ids[:h.n].tolist() == [1, 2, 5]  # equal values: by id


def test_scope_drops_hits_on_the_host():
    cpu = torch.device("cpu")
    masks = R._MaskSet(R.pack_doc_mask(torch.tensor([[1, 1, 0, 1, 0, 1, 1, 1, 1, 1], [0, 0, 1, 0, 1, 0, 0, 0, 0, 0]],
                                                    dtype=torch.bool)), torch.tensor([0, 1], dtype=torch.int32))
    hits = _cpu_hits([0, 2, 5], [3, 2, 0, 4, 2], [1.0, 2.0, 0.5, 0.5, 3.0])
    h = R._check_hits(hits, 2, 10, cpu, masks=masks)
    assert h.offsets.tolist() == [0, 1, 3] and h.ids[:h.n].tolist() == [3, 2, 4]
    ls = R._ListSet(torch.tensor([0, 2, 4]), torch.tensor([3, 9, 4, 0], dtype=torch.int32),
                    torch.tensor([1, 0], dtype=torch.int32), 2, True)
    h = R._check_hits(hits, 2, 10, cpu, ls=ls)  # row 0 searches {4, 0}, row 1 {3, 9}: every hit is outside
    assert h.offsets.tolist() == [0, 0, 0] and h.width == 0
    ls = R._ListSet(torch.tensor([0, 3]), torch.tensor([0, 2, 4], dtype=torch.int32), None, 3, False)
    h = R._check_hits(hits, 2, 10, cpu, ls=ls)
    assert h.offsets.tolist() == [0, 1, 4] and h.ids[:h.n].tolist() == [2, 0, 2, 4]


def test_arguments_are_refused_before_any_work():
    with pytest.raises(ValueError, match="weighted sum only"):
        R.score_topk_groups_hybrid(None, None, 10, None, None, fusion="rrf")
    with pytest.raises(ValueError, match="fusion must be"):
        R.score_topk_hybrid(None, None, 10, None, fusion="max")
    for w in (-1.0, float("nan"), float("inf"), 1e39, True):
        with pytest.raises(ValueError, match="weight"):
            R.score_topk_hybrid(None, None, 10, None, weight=w)
    with pytest.raises(ValueError, match="window"):
        R.score_topk_hybrid(None, None, 10, None, fusion="rrf", window=5000)
    with pytest.raises(ValueError, match="window"):
        R.score_topk_hybrid(None, None, 10, None, window=20)
    with pytest.raises(ValueError, match="k="):
        R.score_topk_hybrid(None, None, 0, None)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def test_ctypes_signatures_match_the_header(lib):
    text = open(HEADER).read()
    i64, i32, vp, f32 = C.c_int64, C.c_int32, C.c_void_p, C.c_float
    assert "vr_fuse_rows" in G.exported_symbols() and "vr_group_pages_fused" in G.exported_symbols()
    assert lib.vr_fuse_rows.argtypes == [vp, vp, i32, i32, vp, vp, vp, vp, i64, i32, f32, i32, i64, vp, vp, vp, vp]
    assert lib.vr_group_pages_fused.argtypes[10] is C.POINTER(L.DocMasks) and lib.vr_group_pages_fused.argtypes[14] is f32
    for name in ("vr_fuse_rows", "vr_group_pages_fused"):
        decl = re.search(rf"int {name}\((.*?)\);", text, re.S).group(1)
        assert len(decl.split(",")) == len(getattr(lib, name).argtypes), name
    assert "#define VR_FUSE_SUM 0" in text and "#define VR_FUSE_RRF 1" in text
    assert (L.VR_FUSE_SUM, L.VR_FUSE_RRF) == (0, 1)


_FAKE = 0x7F0000000000


def _fuse(lib, **kw):
    a = dict(dense_scores=_FAKE, dense_ids=_FAKE + 0x1000, rows=4, kd=10, hit_offsets=_FAKE + 0x2000, hit_ids=_FAKE + 0x3000,
             hit_values=_FAKE + 0x4000, hit_dense=_FAKE + 0x5000, hit_pitch=8, mode=0, weight=1.0, rrf_c=60, width=18,
             out_scores=_FAKE + 0x6000, out_ids=_FAKE + 0x7000, status=_FAKE + 0x8000)
    a.update(kw)
    rc = lib.vr_fuse_rows(*a.values(), None)
    return rc, lib.vr_last_error().decode()


def _grouped(lib, **kw):
    a = dict(q=_FAKE, nq=2, d=_FAKE + 0x1000, nd=100, dim=64, groups=_FAKE + 0x2000, kg=5, offsets=_FAKE + 0x3000,
             pages=_FAKE + 0x4000, G=20, masks=None, hit_offsets=_FAKE + 0x5000, hit_ids=_FAKE + 0x6000,
             hit_values=_FAKE + 0x7000, weight=0.5, piece=8, pieces=1, id_offset=0, out_scores=_FAKE + 0x8000,
             out_pages=_FAKE + 0x9000)
    a.update(kw)
    rc = lib.vr_group_pages_fused(*a.values(), None)
    return rc, lib.vr_last_error().decode()


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
def test_entry_points_refuse_bad_operands(lib):
    assert _fuse(lib)[0] not in (0, 2)          # valid arguments get past validation (no device: the launch fails)
    assert _fuse(lib, mode=1, hit_values=None, hit_dense=None)[0] not in (0, 2)
    for kw, word in ((dict(dense_ids=_FAKE + 0x1004), "dense_ids"), (dict(hit_offsets=None), "hit_offsets"),
                     (dict(hit_ids=_FAKE + 0x3002), "hit_ids"), (dict(out_ids=_FAKE + 0x7004), "out_ids"),
                     (dict(hit_dense=None), "hit_dense"), (dict(status=None), "status"), (dict(mode=2), "mode"),
                     (dict(rows=0), "rows"), (dict(kd=0), "kd"), (dict(kd=4097, width=5000), "kd"), (dict(width=9), "width"),
                     (dict(hit_pitch=0), "hit_pitch"), (dict(weight=-1.0), "weight"), (dict(weight=float("nan")), "weight"),
                     (dict(weight=float("inf")), "weight"), (dict(mode=1, rrf_c=-1), "rrf_c")):
        rc, msg = _fuse(lib, **kw)
        assert rc != 0 and word in msg, (kw, rc, msg)
    assert _grouped(lib)[0] not in (0, 2)
    for kw, word in ((dict(hit_offsets=_FAKE + 0x5004), "hit_offsets"), (dict(hit_values=None), "hit_values"),
                     (dict(d=_FAKE + 0x1004), "d_f32"), (dict(weight=-0.5), "weight"), (dict(weight=float("nan")), "weight"),
                     (dict(kg=0), "kg"), (dict(piece=0), "piece"), (dict(nq=0), "nq"), (dict(G=0), "G")):
        rc, msg = _grouped(lib, **kw)
        assert rc != 0 and word in msg, (kw, rc, msg)
