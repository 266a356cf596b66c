"""Diverse retrieval (maximal marginal relevance) without a GPU: a numpy float32 model of the selection's definition
(DESIGN §4), hand-checked cases, three mutants of the arithmetic that each return a different pick on a fixture built
here, the refusals of vr_mmr_select (C ABI, before any CUDA call, fake pointers) and the Python argument checks (with a
library stub that fails if reached). tests/test_gpu_mmr.py compares the kernel with this model bit for bit."""
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
f32 = np.float32


# ------------------------------------------------------------------------------------------------ the model
def mmr_model(s, ids, gram, lam, k, fma=False, late_ties=False, latest_only=False):
    """One query row. s f32 [F] / ids [F]: the candidates (the first id < 0 ends them); gram f32 [F', F'] (F' the
    candidates): gram[a, b] = sim(c_a, c_b). Returns the picked positions, in pick order. The flags are the mutants:
    fma computes v with one rounding, late_ties gives ties to the later candidate, latest_only takes r from the latest
    pick alone."""
    s = np.asarray(s, f32)
    ids = np.asarray(ids)
    bad = np.nonzero(ids < 0)[0]
    n = int(bad[0]) if bad.size else len(ids)
    npick = min(k, n)
    if npick == 0:
        return []
    lam = f32(lam)
    mu = f32(f32(1) - lam)
    r = np.full(n, -np.inf, f32)
    taken = np.zeros(n, bool)
    picks = [0]
    with np.errstate(invalid="ignore", over="ignore"):
        for _ in range(1, npick):
            p = picks[-1]
            taken[p] = True
            sim = np.asarray(gram, f32)[:n, p]
            r = sim.copy() if latest_only else np.fmax(r, sim)
            if fma:  # lam * s exactly (48 bits), minus the rounded mu * r, rounded once
                v = (lam.astype(np.float64) * s[:n].astype(np.float64) - (mu * r).astype(np.float64)).astype(f32)
            else:
                v = (lam * s[:n]) - (mu * r)
            best = -1
            for j in range(n):
                if taken[j]:
                    continue
                if best < 0:
                    best = j
                    continue
                a, b = v[j], v[best]
                if np.isnan(a):
                    continue
                if np.isnan(b) or a > b or (late_ties and a == b):
                    best = j
            picks.append(best)
    return picks


def rows_of(picks, s, ids, k, id_offset=0):
    """The output row (scores, ids) of a pick list."""
    out_s = np.full(k, -np.inf, f32)
    out_i = np.full(k, -1, np.int64)
    for t, p in enumerate(picks):
        out_s[t], out_i[t] = s[p], ids[p] + id_offset
    return out_s, out_i


def gram_of(E):
    """sim of unit rows by a float32 numpy matmul: the hand-checked cases only need values, not the kernel's bits."""
    return (np.asarray(E, f32) @ np.asarray(E, f32).T).astype(f32)


# ------------------------------------------------------------------------------------------------ hand-checked cases
def test_lambda_one_gives_the_candidate_order():
    rs = np.random.RandomState(0)
    E = rs.randn(30, 16).astype(f32)
    s = np.sort(rs.randn(30).astype(f32))[::-1]
    assert mmr_model(s, np.arange(30), gram_of(E), 1.0, 10) == list(range(10))


def _planted(clusters=4, per=5, dim=32, seed=1):
    """Candidates in score order where each cluster's pages are near-copies, and clusters are nearly orthogonal."""
    rs = np.random.RandomState(seed)
    centers = np.linalg.qr(rs.randn(dim, clusters))[0].T.astype(f32)
    cl = np.repeat(np.arange(clusters), per)
    E = centers[cl] + f32(0.01) * rs.randn(len(cl), dim).astype(f32)
    E /= np.linalg.norm(E, axis=1, keepdims=True)
    # cluster 0 scores highest, and so on: plain top-k fills with cluster 0
    s = np.sort((f32(0.9) - f32(0.1) * cl + f32(0.001) * rs.rand(len(cl))).astype(f32))[::-1]
    return E, s, cl


def test_lambda_zero_covers_every_planted_cluster_first():
    E, s, cl = _planted()
    picks = mmr_model(s, np.arange(len(s)), gram_of(E), 0.0, 4)
    assert sorted(cl[picks].tolist()) == [0, 1, 2, 3]
    assert mmr_model(s, np.arange(len(s)), gram_of(E), 1.0, 4) == [0, 1, 2, 3]  # all of cluster 0
    assert set(cl[:4].tolist()) == {0}


def test_lambda_zero_takes_the_least_similar_candidate():
    s = f32([0.9, 0.8, 0.7, 0.6])
    g = f32([[1, 0.5, 0.2, 0.9], [0.5, 1, 0.3, 0.1], [0.2, 0.3, 1, 0.8], [0.9, 0.1, 0.8, 1]])
    # r after c0: [., .5, .2, .9] -> c2; r: max(.5, .3) = .5, max(.9, .8) = .9 -> c1
    assert mmr_model(s, np.arange(4), g, 0.0, 4) == [0, 2, 1, 3]


def test_ties_go_to_the_lower_position():
    s = f32([0.9, 0.5, 0.5, 0.5])
    g = np.eye(4, dtype=f32)
    g[1, 0] = g[2, 0] = g[3, 0] = 0.25
    assert mmr_model(s, np.arange(4), g, 0.5, 4) == [0, 1, 2, 3]
    # +0 and -0 are equal values: lam * s = +0 and -0
    s0 = f32([1.0, 0.0, -0.0])
    g0 = np.zeros((3, 3), f32)
    assert mmr_model(s0, np.arange(3), g0, 0.5, 3) == [0, 1, 2]
    assert mmr_model(f32([1.0, -0.0, 0.0]), np.arange(3), g0, 0.5, 3) == [0, 1, 2]


def test_nan_ranks_below_every_number_and_inf_above():
    inf = np.inf
    s = f32([inf, inf, 0.3])
    g = f32([[1, inf, inf], [inf, 1, 0], [inf, 0, 1]])
    # v1 = inf - inf = NaN, v2 = 0.15 - inf = -inf: -inf still beats NaN
    assert mmr_model(s, np.arange(3), g, 0.5, 3) == [0, 2, 1]
    # v = +inf wins over any finite value
    s2 = f32([1.0, 0.9, 0.8])
    s2[2] = np.nan  # a NaN score gives a NaN v at any lambda > 0
    assert mmr_model(s2, np.arange(3), np.eye(3, dtype=f32), 0.5, 3) == [0, 1, 2]
    s3 = f32([inf, 0.5, inf])
    assert mmr_model(s3, np.arange(3), np.eye(3, dtype=f32), 0.5, 2) == [0, 2]


def test_nan_similarity_is_ignored_by_r():
    s = f32([0.9, 0.8, 0.7])
    g = f32([[1, np.nan, 0.5], [np.nan, 1, 0.0], [0.5, 0.0, 1]])
    # r1 = fmax(-inf, NaN) = -inf, so v1 = 0.5 * 0.8 - 0.5 * -inf = +inf
    assert mmr_model(s, np.arange(3), g, 0.5, 3) == [0, 1, 2]
    # at lambda = 1, mu * r1 = 0 * -inf = NaN: v1 is NaN and c2 comes first
    assert mmr_model(s, np.arange(3), g, 1.0, 3) == [0, 2, 1]


def test_fewer_candidates_than_k_end_in_the_tail():
    s = f32([0.9, 0.8, -np.inf, -np.inf])
    ids = np.array([7, 3, -1, -1])
    picks = mmr_model(s, ids, np.eye(2, dtype=f32), 0.5, 3)
    assert picks == [0, 1]
    out_s, out_i = rows_of(picks, s, ids, 3, id_offset=100)
    assert out_i.tolist() == [107, 103, -1] and out_s[2] == -np.inf
    assert mmr_model(s[:0], ids[:0], np.zeros((0, 0), f32), 0.5, 3) == []


# ------------------------------------------------------------------------------------------------ mutants
def _fma_fixture():
    """Two candidates whose v differ only in the last bits: each seed draws lam, s_1 > s_2 and r_1, and sets r_2 so that
    the exact values nearly tie. Returns the first seeded fixture on which the fused v changes the pick."""
    for seed in range(2000):
        rs = np.random.RandomState(seed)
        lam = f32(rs.uniform(0.2, 0.8))
        mu = f32(1) - lam
        s1 = f32(rs.uniform(0.3, 0.9))
        s2 = f32(s1 - f32(rs.uniform(1e-4, 1e-2)))
        r1 = f32(rs.uniform(0.1, 0.9))
        r2 = f32(float(r1) - float(lam) * (float(s1) - float(s2)) / float(mu))
        s = f32([1.0, s1, s2])
        g = np.eye(3, dtype=f32)
        g[1, 0] = g[0, 1] = r1
        g[2, 0] = g[0, 2] = r2
        if mmr_model(s, np.arange(3), g, lam, 2) != mmr_model(s, np.arange(3), g, lam, 2, fma=True):
            return s, g, lam
    return None


def test_fused_multiply_add_changes_a_pick():
    fx = _fma_fixture()
    assert fx is not None
    s, g, lam = fx
    assert mmr_model(s, np.arange(3), g, lam, 2) != mmr_model(s, np.arange(3), g, lam, 2, fma=True)


def test_ties_to_the_later_candidate_change_a_pick():
    """Exact duplicate pages: same score, same similarity to every pick."""
    s = f32([0.9, 0.7, 0.7, 0.2])
    g = f32([[1, 0.3, 0.3, 0.1], [0.3, 1, 1, 0.2], [0.3, 1, 1, 0.2], [0.1, 0.2, 0.2, 1]])
    assert mmr_model(s, np.arange(4), g, 0.5, 2) == [0, 1]
    assert mmr_model(s, np.arange(4), g, 0.5, 2, late_ties=True) == [0, 2]


def test_r_from_the_latest_pick_only_changes_a_pick():
    s = f32([0.9, 0.85, 0.5, 0.45])
    g = f32([[1, 0.99, 0.1, 0.2], [0.99, 1, 0.1, 0.2], [0.1, 0.1, 1, 0.3], [0.2, 0.2, 0.3, 1]])
    assert mmr_model(s, np.arange(4), g, 0.5, 3) == [0, 2, 3]
    assert mmr_model(s, np.arange(4), g, 0.5, 3, latest_only=True) == [0, 2, 1]


# ------------------------------------------------------------------------------------------------ C ABI refusals
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
FAKE = 0x7F0000000000
TABLE = {"emb": 16, "cand_scores": 4, "cand_ids": 8, "lambda": 4, "out_scores": 4, "out_ids": 8}


def test_alignment_table_matches_header():
    text = open(HEADER).read()
    m = re.search(r"Alignment \(bytes\) of the vr_mmr_select arguments: (.*?)\*/", text, re.S)
    assert m and {name: int(n) for name, n in re.findall(r"(\w+) (\d+)", m.group(1))} == TABLE


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _call(lib, **over):
    p = {name: FAKE + 0x100000 * (i + 1) for i, name in enumerate(TABLE)}
    a = dict(nd=5000, dim=2304, nq=40, fetch=40, k=10)
    for key, v in over.items():
        (p if key in p else a)[key] = v
    return lib.vr_mmr_select(p["emb"], a["nd"], a["dim"], p["cand_scores"], p["cand_ids"], a["nq"], a["fetch"], p["lambda"],
                             a["k"], 0, p["out_scores"], p["out_ids"], None)


BAD = [
    (dict(nq=0), r"nq=0"),
    (dict(nq=1 << 28), r"nq=268435456"),
    (dict(nd=0), r"nd=0"),
    (dict(dim=0), r"dim=0"),
    (dict(dim=6), r"dim=6"),
    (dict(fetch=0), r"fetch=0"),
    (dict(fetch=129, dim=64), r"fetch=129"),
    (dict(fetch=72, dim=4104), r"fetch=72 x dim=4104"),
    (dict(fetch=1, dim=40000), r"fetch=1 rows of dim=40000 do not fit"),
    (dict(fetch=121, dim=2432), r"fetch=121 rows of dim=2432 do not fit"),
    (dict(fetch=8, dim=36864), r"fetch=8 rows of dim=36864 do not fit"),  # one row a CTA, but not with the pick's row
    (dict(k=0), r"k=0"),
    (dict(k=41), r"k=41"),
]


@no_device
@pytest.mark.parametrize("kw,pattern", BAD, ids=[f"{sorted(k)[0]}-{i}" for i, (k, _) in enumerate(BAD)])
def test_refuses_bad_arguments_before_any_cuda_call(lib, kw, pattern):
    rc = _call(lib, **kw)
    msg = lib.vr_last_error().decode()
    assert rc == 2 and "vr_mmr_select" in msg and re.search(pattern, msg), (rc, msg)


@no_device
@pytest.mark.parametrize("name", list(TABLE))
def test_refuses_each_null_and_misaligned_pointer(lib, name):
    n = TABLE[name]
    base = FAKE + 0x100000 * (list(TABLE).index(name) + 1)
    rc = _call(lib, **{name: base + (4 if n >= 8 else 2)})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b must be {n}-byte aligned", msg), (rc, msg)
    rc = _call(lib, **{name: None})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b must not be NULL", msg), (rc, msg)


@no_device
@pytest.mark.parametrize("dim", [4, 64, 2304, 2432, 4096, 6144, 18000, 20000, 36864, 36868])
def test_python_caps_are_the_entry_points(lib, dim):
    """mmr_fetch_max(dim) is accepted (past validation a call stops at its first CUDA call, status 1) and one more
    candidate is refused."""
    top = R.mmr_fetch_max(dim)
    if top:
        assert _call(lib, dim=dim, fetch=top, k=1) != 2, lib.vr_last_error().decode()
        assert _call(lib, dim=dim, fetch=top, k=top) != 2, lib.vr_last_error().decode()
    assert _call(lib, dim=dim, fetch=top + 1, k=1) == 2
    for f in range(1, top + 1):  # every smaller fetch is accepted too
        assert _call(lib, dim=dim, fetch=f, k=1) != 2, (f, lib.vr_last_error().decode())


def test_fetch_caps():
    assert R.mmr_fetch_max(2304) == 128 and R.mmr_fetch_max(64) == 128
    assert R.mmr_fetch_max(4096) == 72 and R.mmr_fetch_max(20000) == 8 and R.mmr_fetch_max(18000) == 1
    assert R.mmr_fetch_max(36864) == 0 and R.mmr_fetch_max(40000) == 0


# ------------------------------------------------------------------------------------------------ Python refusals
class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name}) although the arguments are invalid")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(L, "_lib", _NoLib())


def _cpu_index(nd=100, d=8):
    return R.CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


@pytest.mark.parametrize("lam,match", [
    (float("nan"), "not be NaN"),
    (np.float32("nan"), "not be NaN"),
    (-0.1, r"\[0, 1\]"),
    (1.5, r"\[0, 1\]"),
    (torch.tensor([0.1, float("nan"), 0.2]), "not be NaN"),
    (torch.tensor([0.1, 1.2, 0.2]), r"\[0, 1\]"),
    (torch.tensor([0.1, 0.2]), r"shape \[3\]"),
    (torch.zeros(3, dtype=torch.float64), "torch.float32"),
    ("0.5", "must be a float"),
    (None, "must be a float"),
    (True, "must be a float"),
])
def test_python_refuses_bad_lambda(stub, lam, match):
    with pytest.raises(ValueError, match=match):
        R._check_lambda(lam, 3, torch.device("cpu"))


def test_python_lambda_forms(stub):
    assert R._check_lambda(0.25, 3, torch.device("cpu")).tolist() == [0.25] * 3
    assert R._check_lambda(1, 2, torch.device("cpu")).dtype == torch.float32
    assert R._check_lambda(torch.tensor([0.0, 1.0]), 2, torch.device("cpu")).tolist() == [0.0, 1.0]


def test_python_fetch_rules(stub):
    assert R._check_fetch(3, None, 2304) == (3, 20)
    assert R._check_fetch(10, None, 2304) == (10, 40)
    assert R._check_fetch(40, None, 2304) == (40, 128)
    assert R._check_fetch(10, None, 4096) == (10, 40) and R._check_fetch(30, None, 4096) == (30, 72)
    assert R._check_fetch(5, 5, 64) == (5, 5)
    for k, fetch, match in [(0, None, "k=0"), (10, 8, "k=10"), (3, 129, "fetch_k=129"), (3, 0, "fetch_k=0"),
                            (129, None, "k=129"), (2.0, None, "k must be an int"), (3, True, "fetch_k must be an int")]:
        with pytest.raises(ValueError, match=match):
            R._check_fetch(k, fetch, 2304)
    with pytest.raises(ValueError, match="dim=40000 is too large"):
        R._check_fetch(1, None, 40000)


def test_python_mmr_select_refuses_bad_candidates(stub):
    idx = _cpu_index()
    s = torch.zeros((2, 8))
    i = torch.zeros((2, 8), dtype=torch.int64)
    bad = [
        (dict(scores=s.double()), "torch.float32"),
        (dict(scores=s[0]), r"\[nq, F\]"),
        (dict(ids=i.float()), "int32 or int64"),
        (dict(ids=i[:, :4]), "shape of scores"),
        (dict(ids=i.clone().fill_(100)), r"\[0, 100\)"),
        (dict(ids=i.clone().fill_(-2)), r"\[0, 100\)"),
        (dict(k=9), "k=9"),
        (dict(k=0), "k=0"),
        (dict(lambda_mult=2.0), r"\[0, 1\]"),
        (dict(lambda_mult=torch.zeros(3)), r"shape \[2\]"),
    ]
    for kw, match in bad:
        a = dict(scores=s, ids=i, k=3, lambda_mult=0.5)
        a.update(kw)
        with pytest.raises(ValueError, match=match):
            R.mmr_select(idx, a["scores"], a["ids"], a["k"], a["lambda_mult"])
    with pytest.raises(ValueError, match="fetch_k=200"):
        R.mmr_select(_cpu_index(d=8), torch.zeros((1, 200)), torch.zeros((1, 200), dtype=torch.int64), 3)


def test_python_score_mmr_refuses_before_the_search(stub):
    idx = _cpu_index()
    with pytest.raises(ValueError, match="fetch_k=129"):
        R.score_mmr(torch.zeros((2, 8)), idx, 3, fetch_k=129)
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        R.score_mmr(torch.zeros((2, 8)), idx, 3, lambda_mult=-1.0)
    with pytest.raises(ValueError, match="CUDA"):
        R.score_mmr(torch.zeros((2, 8)), idx, 3)
