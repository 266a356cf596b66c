"""Per-document caps without a GPU: a numpy model of the capped page top-k and of the inner hits (DESIGN §4) over a given
score matrix, checked against the walk with per-document counters on random matrices with ties, -0 and NaN; the lemma
(the capped answer is the top-k of the union of the top-k documents' top-m pages); four mutants of the construction,
each rejected on a named fixture; the header's alignment line and the refusals of vr_group_pages_topm before any CUDA
call (fake pointers); and the Python argument checks. tests/test_gpu_capped_retrieval.py compares the GPU with these
models."""
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


# ------------------------------------------------------------------------------------------------ the models
def page_order(s, elig=None):
    """The eligible pages with a number for a score, in (score desc, page asc) order (-0 and +0 tie: the page decides)."""
    s = np.asarray(s, np.float32)
    ok = ~np.isnan(s) if elig is None else (np.asarray(elig, bool) & ~np.isnan(s))
    cols = np.nonzero(ok)[0]
    return cols[np.lexsort((cols, -s[cols]))]


def walk_capped(s, groups, k, m, elig=None):
    """The definition: walk the pages in page order, pick a page unless its document already has m picks, stop at k."""
    count, picks = {}, []
    for p in page_order(s, elig):
        g = int(groups[p])
        if count.get(g, 0) < m:
            picks.append(int(p))
            count[g] = count.get(g, 0) + 1
            if len(picks) == k:
                break
    return picks


def top_documents(s, groups, k, elig=None):
    """score_topk_groups' documents: (best score desc, best page asc) = the capped walk with m = 1."""
    return [int(groups[p]) for p in walk_capped(s, groups, k, 1, elig)]


def topm(s, groups, g, m, elig=None):
    """topm(D): D's first m eligible pages in page order."""
    return [int(p) for p in page_order(s, elig) if groups[p] == g][:m]


def inner_hits(s, groups, k, m, elig=None):
    """[(document, its top-m pages)] of the top-k documents."""
    return [(g, topm(s, groups, g, m, elig)) for g in top_documents(s, groups, k, elig)]


def in_page_order(s, pages):
    pages = np.asarray(pages, np.int64)
    s = np.asarray(s, np.float32)
    return [int(p) for p in pages[np.lexsort((pages, -s[pages]))]] if len(pages) else []


def capped_by_lemma(s, groups, k, m, elig=None):
    """The construction: the plain top-k, in page order, of the union of topm(D) over the top-k documents D."""
    return in_page_order(s, [p for _, ps in inner_hits(s, groups, k, m, elig) for p in ps])[:k]


def capped_from_lists(s, groups, k, m, lists, reduce=True):
    """The construction when each top document's pages arrive as several lists (pieces of a long document, or ranks):
    each list's top-m, reduced to the document's top-m (reduce=False: the trap, the top-k straight over the lists)."""
    cand = []
    for g in top_documents(s, groups, k):
        got = [p for part in lists for p in topm_of(s, [q for q in part if groups[q] == g], m)]
        cand += topm_of(s, got, m) if reduce else got
    return in_page_order(s, cand)[:k]


def topm_of(s, pages, m):
    return in_page_order(s, [p for p in pages if not np.isnan(s[p])])[:m]


def rows(s_rows, picks_rows, groups, k):
    """Picks per row -> (scores [nq, k] f32, pages [nq, k] i64, groups [nq, k] i64) with the (-inf, -1, -1) tail."""
    n = len(picks_rows)
    out = (np.full((n, k), -np.inf, np.float32), np.full((n, k), -1, np.int64), np.full((n, k), -1, np.int64))
    for r, picks in enumerate(picks_rows):
        picks = np.asarray(picks, np.int64)
        out[0][r, :len(picks)] = np.asarray(s_rows[r], np.float32)[picks]
        out[1][r, :len(picks)] = picks
        out[2][r, :len(picks)] = np.asarray(groups)[picks]
    return out


# ------------------------------------------------------------------------------------------------ random fixtures
def _fixture(seed, nd=60, nq=30):
    """Scores on a coarse grid (many ties), some -0 next to +0, some NaN; 1 to 12 documents; a random eligibility."""
    rs = np.random.RandomState(seed)
    s = (rs.randint(-4, 5, (nq, nd)) / 4).astype(np.float32)
    s[rs.rand(nq, nd) < 0.1] = -0.0
    s[rs.rand(nq, nd) < 0.05] = np.nan
    groups = rs.randint(0, rs.randint(1, 13), nd)
    elig = rs.rand(nq, nd) < rs.choice([0.3, 0.8, 1.0])
    return s, groups, elig


@pytest.mark.parametrize("seed", range(40))
def test_model_is_the_walk_with_counters(seed):
    s, groups, elig = _fixture(seed)
    for r in range(len(s)):
        for k, m in [(1, 1), (3, 1), (5, 2), (8, 3), (10, 20), (60, 4)]:
            want = []
            count = np.zeros(groups.max() + 1, np.int64)
            for p in sorted(np.nonzero(elig[r] & ~np.isnan(s[r]))[0], key=lambda p: (-float(s[r, p]), p)):
                if count[groups[p]] < m and len(want) < k:
                    want.append(int(p))
                    count[groups[p]] += 1
            assert walk_capped(s[r], groups, k, m, elig[r]) == want, (r, k, m)


@pytest.mark.parametrize("seed", range(40))
def test_lemma_union_of_top_documents_topm(seed):
    s, groups, elig = _fixture(seed)
    for r in range(len(s)):
        for k, m in [(1, 1), (3, 1), (5, 2), (8, 3), (10, 20), (60, 4), (4, 60)]:
            want = walk_capped(s[r], groups, k, m, elig[r])
            assert capped_by_lemma(s[r], groups, k, m, elig[r]) == want, (r, k, m)
            hits = inner_hits(s[r], groups, k, m, elig[r])
            assert all(len({groups[p] for p in ps}) == 1 and ps[0] == walk_capped(s[r], groups, k, 1, elig[r])[j]
                       for j, (_, ps) in enumerate(hits))  # column 0 is the document's best page


@pytest.mark.parametrize("seed", range(20))
def test_cap_one_is_the_documents_and_cap_k_the_pages(seed):
    s, groups, elig = _fixture(seed)
    for r in range(len(s)):
        for k in (1, 4, 9):
            firsts = walk_capped(s[r], groups, k, 1, elig[r])
            assert [groups[p] for p in firsts] == top_documents(s[r], groups, k, elig[r])
            assert walk_capped(s[r], groups, k, k, elig[r]) == [int(p) for p in page_order(s[r], elig[r])][:k]


def test_negative_zero_ties_with_zero_and_nan_is_never_picked():
    s = np.array([0.0, -0.0, np.nan, -0.0, 0.0], np.float32)
    groups = np.array([0, 1, 1, 2, 2])
    assert walk_capped(s, groups, 5, 1) == [0, 1, 3]
    assert walk_capped(s, groups, 5, 2) == [0, 1, 3, 4]
    assert inner_hits(s, groups, 3, 2) == [(0, [0]), (1, [1]), (2, [3, 4])]


# ------------------------------------------------------------------------------------------------ mutants
def _ab(pages_a=12):
    """k = 2, m = 1: document A has pages 0.90, 0.89, 0.88, ...; document B a single page at 0.5."""
    s = np.array([0.90 - 0.01 * i for i in range(pages_a)] + [0.5], np.float32)
    return s, np.array([0] * pages_a + [1])


def test_mutant_candidates_from_the_page_top_k_m():
    s, groups = _ab()
    k, m = 2, 1
    want = walk_capped(s, groups, k, m)
    assert want == [0, 12]
    cand = [int(p) for p in page_order(s)][:k * m]           # the page top-(k m) instead of the top-k documents
    mutant = walk_capped(np.where(np.isin(np.arange(len(s)), cand), s, np.nan), groups, k, m)
    assert mutant != want and capped_by_lemma(s, groups, k, m) == want


def test_mutant_first_pages_by_id():
    s = np.array([0.1, 0.9, 0.8, 0.7, 0.6], np.float32)     # document 0's lowest pages are its worst
    groups = np.array([0, 0, 0, 1, 1])
    k, m = 3, 2
    want = walk_capped(s, groups, k, m)
    assert want == [1, 2, 3]
    by_id = in_page_order(s, [p for g in top_documents(s, groups, k) for p in sorted(np.nonzero(groups == g)[0])[:m]])[:k]
    assert by_id != want and capped_by_lemma(s, groups, k, m) == want


def test_mutant_top_k_straight_over_pieces_or_ranks():
    """m = 2: D has pages 0.9 and 0.8 on one rank (or piece) and 0.7 on the other; E has 0.6. The top-3 of the gathered
    lists is D, D, D."""
    s = np.array([0.9, 0.8, 0.7, 0.6], np.float32)
    groups = np.array([0, 0, 0, 1])
    k, m = 3, 2
    lists = [[0, 1], [2, 3]]
    want = walk_capped(s, groups, k, m)
    assert want == [0, 1, 3]
    assert capped_from_lists(s, groups, k, m, lists) == want
    assert capped_from_lists(s, groups, k, m, lists, reduce=False) == [0, 1, 2]


def test_mutant_over_fetch_four_times_then_cap():
    s, groups = _ab()
    k, m = 2, 1
    fetched = [int(p) for p in page_order(s)][:4 * k]      # search(topk * 4)
    count, mutant = {}, []
    for p in fetched:
        if count.get(groups[p], 0) < m and len(mutant) < k:
            mutant.append(p)
            count[groups[p]] = count.get(groups[p], 0) + 1
    assert mutant != walk_capped(s, groups, k, m) == capped_by_lemma(s, groups, k, m)


# ------------------------------------------------------------------------------------------------ C ABI refusals
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
FAKE = 0x7F0000000000
TABLE = {"q_f32": 4, "d_f32": 16, "groups": 8, "group_offsets": 4, "group_pages": 4, "out_scores": 4, "out_pages": 8}


def test_alignment_table_matches_header():
    text = open(HEADER).read()
    m = re.search(r"Alignment \(bytes\) of the vr_group_pages_topm arguments: (.*?)\*/", text, re.S)
    assert m and {name: int(n) for name, n in re.findall(r"(\w+) (\d+)", m.group(1))} == TABLE


def test_python_and_c_caps_agree():
    text = open(os.path.join(os.path.dirname(HEADER), "..", "visrag_b200", "csrc", "score.cu")).read()
    assert f"constexpr int GROUP_PAGES_MAX = {R.GROUP_PAGES_MAX};" in text
    assert R.GROUP_PAGES_MAX >= 64


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _call(lib, masks=None, **over):
    p = {name: FAKE + 0x100000 * (i + 1) for i, name in enumerate(TABLE)}
    a = dict(nq=40, nd=5000, dim=2304, kg=10, G=700, m=3, piece=64, pieces=2)
    for key, v in over.items():
        (p if key in p else a)[key] = v
    return lib.vr_group_pages_topm(p["q_f32"], a["nq"], p["d_f32"], a["nd"], a["dim"], p["groups"], a["kg"],
                                   p["group_offsets"], p["group_pages"], a["G"], masks, a["m"], a["piece"], a["pieces"], 0,
                                   p["out_scores"], p["out_pages"], None)


BAD = [
    (dict(nq=0), r"nq=0"),
    (dict(nd=0), r"nd=0"),
    (dict(nd=1 << 31), r"nd=2147483648"),
    (dict(dim=0), r"dim=0"),
    (dict(dim=6), r"dim=6"),
    (dict(kg=0), r"kg=0"),
    (dict(nq=1 << 28, kg=8), r"nq=268435456 x kg=8"),
    (dict(G=0), r"G=0"),
    (dict(m=0), r"m=0"),
    (dict(m=257), r"m=257"),
    (dict(piece=0), r"piece=0"),
    (dict(piece=4097), r"piece=4097"),
    (dict(pieces=0), r"pieces=0"),
    (dict(pieces=65536), r"pieces=65536"),
    (dict(dim=50000, piece=4096), r"dim=50000 with piece=4096"),
]


@no_device
@pytest.mark.parametrize("kw,pattern", BAD, ids=[f"{sorted(k)[0]}-{i}" for i, (k, _) in enumerate(BAD)])
def test_refuses_bad_arguments_before_any_cuda_call(lib, kw, pattern):
    rc = _call(lib, **kw)
    msg = lib.vr_last_error().decode()
    assert rc == 2 and "vr_group_pages_topm" in msg and re.search(pattern, msg), (rc, msg)


@no_device
@pytest.mark.parametrize("name", list(TABLE))
def test_refuses_each_null_and_misaligned_pointer(lib, name):
    n = TABLE[name]
    base = FAKE + 0x100000 * (list(TABLE).index(name) + 1)
    if n > 1:
        rc = _call(lib, **{name: base + (4 if n >= 8 else 2)})
        msg = lib.vr_last_error().decode()
        assert rc == 2 and re.search(rf"\b{name}\b must be {n}-byte aligned", msg), (rc, msg)
    rc = _call(lib, **{name: None})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b must not be NULL", msg), (rc, msg)


@no_device
def test_refuses_a_bad_mask_set(lib):
    m = L.DocMasks()
    m.words, m.pitch, m.of_query, m.count = FAKE + 2, 157, None, 1
    assert _call(lib, masks=C.byref(m)) == 2 and "masks->words" in lib.vr_last_error().decode()
    m.words, m.pitch = FAKE, 100                                   # ceil(5000 / 32) = 157 words
    assert _call(lib, masks=C.byref(m)) == 2 and "masks->pitch" in lib.vr_last_error().decode()
    m.pitch, m.count = 157, 3                                      # several masks need of_query
    assert _call(lib, masks=C.byref(m)) == 2 and "masks->of_query" in lib.vr_last_error().decode()
    m.count = 0
    assert _call(lib, masks=C.byref(m)) == 2 and "masks->count" in lib.vr_last_error().decode()


@no_device
def test_valid_arguments_reach_the_device(lib):
    """Past validation a call stops at its first CUDA call (status 1, not the refusal's 2)."""
    for kw in (dict(m=1), dict(m=256), dict(piece=4096, dim=4), dict(pieces=65535), dict(kg=1, pieces=1, piece=1)):
        assert _call(lib, **kw) != 2, (kw, lib.vr_last_error().decode())


# ------------------------------------------------------------------------------------------------ Python refusals
class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name}) although the arguments are invalid")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(L, "_lib", _NoLib())


def _cpu_index(nd=100, d=8):
    return R.CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


@pytest.mark.parametrize("v,match", [(0, "per_group=0"), (-1, "per_group=-1"), (2.0, "per_group must be an int"),
                                     (True, "per_group must be an int"), (None, "per_group must be an int")])
def test_python_refuses_bad_per_group(stub, v, match):
    with pytest.raises(ValueError, match=match):
        R.score_topk_capped(torch.zeros((2, 8)), _cpu_index(), 5, torch.zeros(100, dtype=torch.int64), v)
    with pytest.raises(ValueError, match=match):
        R.sharded_topk_capped(torch.zeros((2, 8)), _cpu_index(), 5, torch.zeros(100, dtype=torch.int64), v, 0)


def test_python_refuses_a_cap_beyond_the_kernel(stub):
    with pytest.raises(ValueError, match="per_group=300"):
        R.score_topk_capped(torch.zeros((2, 8)), _cpu_index(), 400, torch.zeros(100, dtype=torch.int64), 300)


@pytest.mark.parametrize("v,match", [(0, "pages=0"), (257, "pages=257"), (1.5, "pages must be an int")])
def test_python_refuses_bad_pages(stub, v, match):
    for fn in (R.score_topk_groups_pages, R.sharded_topk_groups_pages):
        with pytest.raises(ValueError, match=match):
            fn(torch.zeros((2, 8)), _cpu_index(), 5, torch.zeros(100, dtype=torch.int64), v, 0)
    with pytest.raises(ValueError, match=match):
        R.group_pages_topm(torch.zeros((2, 8)), _cpu_index(), torch.zeros((2, 3), dtype=torch.int64),
                           torch.zeros(100, dtype=torch.int64), v)


def test_python_refuses_cpu_queries(stub):
    with pytest.raises(ValueError, match="CUDA"):
        R.score_topk_capped(torch.zeros((2, 8)), _cpu_index(), 5, torch.zeros(100, dtype=torch.int64), 2)
    with pytest.raises(ValueError, match="CUDA"):
        R.score_topk_groups_pages(torch.zeros((2, 8)), _cpu_index(), 5, torch.zeros(100, dtype=torch.int64), 2)
