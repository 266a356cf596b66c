"""Document range search and deep document top-k without a GPU: a numpy model of the reduction (vr_range_groups) and of
the deep document route against brute force (scan -> per-document max with the lowest page -> filter -> sort) on
random matrices with ties, -0, NaN and sparse groups; four mutants, each rejected on a named fixture; the refusals of
vr_range_groups (C ABI, before any CUDA call, fake pointers) and the Python argument checks (a library stub that fails
if reached)."""
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


# ------------------------------------------------------------------------------------------------ models
def page_key(s, p):
    """group_key_kernel's key: the order bits of the score (-0 as +0) above ~page; larger = earlier in page order."""
    b = np.float32(s).view(np.uint32)
    if b == 0x80000000:
        b = np.uint32(0)
    o = (~b & 0xFFFFFFFF) if b & 0x80000000 else (b | 0x80000000)
    return (int(o) << 32) | (~int(p) & 0xFFFFFFFF)


def reduce_region(scores, ids, groups, first_in_region=False, higher_page=False):
    """The reduction of one region row (entries in any order): {group: (score, page)} of each group's first entry in
    (score desc, page asc) order, with that entry's own score. Mutants: the group's first entry in region order; ties
    going to the higher page."""
    best = {}
    for s, p in zip(scores, ids):
        if np.isnan(s):
            continue
        g = int(groups[p])
        if first_in_region:
            best.setdefault(g, (s, p))
            continue
        key = page_key(s, (~p & 0xFFFFFFFF) if higher_page else p)
        if g not in best or key > best[g][2]:
            best[g] = (s, p, key)
    return {g: v[:2] for g, v in best.items()}


def order(entries):
    """(score, page, group) entries by (score desc, page asc); -0 ties +0."""
    return sorted(entries, key=lambda e: (-float(e[0]), e[1]))


def brute(row, groups, eligible):
    """Every document with an eligible non-NaN page: (its max score with that page's bits, the lowest page with it)."""
    best = {}
    for p in range(len(row)):
        if not eligible[p] or np.isnan(row[p]):
            continue
        g = int(groups[p])
        if g not in best or row[p] > best[g][0]:
            best[g] = (row[p], p)
    return order([(s, p, g) for g, (s, p) in best.items()])


def range_model(row, groups, eligible, t, **mut):
    """A = eligible pages with s >= t, in a shuffled region order; reduced; sorted."""
    region = [p for p in np.random.RandomState(len(row)).permutation(len(row)) if eligible[p] and row[p] >= t]
    red = reduce_region([row[p] for p in region], region, groups, **mut)
    return order([(s, p, g) for g, (s, p) in red.items()])


def deep_model(row, groups, eligible, k, t, count_pages=False):
    """The deep document route for one row with threshold t: the top-k of the reduced region when it holds at least k
    documents (mutant: at least k pages), else None (the row falls back to the scan)."""
    region = [p for p in range(len(row)) if eligible[p] and row[p] >= t]
    red = reduce_region([row[p] for p in region], region, groups)
    if (len(region) if count_pages else len(red)) < k:
        return None
    return order([(s, p, g) for g, (s, p) in red.items()])[:k]


def same(a, b):
    return len(a) == len(b) and all(np.float32(x[0]).view(np.uint32) == np.float32(y[0]).view(np.uint32) and x[1:] == y[1:]
                                    for x, y in zip(a, b))


def random_row(rs, nd):
    row = (rs.randint(-6, 7, nd) / 4).astype(np.float32)                 # many ties
    row[rs.rand(nd) < 0.05] = np.float32(-0.0)
    row[rs.rand(nd) < 0.03] = np.nan
    groups = rs.choice(np.arange(0, 10 * nd, 7), nd // 3 + 1)[rs.randint(0, nd // 3 + 1, nd)]   # sparse ids, G > nd
    return row, groups, rs.rand(nd) < 0.8


@pytest.mark.parametrize("seed", range(40))
def test_reduction_equals_brute_force(seed):
    rs = np.random.RandomState(seed)
    row, groups, eligible = random_row(rs, 60 + seed * 5)
    want = brute(row, groups, eligible)
    for t in (-np.inf, np.float32(-0.0), np.float32(0.0), np.float32(0.5), np.float32(2.0)):
        assert same(range_model(row, groups, eligible, t), [e for e in want if e[0] >= t]), t


@pytest.mark.parametrize("seed", range(40))
def test_deep_route_is_exact_whenever_it_answers(seed):
    rs = np.random.RandomState(100 + seed)
    row, groups, eligible = random_row(rs, 200)
    want = brute(row, groups, eligible)
    for k in (1, 5, 17, 40):
        for t in (np.float32(x) for x in (-1.5, -0.25, 0.0, 0.75, 1.5)):
            got = deep_model(row, groups, eligible, k, t)
            if got is not None:
                assert same(got, want[:k]), (k, t)
        assert deep_model(row, groups, eligible, k, -np.inf) is not None or len(want) < k


# ------------------------------------------------------------------------------------------------ mutants
def test_mutant_first_entry_in_region_order():
    """Fixture "document of two pages, the worse first": the region lists page 3 (0.25) before page 1 (0.75)."""
    groups = np.array([0, 5, 1, 5])
    got = reduce_region(np.float32([0.25, 0.75]), [3, 1], groups, first_in_region=True)
    assert got[5] != reduce_region(np.float32([0.25, 0.75]), [3, 1], groups)[5] == (np.float32(0.75), 1)


def test_mutant_ties_to_the_higher_page():
    """Fixture "equal best pages": pages 2 and 6 of document 4 both score 0.5; the lower page is the best page."""
    groups = np.array([0, 0, 4, 0, 0, 0, 4])
    s, ids = np.float32([0.5, 0.5]), [6, 2]
    assert reduce_region(s, ids, groups)[4][1] == 2
    assert reduce_region(s, ids, groups, higher_page=True)[4][1] == 6


def test_mutant_counting_pages_instead_of_documents():
    """Fixture "one long document fills the region": document 0 has 30 pages at 0.9, documents 1 .. 9 one page each at
    0.1 .. 0.5; t = 0.45 keeps 32 pages of three documents. At k = 5 the page count says "answer", and the answer holds
    two documents where the scan has five."""
    row = np.float32([0.9] * 30 + [0.1, 0.2, 0.3, 0.35, 0.4, 0.45, 0.5, 0.15, 0.25])
    groups = np.array([0] * 30 + list(range(1, 10)))
    eligible = np.ones(len(row), bool)
    want = brute(row, groups, eligible)[:5]
    assert deep_model(row, groups, eligible, 5, np.float32(0.45)) is None
    bad = deep_model(row, groups, eligible, 5, np.float32(0.45), count_pages=True)
    assert bad is not None and not same(bad, want) and len(want) == 5


def test_mutant_canonical_zero_instead_of_the_pages_bits():
    """Fixture "a document at -0": its best page scores -0 (ties +0 by value, but the bits are the page's own). An
    output that rebuilt the score from the key (-0 canonicalised to +0) differs in bits from the scan."""
    groups = np.array([0, 1])
    row = np.float32([-0.0, -0.5])
    red = reduce_region(row, [0, 1], groups)
    assert np.float32(red[0][0]).view(np.uint32) == 0x80000000
    key = page_key(red[0][0], 0)
    from_key = np.uint32(key >> 32) & np.uint32(0x7FFFFFFF)  # what the key holds of a score >= 0: +0
    assert not same([(np.uint32(from_key).view(np.float32), 0, 0)], [(red[0][0], 0, 0)])
    assert same(order([(s, p, g) for g, (s, p) in red.items()]), brute(row, groups, np.ones(2, bool)))


def test_zero_ties_go_to_the_lower_page_with_its_bits():
    groups = np.array([3, 3, 3])
    s, p = reduce_region(np.float32([0.0, -0.0, -0.25]), [1, 0, 2], groups)[3]   # page 1: +0, page 0: -0
    assert p == 0 and np.float32(s).view(np.uint32) == 0x80000000
    s, p = reduce_region(np.float32([-0.0, 0.0, -0.25]), [2, 1, 0], groups)[3]   # page 2: -0, page 1: +0
    assert p == 1 and np.float32(s).view(np.uint32) == 0


# ------------------------------------------------------------------------------------------------ C ABI refusals
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
FAKE = 0x7F0000000000
TABLE = {"scores": 4, "ids": 4, "counts": 4, "doc_groups": 4, "out_scores": 4, "out_ids": 4, "out_counts": 4, "ws": 8}


def test_alignment_table_matches_header():
    text = open(HEADER).read()
    m = re.search(r"Alignment \(bytes\) of the vr_range_groups arguments: (.*?)\*/", text, re.S)
    assert m and {n: int(b) for n, b in re.findall(r"(\w+) (\d+)", m.group(1))} == TABLE


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _call(lib, **over):
    p = {name: FAKE + 0x100000 * (i + 1) for i, name in enumerate(TABLE)}
    a = dict(rows=40, pitch=30000, max_count=20000, nd=30000, G=900, ws_bytes=1 << 40)
    for k, v in over.items():
        (p if k in p else a)[k] = v
    return lib.vr_range_groups(p["scores"], p["ids"], a["pitch"], p["counts"], a["rows"], a["max_count"], p["doc_groups"],
                               a["nd"], a["G"], p["ws"], a["ws_bytes"], p["out_scores"], p["out_ids"], p["out_counts"], None)


BAD = [(dict(rows=0), r"rows=0"), (dict(rows=65536), r"rows=65536"), (dict(nd=0), r"nd=0"),
       (dict(nd=1 << 31), r"nd=2147483648"), (dict(G=0), r"G=0"), (dict(G=-3), r"G=-3"),
       (dict(max_count=-1), r"max_count=-1"), (dict(max_count=30001), r"max_count=30001"),
       (dict(ws_bytes=1000), r"ws of 1000 bytes"), (dict(ws=None), r"ws of")]


@no_device
@pytest.mark.parametrize("kw,pattern", BAD, ids=[f"{sorted(k)[0]}-{i}" for i, (k, _) in enumerate(BAD)])
def test_refuses_bad_arguments_before_any_cuda_call(lib, kw, pattern):
    rc = _call(lib, **kw)
    msg = lib.vr_last_error().decode()
    assert rc == 2 and "vr_range_groups" in msg and re.search(pattern, msg), (rc, msg)


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
    assert rc == 2 and re.search(rf"\b{name}\b", msg), (rc, msg)


@no_device
def test_accepts_valid_arguments_and_sizes_the_workspace(lib):
    assert _call(lib) != 2, lib.vr_last_error().decode()
    assert _call(lib, max_count=4096, ws=None, ws_bytes=0) != 2, lib.vr_last_error().decode()  # shared memory
    assert lib.vr_range_groups_ws_bytes(3, 4096) == 0 and lib.vr_range_groups_ws_bytes(3, 4097) == 3 * 16384 * 12
    assert lib.vr_range_groups_ws_bytes(0, 5) == -1 and lib.vr_range_groups_ws_bytes(1, -1) == -1


# ------------------------------------------------------------------------------------------------ Python refusals
class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name}) although the arguments are invalid")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(L, "_lib", _NoLib())


def _cpu_index(nd=100, d=8):
    return R.CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


def test_python_refuses_bad_arguments(stub):
    idx, g = _cpu_index(), torch.zeros(100, dtype=torch.int32)
    with pytest.raises(ValueError, match="CUDA tensor"):
        R.score_range_groups(torch.zeros((2, 8)), idx, 0.5, g)
    with pytest.raises(ValueError, match="must not be NaN"):
        R._check_min_score(float("nan"), 2, torch.device("cpu"))
    with pytest.raises(ValueError, match="cap"):
        R._check_cap(0)


def test_sampled_documents_take_every_stride_th_group_with_all_its_pages(stub):
    groups = torch.tensor([4, 0, 4, 1, 2, 0, 9, 8, 8], dtype=torch.int32)
    G = 10
    order = torch.sort(groups, stable=True).indices
    offsets = torch.zeros(G + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.bincount(groups, minlength=G), 0)
    gt = R._GroupTable(groups, offsets.to(torch.int32), order.to(torch.int32), G, 2)
    cols, renumbered = R._sample_documents(gt, 4)
    assert cols.tolist() == [1, 5, 0, 2, 7, 8] and renumbered.tolist() == [0, 0, 1, 1, 2, 2]
    assert renumbered.dtype == torch.int32
    cols, renumbered = R._sample_documents(gt, 1)
    assert sorted(cols.tolist()) == list(range(9)) and torch.equal(renumbered, groups[cols])
