"""Candidate lists without a GPU: the refusals of vr_score_lists (C ABI, before any CUDA call, fake pointers), the Python
argument checks (with a library stub that fails if reached), a numpy model of the chunked page and document selection
against a direct sort, a mutant of the document merge that keeps the first k pages per chunk instead of the first k
distinct groups (it returns a wrong top-k on a fixture), and the knowledge base's routing rule."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from visrag_b200 import _lib as L
from visrag_b200 import knowledge_base as KB
from visrag_b200 import retriever as R

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "visrag_b200.h")

# pointer -> alignment its accesses need (vr_score_lists: scalar loads and stores; d_f32 rows are read as float4)
TABLE = {"q_f32": 4, "d_f32": 16, "doc_groups": 4, "out_scores": 4, "out_ids": 8, "out_groups": 8, "status": 4}
LIST_TABLE = {"offsets": 8, "ids": 4, "of_query": 4}


def _header_alignments(what):
    text = open(HEADER).read()
    m = re.search(rf"Alignment \(bytes\) of the {what}: (.*?)\*/", text, re.S)
    assert m, what
    return {name: int(n) for name, n in re.findall(r"(\w+) (\d+)", m.group(1))}


def test_alignment_tables_match_header():
    assert _header_alignments("vr_score_lists arguments") == TABLE
    assert _header_alignments("vr_doc_lists arrays") == LIST_TABLE


# ------------------------------------------------------------------------------------------------ C ABI refusals
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")
FAKE = 0x7F0000000000  # never dereferenced: every call below must stop in argument validation


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def _lists(offsets=FAKE + 0x1000, ids=FAKE + 0x2000, count=3, of_query=FAKE + 0x3000):
    ls = L.DocLists()
    ls.offsets, ls.ids, ls.count, ls.of_query = offsets, ids, count, of_query
    return ls


def _call(lib, lists="default", nq=40, nd=5000, dim=256, width=64, **over):
    p = {name: FAKE + 0x100000 * (i + 1) for i, name in enumerate(TABLE)}
    p.update(over)
    ls = _lists() if lists == "default" else lists
    return lib.vr_score_lists(p["q_f32"], nq, p["d_f32"], nd, dim, None if ls is None else C.byref(ls), width,
                              p["doc_groups"], p["out_scores"], p["out_ids"], p["out_groups"], p["status"], None)


BAD = {
    "lists NULL": (dict(lists=None), r"lists must not be NULL"),
    "offsets NULL": (dict(lists=_lists(offsets=None)), r"lists->offsets must not be NULL"),
    "ids NULL": (dict(lists=_lists(ids=None)), r"lists->ids must not be NULL"),
    "offsets misaligned": (dict(lists=_lists(offsets=FAKE + 0x1004)), r"lists->offsets must be 8-byte aligned"),
    "ids misaligned": (dict(lists=_lists(ids=FAKE + 0x2002)), r"lists->ids must be 4-byte aligned"),
    "of_query misaligned": (dict(lists=_lists(of_query=FAKE + 0x3002)), r"lists->of_query must be 4-byte aligned"),
    "count 0": (dict(lists=_lists(count=0)), r"lists->count=0"),
    "count -1": (dict(lists=_lists(count=-1)), r"lists->count=-1"),
    "count 2 without of_query": (dict(lists=_lists(count=2, of_query=None)), r"lists->of_query is NULL"),
    "width 0": (dict(width=0), r"width=0"),
    "width -3": (dict(width=-3), r"width=-3"),
    "dim 6": (dict(dim=6), r"dim=6"),
    "dim 0": (dict(dim=0), r"dim=0"),
    "nq 0": (dict(nq=0), r"nq=0"),
    "nd 2^31": (dict(nd=1 << 31), r"nd=2147483648"),
    "nd 0": (dict(nd=0), r"nd=0"),
    "q_f32 NULL": (dict(q_f32=None), r"null pointer"),
    "d_f32 NULL": (dict(d_f32=None), r"null pointer"),
    "out_scores NULL": (dict(out_scores=None), r"null pointer"),
    "out_ids NULL": (dict(out_ids=None), r"null pointer"),
    "status NULL": (dict(status=None), r"null pointer"),
    "doc_groups without out_groups": (dict(out_groups=None), r"doc_groups and out_groups"),
    "out_groups without doc_groups": (dict(doc_groups=None), r"doc_groups and out_groups"),
}


@no_device
@pytest.mark.parametrize("bad", sorted(BAD))
def test_score_lists_refuses_bad_arguments_before_any_cuda_call(lib, bad):
    kw, pattern = BAD[bad]
    rc = _call(lib, **kw)
    msg = lib.vr_last_error().decode()
    assert rc == 2, (rc, msg)
    assert "vr_score_lists" in msg and re.search(pattern, msg), msg


@no_device
@pytest.mark.parametrize("name", sorted(TABLE))
def test_score_lists_refuses_each_misaligned_pointer(lib, name):
    n = TABLE[name]
    rc = _call(lib, **{name: FAKE + 0x100000 * (list(TABLE).index(name) + 1) + (4 if n >= 8 else 2)})
    msg = lib.vr_last_error().decode()
    assert rc == 2 and re.search(rf"\b{name}\b must be {n}-byte aligned", msg), (rc, msg)


@no_device
def test_score_lists_accepts_valid_arguments(lib):
    """Shared (count 1, no of_query), per-row (count 3 with of_query), and no groups: past validation, a call without a
    device stops at its first CUDA call (status 1)."""
    for kw in (dict(lists=_lists(count=1, of_query=None)), dict(), dict(doc_groups=None, out_groups=None),
               dict(nd=(1 << 31) - 2, width=1)):
        rc = _call(lib, **kw)
        assert rc != 2, lib.vr_last_error().decode()


# ------------------------------------------------------------------------------------------------ Python refusals
def _cpu_index(nd=100, d=8):
    return R.CorpusIndex(torch.zeros((nd, d)), torch.zeros((nd, d), dtype=torch.float16), torch.zeros(1))


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"the library was reached ({name}) although the arguments are invalid")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(L, "_lib", _NoLib())


_OFF, _IDS = torch.tensor([0, 2, 5]), torch.tensor([1, 2, 3, 4, 99], dtype=torch.int32)


@pytest.mark.parametrize("doc_lists,list_of,nq,match", [
    ((_OFF,), None, 2, "pair"),
    ([_OFF, _IDS, _IDS], None, 2, "pair"),
    ((_OFF.float(), _IDS), None, 2, "doc_lists offsets must be an int32 or int64"),
    ((_OFF, _IDS.to(torch.int16)), None, 2, "doc_lists ids must be an int32 or int64"),
    ((_OFF.view(1, 3), _IDS), None, 2, "doc_lists offsets must have shape 1-D"),
    ((_OFF, _IDS.view(5, 1)), None, 2, "doc_lists ids must have shape 1-D"),
    ((torch.tensor([0]), _IDS[:0]), None, 2, "M \\+ 1 >= 2"),
    ((_OFF + 1, _IDS), None, 2, "must start at 0"),
    ((torch.tensor([0, 3, 2, 5]), _IDS), None, 3, "non-decreasing"),
    ((torch.tensor([0, 2, 4]), _IDS), None, 2, "must end at len\\(ids\\) = 5"),
    ((_OFF, torch.tensor([1, 2, 3, 4, 100])), None, 2, r"ids must lie in \[0, 100\)"),
    ((_OFF, torch.tensor([1, -1, 3, 4, 5])), None, 2, r"ids must lie in \[0, 100\)"),
    ((_OFF, _IDS), None, 3, "2 lists for 3 queries"),
    ((_OFF, _IDS), torch.tensor([0, 1]), 3, r"list_of must have shape \[3\]"),
    ((_OFF, _IDS), torch.tensor([0., 1., 1.]), 3, "list_of must be an int32 or int64"),
    ((_OFF, _IDS), [0, 1, 1], 3, "list_of must be an int32 or int64"),
    ((_OFF, _IDS), torch.tensor([0, 2, 1]), 3, r"list_of must lie in \[0, 2\)"),
    ((_OFF, _IDS), torch.tensor([0, -1, 1]), 3, r"list_of must lie in \[0, 2\)"),
])
def test_python_refuses_bad_lists(stub, doc_lists, list_of, nq, match):
    with pytest.raises(ValueError, match=match):
        R._check_doc_lists(doc_lists, _cpu_index(), nq, list_of)


def test_python_refuses_lists_with_masks_or_list_of_alone(stub):
    q, idx = torch.zeros((2, 8)), _cpu_index()
    m = torch.ones(100, dtype=torch.bool)
    for fn, extra in ((R.score_topk, ()), (R.score_topk_groups, (torch.zeros(100, dtype=torch.int32),))):
        with pytest.raises(ValueError, match="cannot be combined"):
            fn(q, idx, 5, *extra, doc_mask=m, doc_lists=(_OFF, _IDS))
        with pytest.raises(ValueError, match="cannot be combined"):
            fn(q, idx, 5, *extra, mask_of=torch.zeros(2, dtype=torch.int32), doc_lists=(_OFF, _IDS))
        with pytest.raises(ValueError, match="list_of needs doc_lists"):
            fn(q, idx, 5, *extra, list_of=torch.zeros(2, dtype=torch.int32))
    with pytest.raises(ValueError, match="CUDA tensor"):   # the queries are checked as in the masked calls
        R.score_topk(q, idx, 5, doc_lists=(_OFF, _IDS))


def test_python_list_set_defaults(stub):
    idx = _cpu_index()
    one = R._check_doc_lists((torch.tensor([0, 3]), torch.tensor([5, 5, 7])), idx, 4)
    assert one.of_query is None and one.width == 3 and not one.sort and one.ids.dtype == torch.int32
    per = R._check_doc_lists((_OFF, _IDS), idx, 2)
    assert per.of_query.tolist() == [0, 1] and per.width == 3 and not per.sort
    picked = R._check_doc_lists((_OFF, _IDS), idx, 3, torch.tensor([0, 0, 0]))
    assert picked.width == 2 and picked.sort            # the width is that of the lists the queries use
    empty = R._check_doc_lists((torch.tensor([0, 0]), torch.zeros(0, dtype=torch.int64)), idx, 2)
    assert empty.width == 1 and empty.ids.numel() == 1  # a valid pointer that is never read
    m, mo = picked.masks(100)
    assert m.shape == (2, 100) and m[0].nonzero().flatten().tolist() == [1, 2] and mo.tolist() == [0, 0, 0]


# ------------------------------------------------------------------------------------------------ selection model
def first_k_distinct(s, ids, k, key=None):
    """Entries in (score desc, id asc) order, skipping id < 0 and NaN; repeats of an emitted key are skipped (key = id for
    pages, the group for documents). Returns the emitted positions, padded to k with -1."""
    key = ids if key is None else key
    order = sorted((i for i in range(len(s)) if ids[i] >= 0 and not np.isnan(s[i])), key=lambda i: (-s[i], ids[i]))
    out, seen = [], set()
    for i in order:
        if key[i] in seen:
            continue
        seen.add(key[i])
        out.append(i)
        if len(out) == k:
            break
    return out + [-1] * (k - len(out))


def _pick(arrs, pos):
    return [np.array([a[p] if p >= 0 else f for p in pos], dtype=a.dtype) for a, f in zip(arrs, (-np.inf, -1, -1))]


def chunked_pages(s, ids, k, chunk):
    """The list path's page selection: padded to whole chunks, the top-k of each chunk, then the top-k of those."""
    w = -(-len(s) // chunk) * chunk
    s = np.concatenate([s, np.full(w - len(s), -np.inf, np.float32)])
    ids = np.concatenate([ids, np.full(w - len(ids), -1)])
    parts = [_pick((s[c:c + chunk], ids[c:c + chunk]), first_k_distinct(s[c:c + chunk], ids[c:c + chunk], k))
             for c in range(0, w, chunk)]
    s2, i2 = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    return _pick((s2, i2), first_k_distinct(s2, i2, k))


def chunked_groups(s, p, g, k, width=512, per_chunk=None):
    """The list path's document selection: [C, 512] merges repeated until a row fits 512, then the final merge.
    per_chunk: the mutant's per-chunk selection instead of the first k distinct groups."""
    per_chunk = per_chunk or (lambda s, p, g, k: first_k_distinct(s, p, k, g))
    while len(s) > width:
        w = -(-len(s) // width) * width
        s, p, g = (np.concatenate([a, np.full(w - len(a), f, a.dtype)]) for a, f in ((s, -np.inf), (p, -1), (g, -1)))
        parts = [_pick((s[c:c + width], p[c:c + width], g[c:c + width]),
                       per_chunk(s[c:c + width], p[c:c + width], g[c:c + width], k)) for c in range(0, w, width)]
        s, p, g = (np.concatenate([x[j] for x in parts]) for j in range(3))
    return _pick((s, p, g), first_k_distinct(s, p, k, g))


def direct_pages(s, ids, k):
    return _pick((s, ids), first_k_distinct(s, ids, k))


def direct_groups(s, p, g, k):
    """Each group's best listed page (max non-NaN score, lowest page on ties), groups by (score desc, best page asc)."""
    best = {}
    for i in range(len(s)):
        if p[i] < 0 or np.isnan(s[i]):
            continue
        b = best.get(g[i])
        if b is None or s[i] > s[b] or (s[i] == s[b] and p[i] < p[b]):
            best[g[i]] = i
    order = sorted(best.values(), key=lambda i: (-s[i], p[i]))[:k]
    return _pick((s, p, g), order + [-1] * (k - len(order)))


def _fixture(n, nd, seed, groups_of=lambda p: p // 7):
    """A list of n entries (unsorted, with repeats, coarse scores so that ties occur) and its scores, pages and groups."""
    rs = np.random.RandomState(seed)
    pages = rs.randint(0, nd, n)
    pages[rs.rand(n) < 0.1] = pages[0]                       # repeats
    score_of = np.round(rs.randn(nd), 1).astype(np.float32)  # one score per page, coarse: ties between pages
    score_of[rs.rand(nd) < 0.01] = np.nan
    return score_of[pages], pages.astype(np.int64), groups_of(pages).astype(np.int64)


@pytest.mark.parametrize("n,chunk", [(1, 4), (5, 4), (17, 4), (130, 32), (4097, 4096), (9000, 4096), (3000, 128)])
@pytest.mark.parametrize("k", [1, 3, 10, 50])
def test_chunked_page_selection_equals_a_direct_sort(n, chunk, k):
    s, p, _ = _fixture(n, 2000, n * 7 + k)
    for a, b in zip(chunked_pages(s, p, k, chunk), direct_pages(s, p, k)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("n,groups_of", [(1, lambda p: p // 7), (600, lambda p: p // 7), (1500, lambda p: p % 13),
                                         (5000, lambda p: p // 3), (20000, lambda p: (p * 7919) % 997),
                                         (3000, lambda p: p % 5)])
@pytest.mark.parametrize("k", [1, 10, 20, 256])
def test_chunked_group_selection_equals_a_direct_sort(n, groups_of, k):
    """Lists crossing chunk boundaries, documents spread over chunks, k above the groups present (p % 5, p % 13), and
    widths that take one, two and more merge levels (20 000 entries at k = 256: 40 chunks, then 20, 10, 5, 3, 2)."""
    s, p, g = _fixture(n, 8000, n + k, groups_of)
    got, want = chunked_groups(s, p, g, k), direct_groups(s, p, g, k)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert ((got[1] >= 0).sum() == min(k, len(set(g[~np.isnan(s)].tolist()))))


def test_first_k_pages_per_chunk_instead_of_groups_gives_a_wrong_document_topk():
    """Chunk 0 holds 600 high pages of document 0 and the best page of document 1 below them; chunk 1 holds document 2,
    lower still. The first 2 pages of chunk 0 are both document 0's, so the mutant loses document 1."""
    s = np.concatenate([np.linspace(2.0, 1.5, 511, dtype=np.float32), [1.0], np.full(600, 0.5, np.float32)])
    p = np.arange(len(s), dtype=np.int64)
    g = np.concatenate([np.zeros(511), [1], np.full(600, 2)]).astype(np.int64)
    pages_mutant = lambda s, p, g, k: first_k_distinct(s, p, k)  # noqa: E731
    want = direct_groups(s, p, g, 2)
    assert want[2].tolist() == [0, 1]
    assert np.array_equal(chunked_groups(s, p, g, 2)[2], want[2])
    assert chunked_groups(s, p, g, 2, per_chunk=pages_mutant)[2].tolist() == [0, 2]


# ------------------------------------------------------------------------------------------------ routing rule
def test_routing_rule_is_monotone_in_the_list_work():
    for nq, nd in ((1, 125_000), (1, 1_000_000), (10_000, 125_000), (300, 500_000)):
        picks = [KB.list_path_wins(r, nq, nd, 10, False) for r in range(0, 40 * nd, nd // 50)]
        assert picks[0] and not picks[-1]
        assert picks == sorted(picks, reverse=True)       # True ... True False ... False
    assert not KB.list_path_wins(0, 1, 125_000, 257, True) and KB.list_path_wins(0, 1, 125_000, 257, False)


BENCH = [  # (queries, index pages, list rows = scope pages x query tiles, lists measured faster)
    (1, 125_000, 8, True), (1, 125_000, 1000, True), (1, 125_000, 10_000, True), (1, 125_000, 50_000, False),
    (1, 1_000_000, 8, True), (1, 1_000_000, 50_000, True),
    (10_000, 125_000, 100 * 1250, True), (10_000, 125_000, 2000 * 1250, True), (10_000, 125_000, 20_000 * 1250, False),
    (10_000, 125_000, 8 * 10_000, True),
]


@pytest.mark.parametrize("nq,nd,rows,lists_faster", BENCH)
def test_routing_rule_picks_the_faster_path_on_the_measured_workloads(nq, nd, rows, lists_faster):
    assert KB.list_path_wins(rows, nq, nd, 10, False) == lists_faster
    assert KB.list_path_wins(rows, nq, nd, 10, True) == lists_faster


def test_measured_workloads_fall_on_both_sides():
    assert {b[3] for b in BENCH} == {True, False}
