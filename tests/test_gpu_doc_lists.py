"""Candidate lists on the GPU: every row of score_topk / score_topk_groups with doc_lists equals, bit for bit, the masked
call with a mask of exactly the listed pages, through the tensor-core filter and through the fp32 scan (force_exact).
List lengths 0, 1, 127-129, 511-513, 4097 and 20 000 cover every topk_rows kernel choice, the two-level page selection
and one and several levels of the document merge; lists are shared, per query, picked by list_of with repeats, unsorted
and with repeated ids. Also: batch composition, the knowledge base's routing in both directions, and sharded merges."""
import numpy as np
import pytest
import torch

from visrag_b200 import knowledge_base as KB
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu

ND = 30_000


def _unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn((n, d), device="cuda", generator=g), dim=1)


@pytest.fixture(scope="module")
def data():
    D = _unit(ND, 2304, 1)
    D[100] = D[200]          # equal rows: ties broken by id
    D[101] = D[200]
    D[300] = float("nan")   # non-finite rows
    D[301] = float("inf")
    D[302] = -float("inf")
    return D, R.build_index(D), _unit(64, 2304, 2)


def _csr(lists):
    offsets = torch.tensor(np.cumsum([0] + [len(x) for x in lists]), dtype=torch.int64, device="cuda")
    ids = torch.tensor([int(v) for x in lists for v in x], dtype=torch.int32, device="cuda")
    return offsets, ids


def _masks(lists, nd):
    m = torch.zeros((len(lists), nd), dtype=torch.bool, device="cuda")
    for r, x in enumerate(lists):
        if len(x):
            m[r, torch.as_tensor(np.asarray(x, dtype=np.int64), device="cuda")] = True
    return m


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(_bits(x), _bits(y)), (x, y)


def _mask_args(lists, list_of, nd):
    m = _masks(lists, nd)
    if list_of is None and len(lists) == 1:
        return m[0], None
    return m, list_of


def check_pages(Q, index, k, lists, list_of=None, id_offset=0):
    stats = {}
    got = R.score_topk(Q, index, k, id_offset, stats=stats, doc_lists=_csr(lists), list_of=list_of)
    assert stats["path"] == "lists"
    m, mo = _mask_args(lists, list_of, index.nd)
    for force in (True, False):
        _same(got, R.score_topk(Q, index, k, id_offset, force_exact=force, doc_mask=m, mask_of=mo))
    return got


def check_docs(Q, index, k, groups, lists, list_of=None, id_offset=0):
    stats = {}
    got = R.score_topk_groups(Q, index, k, groups, id_offset, stats=stats, doc_lists=_csr(lists), list_of=list_of)
    assert stats["path"] == ("lists" if k <= R.LIST_GROUPS_MAX_K else stats["path"])
    m, mo = _mask_args(lists, list_of, index.nd)
    for force in (True, False):
        _same(got, R.score_topk_groups(Q, index, k, groups, id_offset, force_exact=force, doc_mask=m, mask_of=mo))
    return got


LENGTHS = [0, 1, 127, 128, 129, 511, 512, 513, 4097, 20_000]


def _random_list(rs, n, nd=ND):
    return rs.choice(nd, n, replace=False) if n <= nd else rs.randint(0, nd, n)


@pytest.mark.parametrize("n", LENGTHS)
def test_one_query_shared_list_every_length(data, n):
    _, index, Q = data
    rs = np.random.RandomState(n)
    lst = _random_list(rs, n)
    for k in (1, 10, 200):
        check_pages(Q[:1], index, k, [lst])


def test_per_query_lists_of_every_length_in_one_call(data):
    _, index, Q = data
    rs = np.random.RandomState(5)
    lists = [_random_list(rs, n) for n in LENGTHS]
    check_pages(Q[:len(lists)], index, 10, lists)
    check_pages(Q[:len(lists)], index, 10, lists, id_offset=1_000_000)


def test_shared_lists_through_list_of_with_repeats(data):
    _, index, Q = data
    rs = np.random.RandomState(6)
    lists = [_random_list(rs, n) for n in (0, 3, 129, 600, 5000)]
    list_of = torch.tensor(rs.randint(0, len(lists), Q.shape[0]), dtype=torch.int64, device="cuda")
    check_pages(Q, index, 10, lists, list_of)
    check_pages(Q, index, 10, [lists[3]], torch.zeros(Q.shape[0], dtype=torch.int32, device="cuda"))
    check_pages(Q, index, 10, [lists[3]])   # one list for every query, no list_of


def test_unsorted_lists_with_repeated_ids_edges_ties_and_nonfinite_rows(data):
    _, index, Q = data
    rs = np.random.RandomState(7)
    base = np.concatenate([[0, ND - 1, 100, 101, 200, 300, 301, 302], _random_list(rs, 700)])
    lst = np.concatenate([base, base[::3], [0, 0, ND - 1]])
    rs.shuffle(lst)
    for k in (1, 5, 10, 1000):
        s, i = check_pages(Q[:9], index, k, [lst])
        for row in i.tolist():                       # a repeated id is returned once
            ids = [x for x in row if x >= 0]
            assert len(ids) == len(set(ids))
    # equal rows 100, 101, 200 rank by id whenever they are returned
    s, i = check_pages(Q[:1], index, 3, [[200, 101, 100, 200]])
    assert i[0].tolist()[:3] == [100, 101, 200] or s[0, 0] != s[0, 1]
    # the NaN row is never returned; +inf is first when present
    s, i = check_pages(Q[:1], index, 4, [[300, 301, 302, 5]])
    assert 300 not in i[0].tolist()


def test_k_larger_than_the_list_pads(data):
    _, index, Q = data
    s, i = check_pages(Q[:2], index, 20, [[5, 6, 7], []])
    assert (i[0, 3:] == -1).all() and (i[1] == -1).all() and torch.isinf(s[1]).all()


def test_small_dim(data):
    D, _, _ = data
    D64 = torch.nn.functional.normalize(D[:5000, :64].nan_to_num(0.0, 1.0, -1.0), dim=1).contiguous()
    index = R.build_index(D64)
    Q = _unit(20, 64, 9)
    rs = np.random.RandomState(8)
    lists = [rs.randint(0, 5000, n) for n in (1, 129, 513, 4097)]
    check_pages(Q[:4], index, 10, lists)
    check_pages(Q, index, 10, lists, torch.tensor(rs.randint(0, 4, 20), device="cuda"))
    groups = torch.tensor(np.arange(5000) // 7, dtype=torch.int32, device="cuda")
    check_docs(Q[:4], index, 10, groups, lists)


def _spread_groups(nd, seed):
    """Documents of 1-60 pages whose pages are spread over the whole index (so they cross every merge chunk)."""
    rs = np.random.RandomState(seed)
    g = np.repeat(np.arange(nd), rs.randint(1, 60, nd))[:nd]
    rs.shuffle(g)
    return torch.tensor(g, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("n", LENGTHS)
def test_documents_every_length(data, n):
    _, index, Q = data
    groups = _spread_groups(ND, 3)
    rs = np.random.RandomState(100 + n)
    lst = _random_list(rs, n)
    for k in (1, 10, 20, 256, 257):
        check_docs(Q[:2], index, k, groups, [lst])


def test_documents_per_query_partial_documents_and_list_of(data):
    _, index, Q = data
    groups = _spread_groups(ND, 4)
    rs = np.random.RandomState(12)
    lists = [_random_list(rs, n) for n in LENGTHS]
    check_docs(Q[:len(lists)], index, 10, groups, lists, id_offset=777)
    # documents with only some pages listed, unsorted with repeats, shared through list_of
    contig = torch.tensor(np.arange(ND) // 50, dtype=torch.int32, device="cuda")
    part = np.concatenate([np.arange(50 * d, 50 * d + 10) for d in range(0, 600, 3)])
    part = np.concatenate([part, part[:100], [0, ND - 1]])
    rs.shuffle(part)
    lists = [part, lists[8], [ND - 1, 0, 0]]
    list_of = torch.tensor(rs.randint(0, 3, Q.shape[0]), dtype=torch.int32, device="cuda")
    for k in (1, 10, 40, 256):
        check_docs(Q, index, k, contig, lists, list_of)


def test_rows_do_not_depend_on_batch_composition(data):
    _, index, Q = data
    rs = np.random.RandomState(13)
    lists = [_random_list(rs, n) for n in (7, 129, 513, 4097, 20_000, 1)]
    list_of = torch.tensor(rs.randint(0, len(lists), Q.shape[0]), dtype=torch.int32, device="cuda")
    groups = _spread_groups(ND, 5)
    csr = _csr(lists)
    full = R.score_topk(Q, index, 10, doc_lists=csr, list_of=list_of)
    fullg = R.score_topk_groups(Q, index, 10, groups, doc_lists=csr, list_of=list_of)
    perm = torch.tensor(rs.permutation(Q.shape[0]), device="cuda")
    _same([t[perm] for t in full], R.score_topk(Q[perm], index, 10, doc_lists=csr, list_of=list_of[perm]))
    _same([t[perm] for t in fullg], R.score_topk_groups(Q[perm], index, 10, groups, doc_lists=csr, list_of=list_of[perm]))
    for a, b in ((0, 1), (1, 9), (9, 40), (40, 64)):
        _same([t[a:b] for t in full], R.score_topk(Q[a:b], index, 10, doc_lists=csr, list_of=list_of[a:b]))
        _same([t[a:b] for t in fullg], R.score_topk_groups(Q[a:b], index, 10, groups, doc_lists=csr, list_of=list_of[a:b]))
    for r in (0, 17, 63):   # a row alone, with its own list only
        lone = (torch.tensor([0, len(lists[list_of[r]])], device="cuda"), csr[1][csr[0][list_of[r]]:csr[0][list_of[r] + 1]])
        _same([t[r:r + 1] for t in full], R.score_topk(Q[r:r + 1], index, 10, doc_lists=lone))


def test_sharded_merges_of_list_results(data):
    """Two shards of the index with lists in local ids: sharded_topk(_groups) outside torch.distributed equals
    score_topk(_groups), and merging the shards' results equals the search over the whole index."""
    D, index, Q = data
    rs = np.random.RandomState(14)
    lst = _random_list(rs, 3000)
    groups = _spread_groups(ND, 6)
    whole = R.score_topk(Q, index, 10, doc_lists=_csr([lst]))
    wholeg = R.score_topk_groups(Q, index, 10, groups, doc_lists=_csr([lst]))
    parts, partsg = [], []
    for lo, hi in (R.shard_range(ND, 0, 2), R.shard_range(ND, 1, 2)):
        shard = R.build_index(D[lo:hi].contiguous())
        local = [lst[(lst >= lo) & (lst < hi)] - lo]
        parts.append(R.sharded_topk(Q, shard, 10, lo, doc_lists=_csr(local)))
        _same(parts[-1], R.score_topk(Q, shard, 10, lo, doc_lists=_csr(local)))
        partsg.append(R.sharded_topk_groups(Q, shard, 10, groups[lo:hi].contiguous(), lo, doc_lists=_csr(local)))
    _same(whole, R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1), 10))
    _same(wholeg, R.merge_topk_groups(*[torch.cat([p[j] for p in partsg], 1) for j in range(3)], 10))


# ------------------------------------------------------------------------------------------------ knowledge base
def _kb(tmp_path):
    rs = np.random.RandomState(15)
    n = 3000
    reps = rs.randn(n, 256).astype(np.float32)
    reps /= np.linalg.norm(reps, axis=1, keepdims=True)
    names = [f"doc{i // 20}.pdf_{i % 20}.png" for i in range(n)]
    KB.save_knowledge_base(str(tmp_path), reps, names)
    kb = KB.KnowledgeBase(str(tmp_path))
    kb.remove(names[5:40] + names[700:705])
    extra = rs.randn(50, 256).astype(np.float32)
    kb.add(extra / np.linalg.norm(extra, axis=1, keepdims=True), [f"new.pdf_{i}.png" for i in range(50)])
    return kb, names


def test_knowledge_base_gives_the_same_bits_routed_either_way(tmp_path, monkeypatch):
    kb, names = _kb(tmp_path)
    rs = np.random.RandomState(16)
    Q = rs.randn(40, 256).astype(np.float32)
    small = names[:5] + names[40:95] + ["new.pdf_3.png", "new.pdf_49.png"]   # live pages only
    each = [None if i % 7 == 0 else [names[j] for j in rs.choice(np.r_[40:700, 705:3000], rs.randint(1, 90), replace=False)]
            + ([f"new.pdf_{i}.png"] if i % 3 == 0 else []) for i in range(40)]
    each[5] = each[4]
    calls = [lambda: kb.search(Q, 10, within=small), lambda: kb.search(Q[:1], 300, within=small),
             lambda: kb.search(Q, 10, within_each=each), lambda: kb.search(Q[:3], 25, within_each=[small, None, small[:2]]),
             lambda: kb.search_documents(Q, 5, within=small), lambda: kb.search_documents(Q, 5, within_each=each),
             lambda: kb.search_documents(Q[:2], 300, within_each=[small, None])]
    results = {}
    for route, want in ((0.0, False), (1e12, True)):
        monkeypatch.setattr(KB, "LIST_ROUTE", route)
        seen = []
        orig = KB.list_path_wins
        monkeypatch.setattr(KB, "list_path_wins", lambda *a: seen.append(orig(*a)) or seen[-1])
        results[route] = [c() for c in calls]
        assert seen and any(v == want for v in seen)
        monkeypatch.setattr(KB, "list_path_wins", orig)
    for a, b in zip(results[0.0], results[1e12]):
        _same(a[:2], b[:2])
        if len(a) == 3:
            assert a[2] == b[2]
    removed = {kb.filenames.index(n) for n in names[5:40]}
    for s, i, *_ in results[1e12]:
        assert not removed & set(i.flatten().tolist())
