"""Document range search and deep document top-k on the GPU, bit for bit against a reference built from the library's
fp32 scan (vr_score_exact) with torch: each row's eligible, non-NaN pages ordered by (score desc, page asc), the first
page of each document in that order (its best page, with its own bits), then s >= t (range) or the first k (top-k)."""
import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import knowledge_base as KB
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu

DIM = 64


def _exact(q, index):
    s = torch.empty((q.shape[0], index.nd), dtype=torch.float32, device=q.device)
    L.check(L.lib().vr_score_exact(q.data_ptr(), q.shape[0], index.emb.data_ptr(), index.nd, q.shape[1], s.data_ptr(),
                                   L.stream_ptr()))
    return s


def _doc_rows(s, groups, mask=None, mask_of=None):
    """Per row: (scores, best pages, groups) of every document with an eligible page, by (score desc, best page asc)."""
    out = []
    for r in range(s.shape[0]):
        keep = ~torch.isnan(s[r])
        if mask is not None:
            keep &= mask if mask.dim() == 1 else mask[r if mask_of is None else int(mask_of[r])]
        pages = torch.nonzero(keep).flatten()
        v = s[r, pages]
        o = torch.sort(v, descending=True, stable=True).indices  # pages ascend: equal scores (+0, -0) keep the lower page
        v, pages = v[o], pages[o]
        g = groups[pages].long()
        first = torch.full((int(groups.max()) + 1,), 1 << 40, dtype=torch.int64, device=s.device)
        pos = torch.arange(g.numel(), device=s.device)
        first.scatter_reduce_(0, g, pos, "amin")
        sel = first[g] == pos
        out.append((v[sel], pages[sel], g[sel]))
    return out


def _range_ref(rows, t, id_offset=0):
    t = t.tolist() if isinstance(t, torch.Tensor) else [float(t)] * len(rows)
    offs, ss, pp, gg = [0], [], [], []
    for (v, p, g), tr in zip(rows, t):
        keep = v >= tr
        ss.append(v[keep])
        pp.append(p[keep] + id_offset)
        gg.append(g[keep])
        offs.append(offs[-1] + int(keep.sum()))
    dev = rows[0][0].device
    return torch.tensor(offs, dtype=torch.int64, device=dev), torch.cat(ss), torch.cat(pp), torch.cat(gg)


def _topk_ref(rows, k, id_offset=0):
    dev = rows[0][0].device
    s = torch.full((len(rows), k), float("-inf"), device=dev)
    p = torch.full((len(rows), k), -1, dtype=torch.int64, device=dev)
    g = p.clone()
    for r, (v, pg, gr) in enumerate(rows):
        n = min(k, v.numel())
        s[r, :n], p[r, :n], g[r, :n] = v[:n], pg[:n] + id_offset, gr[:n]
    return s, p, g


def _same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape, (what, i, x.dtype, y.dtype, x.shape, y.shape)
        assert torch.equal(x, y), (what, i, int((x != y).sum()) if x.shape == y.shape else None)


def _corpus(kind, nd, pages, seed, nq):
    """Unit pages in documents of `pages` pages: random, or clustered (the pages of a document near one centre, and
    queries near some documents). Groups are sparse: document j has id 3 j."""
    g = torch.Generator().manual_seed(seed)
    n_docs = -(-nd // pages)
    if kind == "random":
        d = torch.randn((nd, DIM), generator=g)
        q = torch.randn((nq, DIM), generator=g)
    else:
        centres = torch.randn((n_docs, DIM), generator=g)
        d = centres.repeat_interleave(pages, 0)[:nd] + 0.3 * torch.randn((nd, DIM), generator=g)
        q = centres[torch.randint(0, n_docs, (nq,), generator=g)] + 0.5 * torch.randn((nq, DIM), generator=g)
    d /= d.norm(dim=1, keepdim=True)
    q /= q.norm(dim=1, keepdim=True)
    groups = (torch.arange(nd) // pages) * 3
    return q.cuda(), d.cuda(), groups.to(torch.int32).cuda()


def _kth_doc_scores(rows, n):
    return torch.stack([v[min(n, v.numel()) - 1] if v.numel() else torch.tensor(1.0, device=v.device) for v, _, _ in rows])


@pytest.mark.parametrize("nq", [1, 300, 2000])
@pytest.mark.parametrize("kind,pages", [("random", 1), ("random", 8), ("clustered", 8), ("clustered", 64)])
def test_score_range_groups_equals_the_scan(nq, kind, pages):
    q, d, groups = _corpus(kind, 30_000, pages, 10 + pages, nq)
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    for name, t in (("none", 1.5), ("few", _kth_doc_scores(rows, 5)), ("thousands", _kth_doc_scores(rows, 2000))):
        stats = {}
        got = R.score_range_groups(q, index, t, groups, stats=stats)
        want = _range_ref(rows, t)
        _same(got, want, (kind, pages, nq, name))
        assert stats["documents"] == want[1].numel()
        assert stats["path"] == ("exact" if nq * index.nd <= R.SMALL_PROBLEM else "filter+rescore")
    t = _kth_doc_scores(rows, 50)
    _same(R.score_range_groups(q, index, t, groups, force_exact=True, id_offset=7), _range_ref(rows, t, 7), "force_exact")


def test_masks_per_query_masks_id_offset_and_a_small_cap():
    q, d, groups = _corpus("clustered", 40_000, 8, 3, 400)
    index = R.build_index(d)
    s = _exact(q, index)
    gen = torch.Generator(device="cuda").manual_seed(4)
    mask = torch.rand(index.nd, generator=gen, device="cuda") < 0.6
    t = float(s.flatten().kthvalue(s.numel() - 50 * q.shape[0]).values)
    rows = _doc_rows(s, groups, mask)
    _same(R.score_range_groups(q, index, t, groups, doc_mask=mask, id_offset=11), _range_ref(rows, t, 11), "1-D mask")
    masks = torch.rand((5, index.nd), generator=gen, device="cuda") < 0.5
    of = torch.randint(0, 5, (q.shape[0],), generator=gen, device="cuda")
    rows = _doc_rows(s, groups, masks, of)
    want = _range_ref(rows, t)
    _same(R.score_range_groups(q, index, t, groups, doc_mask=masks, mask_of=of), want, "per-query masks")
    stats = {}
    _same(R.score_range_groups(q, index, t, groups, doc_mask=masks, mask_of=of, cap=40, stats=stats), want, "cap 40")
    assert stats["path"] == "filter+rescore" and stats["fallback"] > 0, stats


def test_sparse_groups_beyond_nd_duplicates_and_zero_ties():
    """G > nd (global ids on a shard), planted duplicate pages inside and across documents, and two pages of one
    document scoring exactly 0 for every query: ties go to the lower page. (-0 scores are covered by the kernel test.)"""
    q, d, _ = _corpus("random", 20_000, 1, 5, 300)
    d[100:110] = d[5]                            # duplicates: documents of several equal pages
    d[200] = 0.0
    d[201] = 0.0
    index = R.build_index(d)
    groups = torch.arange(index.nd, device="cuda", dtype=torch.int32) // 4 * 1000 + 999   # G ~ 5 M > nd
    groups[201] = groups[300] = groups[200] + 1000 * 9000  # one document of pages 200 (0, G-local tie), 201 and 300
    groups[200] = groups[201]
    s = _exact(q, index)
    rows = _doc_rows(s, groups)
    for t in (0.0, float("-inf"), -0.05):
        got = R.score_range_groups(q, index, t, groups)
        _same(got, _range_ref(rows, t), f"t={t}")
        assert not (got[2] == 201).any()


def test_nan_pages_never_qualify():
    q, d, groups = _corpus("random", 20_000, 4, 6, 300)
    d[40] = float("nan")
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    for t in (float("-inf"), 0.1):
        got = R.score_range_groups(q, index, t, groups)
        _same(got, _range_ref(rows, t), t)
        assert not torch.isnan(got[1]).any()


def _region_groups(rs, ri, counts, most, groups, G):
    lib = L.lib()
    n, pitch = rs.shape
    gs, gi = torch.empty_like(rs), torch.empty_like(ri)
    gc = torch.empty(n, dtype=torch.int32, device=rs.device)
    wsb = lib.vr_range_groups_ws_bytes(n, most)
    ws = torch.empty(max(wsb // 8, 1), dtype=torch.int64, device=rs.device)
    L.check(lib.vr_range_groups(rs.data_ptr(), ri.data_ptr(), pitch, counts.data_ptr(), n, most, groups.data_ptr(),
                                groups.shape[0], G, ws.data_ptr(), wsb, gs.data_ptr(), gi.data_ptr(), gc.data_ptr(),
                                L.stream_ptr()))
    return gs, gi, gc


@pytest.mark.parametrize("most", [100, 4096, 4097, 20_000])
def test_kernel_on_shuffled_regions_in_and_beyond_shared_memory(most):
    """The kernel alone: rows of shuffled (score, page) entries with many ties, ±0 and entries past the count; its
    output set equals the per-document first entry."""
    gen = torch.Generator(device="cuda").manual_seed(most)
    n, nd, pitch = 40, 50_000, most + 7
    groups = torch.randint(0, 700, (nd,), generator=gen, device="cuda", dtype=torch.int32)
    counts = torch.randint(0, most + 1, (n,), generator=gen, device="cuda", dtype=torch.int32)
    counts[0] = most
    ri = torch.stack([torch.randperm(nd, generator=gen, device="cuda")[:pitch] for _ in range(n)]).to(torch.int32)
    rs = torch.randint(-3, 4, (n, pitch), generator=gen, device="cuda").float() / 4
    rs[rs == 0] = torch.where(torch.rand(int((rs == 0).sum()), generator=gen, device="cuda") < 0.5, 0.0, -0.0)
    gs, gi, gc = _region_groups(rs, ri, counts, most, groups, 700)
    for r in range(n):
        c = int(counts[r])
        v, p = rs[r, :c], ri[r, :c].long()
        o = torch.argsort(p)
        v, p = v[o], p[o]
        o = torch.sort(v, descending=True, stable=True).indices
        v, p = v[o], p[o]
        g = groups[p].long()
        first = torch.full((700,), 1 << 40, dtype=torch.int64, device="cuda")
        pos = torch.arange(g.numel(), device="cuda")
        first.scatter_reduce_(0, g, pos, "amin")
        sel = first[g] == pos
        want = sorted(zip(p[sel].tolist(), v[sel].view(torch.int32).tolist()))
        m = int(gc[r])
        got = sorted(zip(gi[r, :m].long().tolist(), gs[r, :m].view(torch.int32).tolist()))
        assert got == want, r


def test_every_page_of_300k_at_minus_infinity():
    q, d, groups = _corpus("clustered", 300_000, 8, 7, 2)
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    _same(R.score_range_groups(q, index, float("-inf"), groups), _range_ref(rows, float("-inf")), "t = -inf")


# ------------------------------------------------------------------------------------------------ deep document top-k
def _expected_path(k):
    return "deep" if R.DEEP_K_MIN < k <= R.DEEP_K_MAX else "filter+rescore"


@pytest.mark.parametrize("kind,pages", [("random", 1), ("random", 8), ("clustered", 8), ("clustered", 64)])
def test_score_topk_groups_deep_equals_the_scan(kind, pages):
    q, d, groups = _corpus(kind, 40_000, pages, 20 + pages, 300)
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    for k in (17, 64, 100, 1000, 4096):
        stats = {}
        got = R.score_topk_groups(q, index, k, groups, id_offset=5, stats=stats)
        _same(got, _topk_ref(rows, k, 5), (kind, pages, k))
        assert stats["path"] == _expected_path(k), (k, stats)
        if stats["path"] == "deep":
            assert stats["sample_stride"] == k // 8, stats
    exact = R.score_topk_groups(q, index, 100, groups, force_exact=True)
    _same(exact, _topk_ref(rows, 100), "scan at k = 100")


def test_deep_masks_lists_and_k_beyond_the_documents():
    q, d, groups = _corpus("clustered", 40_000, 8, 30, 300)
    index = R.build_index(d)
    s = _exact(q, index)
    gen = torch.Generator(device="cuda").manual_seed(31)
    mask = torch.rand(index.nd, generator=gen, device="cuda") < 0.5
    masks = torch.rand((4, index.nd), generator=gen, device="cuda") < 0.7
    of = torch.randint(0, 4, (q.shape[0],), generator=gen, device="cuda")
    for k in (100, 1000):
        _same(R.score_topk_groups(q, index, k, groups, doc_mask=mask), _topk_ref(_doc_rows(s, groups, mask), k), ("mask", k))
        _same(R.score_topk_groups(q, index, k, groups, doc_mask=masks, mask_of=of),
              _topk_ref(_doc_rows(s, groups, masks, of), k), ("per-query masks", k))
    lists = [torch.nonzero(masks[m]).flatten() for m in range(4)]
    offs = torch.tensor([0] + np.cumsum([x.numel() for x in lists]).tolist(), device="cuda")
    got = R.score_topk_groups(q, index, 600, groups, doc_lists=(offs, torch.cat(lists)), list_of=of)
    _same(got, _topk_ref(_doc_rows(s, groups, masks, of), 600), "lists, k = 600")
    few = torch.zeros(index.nd, dtype=torch.bool, device="cuda")
    few[:2000] = True  # 250 documents, k = 1000
    stats = {}
    _same(R.score_topk_groups(q, index, 1000, groups, doc_mask=few, stats=stats), _topk_ref(_doc_rows(s, groups, few), 1000),
          "k beyond the documents")
    assert stats["path"] == "deep" and stats["fallback"] == q.shape[0], stats


def test_misleading_sample_falls_back():
    """The sampled documents (group ids divisible by k // 8 = 50 at k = 400) score far above the rest for the first 30
    queries: their threshold keeps fewer than k documents, and those rows rerun through the scan."""
    q, d, groups = _corpus("random", 40_000, 4, 40, 400)
    sampled = groups % 50 == 0
    d[sampled] = q[:30].repeat(int(sampled.sum()) // 30 + 1, 1)[:int(sampled.sum())]
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    stats = {}
    got = R.score_topk_groups(q, index, 400, groups, stats=stats)
    _same(got, _topk_ref(rows, 400), "misleading sample")
    assert stats["path"] == "deep" and stats["fallback"] >= 1, stats


def test_row_alone_equals_its_row_in_the_batch():
    q, d, groups = _corpus("clustered", 40_000, 8, 50, 300)
    index = R.build_index(d)
    for k in (100, 1000):
        batch = R.score_topk_groups(q, index, k, groups)
        for r in (0, 150, 299):
            _same(R.score_topk_groups(q[r:r + 1], index, k, groups), tuple(x[r:r + 1] for x in batch), (k, r))


def test_capped_and_inner_hits_at_k_100():
    q, d, groups = _corpus("clustered", 40_000, 8, 60, 300)
    index = R.build_index(d)
    k, m = 100, 3
    hits = R.score_topk_groups_pages(q, index, k, groups, m)
    want = R.score_topk_groups_pages(q, index, k, groups, m, force_exact=True)
    _same(hits, want, "inner hits")
    _same(R.score_topk_capped(q, index, k, groups, m), R.score_topk_capped(q, index, k, groups, m, force_exact=True), "capped")
    _same(hits[:3], _topk_ref(_doc_rows(_exact(q, index), groups), k), "documents of the inner hits")


def test_group_topk_rows_select_plain_and_chunked():
    """vr_group_topk_rows at k > 32 (the radix select over the group rows): the chunked form (3 queries over 100 k
    documents) and the plain form (100 queries), against the reference."""
    q, d, groups = _corpus("random", 200_000, 2, 70, 100)
    index = R.build_index(d)
    rows = _doc_rows(_exact(q, index), groups)
    for k in (33, 100, 4096):
        _same(R.score_topk_groups(q[:3], index, k, groups), _topk_ref(rows[:3], k), ("chunked", k))
        _same(R.score_topk_groups(q, index, k, groups, force_exact=True, id_offset=9), _topk_ref(rows, k, 9), ("plain", k))


# ------------------------------------------------------------------------------------------------ knowledge base
def test_search_documents_above(tmp_path):
    rs = np.random.RandomState(80)
    names = [f"doc{j}.pdf_{i}.png" for j in range(300) for i in range(rs.randint(1, 6))] + [f"loose{i}.png" for i in range(50)]
    reps = rs.randn(len(names), DIM).astype(np.float32)
    reps /= np.linalg.norm(reps, axis=1, keepdims=True)
    KB.save_knowledge_base(str(tmp_path), reps, names)
    kb = KB.KnowledgeBase(str(tmp_path))
    q = torch.from_numpy(reps[rs.randint(0, len(names), 20)] + 0.3 * rs.randn(20, DIM).astype(np.float32)).cuda()
    q /= q.norm(dim=1, keepdim=True)
    kb.remove(names[3:40])
    new = rs.randn(30, DIM).astype(np.float32)
    kb.add(new / np.linalg.norm(new, axis=1, keepdims=True), [f"doc7.pdf_{100 + i}.png" for i in range(15)] +
           [f"fresh.pdf_{i}.png" for i in range(15)])
    within = names[100:400]
    each = [None if i % 3 == 0 else names[40 + 10 * i:240 + 10 * i] for i in range(20)]
    for kw, mask, mask_of in ((dict(), kb._live, None),
                              (dict(within=within), kb._scope_masks([kb._rows(within)])[0], None),
                              (dict(within_each=each), kb._scope_masks([None if s is None else kb._rows(s) for s in each]),
                               torch.arange(20, dtype=torch.int32, device="cuda"))):
        off, s, p, got_names = kb.search_documents_above(q, 0.2, **kw)
        want = R.score_range_groups(q, kb.index, 0.2, kb._doc_groups, doc_mask=mask, mask_of=mask_of)
        _same((off, s, p), want[:3], kw.keys())
        groups = want[3].tolist()
        o = off.tolist()
        assert got_names == [[kb.documents[g] for g in groups[a:b]] for a, b in zip(o[:-1], o[1:])]
        assert off[-1] > 0 and not any(kb._live[p].logical_not().tolist())
