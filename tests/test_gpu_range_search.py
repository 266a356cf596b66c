"""Range search on the GPU: score_range, KnowledgeBase.search_above and KnowledgeBase.near_duplicates against the fp32
scan, bit for bit. The reference is the library's fp32 scan (vr_score_exact, whose bits every path must carry) filtered
by s >= t and ordered by (score desc, id asc) with torch; it is also checked against float64 away from the threshold."""
import os

import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import knowledge_base as KB
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu

DIM = 256


def _corpus(nd, seed, dups=True, dim=DIM):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn((nd, dim), generator=g)
    d /= d.norm(dim=1, keepdim=True)
    if dups:  # exact ties: repeated rows
        d[7::97] = d[3]
    return d.cuda()


def _queries(nq, seed, docs=None, dim=DIM):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((nq, dim), generator=g)
    if docs is not None:  # queries near some docs: a few high scores per query
        q = docs[torch.randint(0, docs.shape[0], (nq,), generator=g)].cpu() + 0.3 * q / q.norm(dim=1, keepdim=True)
    q /= q.norm(dim=1, keepdim=True)
    return q.cuda()


def exact_scores(q, index):
    s = torch.empty((q.shape[0], index.nd), dtype=torch.float32, device=q.device)
    L.check(L.lib().vr_score_exact(q.data_ptr(), q.shape[0], index.emb.data_ptr(), index.nd, q.shape[1], s.data_ptr(),
                                   L.stream_ptr()))
    return s


def reference(q, index, t, mask=None, id_offset=0):
    """CSR of the fp32 scan's rows filtered by s >= t (and the mask), by (score desc, id asc)."""
    s = exact_scores(q, index)
    t = t if isinstance(t, torch.Tensor) else torch.full((q.shape[0],), float(t), device=q.device)
    keep = s >= t[:, None]
    if mask is not None:
        keep &= mask if mask.dim() == 2 else mask[None, :]
    offs, ss, ii = [0], [], []
    for r in range(q.shape[0]):
        idx = torch.nonzero(keep[r]).flatten()
        v = s[r, idx]
        o = torch.sort(v, descending=True, stable=True).indices  # ids ascend, so equal scores keep the lower id first
        ss.append(v[o])
        ii.append(idx[o] + id_offset)
        offs.append(offs[-1] + idx.numel())
    return (torch.tensor(offs, dtype=torch.int64, device=q.device), torch.cat(ss), torch.cat(ii))


def assert_same(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and torch.equal(x, y)


def thresholds_keeping(q, index, n):
    """Per-query thresholds that keep about n docs each (the n-th exact score of each row)."""
    s = exact_scores(q, index)
    return torch.topk(s, n, dim=1).values[:, -1].contiguous()


@pytest.mark.parametrize("nq", [1, 37, 300, 2000])
@pytest.mark.parametrize("keep", ["none", "few", "thousands"])
def test_score_range_equals_the_scan(nq, keep):
    nd = 70_000 if nq < 2000 else 30_000   # several waves of the filter's work items
    docs = _corpus(nd, 1)
    index = R.build_index(docs)
    q = _queries(nq, 2, docs)
    t = {"none": 1.5, "few": None, "thousands": None}[keep]
    if keep == "few":
        t = thresholds_keeping(q, index, 5)
    elif keep == "thousands":
        t = thresholds_keeping(q, index, 2500)
    stats = {}
    got = R.score_range(q, index, t, id_offset=11, stats=stats)
    assert stats["path"] == "filter+rescore" or nq * nd <= R.SMALL_PROBLEM
    assert_same(got, R.score_range(q, index, t, id_offset=11, force_exact=True))
    assert_same(got, reference(q, index, t, id_offset=11))
    if keep == "none":
        assert got[1].numel() == 0
    if keep == "few":
        assert stats.get("fallback", 0) == 0


def test_minus_inf_sorts_every_page_and_plus_inf_returns_nothing():
    nd = 120_000
    docs = _corpus(nd, 3)
    index = R.build_index(docs)
    q = _queries(40, 4)
    stats = {}
    got = R.score_range(q, index, float("-inf"), stats=stats)
    assert stats["path"] == "filter+rescore" and stats["fallback"] == 40  # every row overflows into the scan
    assert torch.equal(got[0], torch.arange(41, device="cuda") * nd)
    assert_same(got, reference(q, index, float("-inf")))
    one = R.score_range(q[:1], index, float("-inf"))  # a small problem: the scan path, one row of 120 k
    assert_same(one, reference(q[:1], index, float("-inf")))
    none = R.score_range(q, index, float("inf"))
    assert torch.equal(none[0], torch.zeros(41, dtype=torch.int64, device="cuda")) and none[1].numel() == 0


def test_masks_and_per_query_thresholds():
    nd, nq = 50_000, 300
    docs = _corpus(nd, 5)
    index = R.build_index(docs)
    q = _queries(nq, 6, docs)
    t = thresholds_keeping(q, index, 40)
    g = torch.Generator(device="cuda").manual_seed(7)
    m1 = torch.rand(nd, generator=g, device="cuda") < 0.3
    got = R.score_range(q, index, t, doc_mask=m1)
    assert_same(got, R.score_range(q, index, t, doc_mask=m1, force_exact=True))
    assert_same(got, reference(q, index, t, m1))
    sets = torch.rand((5, nd), generator=g, device="cuda") < torch.tensor([0.01, 0.1, 0.5, 0.9, 1.0], device="cuda")[:, None]
    of = torch.randint(0, 5, (nq,), generator=g, device="cuda")
    got = R.score_range(q, index, t, doc_mask=sets, mask_of=of)
    assert_same(got, R.score_range(q, index, t, doc_mask=sets, mask_of=of, force_exact=True))
    assert_same(got, reference(q, index, t, sets[of]))


def test_small_capacity_overflows_and_gives_the_same_bits():
    nd, nq = 60_000, 200
    docs = _corpus(nd, 8)
    index = R.build_index(docs)
    q = _queries(nq, 9, docs)
    t = thresholds_keeping(q, index, 30)
    t[::3] = thresholds_keeping(q[::3], index, 600)
    small, big = {}, {}
    a = R.score_range(q, index, t, cap=64, stats=small)
    b = R.score_range(q, index, t, cap=8192, stats=big)
    assert small["fallback"] > 0 and big["fallback"] == 0
    assert_same(a, b)
    assert_same(a, reference(q, index, t))


def test_clustered_corpus_needs_no_fallback():
    """Tight clusters (the layout that flags top-k queries: many near-equal scores) are exact by the margin alone."""
    g = torch.Generator().manual_seed(10)
    centers = torch.randn((50, DIM), generator=g)
    docs = centers[torch.randint(0, 50, (40_000,), generator=g)] + 1e-3 * torch.randn((40_000, DIM), generator=g)
    docs = (docs / docs.norm(dim=1, keepdim=True)).cuda()
    index = R.build_index(docs)
    q = centers[torch.randint(0, 50, (300,), generator=g)]
    q = (q / q.norm(dim=1, keepdim=True)).cuda()
    t = thresholds_keeping(q, index, 300)
    stats = {}
    got = R.score_range(q, index, t, stats=stats)
    assert stats["path"] == "filter+rescore" and stats["fallback"] == 0
    assert_same(got, reference(q, index, t))


def test_query_norm_beyond_fp16_takes_the_scan():
    nd = 40_000
    docs = _corpus(nd, 11)
    index = R.build_index(docs)
    q = _queries(200, 12, docs)
    q[5] *= 70_000.0  # |q| >= 65504: the fp16 copy overflows, no bound
    t = thresholds_keeping(q, index, 20)
    stats = {}
    got = R.score_range(q, index, t, stats=stats)
    assert stats["fallback"] == 1
    assert_same(got, reference(q, index, t))


def test_results_do_not_depend_on_the_batch():
    nd = 50_000
    docs = _corpus(nd, 13)
    index = R.build_index(docs)
    q = _queries(100, 14, docs)
    t = thresholds_keeping(q, index, 25)
    off, s, i = R.score_range(q, index, t)
    for r in (0, 41, 99):
        o1, s1, i1 = R.score_range(q[r:r + 1].clone(), index, t[r:r + 1].clone())
        assert torch.equal(s1, s[off[r]:off[r + 1]]) and torch.equal(i1, i[off[r]:off[r + 1]])


def test_scores_agree_with_float64_away_from_the_threshold():
    nd = 50_000
    docs = _corpus(nd, 15, dups=False)
    index = R.build_index(docs)
    q = _queries(60, 16, docs)
    t = 0.25
    off, s, i = R.score_range(q, index, t)
    s64 = q.double() @ docs.double().T
    for r in range(q.shape[0]):
        got = set(i[off[r]:off[r + 1]].tolist())
        sure = set(torch.nonzero(s64[r] >= t + 1e-6).flatten().tolist())
        maybe = set(torch.nonzero(s64[r] >= t - 1e-6).flatten().tolist())
        assert sure <= got <= maybe


# ------------------------------------------------------------------------------------------------ knowledge base
def _kb(tmp_path, n=30_000, seed=17):
    docs = _corpus(n, seed).cpu().numpy()
    names = [f"doc{j // 10}.pdf_{j % 10}.png" for j in range(n)]
    KB.save_knowledge_base(str(tmp_path), docs, names)
    return KB.KnowledgeBase(str(tmp_path)), docs, names


def test_search_above_matches_score_range(tmp_path):
    kb, docs, names = _kb(tmp_path)
    q = _queries(150, 18, torch.from_numpy(docs).cuda())
    t = thresholds_keeping(q, kb.index, 12)
    assert_same(kb.search_above(q, t), R.score_range(q, kb.index, t))
    within = names[100:5000]
    m = torch.zeros(kb.index.nd, dtype=torch.bool, device="cuda")
    m[100:5000] = True
    assert_same(kb.search_above(q, t, within=within), R.score_range(q, kb.index, t, doc_mask=m))
    each = [names[j * 100:j * 100 + 3000] if j % 3 else None for j in range(150)]
    got = kb.search_above(q, t, within_each=each)
    ar = torch.arange(kb.index.nd, device="cuda")
    masks = torch.stack([(ar >= j * 100) & (ar < j * 100 + 3000) if j % 3 else torch.ones_like(m) for j in range(150)])
    assert_same(got, reference(q, kb.index, t, masks))
    kb.remove(names[:2000])
    alive = torch.ones_like(m)
    alive[:2000] = False
    got = kb.search_above(q, t)
    assert_same(got, reference(q, kb.index, t, alive))
    assert not (got[2] < 2000).any()
    extra = _corpus(500, 19).cpu().numpy()
    kb.add(extra, [f"new{j}.png" for j in range(500)])
    alive = torch.cat([alive, torch.ones(500, dtype=torch.bool, device="cuda")])
    assert_same(kb.search_above(q, t), reference(q, kb.index, t, alive))
    kb.save(str(tmp_path / "saved"))
    kb2 = KB.KnowledgeBase(str(tmp_path / "saved"))
    o1, s1, i1 = kb.search_above(q, t)
    o2, s2, i2 = kb2.search_above(q, t)
    live = torch.nonzero(alive).flatten()
    assert torch.equal(o1, o2) and torch.equal(s1, s2) and torch.equal(live[i2], i1)


def test_near_duplicates(tmp_path):
    n = 20_000
    g = torch.Generator().manual_seed(20)
    docs = torch.randn((n, DIM), generator=g)
    for c in range(40):  # planted clusters of near-identical pages
        members = torch.randint(0, n, (5,), generator=g)
        docs[members] = docs[members[0]] + 0.02 * torch.randn((5, DIM), generator=g)
    docs[100] = docs[200]  # an exact duplicate
    docs = docs / docs.norm(dim=1, keepdim=True)
    names = [f"p{j}.png" for j in range(n)]
    KB.save_knowledge_base(str(tmp_path), docs.numpy(), names)
    kb = KB.KnowledgeBase(str(tmp_path))
    t = 0.99
    a, b, s = kb.near_duplicates(t)
    assert a.numel() > 40 and bool((a < b).all())
    S = exact_scores(kb.index.emb, kb.index)
    assert torch.equal(S.view(torch.int32), S.T.contiguous().view(torch.int32))  # symmetric in bits
    keep = (S >= t) & torch.ones_like(S, dtype=torch.bool).triu(1)
    ra, rb = torch.nonzero(keep, as_tuple=True)
    rs = S[ra, rb]
    order = np.lexsort((rb.cpu().numpy(), -rs.cpu().numpy(), ra.cpu().numpy()))
    order = torch.from_numpy(order).cuda()
    assert torch.equal(a, ra[order]) and torch.equal(b, rb[order]) and torch.equal(s, rs[order])
    s64 = (kb.index.emb.double()[a] * kb.index.emb.double()[b]).sum(1)
    assert bool(((s64 - s.double()).abs() < 1e-5).all())
    within = names[:10_000]
    a2, b2, s2 = kb.near_duplicates(t, within=within)
    sel = (a < 10_000) & (b < 10_000)
    assert torch.equal(a2, a[sel]) and torch.equal(b2, b[sel]) and torch.equal(s2, s[sel])
    kb.remove([names[int(a[0])]])
    a3, b3, _ = kb.near_duplicates(t)
    assert not ((a3 == a[0]) | (b3 == a[0])).any()
