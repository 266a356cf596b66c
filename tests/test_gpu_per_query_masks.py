"""Per-query masks on the H100: with a 2-D doc_mask and mask_of, every row of score_topk / score_topk_groups equals, bit
for bit (torch.equal on scores and ids), the same query called alone with its own mask as a 1-D doc_mask, and the masked
fp32 scan (force_exact). The sizes take the tensor-core filter over several waves, one 256-query block mixes disjoint,
nested, single-page, empty, full and smaller-than-k scopes, and rows r and r + 8 of every warp (the two accumulator rows
of one filter thread) search different masks. Also: flagged queries rerun with their own masks, the filter's lists of
each query hold only its eligible docs, a row does not depend on the other queries, and the knowledge base's
`within_each` and per-shard masks equal their single-scope and whole-index answers."""
import os

import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu


def _plan(nq, nd):
    out = np.zeros(6, np.int32)
    L.check(L.lib().vr_score_plan(nq, nd, out.ctypes.data))
    return dict(zip(("T", "R", "QB", "items", "pairs", "lists"), (int(v) for v in out)))


def _unit(g, n, d):
    return torch.nn.functional.normalize(torch.randn(n, d, device="cuda", generator=g), dim=1)


def _same(a, b, what):
    for x, y in zip(a, b):
        assert torch.equal(x, y), (what, int((x != y).sum()))


def _scopes(nd, g):
    """Mask rows of every kind: full, empty, one page, fewer pages than k, two disjoint blocks, a block nested in another,
    random 10 % and 50 %."""
    m = torch.zeros((10, nd), dtype=torch.bool, device="cuda")
    m[0] = True
    m[2, nd // 3] = True
    m[3, torch.tensor([7, nd // 2, nd - 1], device="cuda")] = True
    m[4, : nd // 4] = True
    m[5, nd // 4: nd // 2] = True
    m[6, nd // 8: nd // 5] = True                        # nested in row 4
    m[7] = torch.rand(nd, device="cuda", generator=g) < 0.1
    m[8] = torch.rand(nd, device="cuda", generator=g) < 0.5
    m[9] = m[7] & m[8]                                   # nested in rows 7 and 8
    return m


def _mask_of(nq, M, g):
    """Rows r and r + 8 of every warp get different masks (r mod M differs for M = 10); later blocks are random."""
    of = torch.randint(0, M, (nq,), device="cuda", generator=g)
    of[:256] = torch.arange(256, device="cuda") % M
    return of


NQ, ND, DIM = 5001, 60000, 128                            # several waves; the fp32 scan runs in row chunks


@pytest.fixture(scope="module")
def setup():
    p = _plan(NQ, ND)
    assert p["items"] > p["pairs"] and p["R"] > 1, p
    g = torch.Generator(device="cuda").manual_seed(90)
    idx = R.build_index(_unit(g, ND, DIM))
    q = _unit(g, NQ, DIM)
    masks = _scopes(ND, g)
    of = _mask_of(NQ, masks.shape[0], g)
    groups = (torch.arange(ND, device="cuda", dtype=torch.int32) * 7919 % 9973) // 5   # documents of scattered pages
    return q, idx, masks, of, groups


SAMPLE = list(range(0, 20)) + [100, 255, 256, 1000, 4095, 5000]


def test_page_rows_equal_single_calls_and_the_masked_fp32_scan(setup):
    q, idx, masks, of, _ = setup
    stats = {}
    got = R.score_topk(q, idx, 10, doc_mask=masks, mask_of=of, stats=stats)
    assert stats["path"] == "filter+rescore" and stats["flagged"] < NQ // 2, stats
    _same(got, R.score_topk(q, idx, 10, doc_mask=masks, mask_of=of, force_exact=True), "fp32 scan")
    for r in SAMPLE:
        alone = R.score_topk(q[r:r + 1], idx, 10, doc_mask=masks[int(of[r])])
        _same((got[0][r:r + 1], got[1][r:r + 1]), alone, f"query {r}, mask {int(of[r])}")
    # the empty scope is all (-inf, -1); the three-page scope ends in (-inf, -1) after three entries
    empty, three = int((of[:256] == 1).nonzero()[0]), int((of[:256] == 3).nonzero()[0])
    assert (got[1][empty] == -1).all() and torch.isinf(got[0][empty]).all()
    assert (got[1][three, :3] >= 0).all() and (got[1][three, 3:] == -1).all()
    assert not torch.equal(got[1][0], got[1][8])


def test_document_rows_equal_single_calls_and_the_masked_fp32_scan(setup):
    q, idx, masks, of, groups = setup
    stats = {}
    got = R.score_topk_groups(q, idx, 10, groups, doc_mask=masks, mask_of=of, stats=stats)
    assert stats["path"] == "filter+rescore", stats
    _same(got, R.score_topk_groups(q, idx, 10, groups, doc_mask=masks, mask_of=of, force_exact=True), "fp32 scan")
    for r in SAMPLE:
        alone = R.score_topk_groups(q[r:r + 1], idx, 10, groups, doc_mask=masks[int(of[r])])
        _same(tuple(t[r:r + 1] for t in got), alone, f"query {r}, mask {int(of[r])}")


def test_one_mask_row_per_query_by_default(setup):
    q, idx, masks, of, _ = setup
    n = 600
    full = masks[of[:n]]                                  # [nq, nd]: mask_of omitted, row i for query i
    _same(R.score_topk(q[:n], idx, 10, doc_mask=full), R.score_topk(q[:n], idx, 10, doc_mask=masks, mask_of=of[:n]), "pages")
    with pytest.raises(ValueError, match="rows for"):
        R.score_topk(q[:n], idx, 10, doc_mask=full[:-1])


def test_a_row_does_not_depend_on_the_other_queries(setup):
    q, idx, masks, of, groups = setup
    n = 1500
    base = R.score_topk(q[:n], idx, 10, doc_mask=masks, mask_of=of[:n])
    perm = torch.randperm(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    pq = R.score_topk(q[perm], idx, 10, doc_mask=masks, mask_of=of[perm])
    _same(tuple(t[perm] for t in base), pq, "permuted queries")
    other = torch.where(torch.arange(n, device="cuda") % 2 == 0, of[:n], (of[:n] + 3) % masks.shape[0])
    changed = R.score_topk(q[:n], idx, 10, doc_mask=masks, mask_of=other)
    keep = torch.arange(0, n, 2, device="cuda")
    _same(tuple(t[keep] for t in base), tuple(t[keep] for t in changed), "other queries' masks changed")
    # a set of one with mask_of all zeros is the 1-D doc_mask call, for pages and documents, filter and scan
    zeros = torch.zeros(n, dtype=torch.int64, device="cuda")
    for kw in ({}, {"force_exact": True}):
        _same(R.score_topk(q[:n], idx, 10, doc_mask=masks[8:9], mask_of=zeros, **kw),
              R.score_topk(q[:n], idx, 10, doc_mask=masks[8], **kw), f"set of one {kw}")
        _same(R.score_topk_groups(q[:n], idx, 10, groups, doc_mask=masks[8:9], mask_of=zeros, **kw),
              R.score_topk_groups(q[:n], idx, 10, groups, doc_mask=masks[8], **kw), f"documents, set of one {kw}")


def test_flagged_queries_rerun_with_their_own_masks():
    rs = np.random.RandomState(91)
    d = 128
    D = rs.randn(40000, d).astype(np.float32)
    Q = rs.randn(1500, d).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    for qi in range(1, 6):                                # 40 near-identical docs per query in one tile: lists overflow
        pert = Q[qi] + rs.randn(40, d).astype(np.float32) * 1e-4
        D[5000 + 300 * qi: 5040 + 300 * qi] = pert / np.linalg.norm(pert, axis=1, keepdims=True)
    masks = torch.from_numpy(rs.rand(3, len(D)) < 0.5).cuda()
    masks[1:, 5000:7000] = True                           # the clusters stay eligible for masks 1 and 2, not for mask 0
    masks[0, 5000:7000] = False
    of = torch.from_numpy(rs.randint(0, 3, len(Q))).cuda()
    of[0], of[1:6] = 0, torch.tensor([1, 2, 1, 2, 1], device="cuda")
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    stats = {}
    got = R.score_topk(q, idx, 10, doc_mask=masks, mask_of=of, stats=stats)
    assert stats["flagged"] > 0, stats
    # which rows flag: the filter + rescoring once more by hand (rows 1-5, whose clusters overflow their lists, do)
    lib = L.lib()
    nq, nd = q.shape[0], idx.nd
    ranges = lib.vr_score_ranges(nq, nd)
    lists = ranges * 2 * lib.vr_score_list_len()
    cand_s = torch.empty((nq, lists), device="cuda")
    cand_i = torch.empty((nq, lists), dtype=torch.int32, device="cuda")
    ms = R._check_doc_mask(masks, idx, nq, of)
    q16 = R.to_f16_rows(q)
    L.check(lib.vr_score_filter_masks(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(),
                                      cand_i.data_ptr(), ms.arg(), L.stream_ptr()))
    out_s = torch.empty((nq, 10), device="cuda")
    out_i = torch.empty((nq, 10), dtype=torch.int64, device="cuda")
    flags = torch.empty(nq, dtype=torch.int32, device="cuda")
    L.check(lib.vr_score_rescore(q.data_ptr(), nq, idx.emb.data_ptr(), nd, d, ranges, cand_s.data_ptr(), cand_i.data_ptr(),
                                 idx.max_norm.data_ptr(), 10, 0, out_s.data_ptr(), out_i.data_ptr(), flags.data_ptr(),
                                 L.stream_ptr()))
    bad = torch.nonzero(flags).flatten()
    assert (of[bad] != of[0]).any(), (bad.tolist(), of[bad].tolist())
    _same(got, R.score_topk(q, idx, 10, doc_mask=masks, mask_of=of, force_exact=True), "clustered")
    for r in bad.tolist()[:8] + [0]:
        _same((got[0][r:r + 1], got[1][r:r + 1]), R.score_topk(q[r:r + 1], idx, 10, doc_mask=masks[int(of[r])]), f"row {r}")


@pytest.mark.parametrize("grouped", [False, True])
def test_candidate_lists_hold_each_querys_eligible_docs_and_cover_its_top16(grouped):
    nq, nd, d = 700, 33333, 256
    g = torch.Generator(device="cuda").manual_seed(92)
    q, idx = _unit(g, nq, d), R.build_index(_unit(g, nd, d))
    masks = torch.rand((9, nd), device="cuda", generator=g) < torch.tensor([[0.02], [0.1], [0.25], [0.5], [0.9],
                                                                            [0.3], [0.05], [0.7], [0.15]], device="cuda")
    of = _mask_of(nq, 9, g)
    lib = L.lib()
    ranges, kt = lib.vr_score_ranges(nq, nd), lib.vr_score_list_len()
    lists = ranges * 2
    cand_s = torch.full((nq, lists * kt), float("nan"), device="cuda")
    cand_i = torch.full((nq, lists * kt), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    ms = R._check_doc_mask(masks, idx, nq, of)
    q16 = R.to_f16_rows(q)
    args = (q16.data_ptr(), nq, idx.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(), cand_i.data_ptr())
    groups = torch.arange(nd, dtype=torch.int32, device="cuda") // 3
    if grouped:
        L.check(lib.vr_score_filter_groups_masks(*args, groups.data_ptr(), ms.arg(), L.stream_ptr()))
    else:
        L.check(lib.vr_score_filter_masks(*args, ms.arg(), L.stream_ptr()))
    torch.cuda.synchronize()
    ci, cs = cand_i.cpu().numpy().reshape(nq, lists, kt), cand_s.cpu().numpy().reshape(nq, lists, kt)
    assert not np.isnan(cs).any() and ((ci == -1) | ((ci >= 0) & (ci < nd))).all()
    elig = masks[of].cpu().numpy()
    rows = np.nonzero(ci >= 0)[0]
    assert elig[rows, ci[ci >= 0]].all()                  # no list holds a doc its own query may not see
    assert (cs[:, :, 1:] <= cs[:, :, :-1]).all()
    approx = (q16.float() @ idx.emb_f16.float().T).cpu().numpy()
    approx[~elig] = -np.inf
    gr = groups.cpu().numpy()
    for r in list(range(16)) + list(np.random.RandomState(0).choice(nq, 30, replace=False)):
        have = set(ci[r][ci[r] >= 0].tolist())
        if grouped:
            have = set(gr[list(have)].tolist())
        a = approx[r]
        if grouped:                                     # best approximate page per group
            best = np.full(gr.max() + 1, -np.inf, np.float32)
            np.maximum.at(best, gr, a)
            a = best
        if np.isinf(a).all():
            assert not have
            continue
        kth = np.sort(a)[-kt]
        must = set(np.nonzero(a > kth + 1e-4)[0].tolist())  # clear members of the query's eligible approximate top-16
        assert must <= have, r


# ---------------------------------------------------------------------------------------------------- knowledge base
def _kb(path, D, names):
    from visrag_b200 import knowledge_base as KB

    KB.save_knowledge_base(str(path), D, names)
    return KB.KnowledgeBase(str(path))


def test_knowledge_base_within_each(tmp_path):
    """300 queries (the filter path) with one scope each: whole PDFs, scattered pages, one page, every live page (None),
    and pages added after a removal. Each row equals the same query searched alone with within=; removed pages are never
    returned; search_documents names only the documents a query found."""
    rs = np.random.RandomState(93)
    D = rs.randn(30000, 256).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    names = [f"doc{i // 100}.pdf_{i % 100}.png" for i in range(len(D))]
    kb = _kb(tmp_path / "kb", D, names)
    gone = sorted(rs.choice(len(D), 3000, replace=False))
    kb.remove([names[i] for i in gone])
    new = rs.randn(500, 256).astype(np.float32) * 1.2
    kb.add(new, [f"new.pdf_{i}.png" for i in range(500)])
    live = set(kb._row)
    pdf = lambda n: [f for f in (f"doc{n}.pdf_{i}.png" for i in range(100)) if f in live]  # noqa: E731
    kinds = [pdf(3), pdf(250), sorted(rs.choice(sorted(live), 4000, replace=False).tolist()), [pdf(7)[0]], None,
             [f"new.pdf_{i}.png" for i in range(0, 500, 3)], pdf(3)[:4] + [f"new.pdf_{i}.png" for i in range(2)]]
    Q = rs.randn(300, 256).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    scopes = [kinds[i % len(kinds)] for i in range(len(Q))]
    s, i = kb.search(Q, 10, within_each=scopes)
    assert i.shape == (300, 10)
    dead = set(gone)
    for r in list(range(20)) + [150, 299]:
        s1, i1 = kb.search(Q[r:r + 1], 10, within=scopes[r])
        n = i1.shape[1]
        assert torch.equal(i[r, :n], i1[0]) and torch.equal(s[r, :n], s1[0]), r
        assert (i[r, n:] == -1).all() and torch.isinf(s[r, n:]).all()
        assert not dead & set(i[r].tolist()), r
    ds, dp, dn = kb.search_documents(Q, 5, within_each=scopes)
    for r in list(range(14)) + [299]:
        s1, p1, n1 = kb.search_documents(Q[r:r + 1], 5, within=scopes[r])
        assert dn[r] == n1[0] and torch.equal(dp[r, :len(n1[0])], p1[0]) and torch.equal(ds[r, :len(n1[0])], s1[0]), r
    assert len(dn[3]) == 1 and dn[3] == ["doc7.pdf"]          # the one-page scope finds one document
    with pytest.raises(ValueError, match="cannot be combined"):
        kb.search(Q[:2], 5, within=pdf(3), within_each=[None, None])
    with pytest.raises(ValueError, match="one scope per query"):
        kb.search(Q[:2], 5, within_each=[None])
    with pytest.raises(KeyError):
        kb.search(Q[:2], 5, within_each=[None, [names[gone[0]]]])


# ---------------------------------------------------------------------------------------------------- shards
def test_per_shard_masks_merge_to_the_whole_index_on_one_gpu():
    g = torch.Generator(device="cuda").manual_seed(94)
    nd, nq, d, world = 30001, 700, 128, 3
    D, q = _unit(g, nd, d), _unit(g, nq, d)
    masks = _scopes(nd, g)
    of = _mask_of(nq, masks.shape[0], g)
    groups = (torch.arange(nd, device="cuda", dtype=torch.int32) // 11)
    whole = R.build_index(D)
    want = R.score_topk(q, whole, 10, doc_mask=masks, mask_of=of)
    want_g = R.score_topk_groups(q, whole, 10, groups, doc_mask=masks, mask_of=of)
    parts, parts_g = [], []
    for r in range(world):
        lo, hi = R.shard_range(nd, r, world)
        shard = R.build_index(D[lo:hi].contiguous())
        m = masks[:, lo:hi].contiguous()
        parts.append(R.sharded_topk(q, shard, 10, lo, doc_mask=m, mask_of=of))
        parts_g.append(R.sharded_topk_groups(q, shard, 10, groups[lo:hi].contiguous(), lo, doc_mask=m, mask_of=of))
    got = R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1), 10)
    _same(got, want, "pages")
    got_g = R.merge_topk_groups(*(torch.cat([p[j] for p in parts_g], 1) for j in range(3)), 10)
    _same(got_g, want_g, "documents")


def _nccl_worker(rank, world, port, out_q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(4322)           # same stream on every rank: corpus, masks, mask_of
        D = torch.nn.functional.normalize(torch.randn(12000, 256, device=dev, generator=g), dim=1)
        Q = torch.nn.functional.normalize(torch.randn(1000, 256, device=dev, generator=g), dim=1)
        masks = torch.rand(4, 12000, device=dev, generator=g) < torch.tensor([[0.3], [0.05], [0.6], [1.0]], device=dev)
        of = torch.randint(0, 4, (1000,), device=dev, generator=g)
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index = R.build_index(D[lo:hi].contiguous())
        s, i = R.sharded_topk(Q, index, 10, lo, doc_mask=masks[:, lo:hi].contiguous(), mask_of=of)
        ok = True
        for r in range(0, 1000, 97):
            cols = torch.nonzero(masks[of[r]]).flatten()
            ref = torch.topk(Q[r] @ D[cols].T, 10)                  # brute-force fp32 scan of the row's eligible docs
            ok &= bool(torch.equal(i[r], cols[ref.indices])) and float((s[r] - ref.values).abs().max()) <= 2e-6
        out_q.put((rank, ok))
    finally:
        dist.destroy_process_group()


def test_sharded_topk_with_per_query_masks_under_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() + 700) % 1000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == [0, 1] and all(r[1] for r in res), res
