"""Document-level retrieval on the H100: score_topk_groups returns exactly (torch.equal) the contract computed from
vr_score_exact scores - each group scored by its best eligible page, ranked by (score desc, best page asc), tail
(-inf, -1, -1) - on the grouped filter path, the exact path and the chunked exact path; page lists fed to the grouped
rescoring stay exact; the knowledge base's search_documents equals a brute-force grouping of its page search."""
import os

import numpy as np
import pytest
import torch

from visrag_b200 import _lib as L
from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu


def _unit(rs, n, d):
    x = rs.randn(n, d).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _exact_scores(q, idx):
    out = torch.empty((q.shape[0], idx.nd), dtype=torch.float32, device=q.device)
    L.check(L.lib().vr_score_exact(q.data_ptr(), q.shape[0], idx.emb.data_ptr(), idx.nd, q.shape[1], out.data_ptr(),
                                   L.stream_ptr()))
    return out


def _reference(q, idx, k, groups: np.ndarray, mask=None, id_offset=0):
    """Walk the pages in (score desc, id asc) order and keep the first page of each group not yet seen."""
    full = _exact_scores(q, idx).cpu().numpy()
    nd = full.shape[1]
    cols = np.arange(nd) if mask is None else np.nonzero(mask)[0]
    out_s = np.full((len(full), k), -np.inf, np.float32)
    out_p = np.full((len(full), k), -1, np.int64)
    out_g = np.full((len(full), k), -1, np.int64)
    for r in range(len(full)):
        s = full[r, cols]
        order = cols[np.lexsort((cols, -s))]
        _, first = np.unique(groups[order], return_index=True)
        pick = order[np.sort(first)][:k]
        n = len(pick)
        out_s[r, :n], out_p[r, :n], out_g[r, :n] = full[r, pick], pick + id_offset, groups[pick]
    return tuple(torch.from_numpy(x).cuda() for x in (out_s, out_p, out_g))


def _same(a, b, what):
    for x, y, name in zip(a, b, ("scores", "pages", "groups")):
        assert torch.equal(x, y), (what, name, int((x != y).sum()))


def _grouped(q, idx, k, groups, mask=None, **kw):
    g = groups if isinstance(groups, torch.Tensor) else torch.from_numpy(groups).cuda()
    m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else torch.from_numpy(mask).cuda())
    return R.score_topk_groups(q, idx, k, g, doc_mask=m, **kw)


def _layouts(rs, nd):
    return {"contiguous 8": np.arange(nd) // 8, "contiguous 64": np.arange(nd) // 64,
            "random non-contiguous": rs.randint(0, nd // 5, nd), "one page per group": np.arange(nd)}


def test_every_path_equals_the_contract():
    """nd = 9999 (not a multiple of 32 or 256), id_offset: the filter path (700 queries), the exact path (force_exact) and
    the chunked exact path (3 queries over many groups)."""
    rs = np.random.RandomState(50)
    Q, D = _unit(rs, 700, 256), _unit(rs, 9999, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for name, groups in _layouts(rs, len(D)).items():
        want = _reference(q, idx, 10, groups, id_offset=123)
        stats = {}
        _same(_grouped(q, idx, 10, groups, id_offset=123, stats=stats), want, name)
        assert stats["path"] == "filter+rescore", stats
        _same(_grouped(q, idx, 10, groups, id_offset=123, force_exact=True), want, f"{name}, exact")
        _same(_grouped(q[:3], idx, 10, groups, id_offset=123), tuple(x[:3] for x in want), f"{name}, 3 queries")


def test_one_page_per_group_equals_score_topk():
    rs = np.random.RandomState(51)
    Q, D = _unit(rs, 1000, 256), _unit(rs, 20001, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    groups = torch.arange(len(D), device="cuda")
    for kw in ({}, {"force_exact": True}):
        s, p, g = R.score_topk_groups(q, idx, 10, groups, **kw)
        s2, i2 = R.score_topk(q, idx, 10, **kw)
        assert torch.equal(s, s2) and torch.equal(p, i2) and torch.equal(g, p), kw
    s, p, g = R.score_topk_groups(q[:1], idx, 10, groups)
    s2, i2 = R.score_topk(q[:1], idx, 10)
    assert torch.equal(s, s2) and torch.equal(p, i2)


def test_mask_fewer_groups_than_k_and_k_beyond_G():
    rs = np.random.RandomState(52)
    Q, D = _unit(rs, 600, 128), _unit(rs, 12000, 128)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    groups = np.arange(len(D)) // 16
    masks = {"random 30 %": rs.rand(len(D)) < 0.3, "three groups": np.isin(groups, [4, 300, 749]),
             "random 1 %": rs.rand(len(D)) < 0.01}
    for name, m in masks.items():
        want = _reference(q, idx, 10, groups, m)
        for kw in ({}, {"force_exact": True}):
            _same(_grouped(q, idx, 10, groups, m, **kw), want, (name, kw))
        _same(_grouped(q[:2], idx, 10, groups, m), tuple(x[:2] for x in want), (name, "2 queries"))
    few = np.arange(len(D)) // 3000                                    # G = 4 < k
    want = _reference(q, idx, 10, few)
    assert (want[2][:, 4:] == -1).all()
    for kw in ({}, {"force_exact": True}):
        _same(_grouped(q, idx, 10, few, **kw), want, ("k > G", kw))


def _clustered(rs, n_docs, pages, d, nq, noise=0.02):
    """Each document is a centre plus small noise, its pages stored next to each other; queries lie near centres."""
    c = _unit(rs, n_docs, d)
    D = np.repeat(c, pages, axis=0) + noise * rs.randn(n_docs * pages, d).astype(np.float32) / np.sqrt(d)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q = c[rs.randint(0, n_docs, nq)] + 0.5 * rs.randn(nq, d).astype(np.float32) / np.sqrt(d)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return Q.astype(np.float32), D.astype(np.float32), np.arange(n_docs * pages) // pages


def test_clustered_contiguous_documents():
    rs = np.random.RandomState(53)
    Q, D, groups = _clustered(rs, 500, 64, 128, 2000)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    gt = R._group_table(torch.from_numpy(groups).cuda(), idx)
    want = _reference(q, idx, 10, groups)
    stats = {}
    _same(_grouped(q, idx, 10, groups, stats=stats), want, "grouped filter")
    assert stats["path"] == "filter+rescore" and stats["flagged"] == 0, stats
    # page lists crowd every range's list with one document: the proof fails, the fallback keeps the answer exact
    stats = {}
    got = R._score_topk_groups(q, idx, 10, 0, False, stats, gt, None, page_lists=True)
    _same(got, want, "page lists")
    assert stats["flagged"] > len(Q) // 2, stats


def test_one_document_holds_every_querys_top64_pages():
    rs = np.random.RandomState(54)
    d = 128
    Q, D = _unit(rs, 800, d), _unit(rs, 30000, d)
    centre = Q.mean(0)
    centre /= np.linalg.norm(centre)
    pert = centre + 0.01 * rs.randn(100, d).astype(np.float32) / np.sqrt(d)
    D[7000:7100] = pert / np.linalg.norm(pert, axis=1, keepdims=True)
    Q = Q * 0.3 + centre
    Q = (Q / np.linalg.norm(Q, axis=1, keepdims=True)).astype(np.float32)
    groups = np.arange(len(D)) // 100
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    top = R.score_topk(q, idx, 64, force_exact=True)[1].cpu().numpy()
    assert ((top >= 7000) & (top < 7100)).all()
    for kw in ({}, {"force_exact": True}):
        _same(_grouped(q, idx, 10, groups, **kw), _reference(q, idx, 10, groups), str(kw))


@pytest.mark.parametrize("nq,nd,d", [(700, 33333, 256), (2600, 9000, 64)])
def test_grouped_lists_are_sorted_group_distinct_and_hold_each_top_group(nq, nd, d):
    rs = np.random.RandomState(nq)
    Q, D = _unit(rs, nq, d), _unit(rs, nd, d)
    groups = rs.randint(0, nd // 6, nd).astype(np.int32)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    lib = L.lib()
    ranges, kt = lib.vr_score_ranges(nq, nd), lib.vr_score_list_len()
    lists = ranges * 2
    cand_s = torch.full((nq, lists * kt), float("nan"), device="cuda")
    cand_i = torch.full((nq, lists * kt), 0x7F7F7F7F, dtype=torch.int32, device="cuda")
    g = torch.from_numpy(groups).cuda()
    q16 = R.to_f16_rows(q)
    L.check(lib.vr_score_filter_groups(q16.data_ptr(), nq, idx.emb_f16.data_ptr(), nd, d, ranges, cand_s.data_ptr(),
                                       cand_i.data_ptr(), g.data_ptr(), None, L.stream_ptr()))
    torch.cuda.synchronize()
    ci, cs = cand_i.cpu().numpy().reshape(nq, lists, kt), cand_s.cpu().numpy().reshape(nq, lists, kt)
    assert not np.isnan(cs).any() and ((ci == -1) | ((ci >= 0) & (ci < nd))).all()
    assert (cs[:, :, 1:] <= cs[:, :, :-1]).all()
    assert (np.isinf(cs) == (ci == -1))[:, :-1].all()
    for r in range(nq):
        for li in range(lists - 1):
            gl = groups[ci[r, li][ci[r, li] >= 0]]
            assert len(gl) == len(set(gl.tolist())), (r, li)
    plan = np.zeros(6, np.int32)
    L.check(lib.vr_score_plan(nq, nd, plan.ctypes.data))
    T, Rn = int(plan[0]), int(plan[1])
    approx = (q16.float() @ idx.emb_f16.float().T).cpu().numpy()
    for r in rs.choice(nq, 30, replace=False):
        for rr in range(Rn):
            listed = {int(groups[p]): (float(v), int(p)) for v, p in zip(cs[r, rr], ci[r, rr]) if p >= 0}
            lo, hi = 256 * (T * rr // Rn), min(nd, 256 * (T * (rr + 1) // Rn))
            a = approx[r, lo:hi]
            best = {}
            for j in np.argsort(-a, kind="stable"):
                best.setdefault(int(groups[lo + j]), (float(a[j]), lo + j))
            tops = sorted(best.items(), key=lambda x: -x[1][0])
            if len(tops) <= kt:
                continue
            kth = tops[kt - 1][1][0]
            for grp, (sc, p) in tops[:kt]:
                if sc > kth + 1e-4 and sc > cs[r, lists - 1, 0] + 1e-4:   # clear members, above the final tau
                    assert grp in listed and abs(listed[grp][0] - sc) <= 1e-4, (r, rr, grp)
                    second = [v for v in a[groups[lo:hi] == grp] if v < sc]
                    if not second or max(second) < sc - 1e-4:            # a clear best page
                        assert listed[grp][1] == p, (r, rr, grp)


def test_query_alone_equals_its_row_in_a_batch_of_100():
    rs = np.random.RandomState(55)
    Q, D, groups = _clustered(rs, 6250, 8, 256, 100)           # 100 x 50 000 pages: the filter path
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    stats = {}
    s, p, g = _grouped(q, idx, 7, groups, stats=stats)
    assert stats["path"] == "filter+rescore"
    exact = _grouped(q, idx, 7, groups, force_exact=True)
    _same((s, p, g), exact, "filter vs exact")
    for r in (0, 42, 99):
        _same(_grouped(q[r:r + 1], idx, 7, groups), (s[r:r + 1], p[r:r + 1], g[r:r + 1]), f"query {r}")


def test_bad_doc_groups_are_refused():
    rs = np.random.RandomState(56)
    idx = R.build_index(_unit(rs, 1000, 64))
    q = torch.from_numpy(_unit(rs, 3, 64)).cuda()
    for bad in (torch.zeros(999, dtype=torch.int64, device="cuda"), torch.zeros(1000, dtype=torch.float32, device="cuda"),
                torch.zeros(1000, dtype=torch.int64), torch.full((1000,), -1, dtype=torch.int64, device="cuda")):
        with pytest.raises(ValueError):
            R.score_topk_groups(q, idx, 5, bad)


# ---------------------------------------------------------------------------------------------------- knowledge base


def test_search_documents_equals_grouping_the_page_search(tmp_path):
    from visrag_b200 import knowledge_base as KB

    rs = np.random.RandomState(57)
    D = _unit(rs, 20000, 256)
    names = [f"doc{i // 40}.pdf_{i % 40}.png" for i in range(len(D) - 100)] + [f"img{i}.jpeg" for i in range(100)]
    KB.save_knowledge_base(str(tmp_path / "kb"), D, names)
    kb = KB.KnowledgeBase(str(tmp_path / "kb"))
    Q = _unit(rs, 300, 256)

    def brute(kb, nq, k, within=None):
        """vr_score_exact scores of the searched pages, walked in (score desc, page asc) order, first page per document."""
        if within is None:
            rows = torch.nonzero(kb._live).flatten().tolist()
        else:
            rows = sorted(kb.filenames.index(f) for f in within)
        full = _exact_scores(torch.from_numpy(Q[:nq]).cuda(), kb.index).cpu().numpy()
        cols = np.array(rows)
        out_s, out_p, out_n = [], [], []
        for row in full:
            order = cols[np.lexsort((cols, -row[cols]))]
            seen, rs_, rp, rn = set(), [], [], []
            for pi in order:
                doc = KB.document_of(kb.filenames[pi])
                if doc not in seen:
                    seen.add(doc)
                    rs_.append(float(row[pi])), rp.append(int(pi)), rn.append(doc)
                    if len(rn) == k:
                        break
            out_s.append(rs_), out_p.append(rp), out_n.append(rn)
        return out_s, out_p, out_n

    def check(what, within=None):
        for nq in (1, 300):
            s, p, n = kb.search_documents(Q[:nq], 10, within=within)
            bs, bp, bn = brute(kb, nq, 10, within)
            assert n == bn and p.cpu().tolist() == bp and s.cpu().tolist() == bs, (what, nq)

    check("all")
    check("within", [f"doc{j}.pdf_{i}.png" for j in range(30, 60) for i in range(0, 40, 3)] + ["img5.jpeg"])
    kb.remove([f"doc{j}.pdf_{i}.png" for j in range(0, 200) for i in range(40)] + ["img7.jpeg"])
    check("remove")
    new = _unit(rs, 500, 256)
    kb.add(new, [f"doc3.pdf_{40 + i}.png" for i in range(250)] + [f"fresh.pdf_{i}.png" for i in range(250)])
    assert "doc3.pdf" in kb.documents[:200] and kb.documents[-1] == "fresh.pdf"
    check("add")
    top = kb.retrieve_documents(Q[:1], 3)
    _, p, n = kb.search_documents(Q[:1], 3)
    assert top == [(a, os.path.join(str(tmp_path / "kb"), kb.filenames[b])) for a, b in zip(n[0], p[0].tolist())]
    kb.save(str(tmp_path / "saved"))
    again = KB.KnowledgeBase(str(tmp_path / "saved"))
    for nq in (1, 300):
        s, p, n = kb.search_documents(Q[:nq], 10)
        s2, p2, n2 = again.search_documents(Q[:nq], 10)
        assert n == n2 and torch.equal(s.cpu(), s2.cpu()), nq


@pytest.mark.parametrize("world,k", [(3, 10), (4, 40), (2, 256)])
def test_per_shard_group_lists_merge_to_the_whole_index_on_one_gpu(world, k):
    """The corpus sharded in-process (as sharded_topk_groups shards it across ranks), documents of 70 pages straddling the
    shard boundaries, and one document's pages repeated on both sides of a boundary (equal scores on two shards: the lower
    page wins). world * k = 30, 160 and 512: both forms of the merge kernel (<= 128 and <= 512 entries per row)."""
    rs = np.random.RandomState(58 + world)
    nd, d = 12000, 128
    D = _unit(rs, nd, d)
    groups = np.arange(nd) // 70
    lo1 = nd // world
    D[lo1 + 3] = D[lo1 - 5]                                    # the same page on two shards, one document
    groups[lo1 + 3] = groups[lo1 - 5]
    Q = _unit(rs, 700, d)
    Q[:50] = D[lo1 - 5] + 0.01 * rs.randn(50, d).astype(np.float32)   # queries whose best page is the repeated one
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    q, g = torch.from_numpy(Q).cuda(), torch.from_numpy(groups).cuda()
    parts = []
    for r in range(world):
        lo, hi = R.shard_range(nd, r, world)
        parts.append(R.score_topk_groups(q, R.build_index(D[lo:hi]), k, g[lo:hi].contiguous(), lo))
    cat = [torch.cat([p[i] for p in parts], 1) for i in range(3)]
    assert cat[0].shape[1] == world * k
    got = R.merge_topk_groups(*cat, k)
    want = R.score_topk_groups(q, R.build_index(D), k, g)
    _same(got, want, (world, k))
    _same(want, _reference(q, R.build_index(D), k, groups), "whole index vs contract")
    assert (want[1][:50, 0] == lo1 - 5).all()
    too_many = [x.repeat(1, R.MERGE_GROUPS_MAX // x.shape[1] + 1) for x in cat]
    with pytest.raises(ValueError):
        R.merge_topk_groups(*too_many, k)


def test_exact_path_with_large_documents_and_one_group():
    """Documents of 5000 pages and a single group of every page: the atomic-key reduction spreads them over the grid."""
    rs = np.random.RandomState(59)
    Q, D = _unit(rs, 3, 64), _unit(rs, 100003, 64)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for groups in (np.arange(len(D)) // 5000, np.zeros(len(D), np.int64)):
        want = _reference(q, idx, 10, groups)
        _same(_grouped(q, idx, 10, groups), want, int(groups.max()))
        m = rs.rand(len(D)) < 0.3
        _same(_grouped(q, idx, 10, groups, m), _reference(q, idx, 10, groups, m), ("masked", int(groups.max())))


def _nccl_worker(rank, world, port, out_q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(4322)
        D = torch.nn.functional.normalize(torch.randn(12000, 256, device=dev, generator=g), dim=1)
        Q = torch.nn.functional.normalize(torch.randn(1000, 256, device=dev, generator=g), dim=1)
        groups = torch.arange(12000, device=dev) // 70        # 6000 is no multiple of 70: a document straddles the shards
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index = R.build_index(D[lo:hi].contiguous())
        s, p, gr = R.sharded_topk_groups(Q, index, 10, groups[lo:hi].contiguous(), lo)
        full = R.build_index(D)
        s2, p2, g2 = R.score_topk_groups(Q, full, 10, groups)
        ok = bool(torch.equal(p, p2) and torch.equal(gr, g2) and torch.equal(s, s2))
        out_q.put((rank, ok))
    finally:
        dist.destroy_process_group()


def test_sharded_topk_groups_with_documents_across_the_shard_boundary_under_nccl():
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
