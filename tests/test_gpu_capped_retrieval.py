"""Per-document caps on the H100: score_topk_capped and score_topk_groups_pages return exactly (torch.equal) the
contract computed from vr_score_exact scores with the models of tests/test_capped_retrieval_host.py - on the filter
path, force_exact and the chunked exact path, with masks, per-query masks and candidate lists, long documents split
into pieces, NaN / inf rows, sharded corpora and the knowledge base."""
import os

import numpy as np
import pytest
import torch

from tests.test_capped_retrieval_host import page_order, walk_capped
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


def _contract(q, idx, k, m, groups, elig=None, id_offset=0):
    """From vr_score_exact rows: the capped top-k (scores, pages, groups) [nq, k] and the inner hits (document scores,
    best pages, groups [nq, k], page scores, pages [nq, k, m]). elig: None, bool [nd] or bool [nq, nd]."""
    full = _exact_scores(q, idx).cpu().numpy()
    nq = len(full)
    groups = np.asarray(groups)
    cap = (np.full((nq, k), -np.inf, np.float32), np.full((nq, k), -1, np.int64), np.full((nq, k), -1, np.int64))
    docs = tuple(np.copy(x) for x in cap)
    ps, pp = np.full((nq, k, m), -np.inf, np.float32), np.full((nq, k, m), -1, np.int64)
    for r in range(nq):
        e = None if elig is None else (elig if elig.ndim == 1 else elig[r])
        s = full[r]
        picks = walk_capped(s, groups, k, m, e)
        cap[0][r, :len(picks)], cap[1][r, :len(picks)], cap[2][r, :len(picks)] = s[picks], np.add(picks, id_offset), groups[picks]
        best = walk_capped(s, groups, k, 1, e)
        docs[0][r, :len(best)], docs[1][r, :len(best)], docs[2][r, :len(best)] = s[best], np.add(best, id_offset), groups[best]
        order = page_order(s, e)
        go = groups[order]
        for j, b in enumerate(best):
            top = order[go == groups[b]][:m]
            ps[r, j, :len(top)], pp[r, j, :len(top)] = s[top], top + id_offset
    t = lambda x: torch.from_numpy(x).cuda()  # noqa: E731
    return tuple(map(t, cap)), tuple(map(t, docs + (ps, pp)))


def _same(a, b, what):
    assert len(a) == len(b)
    for j, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x, y), (what, j, int((x != y).sum()) if x.shape == y.shape else x.shape)


def _layouts(rs, nd):
    return {"contiguous 8": np.arange(nd) // 8, "contiguous 64": np.arange(nd) // 64,
            "random non-contiguous": rs.randint(0, nd // 5, nd), "one page per group": np.arange(nd)}


def _both(q, idx, k, m, g, **kw):
    return R.score_topk_capped(q, idx, k, g, m, **kw), R.score_topk_groups_pages(q, idx, k, g, m, **kw)


def test_every_path_equals_the_contract():
    """nd = 9999 (not a multiple of 32 or 256), id_offset 123: the filter path (700 queries), force_exact, and the
    chunked exact path (3 queries)."""
    rs = np.random.RandomState(80)
    Q, D = _unit(rs, 700, 256), _unit(rs, 9999, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for name, groups in _layouts(rs, len(D)).items():
        g = torch.from_numpy(groups).cuda()
        for m in (2, 3):
            cap, hits = _contract(q, idx, 10, m, groups, id_offset=123)
            stats = {}
            got = _both(q, idx, 10, m, g, id_offset=123, stats=stats)
            assert stats["path"] == "filter+rescore", stats
            _same(got[0], cap, (name, m, "capped"))
            _same(got[1], hits, (name, m, "inner hits"))
            got = _both(q, idx, 10, m, g, id_offset=123, force_exact=True)
            _same(got[0], cap, (name, m, "capped, exact"))
            _same(got[1], hits, (name, m, "inner hits, exact"))
            got = _both(q[:3], idx, 10, m, g, id_offset=123)
            _same(got[0], tuple(x[:3] for x in cap), (name, m, "capped, 3 queries"))
            _same(got[1], tuple(x[:3] for x in hits), (name, m, "inner hits, 3 queries"))


def test_masks_per_query_masks_and_lists():
    rs = np.random.RandomState(81)
    nq, nd = 600, 12001
    Q, D = _unit(rs, nq, 128), _unit(rs, nd, 128)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    groups = np.arange(nd) // 16
    g = torch.from_numpy(groups).cuda()
    one = rs.rand(nd) < 0.3
    cap, hits = _contract(q, idx, 10, 3, groups, one)
    for kw in ({}, {"force_exact": True}):
        got = _both(q, idx, 10, 3, g, doc_mask=torch.from_numpy(one).cuda(), **kw)
        _same(got[0], cap, ("1-D mask", kw))
        _same(got[1], hits, ("1-D mask", kw))
    M = rs.rand(5, nd) < np.array([0.02, 0.1, 0.3, 0.6, 1.0])[:, None]
    of = rs.randint(0, 5, nq)
    cap, hits = _contract(q, idx, 10, 3, groups, M[of])
    got = _both(q, idx, 10, 3, g, doc_mask=torch.from_numpy(M).cuda(), mask_of=torch.from_numpy(of).cuda())
    _same(got[0], cap, "per-query masks")
    _same(got[1], hits, "per-query masks")
    lists = [np.nonzero(row)[0] for row in M[:3]]
    lists[0] = np.concatenate([lists[0], lists[0][:5]])  # a repeated id counts once
    offsets = torch.tensor(np.cumsum([0] + [len(x) for x in lists]), dtype=torch.int64, device="cuda")
    ids = torch.from_numpy(np.concatenate(lists).astype(np.int32)).cuda()
    of = rs.randint(0, 3, nq)
    cap, hits = _contract(q, idx, 10, 3, groups, M[:3][of])
    stats = {}
    got = _both(q, idx, 10, 3, g, doc_lists=(offsets, ids), list_of=torch.from_numpy(of).cuda(), stats=stats)
    assert stats["path"] == "lists", stats
    _same(got[0], cap, "doc_lists")
    _same(got[1], hits, "doc_lists")


def test_cap_one_is_the_documents_and_cap_k_the_pages():
    rs = np.random.RandomState(82)
    Q, D = _unit(rs, 1000, 256), _unit(rs, 20001, 256)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    g = torch.from_numpy(rs.randint(0, 3000, len(D))).cuda()
    for kw in ({}, {"force_exact": True}):
        docs = R.score_topk_groups(q, idx, 10, g, **kw)
        _same(R.score_topk_capped(q, idx, 10, g, 1, **kw), docs, ("m = 1", kw))
        s, i = R.score_topk(q, idx, 10, **kw)
        for m in (10, 11, 1000):
            got = R.score_topk_capped(q, idx, 10, g, m, **kw)
            _same(got[:2], (s, i), ("m >= k", m, kw))
            assert torch.equal(got[2], g[i].long()), kw
        hits = R.score_topk_groups_pages(q, idx, 10, g, 4, **kw)
        _same(hits[:3], docs, ("inner hits documents", kw))
        assert torch.equal(hits[3][:, :, 0], docs[0]) and torch.equal(hits[4][:, :, 0], docs[1]), kw


def _clustered(rs, n_docs, pages, d, nq, noise=0.02):
    c = _unit(rs, n_docs, d)
    D = np.repeat(c, pages, axis=0) + noise * rs.randn(n_docs * pages, d).astype(np.float32) / np.sqrt(d)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q = c[rs.randint(0, n_docs, nq)] + 0.5 * rs.randn(nq, d).astype(np.float32) / np.sqrt(d)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return Q.astype(np.float32), D.astype(np.float32), np.arange(n_docs * pages) // pages


def test_clustered_contiguous_documents():
    """Documents of 64 near-identical contiguous pages: the layout where page lists flag."""
    rs = np.random.RandomState(83)
    Q, D, groups = _clustered(rs, 500, 64, 128, 2000)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    g = torch.from_numpy(groups).cuda()
    for m in (2, 5):
        cap, hits = _contract(q, idx, 10, m, groups)
        got = _both(q, idx, 10, m, g)
        _same(got[0], cap, ("clustered capped", m))
        _same(got[1], hits, ("clustered inner hits", m))
    top = R.score_topk(q, idx, 10)[1]
    assert (g[top] == g[top[:, :1]]).all(1).float().mean() > 0.5   # plain top-k: mostly one document per row


def test_documents_longer_than_a_piece_and_one_group_of_every_page():
    rs = np.random.RandomState(84)
    Q, D = _unit(rs, 5, 64), _unit(rs, 40003, 64)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for groups in (np.arange(len(D)) // 5000, np.zeros(len(D), np.int64), rs.randint(0, 3, len(D))):
        g = torch.from_numpy(groups).cuda()
        gt = R._group_table(g, idx)
        assert gt.max_pages > R.GROUP_PIECE
        mask = rs.rand(len(D)) < 0.3
        for m, elig in ((3, None), (64, None), (7, mask)):
            cap, hits = _contract(q, idx, 10, m, groups, elig)
            dm = None if elig is None else torch.from_numpy(elig).cuda()
            got = _both(q, idx, 10, m, g, doc_mask=dm)
            _same(got[0], cap, (int(groups.max()), m, "capped"))
            _same(got[1], hits, (int(groups.max()), m, "inner hits"))


def test_fewer_documents_than_k_and_nonfinite_rows():
    rs = np.random.RandomState(85)
    Q, D = _unit(rs, 600, 128), _unit(rs, 12000, 128)
    D[17] = np.nan
    D[5000, :3] = np.inf
    D[9000] = -D[9000] * np.inf
    Q[3] = np.nan
    Q[4, 0] = np.inf
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    for groups in (np.arange(len(D)) // 3000, np.arange(len(D)) // 8):     # G = 4 < k, and 1500 documents
        g = torch.from_numpy(groups).cuda()
        for m in (2, 3):
            cap, hits = _contract(q, idx, 10, m, groups)
            for kw in ({}, {"force_exact": True}):
                got = _both(q, idx, 10, m, g, **kw)
                _same(got[0], cap, (int(groups.max()), m, kw, "capped"))
                _same(got[1], hits, (int(groups.max()), m, kw, "inner hits"))
    cap, _ = _contract(q, idx, 10, 2, np.arange(len(D)) // 3000)
    assert (cap[1][:, 8:] == -1).all() and (cap[1][5:, :8] >= 0).all()   # four documents of two pages: eight picks


def test_query_alone_equals_its_row_in_a_batch_of_100():
    rs = np.random.RandomState(86)
    Q, D, groups = _clustered(rs, 6250, 8, 256, 100)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    g = torch.from_numpy(groups).cuda()
    stats = {}
    cap, hits = _both(q, idx, 7, 3, g, stats=stats)
    assert stats["path"] == "filter+rescore"
    for r in (0, 42, 99):
        a, b = _both(q[r:r + 1], idx, 7, 3, g)
        _same(a, tuple(x[r:r + 1] for x in cap), f"capped, query {r}")
        _same(b, tuple(x[r:r + 1] for x in hits), f"inner hits, query {r}")


def test_group_pages_topm_takes_groups_from_any_source():
    rs = np.random.RandomState(87)
    Q, D = _unit(rs, 50, 64), _unit(rs, 3000, 64)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    groups = np.arange(len(D)) // 30
    gsel = torch.from_numpy(rs.randint(-3, 110, (50, 6))).cuda()       # -3..-1 and 100..109: empty documents
    s, p = R.group_pages_topm(q, idx, gsel, torch.from_numpy(groups).cuda(), 4, id_offset=7)
    full = _exact_scores(q, idx).cpu().numpy()
    for r in range(50):
        order = page_order(full[r])
        for j, gg in enumerate(gsel[r].tolist()):
            top = order[groups[order] == gg][:4] if gg >= 0 else order[:0]
            want_p = np.full(4, -1, np.int64)
            want_s = np.full(4, -np.inf, np.float32)
            want_p[:len(top)], want_s[:len(top)] = top + 7, full[r, top]
            assert p[r, j].tolist() == want_p.tolist() and np.array_equal(s[r, j].cpu().numpy(), want_s), (r, j)


# ---------------------------------------------------------------------------------------------------- sharded
def _merge_shards(q, D, groups, world, k, m):
    """The sharded procedure in one process: global documents from the per-shard lists, each shard's stage with global
    group ids, per-(row, slot) top-m over the shards, then the capped top-k."""
    g = torch.from_numpy(groups).cuda()
    nd, nq = len(D), q.shape[0]
    shards = [(R.shard_range(nd, r, world), R.build_index(D[slice(*R.shard_range(nd, r, world))])) for r in range(world)]
    parts = [R.score_topk_groups(q, ix, k, g[lo:hi].contiguous(), lo) for (lo, hi), ix in shards]
    docs = R.merge_topk_groups(*[torch.cat([p[i] for p in parts], 1) for i in range(3)], k)
    lists = [R.group_pages_topm(q, ix, docs[2], g[lo:hi].contiguous(), m, id_offset=lo) for (lo, hi), ix in shards]
    s = torch.stack([x[0] for x in lists], 2).reshape(nq * k, world * m)
    p = torch.stack([x[1] for x in lists], 2).reshape(nq * k, world * m)
    ps, pp = (t.view(nq, k, m) for t in R.merge_topk(s, p, m))
    grp = docs[2][:, :, None].expand(nq, k, m).reshape(nq, k * m)
    return R._capped_merge(ps.view(nq, k * m), pp.view(nq, k * m), grp, k), docs + (ps, pp)


@pytest.mark.parametrize("world,k,m", [(2, 10, 2), (3, 10, 3), (4, 20, 5)])
def test_per_shard_results_merge_to_the_whole_index_on_one_gpu(world, k, m):
    """Documents of 70 pages straddle the shard boundaries."""
    rs = np.random.RandomState(88 + world)
    nd, d = 12000, 128
    Q, D, groups = _clustered(rs, nd // 60, 60, d, 700)
    groups = np.arange(nd) // 70
    q = torch.from_numpy(Q).cuda()
    cap, hits = _merge_shards(q, D, groups, world, k, m)
    g = torch.from_numpy(groups).cuda()
    whole = _both(q, R.build_index(D), k, m, g)
    _same(cap, whole[0], ("capped", world))
    _same(hits, whole[1], ("inner hits", world))
    _same(whole[0], _contract(q, R.build_index(D), k, m, groups)[0], "whole index vs contract")


def _nccl_worker(rank, world, port, out_q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(4323)
        D = torch.nn.functional.normalize(torch.randn(12000, 256, device=dev, generator=g), dim=1)
        Q = torch.nn.functional.normalize(torch.randn(1000, 256, device=dev, generator=g), dim=1)
        groups = torch.arange(12000, device=dev) // 70
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index = R.build_index(D[lo:hi].contiguous())
        full = R.build_index(D)
        ok = True
        for m in (2, 3, 10):
            a = R.sharded_topk_capped(Q, index, 10, groups[lo:hi].contiguous(), m, lo)
            b = R.score_topk_capped(Q, full, 10, groups, m)
            ok &= all(torch.equal(x, y) for x, y in zip(a, b))
        a = R.sharded_topk_groups_pages(Q, index, 10, groups[lo:hi].contiguous(), 3, lo)
        b = R.score_topk_groups_pages(Q, full, 10, groups, 3)
        ok &= all(torch.equal(x, y) for x, y in zip(a, b))
        out_q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_sharded_capped_and_inner_hits_under_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() + 800) % 1000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == [0, 1] and all(r[1] for r in res), res


def test_sharded_forms_on_one_process_equal_the_plain_calls():
    rs = np.random.RandomState(90)
    Q, D = _unit(rs, 300, 128), _unit(rs, 9000, 128)
    q, idx = torch.from_numpy(Q).cuda(), R.build_index(D)
    g = torch.from_numpy(np.arange(len(D)) // 9).cuda()
    for m in (2, 12):
        _same(R.sharded_topk_capped(q, idx, 10, g, m, 5), R.score_topk_capped(q, idx, 10, g, m, 5), m)
    _same(R.sharded_topk_groups_pages(q, idx, 10, g, 3, 5), R.score_topk_groups_pages(q, idx, 10, g, 3, 5), "pages")


# ---------------------------------------------------------------------------------------------------- knowledge base
def test_knowledge_base_equals_a_walk_of_its_page_search(tmp_path):
    from visrag_b200 import knowledge_base as KB

    rs = np.random.RandomState(91)
    D = _unit(rs, 20000, 256)
    names = [f"doc{i // 40}.pdf_{i % 40}.png" for i in range(len(D) - 100)] + [f"img{i}.jpeg" for i in range(100)]
    KB.save_knowledge_base(str(tmp_path / "kb"), D, names)
    kb = KB.KnowledgeBase(str(tmp_path / "kb"))
    Q = _unit(rs, 300, 256)

    def brute(nq, k, m, scopes):
        """vr_score_exact scores of each query's searched pages (its scope's live pages), walked in (score desc, page
        asc) order with per-document counters."""
        full = _exact_scores(torch.from_numpy(Q[:nq]).cuda(), kb.index).cpu().numpy()
        live = torch.nonzero(kb._live).flatten().tolist()
        cap, hits = [], []
        for r in range(nq):
            cols = np.array(live if scopes[r] is None else sorted(kb.filenames.index(f) for f in scopes[r]))
            count, picks, docs = {}, [], {}
            for p in cols[np.lexsort((cols, -full[r, cols]))]:
                doc, sc = KB.document_of(kb.filenames[p]), float(full[r, p])
                if count.get(doc, 0) < m and len(picks) < k:
                    picks.append((sc, int(p)))
                    count[doc] = count.get(doc, 0) + 1
                if doc not in docs and len(docs) < k:
                    docs[doc] = []
                if doc in docs and len(docs[doc]) < m:
                    docs[doc].append((sc, int(p)))
            cap.append(picks)
            hits.append(list(docs.items()))
        return cap, hits

    def check(what, within=None, each=False):
        for nq in (1, 300):
            scopes = [within] * nq if not each else [None if r % 3 == 0 else within for r in range(nq)]
            for m in (1, 2, 3):
                cap, hits = brute(nq, 10, m, scopes)
                kw = dict(within_each=scopes) if each else dict(within=within)
                s, p = kb.search(Q[:nq], 10, per_document=m, **kw)
                got = [[(a, b) for a, b in zip(sr, pr) if b >= 0] for sr, pr in zip(s.cpu().tolist(), p.cpu().tolist())]
                assert got == cap, (what, nq, m)
                ds, ps, pp, names = kb.search_document_pages(Q[:nq], 10, m, **kw)
                for r in range(nq):
                    want = hits[r]
                    assert names[r] == [d for d, _ in want], (what, nq, m, r)
                    for j, (_, pages) in enumerate(want):
                        row = [(a, b) for a, b in zip(ps[r, j].cpu().tolist(), pp[r, j].cpu().tolist()) if b >= 0]
                        assert row == pages and ds[r, j].item() == pages[0][0], (what, nq, m, r, j)

    within = [f"doc{j}.pdf_{i}.png" for j in range(30, 60) for i in range(0, 40, 4)] + ["img5.jpeg"]  # kept by remove
    check("all")
    check("within", within)
    check("within_each", within, each=True)
    kb.remove([f"doc{j}.pdf_{i}.png" for j in range(0, 200) for i in range(40) if i % 2] + ["img7.jpeg"])
    check("remove")
    check("remove, within_each", within, each=True)
    paths = kb.retrieve(Q[:1], 10, per_document=1)
    _, p = kb.search(Q[:1], 10, per_document=1)
    assert paths == [os.path.join(str(tmp_path / "kb"), kb.filenames[i]) for i in p[0].tolist() if i >= 0]
    short = kb.retrieve(Q[:1], 10, within=["doc40.pdf_0.png", "doc40.pdf_2.png", "img3.jpeg"], per_document=1)
    assert len(short) == 2                                           # two documents: the caps leave two pages
    pages = kb.retrieve_document_pages(Q[:1], 3, 2)
    _, _, pp, names = kb.search_document_pages(Q[:1], 3, 2)
    assert pages == [(n, [os.path.join(str(tmp_path / "kb"), kb.filenames[i]) for i in row if i >= 0])
                     for n, row in zip(names[0], pp[0].tolist())]
