"""Sharded range search, document range search, hybrid retrieval and MMR on the H100: one index split into W uneven
shards on one GPU, every rank's local stage run, the exchange replaced by concatenation in rank order, and the merge
run; the result must equal (torch.equal on scores, ids and groups) the plain call on the concatenated index. Also the
world-1 forms without torch.distributed and a two-process NCCL run of all five functions."""
import os

import numpy as np
import pytest
import torch

from visrag_b200 import retriever as R

pytestmark = pytest.mark.gpu

SIZES = {2: [21000, 39000], 3: [25000, 200, 34800], 5: [30000, 100, 12000, 17000, 900]}  # 60 000 pages; < 256: scan


def _same(a, b, what):
    assert len(a) == len(b), what
    for j, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and x.dtype == y.dtype and torch.equal(x, y), \
            (what, j, int((x != y).sum()) if x.shape == y.shape else (x.shape, y.shape))


def _data(kind, nq=200, nd=60000, d=128, seed=0):
    """Unit rows: random, or clustered (40 centres, small noise, every 97th page a copy of the page before it)."""
    rs = np.random.RandomState(seed)
    if kind == "random":
        D = rs.randn(nd, d).astype(np.float32)
        Q = rs.randn(nq, d).astype(np.float32)
    else:
        C = rs.randn(40, d).astype(np.float32)
        D = C[rs.randint(0, 40, nd)] + 0.15 * rs.randn(nd, d).astype(np.float32)
        D[97::97] = D[96:-1:97][:len(D[97::97])]
        Q = C[rs.randint(0, 40, nq)] + 0.3 * rs.randn(nq, d).astype(np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return torch.from_numpy(Q).cuda(), torch.from_numpy(D).cuda()


def _shards(D, world):
    sizes = SIZES[world]
    los = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    out = [(int(lo), int(lo + n), R.build_index(D[lo:lo + n].contiguous())) for lo, n in zip(los, sizes)]
    spans = torch.tensor([[lo, hi - lo] for lo, hi, _ in out], dtype=torch.int64)
    return out, spans


def _cut(m, lo, hi):
    return None if m is None else m[..., lo:hi].contiguous()


# ------------------------------------------------------------------------------------------------------
# Range search and document range search
# ------------------------------------------------------------------------------------------------------
def _sharded_range(q, shards, t, groups=None, mask=None, mask_of=None, cap=None):
    parts = []
    for lo, hi, ix in shards:
        if groups is None:
            parts.append(R._range_entries(*R.score_range(q, ix, t, lo, _cut(mask, lo, hi), mask_of, cap=cap)))
        else:
            parts.append(R._range_entries(*R.score_range_groups(q, ix, t, groups[lo:hi].contiguous(), lo, _cut(mask, lo, hi),
                                                                mask_of, cap=cap)))
    return R._merge_range(*R.concat_csr(parts), groups is not None)


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_range_search_merges_to_the_whole_index(world, kind):
    q, D = _data(kind, seed=world)
    whole = R.build_index(D)
    shards, _ = _shards(D, world)
    t_row = torch.full((q.shape[0],), 0.25 if kind == "random" else 0.8, device="cuda")
    t_row[::7] = 2.0                                   # rows with no result
    t_row[5] = 0.0                                     # a row with far more candidates than cap 2000: it falls back
    for t, cap, what in ((0.25 if kind == "random" else 0.85, None, "float"), (t_row, 2000, "per-query")):
        stats = {}
        want = R.score_range(q, whole, t, cap=cap, stats=stats)
        assert stats["path"] == "filter+rescore" and (cap is None or stats["fallback"] >= 1), stats
        _same(_sharded_range(q, shards, t, cap=cap), want, (what, world, kind))
    _same(_sharded_range(q[:8], shards, float("-inf")), R.score_range(q[:8], whole, float("-inf")), "-inf")
    rs = np.random.RandomState(world)
    mask = torch.from_numpy(rs.rand(D.shape[0]) < 0.6).cuda()
    _same(_sharded_range(q, shards, 0.2, mask=mask), R.score_range(q, whole, 0.2, doc_mask=mask), "mask")
    masks = torch.from_numpy(rs.rand(3, D.shape[0]) < 0.5).cuda()
    of = torch.from_numpy(rs.randint(0, 3, q.shape[0])).cuda()
    _same(_sharded_range(q, shards, t_row, mask=masks, mask_of=of), R.score_range(q, whole, t_row, doc_mask=masks, mask_of=of),
          "per-query masks")


def _documents(nd, world, D):
    """70-page documents straddling the shard boundaries, one document spanning the first three shards (for W = 2: both),
    and inside it a page on the first shard copied to the last shard (equal best scores on two ranks)."""
    groups = np.arange(nd) // 70
    sizes = SIZES[world]
    b0 = sizes[0]
    span_hi = b0 + sizes[1] + 50 if world > 2 else b0 + 50
    groups[b0 - 50:span_hi] = nd                        # one document over shards 0, 1 (and 2)
    D[span_hi - 1] = D[b0 - 40]
    return torch.from_numpy(groups).cuda()


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_document_range_search_merges_to_the_whole_index(world, kind):
    q, D = _data(kind, seed=10 + world)
    groups = _documents(D.shape[0], world, D)
    whole = R.build_index(D)
    shards, _ = _shards(D, world)
    t = 0.2 if kind == "random" else 0.8
    want = R.score_range_groups(q, whole, t, groups)
    _same(_sharded_range(q, shards, t, groups), want, ("documents", world, kind))
    # the copied page: the document's two best pages have one score, on two ranks; the lower page wins
    nd = D.shape[0]
    q2 = D[[SIZES[world][0] - 40]].clone()
    got = _sharded_range(q2, shards, 0.5, groups)
    _same(got, R.score_range_groups(q2, whole, 0.5, groups), "tie")
    assert int(got[2][(got[3] == nd).nonzero()[0, 0]]) == SIZES[world][0] - 40
    rs = np.random.RandomState(world)
    masks = torch.from_numpy(rs.rand(4, nd) < 0.5).cuda()
    of = torch.from_numpy(rs.randint(0, 4, q.shape[0])).cuda()
    t_row = torch.full((q.shape[0],), t, device="cuda")
    t_row[::5] = 5.0
    _same(_sharded_range(q, shards, t_row, groups, masks, of, cap=3000),
          R.score_range_groups(q, whole, t_row, groups, doc_mask=masks, mask_of=of, cap=3000), "documents, masks")
    _same(_sharded_range(q[:6], shards, float("-inf"), groups), R.score_range_groups(q[:6], whole, float("-inf"), groups),
          "documents, -inf")


# ------------------------------------------------------------------------------------------------------
# Hybrid retrieval
# ------------------------------------------------------------------------------------------------------
def _hits(rs, nq, nd, per_row, where=None):
    """Global hits: per_row random pages a row (from `where` when given), values in [0, 1)."""
    ids, offs = [], [0]
    pool = np.arange(nd) if where is None else where
    for _ in range(nq):
        n = rs.randint(0, per_row + 1)
        ids.append(rs.choice(pool, n, replace=False))
        offs.append(offs[-1] + n)
    ids = np.concatenate(ids)
    return (torch.tensor(offs, dtype=torch.int64).cuda(), torch.from_numpy(ids.astype(np.int64)).cuda(),
            torch.from_numpy(rs.rand(len(ids)).astype(np.float32)).cuda())


def _hybrid_pages(q, shards, spans, k, hits, w, fusion, window, mask):
    nq = q.shape[0]
    if fusion == "sum":
        parts = []
        for r, (lo, hi, ix) in enumerate(shards):
            _, masks, ls = R._scope(q, ix, _cut(mask, lo, hi), None, None, None)
            local = R._local_hits(hits, nq, spans, r, ix, masks, ls)
            parts.append(R.score_topk_hybrid(q, ix, k, local, w, id_offset=lo, doc_mask=_cut(mask, lo, hi)))
        return R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1), k)
    dense = [R.score_topk(q, ix, window, lo, doc_mask=_cut(mask, lo, hi)) for lo, hi, ix in shards]
    ds, di = R.merge_topk(torch.cat([p[0] for p in dense], 1), torch.cat([p[1] for p in dense], 1), window)
    marks = sum(R._hit_marks(hits, nq, lo, ix, R._scope(q, ix, _cut(mask, lo, hi), None, None, None)[1], None)
                for lo, hi, ix in shards)
    return R._rrf_merge(q, ds, di, hits, marks > 0, k, 60, int(spans[:, 1].sum()), None)


def _hybrid_documents(q, shards, spans, k, groups, hits, w, mask):
    parts = []
    for r, (lo, hi, ix) in enumerate(shards):
        _, masks, ls = R._scope(q, ix, _cut(mask, lo, hi), None, None, None)
        local = R._local_hits(hits, q.shape[0], spans, r, ix, masks, ls)
        parts.append(R.score_topk_groups_hybrid(q, ix, k, groups[lo:hi].contiguous(), local, w, id_offset=lo,
                                                doc_mask=_cut(mask, lo, hi)))
    return R.merge_topk_groups(*[torch.cat([p[j] for p in parts], 1) for j in range(3)], k)


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_hybrid_merges_to_the_whole_index(world, kind):
    q, D = _data(kind, seed=20 + world)
    nq, nd = q.shape[0], D.shape[0]
    groups = _documents(nd, world, D)
    whole = R.build_index(D)
    shards, spans = _shards(D, world)
    rs = np.random.RandomState(world)
    mask = torch.from_numpy(rs.rand(nd) < 0.7).cuda()
    cases = {"every shard": _hits(rs, nq, nd, 40),
             "none": _hits(rs, nq, nd, 0),
             "last shard only": _hits(rs, nq, nd, 30, np.arange(nd - SIZES[world][-1], nd))}
    for name, hits in cases.items():
        for m in (None, mask):  # the mask drops hits outside it
            for fusion, window in (("sum", None), ("rrf", 10), ("rrf", 1000)):
                want = R.score_topk_hybrid(q, whole, 10, hits, 0.3, fusion, window, doc_mask=m)
                got = _hybrid_pages(q, shards, spans, 10, hits, 0.3, fusion, window, m)
                _same(got, want, (name, m is not None, fusion, window, world))
            want = R.score_topk_groups_hybrid(q, whole, 10, groups, hits, 0.3, doc_mask=m)
            _same(_hybrid_documents(q, shards, spans, 10, groups, hits, 0.3, m), want, (name, m is not None, "docs", world))


# ------------------------------------------------------------------------------------------------------
# MMR
# ------------------------------------------------------------------------------------------------------
def _sharded_mmr(q, shards, spans, k, lam, fetch):
    world, nq = len(shards), q.shape[0]
    dense = [R.score_topk(q, ix, fetch, lo) for lo, hi, ix in shards]
    s, i = R.merge_topk(torch.cat([p[0] for p in dense], 1), torch.cat([p[1] for p in dense], 1), fetch)
    routes = R._mmr_routes(i, spans, world)
    sends = [torch.split(R._mmr_send(ix, i, spans, r), routes[:, r].tolist()) for r, (_, _, ix) in enumerate(shards)]
    lam = torch.full((nq,), lam, device="cuda")
    out = []
    for r in range(world):
        lo, hi = R.shard_range(nq, r, world)
        recv = torch.cat([sends[src][r] for src in range(world)])
        out.append(R._mmr_block(s[lo:hi], i[lo:hi], recv, spans, k, lam[lo:hi]))
    return torch.cat([o[0] for o in out]), torch.cat([o[1] for o in out])


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["random", "clustered"])
def test_mmr_merges_to_the_whole_index(world, kind):
    q, D = _data(kind, nq=90, seed=30 + world)
    whole = R.build_index(D)
    shards, spans = _shards(D, world)
    for lam in (0.0, 0.5, 1.0):
        for fetch, k in ((20, 8), (128, 30)):
            want = R.score_mmr(q, whole, k, lam, fetch)
            _same(_sharded_mmr(q, shards, spans, k, lam, fetch), want, (lam, fetch, world, kind))
    # a shard that holds none of a query's candidates: the 100-page shard of W = 5 against a far query
    s, i = R.score_topk(q, whole, 20)
    assert bool(((i >= 30000) & (i < 30100)).sum(1).eq(0).any())


# ------------------------------------------------------------------------------------------------------
# World 1 and NCCL
# ------------------------------------------------------------------------------------------------------
def test_world_one_returns_the_plain_calls():
    q, D = _data("random", nq=50, nd=20000, seed=40)
    ix = R.build_index(D)
    g = torch.arange(D.shape[0], device="cuda") // 9
    rs = np.random.RandomState(40)
    hits = _hits(rs, 50, D.shape[0], 20)
    _same(R.sharded_range(q, ix, 0.2, 0), R.score_range(q, ix, 0.2), "range")
    _same(R.sharded_range_groups(q, ix, 0.2, g, 0), R.score_range_groups(q, ix, 0.2, g), "range groups")
    for fusion, window in (("sum", None), ("rrf", 100)):
        _same(R.sharded_topk_hybrid(q, ix, 10, hits, 0, fusion=fusion, window=window, weight=0.5),
              R.score_topk_hybrid(q, ix, 10, hits, 0.5, fusion, window), fusion)
    _same(R.sharded_topk_groups_hybrid(q, ix, 600, g, hits, 0), R.score_topk_groups_hybrid(q, ix, 600, g, hits), "docs")
    _same(R.sharded_mmr(q, ix, 5, 0.5, 20, 0), R.score_mmr(q, ix, 5, 0.5, 20), "mmr")
    # an id_offset shifts the pages out and the hits in
    shifted = (hits[0], hits[1] + 7, hits[2])
    a, b = R.sharded_topk_hybrid(q, ix, 10, shifted, 7), R.score_topk_hybrid(q, ix, 10, hits, id_offset=7)
    _same(a, b, "id_offset")


def _nccl_worker(rank, world, port, out_q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        dev = f"cuda:{rank}"
        g = torch.Generator(device=dev).manual_seed(4324)
        D = torch.nn.functional.normalize(torch.randn(24000, 256, device=dev, generator=g), dim=1)
        Q = torch.nn.functional.normalize(torch.randn(500, 256, device=dev, generator=g), dim=1)
        groups = torch.arange(24000, device=dev) // 70        # 12000 is no multiple of 70: a document straddles the shards
        n = torch.randint(0, 30, (500,), device=dev, generator=g)
        offsets = torch.zeros(501, dtype=torch.int64, device=dev)
        offsets[1:] = torch.cumsum(n, 0)
        ids = torch.cat([torch.randperm(24000, device=dev, generator=g)[:int(c)] for c in n.tolist()])
        hits = (offsets, ids, torch.rand(ids.shape[0], device=dev, generator=g))
        lo, hi = R.shard_range(D.shape[0], rank, world)
        index, full = R.build_index(D[lo:hi].contiguous()), R.build_index(D)
        mine = groups[lo:hi].contiguous()
        res = {}
        res["range"] = (R.sharded_range(Q, index, 0.15, lo), R.score_range(Q, full, 0.15))
        res["range_groups"] = (R.sharded_range_groups(Q, index, 0.15, mine, lo), R.score_range_groups(Q, full, 0.15, groups))
        res["hybrid sum"] = (R.sharded_topk_hybrid(Q, index, 10, hits, lo, weight=0.4), R.score_topk_hybrid(Q, full, 10, hits, 0.4))
        res["hybrid rrf"] = (R.sharded_topk_hybrid(Q, index, 10, hits, lo, fusion="rrf", window=200),
                             R.score_topk_hybrid(Q, full, 10, hits, fusion="rrf", window=200))
        res["hybrid docs"] = (R.sharded_topk_groups_hybrid(Q, index, 10, mine, hits, lo, weight=0.4),
                              R.score_topk_groups_hybrid(Q, full, 10, groups, hits, 0.4))
        res["mmr"] = (R.sharded_mmr(Q, index, 10, 0.5, 40, lo), R.score_mmr(Q, full, 10, 0.5, 40))
        bad = [name for name, (a, b) in res.items() if not all(torch.equal(x, y) for x, y in zip(a, b))]
        out_q.put((rank, bad))
    finally:
        dist.destroy_process_group()


def test_sharded_retrieval_under_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() + 900) % 1000
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == [0, 1] and all(not r[1] for r in res), res
