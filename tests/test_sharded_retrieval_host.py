"""Host-side parts of the sharded range search, document range search, hybrid retrieval and MMR: gloo runs at world 2
and 3 of the exchanges (the variable-length CSR gather, the MMR row routing, the RRF scope-mark combine) against plain
concatenation in rank order, and the refusals (shard ranges, hits, RRF over documents, world * k over the group merge)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from visrag_b200 import retriever as R


def _csr(rs, nq, max_len, empty=False):
    """A random CSR (offsets, entries int64 [n, 3]) with empty rows; empty=True: no entry at all."""
    lens = np.where(rs.rand(nq) < 0.3, 0, rs.randint(0, max_len + 1, nq)) * (0 if empty else 1)
    offsets = torch.zeros(nq + 1, dtype=torch.int64)
    offsets[1:] = torch.from_numpy(np.cumsum(lens))
    entries = torch.from_numpy(rs.randint(-2**40, 2**40, (int(lens.sum()), 3)))
    return offsets, entries


def _rank_csr(seed, rank, nq):
    rs = np.random.RandomState(seed + 17 * rank)
    return _csr(rs, nq, 9, empty=(rank == 1))  # rank 1 holds nothing


def _by_rows(offsets, entries):
    return [entries[int(offsets[r]):int(offsets[r + 1])] for r in range(offsets.shape[0] - 1)]


def _hits(rs, nq, total, per_row):
    ids, offs = [], [0]
    for _ in range(nq):
        n = rs.randint(0, per_row + 1)
        ids.append(rs.choice(total, n, replace=False))
        offs.append(offs[-1] + n)
    ids = np.concatenate(ids)
    return (torch.tensor(offs, dtype=torch.int64), torch.from_numpy(ids.astype(np.int64)),
            torch.from_numpy(rs.rand(len(ids)).astype(np.float32)))


def _spans(sizes):
    lo = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    return torch.tensor(np.stack([lo, sizes], 1), dtype=torch.int64)


def _worker(rank, world, port, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fails = []
        # 1. the variable-length CSR gather, with a rank and rows that hold nothing, and nq = 0
        for nq in (7, 1, 0):
            parts = [_rank_csr(3, r, nq) for r in range(world)]
            off, ent, heads = R.gather_csr(*parts[rank], head=torch.tensor([rank, 10 * rank]))
            want_off, want_ent = R.concat_csr(parts)
            rows = [torch.cat([_by_rows(*p)[r] for p in parts]) for r in range(nq)]
            if not (torch.equal(off, want_off) and torch.equal(ent, want_ent) and heads.tolist() == [[r, 10 * r] for r in range(world)]
                    and all(torch.equal(a, b) for a, b in zip(_by_rows(off, ent), rows))):
                fails.append(("csr", nq))
        # 2. MMR row routing: uneven shards (one empty), -1 candidates, uneven query blocks
        sizes = np.array([31, 0, 12]) if world == 3 else np.array([29, 14])
        spans, dim = _spans(sizes), 8
        total = int(sizes.sum())
        emb = torch.from_numpy(np.random.RandomState(8).randn(total, dim).astype(np.float32))
        for nq, fetch in ((7, 6), (2, 5)):  # nq = 2 < world 3: a rank without queries
            rs = np.random.RandomState(nq)
            ids = torch.from_numpy(np.stack([np.concatenate([rs.choice(total, m, replace=False), -np.ones(fetch - m, np.int64)])
                                             for m in rs.randint(0, fetch + 1, nq)]))
            lo = int(spans[rank, 0])
            index = R.CorpusIndex(emb[lo:lo + int(sizes[rank])].contiguous(), None, None)
            routes = R._mmr_routes(ids, spans, world)
            recv = R._all_to_all_rows(R._mmr_send(index, ids, spans, rank), routes[:, rank].tolist(), routes[rank].tolist(), None)
            qlo, qhi = R.shard_range(nq, rank, world)
            buf, pos = R._mmr_place(ids[qlo:qhi], recv, spans)
            block = ids[qlo:qhi]
            ok = torch.equal(pos >= 0, block >= 0) and torch.equal(buf[pos[pos >= 0]], emb[block[block >= 0]])
            ok &= int(routes.sum()) == int((ids >= 0).sum()) and recv.shape[0] == int((block >= 0).sum())
            # the picks' gather (gather_queries over int64 blocks) restores query order
            picks = torch.stack([block, block + 1], -1).view(qhi - qlo, 2 * fetch)
            ok &= torch.equal(R.gather_queries(picks, nq).view(nq, fetch, 2)[..., 0], ids)
            if not ok:
                fails.append(("mmr", nq, fetch))
        # 3. the RRF scope marks: only a hit's owner applies the scope; the all-reduce gives the whole index's answer
        nq = 6
        rs = np.random.RandomState(11)
        hits = _hits(rs, nq, total, 12)
        whole = R.CorpusIndex(emb, None, None)
        mask = torch.from_numpy(rs.rand(nq, total) < 0.5)
        lo = int(spans[rank, 0])
        index = R.CorpusIndex(emb[lo:lo + int(sizes[rank])].contiguous(), None, None)
        for scoped in (False, True):
            masks = R._check_doc_mask(mask[:, lo:lo + int(sizes[rank])], index, nq) if scoped and sizes[rank] else None
            keep = R._combine_marks(R._hit_marks(hits, nq, lo, index, masks, None), None)
            rows = R._hit_rows(hits[0], hits[1].shape[0], nq)
            want = R._hits_in_scope(rows, hits[1], total, R._check_doc_mask(mask, whole, nq) if scoped else None, None)
            if not torch.equal(keep, want):
                fails.append(("rrf marks", scoped))
        # 4. the document merge limit holds at world > 1, checked before any work
        try:
            R.sharded_topk_groups_hybrid(torch.zeros(2, 8), index, R.MERGE_GROUPS_MAX // world + 1, torch.zeros(1),
                                         hits, lo)
            fails.append("world * k")
        except ValueError as e:
            if "world * k" not in str(e):
                fails.append(("world * k", str(e)))
        out_q.put((rank, fails))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_exchanges_under_gloo(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 37 * world) % 2000
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(60)
    assert sorted(r[0] for r in res) == list(range(world))
    assert all(not r[1] for r in res), res


def test_concat_csr_lays_rows_out_in_part_order():
    rs = np.random.RandomState(1)
    parts = [_csr(rs, 5, 4) for _ in range(3)] + [_csr(rs, 5, 4, empty=True)]
    off, ent = R.concat_csr(parts)
    for r, row in enumerate(_by_rows(off, ent)):
        assert torch.equal(row, torch.cat([_by_rows(*p)[r] for p in parts]))
    # entries past a part's offsets[-1] (the padding of the gather) are ignored
    padded = [(o, torch.cat([e, torch.full((3, 3), 7)])) for o, e in parts]
    assert all(torch.equal(a, b) for a, b in zip(R.concat_csr(padded), (off, ent)))


def test_shard_ranges_must_follow_each_other_from_page_zero():
    assert R._check_spans(_spans(np.array([4, 0, 6]))).tolist() == [4, 4, 10]
    for bad in ([[0, 5], [4, 3]],           # overlapping
                [[0, 5], [6, 3]],           # a gap
                [[5, 3], [0, 5]],           # out of rank order
                [[1, 5], [6, 2]],           # not from page 0
                [[0, 5], [5, -1]]):
        with pytest.raises(ValueError, match="follow each other"):
            R._check_spans(torch.tensor(bad))
    with pytest.raises(ValueError, match="2\\^31"):
        R._check_spans(torch.tensor([[0, 2**30], [2**30, 2**30]]))


def test_local_hits_are_checked_against_the_whole_corpus():
    spans = _spans(np.array([6, 4, 5]))
    emb = torch.zeros(15, 8)
    idx = [R.CorpusIndex(emb[lo:lo + n].contiguous(), None, None) for lo, n in spans.tolist()]
    hits = (torch.tensor([0, 3, 5]), torch.tensor([14, 2, 7, 6, 0]), torch.tensor([1.0, 2.0, 3.0, 4.0, -0.0]))
    got = [R._local_hits(hits, 2, spans, r, idx[r], None, None) for r in range(3)]
    # rank 0: pages 2 (row 0), 0 (row 1); rank 1: 7 (row 0), 6 (row 1) as 1 and 0; rank 2: 14 (row 0) as 4
    assert [g[0].tolist() for g in got] == [[0, 1, 2], [0, 1, 2], [0, 1, 1]]
    assert [g[1].tolist() for g in got] == [[2, 0], [1, 0], [4]]
    assert [g[2].tolist() for g in got] == [[2.0, 0.0], [3.0, 4.0], [1.0]]
    assert all(g[1].dtype == torch.int32 for g in got)
    bad = {"repeat": (torch.tensor([0, 2]), torch.tensor([8, 8]), torch.tensor([1.0, 1.0])),
           "range": (torch.tensor([0, 1]), torch.tensor([15]), torch.tensor([1.0])),
           "negative id": (torch.tensor([0, 1]), torch.tensor([-1]), torch.tensor([1.0])),
           "negative": (torch.tensor([0, 1]), torch.tensor([3]), torch.tensor([-1.0])),
           "nan": (torch.tensor([0, 1]), torch.tensor([3]), torch.tensor([float("nan")])),
           "offsets": (torch.tensor([0, 2]), torch.tensor([3]), torch.tensor([1.0]))}
    for name, h in bad.items():
        for r in range(3):  # every rank refuses, whichever rank holds the page
            with pytest.raises(ValueError):
                R._local_hits(h, 1, spans, r, idx[r], None, None)
    with pytest.raises(ValueError, match="triple"):
        R._hit_marks((torch.tensor([0, 1]), torch.tensor([3])), 1, 0, idx[0], None, None)


def test_rrf_over_documents_and_bad_weights_are_refused():
    idx = R.CorpusIndex(torch.zeros(4, 8), None, None)
    hits = (torch.tensor([0, 0]), torch.zeros(0, dtype=torch.int64), torch.zeros(0))
    with pytest.raises(ValueError, match="weighted sum only"):
        R.sharded_topk_groups_hybrid(torch.zeros(1, 8), idx, 5, torch.zeros(4, dtype=torch.int64), hits, 0, fusion="rrf")
    for w in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="weight"):
            R.sharded_topk_hybrid(torch.zeros(1, 8), idx, 5, hits, 0, weight=w)
        with pytest.raises(ValueError, match="weight"):
            R.sharded_topk_groups_hybrid(torch.zeros(1, 8), idx, 5, torch.zeros(4, dtype=torch.int64), hits, 0, weight=w)
    with pytest.raises(ValueError, match="fusion"):
        R.sharded_topk_hybrid(torch.zeros(1, 8), idx, 5, hits, 0, fusion="max")


def test_mmr_routes_count_each_candidate_once():
    spans = _spans(np.array([3, 7, 0, 5]))
    ids = torch.tensor([[0, 9, 12, -1], [4, 3, -1, -1], [14, 2, 1, 10], [-1, -1, -1, -1], [5, 6, 7, 8]])
    routes = R._mmr_routes(ids, spans, 4)   # query blocks [0, 2), [2, 3), [3, 4), [4, 5)
    assert routes.tolist() == [[1, 3, 0, 1], [2, 0, 0, 2], [0, 0, 0, 0], [0, 4, 0, 0]]
