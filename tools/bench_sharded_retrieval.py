"""What the sharded range search, document range search, hybrid retrieval and MMR cost on one GPU, with W = 8 emulated
shards: 10 k queries (and one query) over 125 k pages split into 8 shards of 15 625, dim 2304, 8-page documents, in a
RANDOM and a CLUSTERED layout. For each function it reports the local stage of one shard (median and max over the
shards: on 8 GPUs the ranks run theirs at once), the merge that every rank runs after the exchange (the exchange
replaced by concatenation in rank order, as tests/test_gpu_sharded_retrieval.py does), the plain call on the whole
index, whether the merged result equals it bit for bit, and the bytes each collective moves, computed from the shapes
(bytes a rank receives). Collective times need one GPU per rank: with two or more GPUs the NCCL arm times each function
end to end on all of them; otherwise they print "not measured". Range search takes each query's threshold at its
100th best score over the whole index. The card's name, power limit and SM clock are printed with every line.
  python tools/bench_sharded_retrieval.py [--rounds 3] [--out results.jsonl]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_grouped_retrieval import card, corpus  # noqa: E402
from tools.bench_hybrid_retrieval import make_hits  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

WORLD, ND, DIM, K, FETCH, WINDOW, N_HITS = 8, 125_000, 2304, 10, 40, 100, 100


def ms(fn, rounds):
    """Median and max of `rounds` CUDA-event timings of fn() after one warm-up call."""
    out = fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    t.sort()
    return out, round(t[len(t) // 2], 3)


def equal(a, b):
    return all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


def bench(layout, nq, rounds, out, gpu):
    Q, D, groups = corpus(ND, DIM, 8, layout, nq, seed=3)
    whole = R.build_index(D)
    spans = torch.tensor([[lo, hi - lo] for lo, hi in (R.shard_range(ND, r, WORLD) for r in range(WORLD))])
    shards = [(int(lo), int(lo + n), R.build_index(D[lo:lo + n].contiguous())) for lo, n in spans.tolist()]
    hits = make_hits(nq, ND, N_HITS, seed=5)
    hits = (hits[0], hits[1].long(), hits[2])
    t = R.score_topk(Q, whole, 100)[0][:, -1].contiguous()
    lam = torch.full((nq,), 0.5, device="cuda")
    res = {}

    def local_times(fn):
        parts, times = [], []
        for r, (lo, hi, ix) in enumerate(shards):
            p, m = ms(lambda: fn(r, lo, hi, ix), rounds)
            parts.append(p)
            times.append(m)
        times.sort()
        return parts, {"local_ms_per_shard_median": times[len(times) // 2], "local_ms_per_shard_max": times[-1]}

    # range search and document range search
    for name, grouped in (("range", False), ("range_groups", True)):
        if grouped:
            parts, info = local_times(lambda r, lo, hi, ix: R._range_entries(*R.score_range_groups(
                Q, ix, t, groups[lo:hi].contiguous(), lo)))
            plain, info["whole_index_ms"] = ms(lambda: R.score_range_groups(Q, whole, t, groups), rounds)
        else:
            parts, info = local_times(lambda r, lo, hi, ix: R._range_entries(*R.score_range(Q, ix, t, lo)))
            plain, info["whole_index_ms"] = ms(lambda: R.score_range(Q, whole, t), rounds)
        got, info["merge_ms"] = ms(lambda: R._merge_range(*R.concat_csr(parts), grouped), rounds)
        largest = max(int(p[0][-1]) for p in parts)
        info.update(equal=equal(got, plain), entries=int(got[0][-1]),
                    bytes={"all_gather counts": WORLD * (nq + 2) * 8, "all_gather entries": WORLD * largest * (24 if grouped else 16)})
        res[name] = info

    # hybrid retrieval: weighted sum over pages and documents, RRF over pages
    parts, info = local_times(lambda r, lo, hi, ix: R.score_topk_hybrid(Q, ix, K, R._local_hits(hits, nq, spans, r, ix, None,
                                                                                               None), id_offset=lo))
    got, info["merge_ms"] = ms(lambda: R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1),
                                                    K), rounds)
    plain, info["whole_index_ms"] = ms(lambda: R.score_topk_hybrid(Q, whole, K, hits), rounds)
    info.update(equal=equal(got, plain), bytes={"all_gather spans": WORLD * 16, "all_gather partials": WORLD * nq * K * 16})
    res["hybrid_sum"] = info

    parts, info = local_times(lambda r, lo, hi, ix: R.score_topk_groups_hybrid(
        Q, ix, K, groups[lo:hi].contiguous(), R._local_hits(hits, nq, spans, r, ix, None, None), id_offset=lo))
    got, info["merge_ms"] = ms(lambda: R.merge_topk_groups(*[torch.cat([p[j] for p in parts], 1) for j in range(3)], K),
                               rounds)
    plain, info["whole_index_ms"] = ms(lambda: R.score_topk_groups_hybrid(Q, whole, K, groups, hits), rounds)
    info.update(equal=equal(got, plain), bytes={"all_gather spans": WORLD * 16, "all_gather partials": WORLD * nq * K * 24})
    res["hybrid_documents_sum"] = info

    parts, info = local_times(lambda r, lo, hi, ix: (R.score_topk(Q, ix, WINDOW, lo),
                                                     R._hit_marks(hits, nq, lo, ix, None, None)))

    def rrf_merge():
        ds, di = R.merge_topk(torch.cat([p[0][0] for p in parts], 1), torch.cat([p[0][1] for p in parts], 1), WINDOW)
        return R._rrf_merge(Q, ds, di, hits, sum(p[1] for p in parts) > 0, K, 60, ND, None)
    got, info["merge_ms"] = ms(rrf_merge, rounds)
    plain, info["whole_index_ms"] = ms(lambda: R.score_topk_hybrid(Q, whole, K, hits, fusion="rrf", window=WINDOW), rounds)
    info.update(equal=equal(got, plain), bytes={"all_gather spans": WORLD * 16, "all_gather dense": WORLD * nq * WINDOW * 16,
                                                "all_reduce marks (payload)": hits[1].shape[0] * 4})
    res["hybrid_rrf"] = info

    # MMR: candidates per shard; the merge is the candidates' merge, the routing and one rank's selection
    parts, info = local_times(lambda r, lo, hi, ix: R.score_topk(Q, ix, FETCH, lo))
    s, i = R.merge_topk(torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1), FETCH)
    routes = R._mmr_routes(i, spans, WORLD)
    sends = [torch.split(R._mmr_send(ix, i, spans, r), routes[:, r].tolist()) for r, (_, _, ix) in enumerate(shards)]
    picks, sel = [], []
    for r in range(WORLD):
        lo, hi = R.shard_range(nq, r, WORLD)
        recv = torch.cat([sends[src][r] for src in range(WORLD)])
        p, m = ms(lambda: R._mmr_block(s[lo:hi], i[lo:hi], recv, spans, K, lam[lo:hi]), rounds)
        picks.append(p)
        sel.append(m)
    _, info["merge_candidates_ms"] = ms(lambda: R.merge_topk(torch.cat([p[0] for p in parts], 1),
                                                             torch.cat([p[1] for p in parts], 1), FETCH), rounds)
    info["select_ms_per_rank_max"] = max(sel)
    got = (torch.cat([p[0] for p in picks]), torch.cat([p[1] for p in picks]))
    plain, info["whole_index_ms"] = ms(lambda: R.score_mmr(Q, whole, K, 0.5, FETCH), rounds)
    per = -(-nq // WORLD)
    info.update(equal=equal(got, plain),
                bytes={"all_gather spans": WORLD * 16, "all_gather candidates": WORLD * nq * FETCH * 16,
                       "all_to_all rows (largest rank)": int(routes.sum(1).max()) * DIM * 4,
                       "all_gather picks": WORLD * per * K * 16})
    res["mmr"] = info

    for name, info in res.items():
        info["collective_ms"] = "not measured" if torch.cuda.device_count() < 2 else "see the nccl lines"
        line = {"card": gpu, "workload": f"{layout} {nq}q x {ND}p, {WORLD} shards, dim {DIM}", "function": name, **info}
        print(json.dumps(line), flush=True)
        if out:
            out.write(json.dumps(line) + "\n")


def _nccl_worker(rank, world, port, rounds, q_out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        for layout in ("random", "clustered"):
            Q, D, groups = corpus(ND, DIM, 8, layout, 10_000, seed=3)
            lo, hi = R.shard_range(ND, rank, world)
            ix, mine = R.build_index(D[lo:hi].contiguous()), groups[lo:hi].contiguous()
            hits = make_hits(10_000, ND, N_HITS, seed=5)
            hits = (hits[0], hits[1].long(), hits[2])
            t = 0.5 if layout == "clustered" else 0.08
            fns = {"range": lambda: R.sharded_range(Q, ix, t, lo),
                   "range_groups": lambda: R.sharded_range_groups(Q, ix, t, mine, lo),
                   "hybrid_sum": lambda: R.sharded_topk_hybrid(Q, ix, K, hits, lo),
                   "hybrid_documents_sum": lambda: R.sharded_topk_groups_hybrid(Q, ix, K, mine, hits, lo),
                   "hybrid_rrf": lambda: R.sharded_topk_hybrid(Q, ix, K, hits, lo, fusion="rrf", window=WINDOW),
                   "mmr": lambda: R.sharded_mmr(Q, ix, K, 0.5, FETCH, lo)}
            for name, fn in fns.items():
                dist.barrier()
                _, m = ms(fn, rounds)
                if rank == 0:
                    q_out.put({"workload": f"{layout} 10000q x {ND}p over {world} GPUs (nccl)", "function": name,
                               "end_to_end_ms": m})
    finally:
        q_out.put(None)
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sharded_retrieval measures the GPU: no CUDA device"
    out = open(args.out, "w") if args.out else None
    gpu = card()
    for layout in ("random", "clustered"):
        for nq in (10_000, 1):
            bench(layout, nq, args.rounds, out, gpu)
            torch.cuda.empty_cache()
    world = torch.cuda.device_count()
    if world < 2:
        print(json.dumps({"card": gpu, "nccl": "not measured: one GPU"}), flush=True)
        return
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29600 + os.getpid() % 1000, args.rounds, q))
             for r in range(world)]
    for p in procs:
        p.start()
    done = 0
    while done < world:
        line = q.get(timeout=1800)
        if line is None:
            done += 1
            continue
        line = {"card": gpu, **line}
        print(json.dumps(line), flush=True)
        if out:
            out.write(json.dumps(line) + "\n")
    for p in procs:
        p.join(60)


if __name__ == "__main__":
    main()
