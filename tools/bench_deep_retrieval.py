"""What deep top-k costs (retriever.score_topk at k up to 1000), dim 2304. Arms, alternating inside every round: the
default routes ("new": the radix select vr_select_rows for k > SELECT_K_MIN, the deep route for DEEP_K_MIN < k <=
DEEP_K_MAX); the k-pass selection everywhere ("k-pass": SELECT_K_MIN and DEEP_K_MIN raised past k, the routes of the
parent commit); and torch outside the library (fp32 matmul + torch.topk over row blocks). Workloads: 10 k queries x
125 k random unit pages, and planted near-duplicate clusters (5 noisy copies of each of 25 k pages) with queries near
pages; 1 query x 125 k and x 1 M random pages. Each line: median (min - max) ms per arm over the rounds, the new arm's
stats (path, fallback rows, stage times), and whether every arm's ids equal the fp32 scan's (torch may differ: cuBLAS
sums in another order). The card's name, power limit and SM clocks are read in the same run.
  python tools/bench_deep_retrieval.py [--rounds 3] [--ks 10,32,100,128,1000] [--out results.jsonl]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import retriever as R  # noqa: E402

DIM = 2304


def unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):
        x = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
        out[r0:r0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1)
    return out


def clustered(n, per, d, seed):
    c = unit(n // per, d, seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    for r0 in range(0, n, 65536):
        m = min(65536, n - r0)
        x = c[torch.arange(r0, r0 + m, device="cuda") // per] + 0.05 * torch.randn((m, d), device="cuda", generator=g) / d ** 0.5
        out[r0:r0 + m] = torch.nn.functional.normalize(x, dim=1)
    return out


def near(docs, nq, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pick = torch.randint(0, docs.shape[0], (nq,), device="cuda", generator=g)
    return torch.nn.functional.normalize(docs[pick] + 0.3 * unit(nq, docs.shape[1], seed + 1), dim=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def torch_topk(q, idx, k):
    s, i = [], []
    step = max(1, (1 << 28) // idx.nd)
    for r0 in range(0, q.shape[0], step):
        v, j = torch.topk(q[r0:r0 + step] @ idx.emb.T, min(k, idx.nd), dim=1)
        s.append(v)
        i.append(j)
    return torch.cat(s), torch.cat(i)


def kpass(q, idx, k):
    saved = R.SELECT_K_MIN, R.DEEP_K_MIN
    R.SELECT_K_MIN = R.DEEP_K_MIN = 1 << 30
    try:
        return R.score_topk(q, idx, k)
    finally:
        R.SELECT_K_MIN, R.DEEP_K_MIN = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ks", default="10,32,100,128,1000")
    ap.add_argument("--workloads", default="random,clustered,1x125k,1x1M")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    print("card:", card(), flush=True)
    lines = []
    for wl in a.workloads.split(","):
        if wl == "random":
            D, Q = unit(125_000, DIM, 1), unit(10_000, DIM, 2)
        elif wl == "clustered":
            D = clustered(125_000, 5, DIM, 3)
            Q = near(D, 10_000, 4)
        elif wl == "1x125k":
            D, Q = unit(125_000, DIM, 5), unit(1, DIM, 6)
        else:
            D, Q = unit(1_000_000, DIM, 7), unit(1, DIM, 8)
        idx = R.build_index(D)
        del D
        for k in ks:
            arms = {"new": lambda: R.score_topk(Q, idx, k), "k-pass": lambda: kpass(Q, idx, k),
                    "torch": lambda: torch_topk(Q, idx, k)}
            ref = R.score_topk(Q, idx, k, force_exact=True)  # the fp32 scan (its selection as routed)
            times = {n: [] for n in arms}
            same = {}
            for name, fn in arms.items():  # warm-up, and the ids check
                _, out = timed(fn)
                same[name] = bool(torch.equal(out[1], ref[1]))
            for _ in range(a.rounds):
                for name, fn in arms.items():
                    times[name].append(timed(fn)[0])
            stats = {"stages": {}}
            R.score_topk(Q, idx, k, stats=stats)
            torch.cuda.synchronize()
            R.resolve_stages(stats)
            rec = dict(workload=wl, nq=Q.shape[0], nd=idx.nd, k=k, same_ids=same,
                       ms={n: [statistics.median(t), min(t), max(t)] for n, t in times.items()},
                       path=stats.get("path"), fallback=stats.get("fallback", stats.get("flagged")),
                       stages={n: round(v, 3) for n, v in stats["stages"].items()})
            lines.append(rec)
            print(json.dumps(rec), flush=True)
        del idx
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
