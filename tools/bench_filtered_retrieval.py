"""What a doc mask costs. Workloads: one GPU's shard of bench.py's configs[3] leg (10 k queries x 125 k docs, k = 10,
the tensor-core filter path) and one query over 125 k and over 1 M docs (the fp32 scan with the chunked top-k). Arms: no
mask, an all-ones mask, and random masks keeping 50 %, 10 % and 1 % of the docs. The arms alternate inside every round, so
drift of the shared machine falls on all of them alike; each arm reports its median and spread over the rounds, and the
card's name and power limit are read in the same process. Prints one JSON line per (workload, arm), plus one for the card.
  python tools/bench_filtered_retrieval.py [--rounds 10] [--out results.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import retriever as R  # noqa: E402

ARMS = ("none", "all", "50%", "10%", "1%")


def unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):  # chunked: randn + normalise without a second full-size temporary
        x = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
        out[r0:r0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def masks(nd, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand(nd, device="cuda", generator=g)
    return {"none": None, "all": torch.ones(nd, dtype=torch.bool, device="cuda"), "50%": u < 0.5, "10%": u < 0.1,
            "1%": u < 0.01}


def run(name, Q, index, k, rounds, reps, out):
    ms = masks(index.nd, 7)
    stats = {a: {} for a in ARMS}
    for a in ARMS:                                   # warm-up of every arm's shapes and kernels
        R.score_topk(Q, index, k, doc_mask=ms[a], stats=stats[a])
    torch.cuda.synchronize()
    base = R.score_topk(Q, index, k)
    ones = R.score_topk(Q, index, k, doc_mask=ms["all"])
    same = bool(torch.equal(base[0], ones[0]) and torch.equal(base[1], ones[1]))
    times = {a: [] for a in ARMS}
    for _ in range(rounds):
        for a in ARMS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                R.score_topk(Q, index, k, doc_mask=ms[a])
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / reps)
    for a in ARMS:
        t = sorted(times[a])
        line = {"workload": name, "mask": a, "queries": Q.shape[0], "docs": index.nd, "k": k,
                "eligible": index.nd if ms[a] is None else int(ms[a].sum()), "ms_median": round(t[len(t) // 2], 3),
                "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3), "path": stats[a].get("path"),
                "flagged": stats[a].get("flagged"), "all_ones_equals_no_mask": same}
        print(json.dumps(line), flush=True)
        out.append(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpus", type=int, default=125000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--big", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=2304)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_filtered_retrieval needs a CUDA device")
    out = [{"card": card()}]
    print(json.dumps(out[0]), flush=True)

    D = unit(a.corpus, a.dim, 1)
    index = R.build_index(D)
    run("configs[3] shard: filter path", unit(a.queries, a.dim, 2), index, a.k, a.rounds, 1, out)
    run("one query", unit(1, a.dim, 4), index, a.k, a.rounds, 20, out)
    del D, index
    torch.cuda.empty_cache()
    D = unit(a.big, a.dim, 3)
    index = R.build_index(D)
    run("one query", unit(1, a.dim, 5), index, a.k, a.rounds, 10, out)
    if a.out:
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in out))


if __name__ == "__main__":
    main()
