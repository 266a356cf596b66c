"""What document-level retrieval costs. Workloads, each timed as page-level `score_topk` against `score_topk_groups`:
one GPU's shard of bench.py's configs[3] leg (10 k queries x 125 k pages at dim 2304, k = 10, the tensor-core filter
path) with documents of 1, 8 and 64 contiguous pages, in a CLUSTERED layout (each document a centre plus small noise,
queries near document centres: the layout of a knowledge base built from PDFs, where page lists fill up with one
document) and a RANDOM layout (pages independent); then one query over 125 k and over 1 M pages (the exact path), with
documents of 8 and of 1024 pages. Each filter-path line also gives the stage times of one untimed call of each arm
(CUDA events: the filter and the rescoring), which is where the difference between the arms lies.
For the clustered layout it also reports the fraction of queries whose proof fails (and rerun through the exact path)
with the group-distinct filter and with page lists fed to the grouped rescoring. The arms alternate inside every round,
so drift of the shared machine falls on both; each reports its median and spread over the rounds, and the card's name
and power limit are read in the same process. Prints one JSON line per (workload, arm), plus one for the card.
  python tools/bench_grouped_retrieval.py [--rounds 5] [--out results.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import retriever as R  # noqa: E402


def unit(x):
    return torch.nn.functional.normalize(x, dim=1)


def randn(n, d, g):
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):  # chunked: no second full-size temporary
        out[r0:r0 + min(65536, n - r0)] = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
    return out


def corpus(n, d, pages, layout, nq, seed):
    """(queries, pages, doc_groups): contiguous documents of `pages` pages."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    groups = torch.arange(n, device="cuda") // pages
    if layout == "random":
        return unit(randn(nq, d, g)), unit(randn(n, d, g)), groups
    n_docs = (n + pages - 1) // pages
    centres = unit(randn(n_docs, d, g))
    D = randn(n, d, g)
    for r0 in range(0, n, 65536):
        r1 = min(n, r0 + 65536)
        D[r0:r1] = unit(centres[groups[r0:r1]] + D[r0:r1] * (0.3 / d ** 0.5))
    pick = torch.randint(0, n_docs, (nq,), device="cuda", generator=g)
    Q = unit(centres[pick] + randn(nq, d, g) * (1.0 / d ** 0.5))
    return Q, D, groups


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, rounds, reps):
    arms = list(fn)
    times = {a: [] for a in arms}
    for a in arms:
        fn[a]()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn[a]()
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / reps)
    return {a: sorted(t) for a, t in times.items()}


def run(name, Q, index, groups, k, rounds, reps, out, proof=False):
    st = {"pages": {}, "groups": {}}
    fn = {"pages": lambda: R.score_topk(Q, index, k, stats=st["pages"]),
          "groups": lambda: R.score_topk_groups(Q, index, k, groups, stats=st["groups"])}
    times = timed(fn, rounds, reps)
    extra = {}
    if proof:
        gt = R._group_table(groups, index)
        sp = {}
        with torch.no_grad():
            R._score_topk_groups(Q, index, k, 0, False, sp, gt, None, page_lists=True)
        extra = {"flagged_grouped_filter": st["groups"].get("flagged", 0) / Q.shape[0],
                 "flagged_page_lists": sp["flagged"] / Q.shape[0]}
    stages = {}
    for a in fn:                                     # one more call per arm with stage events, outside the timed rounds
        sa = {"stages": {}}
        (R.score_topk(Q, index, k, stats=sa) if a == "pages" else R.score_topk_groups(Q, index, k, groups, stats=sa))
        torch.cuda.synchronize()
        stages[a] = {n: round(v, 3) for n, v in R.resolve_stages(sa).items()}
    for a in fn:
        t = times[a]
        line = {"workload": name, "arm": a, "queries": Q.shape[0], "pages": index.nd, "k": k,
                "ms_median": round(t[len(t) // 2], 3), "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3),
                "path": st[a].get("path"), "flagged": st[a].get("flagged"), "stages_ms": stages[a], **extra}
        print(json.dumps(line), flush=True)
        out.append(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpus", type=int, default=125000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--big", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=2304)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grouped_retrieval needs a CUDA device")
    out = [{"card": card()}]
    print(json.dumps(out[0]), flush=True)
    for layout in ("clustered", "random"):
        for pages in (1, 8, 64):
            Q, D, groups = corpus(a.corpus, a.dim, pages, layout, a.queries, 10 + pages)
            index = R.build_index(D)
            del D
            run(f"configs[3] shard, {layout}, {pages} pages per document", Q, index, groups, a.k, a.rounds, 1, out,
                proof=layout == "clustered")
            del Q, index
            torch.cuda.empty_cache()
    for n, reps, pages in ((a.corpus, 20, 8), (a.big, 10, 8), (a.big, 10, 1024)):
        Q, D, groups = corpus(n, a.dim, pages, "clustered", 1, 7)
        index = R.build_index(D)
        del D
        run(f"one query, clustered, {pages} pages per document", Q, index, groups, a.k, a.rounds, reps, out)
        del Q, index
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in out))


if __name__ == "__main__":
    main()
