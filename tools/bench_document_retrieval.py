"""What document retrieval costs, dim 2304: score_topk_groups at k up to 1000 and score_range_groups.
Document top-k, arms alternating inside every round: the default routes ("new": the deep document route for DEEP_K_MIN <
k <= DEEP_K_MAX and for filter-flagged rows past SELECT_K_MIN); "before": SELECT_K_MIN and DEEP_K_MIN raised past k inside
this script, so flagged rows rerun through the scan as in the parent commit (the scan's group selection itself is C code
and stays the radix select for k > 32, so this arm is faster than the parent's at k > 32). Every arm's pages must equal
the scan's (force_exact).
Document range search at thresholds keeping about 10, 100 and 1000 documents a query (the n-th document score of each
row), arms: the default, force_exact, and torch outside the library (fp32 matmul, a scatter-max of the scores per
document, a sort), which must find the same documents.
Workloads: 10 k queries x 125 k pages, random or clustered (the pages of a document near one centre, queries near
pages), in documents of 1, 8 and 64 pages; 1 query x 125 k and x 1 M random pages in documents of 8. Each line: median
(min - max) ms per arm over the rounds, the new arm's stats (path, fallback rows, stage times). The card's name, power
limit and SM clocks are read in the same run.
  python tools/bench_document_retrieval.py [--rounds 3] [--ks 10,32,100,1000] [--workloads random-1,...] [--out f.jsonl]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_deep_retrieval import card, timed, unit  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

DIM = 2304
WORKLOADS = "random-1,random-8,random-64,clustered-1,clustered-8,clustered-64,1x125k,1x1M"


def corpus(wl):
    """(queries, pages, doc_groups) of a workload."""
    if wl.startswith("1x"):
        nd = 125_000 if wl == "1x125k" else 1_000_000
        return unit(1, DIM, 6), unit(nd, DIM, 7), torch.arange(nd, device="cuda", dtype=torch.int32) // 8
    kind, per = wl.split("-")
    per, nd, nq = int(per), 125_000, 10_000
    groups = torch.arange(nd, device="cuda", dtype=torch.int32) // per
    if kind == "random":
        return unit(nq, DIM, 2), unit(nd, DIM, 1), groups
    c = unit(-(-nd // per), DIM, 3)
    D = torch.empty((nd, DIM), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(4)
    for r0 in range(0, nd, 65536):
        m = min(65536, nd - r0)
        x = c[groups[r0:r0 + m].long()] + 0.5 * torch.randn((m, DIM), device="cuda", generator=g) / DIM ** 0.5
        D[r0:r0 + m] = torch.nn.functional.normalize(x, dim=1)
    pick = torch.randint(0, nd, (nq,), device="cuda", generator=g)
    Q = torch.nn.functional.normalize(D[pick] + 0.3 * unit(nq, DIM, 5), dim=1)
    return Q, D, groups


def before(q, idx, k, groups):
    saved = R.SELECT_K_MIN, R.DEEP_K_MIN
    R.SELECT_K_MIN = R.DEEP_K_MIN = 1 << 30
    try:
        return R.score_topk_groups(q, idx, k, groups)
    finally:
        R.SELECT_K_MIN, R.DEEP_K_MIN = saved


def torch_range(q, idx, t, groups, G):
    """fp32 matmul, scatter-max of the scores per document, the documents >= t sorted by score: CSR (offsets, scores,
    groups)."""
    offs, ss, gg = [0], [], []
    step = max(1, (1 << 27) // max(idx.nd, G))
    gl = groups.long()
    for r0 in range(0, q.shape[0], step):
        s = q[r0:r0 + step] @ idx.emb.T
        best = torch.full((s.shape[0], G), float("-inf"), device=s.device).scatter_reduce_(
            1, gl.expand(s.shape[0], -1), s, "amax")
        keep = best >= t[r0:r0 + step, None]
        rows, g = torch.nonzero(keep).unbind(1)
        v = best[rows, g]
        o = torch.sort(v, descending=True, stable=True).indices
        o = o[torch.sort(rows[o], stable=True).indices]  # by row, then score desc
        ss.append(v[o])
        gg.append(g[o])
        offs.append(keep.sum(1))
    counts = torch.cat(offs[1:])
    return torch.cat([counts.new_zeros(1), torch.cumsum(counts, 0)]), torch.cat(ss), torch.cat(gg)


def rec_of(times, stats, **kw):
    return dict(kw, ms={n: [round(statistics.median(t), 3), round(min(t), 3), round(max(t), 3)] for n, t in times.items()},
                path=stats.get("path"), fallback=stats.get("fallback", stats.get("flagged")),
                stages={n: round(v, 3) for n, v in stats.get("stages", {}).items()})


def run(arms, rounds):
    times = {n: [] for n in arms}
    outs = {n: timed(fn)[1] for n, fn in arms.items()}  # warm-up, and the outputs checked
    for _ in range(rounds):
        for name, fn in arms.items():
            times[name].append(timed(fn)[0])
    return times, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ks", default="10,32,100,1000")
    ap.add_argument("--keeps", default="10,100,1000")
    ap.add_argument("--workloads", default=WORKLOADS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    lines = []
    for wl in a.workloads.split(","):
        Q, D, groups = corpus(wl)
        idx = R.build_index(D)
        del D
        G = int(groups.max()) + 1
        for k in [int(x) for x in a.ks.split(",")] if a.ks else []:
            ref = R.score_topk_groups(Q, idx, k, groups, force_exact=True)
            times, outs = run({"new": lambda: R.score_topk_groups(Q, idx, k, groups),
                               "before": lambda: before(Q, idx, k, groups)}, a.rounds)
            stats = {"stages": {}}
            R.score_topk_groups(Q, idx, k, groups, stats=stats)
            torch.cuda.synchronize()
            R.resolve_stages(stats)
            rec = rec_of(times, stats, op="topk", workload=wl, nq=Q.shape[0], nd=idx.nd, k=k,
                         same_pages={n: bool(torch.equal(o[1], ref[1])) for n, o in outs.items()})
            lines.append(rec)
            print(json.dumps(rec), flush=True)
            del ref, outs
        for keep in [int(x) for x in a.keeps.split(",")] if a.keeps else []:
            top = R.score_topk_groups(Q, idx, keep, groups, force_exact=True)[0]
            t = top[:, -1].contiguous()
            times, outs = run({"new": lambda: R.score_range_groups(Q, idx, t, groups),
                               "force_exact": lambda: R.score_range_groups(Q, idx, t, groups, force_exact=True),
                               "torch": lambda: torch_range(Q, idx, t, groups, G)}, a.rounds)
            stats = {"stages": {}}
            R.score_range_groups(Q, idx, t, groups, stats=stats)
            new, ex, tr = outs["new"], outs["force_exact"], outs["torch"]
            rec = rec_of(times, stats, op="range", workload=wl, nq=Q.shape[0], nd=idx.nd, keep=keep,
                         documents=int(new[0][-1]), same_as_scan=all(torch.equal(x, y) for x, y in zip(new, ex)),
                         torch_same_documents=bool(torch.equal(tr[0], new[0])) and bool(torch.equal(
                             torch.sort(tr[2]).values, torch.sort(new[3]).values)))
            lines.append(rec)
            print(json.dumps(rec), flush=True)
            del outs, new, ex, tr
        del idx
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
