"""What per-document caps cost. Arms, alternated inside every round: page-level `score_topk(k)`, document-level
`score_topk_groups(k)`, the capped page top-k `score_topk_capped(k, m)` for m = 2 and 3, the inner hits
`score_topk_groups_pages(k, 3)`, and a torch arm outside the library (fp32 matmul, stable sort by score, then the greedy
walk with per-document counters, m = 2). Workloads (dim 2304, k = 10): one GPU's shard of bench.py's configs[3] leg
(10 k queries x 125 k pages, the tensor-core filter path) and one query over 125 k and over 1 M pages, each in a
CLUSTERED layout (each document a centre plus small noise, queries near document centres: a knowledge base of PDFs) and a
RANDOM layout, with contiguous documents of 1, 8 and 64 pages. Each line gives the median and min-max over the rounds
and the stage times of one untimed call (CUDA events: documents / pages / merge). The torch arm's picks are compared
with the m = 2 arm's: rows_differ counts the rows that differ, and tie_gap the largest gap between the two arms' fp32
scores at a row's first differing slot (a gap of a few ulps is a tie the torch summation order decided). The card's
name, power limit and SM clock are read in the same process. Prints one JSON line per (workload, arm), plus the card.
  python tools/bench_capped_retrieval.py [--rounds 5] [--out results.jsonl]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_grouped_retrieval import card, corpus, timed  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

TORCH_ROWS = 256  # queries per pass of the torch arm: [rows, nd] fp32 scores and their sort


def torch_capped(Q, D, groups, k, m):
    """fp32 matmul, stable sort by score (desc; equal scores keep the lower page first), then the walk: a page is picked
    when fewer than m earlier pages of its document are (its occurrence rank within its document in sorted order is
    < m), and the first k picked pages are the answer."""
    nq, nd = Q.shape[0], D.shape[0]
    out_s = torch.full((nq, k), float("-inf"), device=Q.device)
    out_p = torch.full((nq, k), -1, dtype=torch.int64, device=Q.device)
    pos = torch.arange(nd, device=Q.device)
    for r0 in range(0, nq, TORCH_ROWS):
        s = Q[r0:r0 + TORCH_ROWS] @ D.T
        s = torch.where(torch.isnan(s), float("-inf"), s)
        ss, order = torch.sort(s, dim=1, descending=True, stable=True)
        gs = groups[order]
        gsorted, by_group = torch.sort(gs, dim=1, stable=True)            # runs of one document, in page order
        start = torch.ones_like(gsorted, dtype=torch.bool)
        start[:, 1:] = gsorted[:, 1:] != gsorted[:, :-1]
        first = torch.cummax(torch.where(start, pos, 0), dim=1).values
        occ = torch.empty_like(by_group)
        occ.scatter_(1, by_group, pos - first)
        keep = occ < m
        rank = torch.cumsum(keep, dim=1)
        sel = keep & (rank <= k)
        n = sel.sum(1)
        idx = torch.sort(torch.where(sel, pos, nd), dim=1).values[:, :k]   # positions of the picks, in order
        valid = torch.arange(k, device=Q.device)[None, :] < n[:, None]
        idx = idx.clamp(max=nd - 1)
        out_s[r0:r0 + TORCH_ROWS] = torch.where(valid, torch.gather(ss, 1, idx), float("-inf"))
        out_p[r0:r0 + TORCH_ROWS] = torch.where(valid, torch.gather(order, 1, idx), -1)
    return out_s, out_p


def run(name, Q, D, index, groups, k, rounds, reps, out, torch_arm=True):
    st = {a: {} for a in ("pages", "groups", "capped_2", "capped_3", "inner_hits_3")}
    fn = {"pages": lambda s: R.score_topk(Q, index, k, stats=s),
          "groups": lambda s: R.score_topk_groups(Q, index, k, groups, stats=s),
          "capped_2": lambda s: R.score_topk_capped(Q, index, k, groups, 2, stats=s),
          "capped_3": lambda s: R.score_topk_capped(Q, index, k, groups, 3, stats=s),
          "inner_hits_3": lambda s: R.score_topk_groups_pages(Q, index, k, groups, 3, stats=s)}
    arms = {a: (lambda a=a: fn[a](st[a])) for a in fn}
    if torch_arm:
        arms["torch_capped_2"] = lambda: torch_capped(Q, D, groups, k, 2)
    times = timed(arms, rounds, reps)
    stages = {}
    for a in fn:                                     # one more call per arm with stage events, outside the timed rounds
        sa = {"stages": {}}
        fn[a](sa)
        torch.cuda.synchronize()
        stages[a] = {n: round(v, 3) for n, v in R.resolve_stages(sa).items()}
    extra = {}
    if torch_arm:
        s_lib, p_lib, _ = R.score_topk_capped(Q, index, k, groups, 2)
        s_t, p_t = torch_capped(Q, D, groups, k, 2)
        diff = (p_lib != p_t).any(1)
        gap = 0.0
        if bool(diff.any()):
            rows = torch.nonzero(diff).flatten()
            j = (p_lib[rows] != p_t[rows]).int().argmax(1)
            gap = float((s_lib[rows, j] - s_t[rows, j]).abs().max())
        extra = {"rows_differ": int(diff.sum()), "tie_gap": gap}
    for a in arms:
        t = times[a]
        line = {"workload": name, "arm": a, "queries": Q.shape[0], "pages": index.nd, "k": k,
                "ms_median": round(t[len(t) // 2], 3), "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3),
                "path": st.get(a, {}).get("path"), "flagged": st.get(a, {}).get("flagged"),
                "stages_ms": stages.get(a), **(extra if a == "torch_capped_2" else {})}
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
        raise SystemExit("bench_capped_retrieval needs a CUDA device")
    out = [{"card": card()}]
    print(json.dumps(out[0]), flush=True)
    for layout in ("clustered", "random"):
        for pages in (1, 8, 64):
            for n, nq, reps in ((a.corpus, a.queries, 1), (a.corpus, 1, 20), (a.big, 1, 10)):
                Q, D, groups = corpus(n, a.dim, pages, layout, nq, 10 + pages)
                index = R.build_index(D)
                what = f"{nq} queries x {n} pages" if nq > 1 else f"one query x {n} pages"
                run(f"{what}, {layout}, {pages} pages per document", Q, D, index, groups, a.k, a.rounds, reps, out)
                del Q, D, index
                torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in out))


if __name__ == "__main__":
    main()
