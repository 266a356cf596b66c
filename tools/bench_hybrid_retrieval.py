"""What exact hybrid retrieval costs, and what the over-fetch recipe it replaces gets wrong. Arms, alternated inside
every round: the dense `score_topk(k)`, `score_topk_hybrid` by weighted sum and by RRF (window = k), the document form
`score_topk_groups_hybrid` (8-page documents), and a torch arm outside the library (fp32 matmul, scatter of the hits,
fl(s + fl(w v)), stable sort). Workloads (dim 2304, k = 10, weight 1): 10 k queries x 125 k pages (the tensor-core filter
path) and one query over 125 k and over 1 M pages, in a RANDOM and a CLUSTERED layout, with hit lists of 10, 100 and
1 000 distinct pages per query (values uniform in [0, 0.5], comparable with the cosine scores). Each line gives the
median and min-max over the rounds, the stage times of one untimed call (CUDA events: dense / lists / fuse / select) and
the mean fused candidates per row. For the weighted sum it also reports the rows where over-fetching search(4k), joining
the hits found there and re-sorting returns other top-k ids than the exact answer (overfetch_rows_differ), the same at
weights 0.05 and 0.01, where the weighted values are on the scale of the dense scores' spread, and the rows
where the torch arm's ids differ (torch_rows_differ; ties its summation order decides). The card's name, power limit and
SM clock are read in the same process. Prints one JSON line per (workload, arm), plus the card.
  python tools/bench_hybrid_retrieval.py [--rounds 3] [--out results.jsonl]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_grouped_retrieval import card, corpus, timed  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

TORCH_ROWS = 256  # queries per pass of the torch arm
K, W = 10, 1.0
LOW_WEIGHTS = (0.05, 0.01)


def make_hits(nq, nd, n, seed):
    """n distinct pages per query: a + j b (mod nd) with b coprime to nd; values uniform in [0, 0.5)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(0, nd, (nq, 1), device="cuda", generator=g)
    b = torch.randint(1, nd, (nq, 1), device="cuda", generator=g)
    nd_t = torch.tensor(nd, device="cuda")
    for _ in range(64):  # step b until it is coprime with nd
        bad = torch.gcd(b, nd_t) != 1
        if not bool(bad.any()):
            break
        b = torch.where(bad, b % (nd - 1) + 1, b)
    b = torch.where(torch.gcd(b, nd_t) == 1, b, torch.ones_like(b))
    ids = (a + torch.arange(n, device="cuda")[None, :] * b) % nd
    vals = torch.rand((nq, n), device="cuda", generator=g) * 0.5
    offsets = torch.arange(0, nq * n + 1, n, device="cuda", dtype=torch.int64)
    return offsets, ids.flatten().to(torch.int32), vals.flatten().contiguous()


def scatter_hits(hits, r0, r1, nd):
    off, ids, vals = hits
    a, b = int(off[r0]), int(off[r1])
    V = torch.zeros((r1 - r0, nd), device="cuda")
    row = torch.repeat_interleave(torch.arange(r1 - r0, device="cuda"), off[r0 + 1:r1 + 1] - off[r0:r1])
    V[row, ids[a:b].long()] = vals[a:b]
    return V


def torch_hybrid(Q, D, hits, k, w):
    nq, nd = Q.shape[0], D.shape[0]
    out_s = torch.empty((nq, k), device="cuda")
    out_i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    for r0 in range(0, nq, TORCH_ROWS):
        r1 = min(nq, r0 + TORCH_ROWS)
        f = Q[r0:r1] @ D.T + w * scatter_hits(hits, r0, r1, nd)
        s, i = torch.sort(f, dim=1, descending=True, stable=True)
        out_s[r0:r1], out_i[r0:r1] = s[:, :k], i[:, :k]
    return out_s, out_i


def overfetch_join(Q, index, hits, k, w):
    """search(4k), then each fetched page's external score from the hits (0 when it has none), re-sorted."""
    s, i = R.score_topk(Q, index, 4 * k)
    off, ids, vals = hits
    nq = Q.shape[0]
    row = torch.repeat_interleave(torch.arange(nq, device="cuda"), off[1:] - off[:-1])
    key_h = row * index.nd + ids.long()
    kh, order = torch.sort(key_h)
    key_f = torch.arange(nq, device="cuda")[:, None] * index.nd + i.clamp(min=0)
    at = torch.searchsorted(kh, key_f).clamp(max=kh.numel() - 1)
    v = torch.where(kh[at] == key_f, vals[order][at], 0.0)
    f = torch.where(i >= 0, s + w * v, float("-inf"))
    fs, o = torch.sort(f, dim=1, descending=True, stable=True)  # equal scores: keep search order (id asc within ties)
    return fs[:, :k], torch.gather(i, 1, o[:, :k])


def run(name, Q, D, index, groups, hits, rounds, reps, out, torch_arm):
    st = {a: {} for a in ("dense", "hybrid_sum", "hybrid_rrf", "documents_sum")}
    fn = {"dense": lambda s: R.score_topk(Q, index, K, stats=s),
          "hybrid_sum": lambda s: R.score_topk_hybrid(Q, index, K, hits, W, stats=s),
          "hybrid_rrf": lambda s: R.score_topk_hybrid(Q, index, K, hits, fusion="rrf", stats=s),
          "documents_sum": lambda s: R.score_topk_groups_hybrid(Q, index, K, groups, hits, W, stats=s)}
    arms = {a: (lambda a=a: fn[a](st[a])) for a in fn}
    if torch_arm:
        arms["torch_sum"] = lambda: torch_hybrid(Q, D, hits, K, W)
    times = timed(arms, rounds, reps)
    stages, cands = {}, {}
    for a in fn:
        sa = {"stages": {}}
        fn[a](sa)
        torch.cuda.synchronize()
        stages[a] = {n: round(v, 3) for n, v in R.resolve_stages(sa).items()}
        if "candidates" in sa:
            cands[a] = round(float(sa["candidates"].float().mean()), 1)
    s_x, i_x = R.score_topk_hybrid(Q, index, K, hits, W)
    _, i_o = overfetch_join(Q, index, hits, K, W)
    extra = {"overfetch_rows_differ": int((i_o != i_x).any(1).sum())}
    for w in LOW_WEIGHTS:  # external scores on the scale of the dense scores' spread
        _, i_xw = R.score_topk_hybrid(Q, index, K, hits, w)
        _, i_ow = overfetch_join(Q, index, hits, K, w)
        extra[f"overfetch_rows_differ_w{w}"] = int((i_ow != i_xw).any(1).sum())
    if torch_arm:
        _, i_t = torch_hybrid(Q, D, hits, K, W)
        extra["torch_rows_differ"] = int((i_t != i_x).any(1).sum())
    for a, t in times.items():
        line = {"workload": name, "arm": a, "ms_median": round(t[len(t) // 2], 3), "ms_min": round(t[0], 3),
                "ms_max": round(t[-1], 3), "stages": stages.get(a), "candidates_per_row": cands.get(a)}
        if a == "hybrid_sum":
            line.update(extra)
        print(json.dumps(line), flush=True)
        if out:
            out.write(json.dumps(line) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_hybrid_retrieval measures the GPU: no CUDA device"
    out = open(args.out, "w") if args.out else None
    print(json.dumps({"card": card()}), flush=True)
    d = 2304
    for layout in ("random", "clustered"):
        for nq, nd, reps, torch_arm in ((10_000, 125_000, 1, True), (1, 125_000, 20, True), (1, 1_000_000, 10, True)):
            Q, D, groups = corpus(nd, d, 8, layout, nq, seed=1)
            index = R.build_index(D)
            for n in (10, 100, 1000):
                hits = make_hits(nq, nd, n, seed=n)
                run(f"{layout} {nq}q x {nd}p, {n} hits", Q, D, index, groups.to(torch.int32), hits, args.rounds, reps, out,
                    torch_arm)
            del Q, D, groups, index
            torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
