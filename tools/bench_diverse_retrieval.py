"""What diverse retrieval costs (retriever.score_mmr: score_topk(fetch_k) + vr_mmr_select), dim 2304. Arms, alternating
inside every round: score_topk(k); score_mmr(k, fetch_k) with the CUDA-event times of its two stages (candidates,
select); and a torch arm outside the library on the same candidates (gather the candidate rows, a bmm Gram, a k-step
greedy loop), which reports whether its picks match the kernel's (they may not: cuBLAS sums in another order).
Workloads: random unit pages, 1 query x 125 k and x 1 M pages, 10 k queries x 125 k pages; planted near-duplicate
clusters (125 k pages, 5 noisy copies of each of 25 k pages), 1 query and 10 k queries; (k, fetch_k) in {(3, 20),
(10, 40), (10, 128)}. Each line gives the median (min - max) of every arm over the rounds, the select stage's share of
its HBM bound (nq * fetch_k * dim * 4 bytes at 3.35 TB/s), and on the clustered corpus the mean number of distinct
clusters in each arm's k pages. The card's name, power limit and SM clocks are read in the same run.
  python tools/bench_diverse_retrieval.py [--rounds 5] [--out results.jsonl]"""
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
HBM = 3.35e12  # bytes/s, H100 SXM data sheet
LAMBDA = 0.5
SHAPES = [(3, 20), (10, 40), (10, 128)]


def unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):
        x = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
        out[r0:r0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1)
    return out


def clustered(n, per, d, seed):
    """n pages: `per` noisy copies (noise norm 0.05) of each of n / per random unit pages; cluster of page j = j // per."""
    c = unit(n // per, d, seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    for r0 in range(0, n, 65536):
        m = min(65536, n - r0)
        x = c[torch.arange(r0, r0 + m, device="cuda") // per] + 0.05 * torch.randn((m, d), device="cuda", generator=g) / d ** 0.5
        out[r0:r0 + m] = torch.nn.functional.normalize(x, dim=1)
    return out


def near(docs, nq, seed):
    """Queries near random pages (page + noise of norm 0.3)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pick = torch.randint(0, docs.shape[0], (nq,), device="cuda", generator=g)
    return torch.nn.functional.normalize(docs[pick] + 0.3 * unit(nq, docs.shape[1], seed + 1), dim=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def torch_mmr(emb, s, i, k, lam, rows=1024):
    """Greedy MMR in torch on given candidates (all valid): gather, bmm Gram, k steps of masked argmax."""
    out = []
    mu = 1.0 - lam
    for r0 in range(0, s.shape[0], rows):
        ss, ii = s[r0:r0 + rows], i[r0:r0 + rows]
        x = emb[ii]                                    # [n, F, dim]
        gram = torch.bmm(x, x.transpose(1, 2))         # [n, F, F]
        n, F = ss.shape
        ar = torch.arange(n, device=s.device)
        taken = torch.zeros((n, F), dtype=torch.bool, device=s.device)
        red = torch.full((n, F), float("-inf"), device=s.device)
        p = torch.zeros(n, dtype=torch.int64, device=s.device)
        picks = [p]
        for _ in range(1, k):
            taken[ar, p] = True
            red = torch.maximum(red, gram[ar, :, p])
            v = torch.where(taken, float("-inf"), lam * ss - mu * red)
            p = torch.argmax(v, dim=1)
            picks.append(p)
        out.append(torch.gather(ii, 1, torch.stack(picks, 1)))
    return torch.cat(out)


def med(xs):
    return {"median_ms": round(statistics.median(xs), 4), "min_ms": round(min(xs), 4), "max_ms": round(max(xs), 4)}


def run(name, index, q, k, fetch, rounds, clusters_of=None):
    nq = q.shape[0]
    cand = R.score_topk(q, index, fetch)
    stats = {"stages": {}}
    arms = {
        "topk": lambda: R.score_topk(q, index, k)[1],
        "mmr": lambda: R.score_mmr(q, index, k, LAMBDA, fetch_k=fetch, stats=stats)[1],
        "torch": lambda: torch_mmr(index.emb, cand[0], cand[1], k, LAMBDA),
    }
    outs = {a: f() for a, f in arms.items()}  # warm-up, and the outputs compared below
    torch.cuda.synchronize()
    stats.clear()
    stats["stages"] = {}
    times = {a: [] for a in arms}
    cand_ms, sel_ms = [], []
    for _ in range(rounds):
        for a, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1))
            if a == "mmr":
                st = R.resolve_stages(stats)
                cand_ms.append(st["candidates"])
                sel_ms.append(st["select"])
                stats["stages"] = {}
    bound_ms = nq * fetch * DIM * 4 / HBM * 1e3
    line = {"workload": name, "nq": nq, "nd": index.nd, "k": k, "fetch_k": fetch, "lambda": LAMBDA,
            **{a: med(t) for a, t in times.items()},
            "mmr_candidates": med(cand_ms), "mmr_select": med(sel_ms),
            "select_hbm_bound_ms": round(bound_ms, 4),
            "select_share_of_hbm_bound": round(bound_ms / statistics.median(sel_ms), 3),
            "torch_picks_match": bool(torch.equal(outs["torch"], outs["mmr"])),
            "torch_rows_matching": round(float((outs["torch"] == outs["mmr"]).all(1).float().mean()), 4)}
    if clusters_of is not None:
        for a in arms:
            c = clusters_of[outs[a]]
            distinct = (torch.sort(c, 1).values.diff(dim=1) != 0).sum(1) + 1
            line[f"{a}_distinct_clusters"] = round(float(distinct.float().mean()), 3)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    head = {"card": card(), "torch": torch.__version__, "dim": DIM}
    print(json.dumps(head), flush=True)
    lines = [head]
    corpora = [
        ("random 125k", lambda: unit(125_000, DIM, 1), None, [1, 10_000]),
        ("random 1M", lambda: unit(1_000_000, DIM, 2), None, [1]),
        ("clusters 125k", lambda: clustered(125_000, 5, DIM, 3), 5, [1, 10_000]),
    ]
    for cname, make, per, nqs in corpora:
        docs = make()
        index = R.build_index(docs)
        clusters_of = torch.arange(index.nd, device="cuda") // per if per else None
        for nq in nqs:
            q = near(docs, nq, 10 + nq) if per else unit(nq, DIM, 10 + nq)
            for k, fetch in SHAPES:
                line = run(f"{cname} x {nq} queries", index, q, k, fetch, args.rounds, clusters_of)
                print(json.dumps(line), flush=True)
                lines.append(line)
        del index, docs
        torch.cuda.empty_cache()
    head_after = {"card_after": card()}
    print(json.dumps(head_after), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for line in lines + [head_after]:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
