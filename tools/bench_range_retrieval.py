"""What range search costs (retriever.score_range, KnowledgeBase.near_duplicates), dim 2304. Arms, alternating inside every
round: the default path (the tensor-core range filter + exact rescoring, the scan for small problems and overflowed
rows), force_exact (the fp32 scan path), and a plain torch baseline outside the library (fp32 matmul, s >= t, a stable
sort per row). Workloads: one query over 125 k and 1 M pages with thresholds keeping about 10, 1 k and 10 k pages; 10 k
queries over 125 k pages with thresholds keeping about 10, 100, 1 000, 10 000 and 30 000 pages per query (the last two
on either side of the filter path's capacity); near_duplicates over 125 k pages
with planted clusters. Each line gives the median (min - max) of every arm over the rounds, whether the library arms gave
the same bits and whether the torch baseline found the same ids, the path, the candidates and the rows that fell back
to the scan. The card's name, power limit and SM clocks are read in the same run.
  python tools/bench_range_retrieval.py [--rounds 5] [--out results.jsonl] [--cap N] [--skip-near-duplicates]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import knowledge_base as KB  # noqa: E402
from visrag_b200 import retriever as R  # noqa: E402

DIM = 2304


def unit(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device="cuda")
    for r0 in range(0, n, 65536):
        x = torch.randn((min(65536, n - r0), d), device="cuda", generator=g)
        out[r0:r0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def torch_range(Q, D, t, rows=512):
    """fp32 matmul, s >= t, stable sort by score desc: CSR (offsets, scores, ids)."""
    offs, ss, ii = [torch.zeros(1, dtype=torch.int64, device="cuda")], [], []
    for r0 in range(0, Q.shape[0], rows):
        s = Q[r0:r0 + rows] @ D.T
        keep = s >= t[r0:r0 + rows, None]
        v, idx = torch.sort(torch.where(keep, s, float("-inf")), dim=1, descending=True, stable=True)
        n = keep.sum(1)
        take = torch.arange(s.shape[1], device="cuda")[None, :] < n[:, None]
        ss.append(v[take])
        ii.append(idx[take])
        offs.append(offs[-1][-1:] + torch.cumsum(n, 0))
    return torch.cat(offs), torch.cat(ss), torch.cat(ii)


def thresholds(Q, D, keep, rows=512):
    """The keep-th largest fp32 score of each query (so about `keep` pages pass)."""
    return torch.cat([torch.topk(Q[r0:r0 + rows] @ D.T, keep, dim=1).values[:, -1] for r0 in range(0, Q.shape[0], rows)])


def timed(fn, rounds, arms):
    times = {a: [] for a in arms}
    outs = {a: fn(a) for a in arms}  # warm-up, and the outputs compared below
    torch.cuda.synchronize()
    for _ in range(rounds):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(a)
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1))
    return times, outs


def report(name, times, outs, stats, extra, out):
    same = all(torch.equal(x, y) for x, y in zip(outs["default"], outs["force_exact"]))
    line = {"workload": name, **extra, "library_arms_identical": same}
    if "torch" in outs:
        line["torch_ids_identical"] = bool(torch.equal(outs["torch"][0], outs["default"][0]) and
                                           torch.equal(outs["torch"][2], outs["default"][2]))
    for a, t in times.items():
        t = sorted(t)
        line[a] = f"{t[len(t) // 2]:.2f} ({t[0]:.2f}-{t[-1]:.2f}) ms"
    line.update({k: stats.get(k) for k in ("path", "candidates", "fallback", "cap")})
    print(json.dumps(line), flush=True)
    out.append(line)


def range_workload(name, Q, index, keep, rounds, cap, out):
    t = thresholds(Q, index.emb, keep)
    stats = {}

    def fn(arm):
        if arm == "torch":
            return torch_range(Q, index.emb, t)
        return R.score_range(Q, index, t, force_exact=arm == "force_exact", cap=cap, stats=stats if arm == "default" else None)

    times, outs = timed(fn, rounds, ("default", "force_exact", "torch"))
    results = int(outs["default"][1].numel())
    report(name, times, outs, stats, {"queries": Q.shape[0], "pages": index.nd, "kept_per_query": results / Q.shape[0]}, out)


def near_duplicates_workload(n, rounds, out):
    g = torch.Generator(device="cuda").manual_seed(5)
    docs = unit(n, DIM, 4)
    for _ in range(2000):  # clusters of 2-8 near-identical pages (a repeated cover, a slide template)
        m = torch.randint(0, n, (int(torch.randint(2, 9, (1,), generator=g, device="cuda")),), generator=g, device="cuda")
        docs[m] = torch.nn.functional.normalize(docs[m[:1]] + 0.002 * torch.randn((m.numel(), DIM), generator=g, device="cuda"),
                                                dim=1)
    t = 0.98
    with tempfile.TemporaryDirectory() as tmp:
        KB.save_knowledge_base(tmp, docs.cpu().numpy(), [f"p{j}.png" for j in range(n)])
        kb = KB.KnowledgeBase(tmp)
    del docs
    emb = kb.index.emb
    stats = {}

    def fn(arm):
        if arm == "default":
            return kb.near_duplicates(t)
        parts = []
        for r0 in range(0, n, kb.NEAR_DUPLICATE_ROWS):
            sel = torch.arange(r0, min(n, r0 + kb.NEAR_DUPLICATE_ROWS), device="cuda")
            if arm == "force_exact":
                off, s, b = R.score_range(emb[sel], kb.index, t, force_exact=True)
            else:
                off, s, b = torch_range(emb[sel], emb, torch.full((sel.numel(),), t, device="cuda"))
            a = torch.repeat_interleave(sel, off[1:] - off[:-1])
            k = b > a
            parts.append((a[k], b[k], s[k]))
        return tuple(torch.cat([p[j] for p in parts]) for j in range(3))

    R.score_range(emb[:kb.NEAR_DUPLICATE_ROWS], kb.index, t, stats=stats)  # the path and candidates of one chunk
    times, outs = timed(fn, rounds, ("default", "force_exact", "torch"))
    same = all(torch.equal(x, y) for x, y in zip(outs["default"], outs["force_exact"]))
    line = {"workload": "near_duplicates", "pages": n, "min_score": t, "pairs": int(outs["default"][0].numel()),
            "library_arms_identical": same,
            "torch_pairs_identical": bool(torch.equal(outs["torch"][0], outs["default"][0]) and
                                          torch.equal(outs["torch"][1], outs["default"][1]))}
    for a, tt in times.items():
        tt = sorted(tt)
        line[a] = f"{tt[len(tt) // 2]:.1f} ({tt[0]:.1f}-{tt[-1]:.1f}) ms"
    line.update({k: stats.get(k) for k in ("path", "candidates", "fallback", "cap")})
    print(json.dumps(line), flush=True)
    out.append(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cap", type=int, default=None)
    ap.add_argument("--skip-near-duplicates", action="store_true")
    ap.add_argument("--only", default=None, help="comma-separated workload name prefixes")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    out = [{"card": card()}]
    print(json.dumps(out[0]), flush=True)
    want = lambda name: args.only is None or any(name.startswith(p) for p in args.only.split(","))  # noqa: E731
    for nd in (125_000, 1_000_000):
        if not want(f"1x{nd // 1000}k"):
            continue
        index = R.build_index(unit(nd, DIM, 1))
        q = unit(1, DIM, 2)
        for keep in (10, 1000, 10_000):
            range_workload(f"1x{nd // 1000}k keep {keep}", q, index, keep, args.rounds, args.cap, out)
        del index
        torch.cuda.empty_cache()
    if want("10kx125k"):
        index = R.build_index(unit(125_000, DIM, 1))
        q = unit(10_000, DIM, 3)
        for keep in (10, 100, 1000, 10_000, 30_000):  # the last two: below and above the capacity
            range_workload(f"10kx125k keep {keep}", q, index, keep, args.rounds, args.cap, out)
        del index
        torch.cuda.empty_cache()
    if not args.skip_near_duplicates and want("near"):
        near_duplicates_workload(125_000, args.rounds, out)
    out.append({"card": card()})
    print(json.dumps(out[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in out) + "\n")


if __name__ == "__main__":
    main()
