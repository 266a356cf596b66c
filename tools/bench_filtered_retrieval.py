"""What a doc mask costs. Workloads: one GPU's shard of bench.py's configs[3] leg (10 k queries x 125 k docs, k = 10,
the tensor-core filter path) and one query over 125 k and over 1 M docs (the fp32 scan with the chunked top-k). Arms: no
mask, an all-ones mask, and random masks keeping 50 %, 10 % and 1 % of the docs. The arms alternate inside every round, so
drift of the shared machine falls on all of them alike; each arm reports its median and spread over the rounds, and the
card's name and power limit are read in the same process. Prints one JSON line per (workload, arm), plus one for the card.
Per-query masks (--per-query, on the configs[3] shard): every query with its own mask in one call, against what it costs
without them: 100 random scopes of 10 % (one shared-mask call per scope), and a run of 8 pages per query (M = nq; a loop
of single-query calls over the first 1 000 queries, reported as measured), with the unmasked call for reference.
Candidate lists (--lists): the list path (doc_lists) and the masked path (doc_mask) alternate on the same scopes, dim 2304,
k = 10: one query over 125 k and 1 M pages with a shared scope of 8, 1 k, 10 k and 50 k pages; 10 k queries x 125 k pages
with one shared scope of 100, 2 k and 20 k pages; 10 k queries each with its own 8-page scope (the masked arm packs the
[nq, nd] bool masks inside the call); and the document-level form of the first and third. Each line also gives the
knowledge base's routing rule for the workload (list rows, the masked side, and the path it picks).
  python tools/bench_filtered_retrieval.py [--rounds 10] [--out results.jsonl] [--per-query] [--lists] [--skip-shared]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import knowledge_base as KB  # noqa: E402
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
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


def _timed(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def run_per_query(Q, index, k, rounds, out, loop_queries=1000):
    """Alternating arms: per-query masks in one call vs the calls they replace, and the unmasked call."""
    nq, nd = Q.shape[0], index.nd
    g = torch.Generator(device="cuda").manual_seed(11)
    scopes = torch.rand((100, nd), device="cuda", generator=g) < 0.1
    of = torch.randint(0, 100, (nq,), device="cuda", generator=g)
    members = [torch.nonzero(of == m).flatten() for m in range(100)]
    start = torch.randint(0, nd - 8, (nq,), device="cuda", generator=g)
    own = torch.zeros((nq, nd), dtype=torch.bool, device="cuda")
    own[torch.arange(nq, device="cuda")[:, None], start[:, None] + torch.arange(8, device="cuda")] = True

    def per_scope_calls():
        for m in range(100):
            if members[m].numel():
                R.score_topk(Q[members[m]], index, k, doc_mask=scopes[m])

    def single_calls():
        for r in range(loop_queries):
            R.score_topk(Q[r:r + 1], index, k, doc_mask=own[r])

    arms = {"100 scopes of 10%: per-query masks": lambda: R.score_topk(Q, index, k, doc_mask=scopes, mask_of=of),
            "100 scopes of 10%: one call per scope": per_scope_calls,
            "8 pages each: per-query masks": lambda: R.score_topk(Q, index, k, doc_mask=own),
            f"8 pages each: single-query calls, first {loop_queries}": single_calls,
            "no mask": lambda: R.score_topk(Q, index, k)}
    stats = {}
    for a, fn in arms.items():                       # warm-up
        fn()
    R.score_topk(Q, index, k, doc_mask=scopes, mask_of=of, stats=stats.setdefault("scopes", {}))
    R.score_topk(Q, index, k, doc_mask=own, stats=stats.setdefault("own", {}))
    # the per-query rows equal the calls they replace
    s, i = R.score_topk(Q, index, k, doc_mask=scopes, mask_of=of)
    same = all(torch.equal(i[members[m]], R.score_topk(Q[members[m]], index, k, doc_mask=scopes[m])[1]) for m in range(0, 100, 9))
    s8, i8 = R.score_topk(Q, index, k, doc_mask=own)
    same &= all(torch.equal(i8[r:r + 1], R.score_topk(Q[r:r + 1], index, k, doc_mask=own[r])[1]) for r in range(0, nq, 997))
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            times[a].append(_timed(fn))
    for a in arms:
        t = sorted(times[a])
        line = {"workload": "per-query masks", "arm": a, "queries": nq, "docs": nd, "k": k,
                "ms_median": round(t[len(t) // 2], 3), "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3),
                "rows_equal_the_calls_they_replace": same,
                "stats": stats["scopes" if a.startswith("100") else "own"] if a.endswith("per-query masks") else None}
        print(json.dumps(line), flush=True)
        out.append(line)


def _lists_of(scopes):
    """[M] int64 index tensors -> doc_lists (offsets, ids)."""
    offsets = torch.zeros(len(scopes) + 1, dtype=torch.int64, device="cuda")
    offsets[1:] = torch.cumsum(torch.tensor([len(x) for x in scopes], device="cuda"), 0)
    return offsets, torch.cat(scopes).to(torch.int32)


def run_lists(name, Q, index, k, scopes, list_of, rounds, out, groups=None, reps=1):
    """The list path and the masked path alternating on the same scopes (scopes: [M] index tensors; list_of: None when
    one scope serves every query, or when M == nq and query i has scope i)."""
    nq, nd = Q.shape[0], index.nd
    lists = _lists_of(scopes)
    if list_of is None and len(scopes) == 1:
        mask = torch.zeros(nd, dtype=torch.bool, device="cuda")
        mask[scopes[0]] = True
    else:
        mask = torch.zeros((len(scopes), nd), dtype=torch.bool, device="cuda")
        mask[torch.repeat_interleave(torch.arange(len(scopes), device="cuda"), lists[0][1:] - lists[0][:-1]), lists[1].long()] = True
    if groups is None:
        arms = {"lists": lambda st=None: R.score_topk(Q, index, k, stats=st, doc_lists=lists, list_of=list_of),
                "masked": lambda st=None: R.score_topk(Q, index, k, stats=st, doc_mask=mask, mask_of=list_of)}
    else:
        arms = {"lists": lambda st=None: R.score_topk_groups(Q, index, k, groups, stats=st, doc_lists=lists, list_of=list_of),
                "masked": lambda st=None: R.score_topk_groups(Q, index, k, groups, stats=st, doc_mask=mask, mask_of=list_of)}
    stats = {a: {} for a in arms}
    res = {a: fn(stats[a]) for a, fn in arms.items()}   # warm-up, and the results of both
    same = all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(res["lists"], res["masked"]))
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            times[a].append(_timed(fn, reps))
    tiles = torch.bincount(list_of.long(), minlength=len(scopes)).tolist() if list_of is not None else [nq] * len(scopes)
    if list_of is None and len(scopes) > 1:
        tiles = [1] * len(scopes)
    list_rows = sum(len(x) * -(-t // KB.LIST_TILE) for x, t in zip(scopes, tiles))
    for a in arms:
        t = sorted(times[a])
        line = {"workload": name, "arm": a, "level": "pages" if groups is None else "documents", "queries": nq, "docs": nd,
                "k": k, "scope_pages": sorted({len(x) for x in scopes})[:3], "ms_median": round(t[len(t) // 2], 3),
                "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3), "path": stats[a].get("path"),
                "same_bits": same, "list_rows": list_rows, "masked_rows": nd * -(-nq // 256),
                "rule_picks_lists": KB.list_path_wins(list_rows, nq, nd, k, groups is not None)}
        print(json.dumps(line), flush=True)
        out.append(line)


def lists_workloads(a, out):
    k, rounds = a.k, a.rounds
    for nd in (a.corpus, a.big):
        D = unit(nd, a.dim, 1 if nd == a.corpus else 3)
        index = R.build_index(D)
        del D
        g = torch.Generator(device="cuda").manual_seed(17)
        groups = (torch.arange(nd, device="cuda", dtype=torch.int32) // 20)[torch.randperm(nd, device="cuda", generator=g)]
        q1 = unit(1, a.dim, 4)
        for n in (8, 1000, 10_000, 50_000):
            scope = torch.randperm(nd, device="cuda", generator=g)[:n]
            run_lists("one query, shared scope", q1, index, k, [scope], None, rounds, out, reps=10)
            if nd == a.corpus:
                run_lists("one query, shared scope", q1, index, k, [scope], None, rounds, out, groups=groups, reps=10)
        if nd == a.corpus:
            Q = unit(a.queries, a.dim, 2)
            for n in (100, 2000, 20_000):
                scope = torch.randperm(nd, device="cuda", generator=g)[:n]
                run_lists("10 k queries, one shared scope", Q, index, k, [scope], None, rounds, out)
            start = torch.randint(0, nd - 8, (a.queries,), device="cuda", generator=g)
            own = list((start[:, None] + torch.arange(8, device="cuda")).unbind(0))
            run_lists("10 k queries, own 8-page scope each", Q, index, k, own, None, rounds, out)
            run_lists("10 k queries, own 8-page scope each", Q, index, k, own, None, rounds, out, groups=groups)
            del Q, own
        del index, groups
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpus", type=int, default=125000)
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--big", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=2304)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--per-query", action="store_true", help="also measure per-query masks on the configs[3] shard")
    ap.add_argument("--skip-shared", action="store_true", help="skip the shared-mask workloads")
    ap.add_argument("--lists", action="store_true", help="measure candidate lists against masks")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_filtered_retrieval needs a CUDA device")
    out = [{"card": card()}]
    print(json.dumps(out[0]), flush=True)

    if a.lists:
        lists_workloads(a, out)
    D = unit(a.corpus, a.dim, 1)
    index = R.build_index(D)
    if not a.skip_shared:
        run("configs[3] shard: filter path", unit(a.queries, a.dim, 2), index, a.k, a.rounds, 1, out)
        run("one query", unit(1, a.dim, 4), index, a.k, a.rounds, 20, out)
    if a.per_query:
        run_per_query(unit(a.queries, a.dim, 2), index, a.k, a.rounds, out)
    if not a.skip_shared:
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
