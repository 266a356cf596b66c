"""Query encoding with and without the prefix cache (VisRAGEngine(prefix_cache=...)) on the full-size model: two engines
with the same weights, timed in alternating windows in one process, on
  * bench.py's query leg: synth_queries(1000, 7) in batches of 500;
  * batches of 16 (the reference evaluation's per-device batch), CUDA-graph path;
  * 64 single queries once the entry exists (graph path);
  * a sweep of the prefix length P with a fixed suffix, batches of 16: where the cached path starts to pay, which sets
    host.PREFIX_MIN_TOKENS.
Prints one JSON line: queries/s per window and the median per arm, LM tokens computed per query, the SM clock and power
drawn after each window, the card and its power limit. Asserts that both arms' embeddings are equal.
  python tools/bench_prefix.py [--windows 3]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import host  # noqa: E402
from visrag_b200.config import VisRAGConfig  # noqa: E402
from visrag_b200.encoder import VisRAGEngine  # noqa: E402
from visrag_b200.host import prepare_batch, select_prefix  # noqa: E402
from visrag_b200.synth import synth_queries  # noqa: E402
from visrag_b200.tokenizer_stub import StubTokenizer  # noqa: E402
from visrag_b200.weights import random_state_dict_device  # noqa: E402


def smi(fields):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    return [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else None


def lm_tokens_per_query(batches, tok, cfg, eng):
    """LM tokens an engine computes per query: all of them without the cache; with it, the suffixes of batches that hit
    an entry (entries are created outside the timed windows)."""
    total = n = 0
    for qs in batches:
        pb = prepare_batch(qs, [None] * len(qs), tok, cfg, 2048)
        sel = select_prefix(pb, list(eng._prefixes)) if eng.prefix_cache else None
        total += int(pb.cu_seqlens[-1]) - (len(sel[0]) * len(qs) if sel else 0)
        n += len(qs)
    return total / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3, help="timed windows per arm and workload")
    a = ap.parse_args()
    cfg = VisRAGConfig.full()
    tok = StubTokenizer(cfg.vocab)
    sd = random_state_dict_device(cfg, 2024, "cuda:0")
    arms = {"cache_on": VisRAGEngine(cfg, sd, prefix_cache=True), "cache_off": VisRAGEngine(cfg, sd, prefix_cache=False)}
    del sd
    torch.cuda.empty_cache()

    qs = synth_queries(1000, 7)
    pfx_single = synth_queries(64, 11)
    workloads = {
        "bench_leg_b500": [qs[i:i + 500] for i in range(0, 1000, 500)],
        "batch16": [qs[i:i + 16] for i in range(0, 256, 16)],
        "single": [[q] for q in pfx_single],
    }
    rs = np.random.RandomState(5)
    for P in (4, 8, 16, 32, 57):     # P tokens of prefix = BOS + P - 1 characters; 48-character suffixes
        pfx = "".join(rs.choice(list("abcdefghijklmnopqrstuvwxyz"), P - 1))
        sq = [pfx + "ABCDEFGHIJKLMNOP"[i % 16] + "".join(rs.choice(list("abcdefghij "), 47)) for i in range(256)]
        workloads[f"sweep_P{P}_b16"] = [sq[i:i + 16] for i in range(0, 256, 16)]

    def run(eng, batches):
        return torch.cat([eng.encode(b, [None] * len(b), tok) for b in batches])

    # the sweep measures prefixes below the shipped threshold too: every shared prefix of a batch gets an entry here
    host.PREFIX_MIN_TOKENS = 1
    card = smi("name,power.limit,clocks.max.sm")
    out = {"card": card[0] if card else None, "power_limit_w": card[1] if card else None,
           "max_sm_clock_mhz": card[2] if card else None, "workloads": {}}
    for name, batches in workloads.items():
        n_q = sum(len(b) for b in batches)
        res = {}
        for arm, eng in arms.items():
            eng.encode(qs[:16], [None] * 16, tok)     # the instruction's entry exists before single queries run
            for _ in range(2):                         # warm every shape (graphs: eager, then capture)
                run(eng, batches)
            res[arm] = {"qps": [], "sm_mhz": [], "power_w": []}
        embs = {}
        for w in range(a.windows):
            for arm in (arms if w % 2 == 0 else list(reversed(arms))):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e = run(arms[arm], batches)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                s = smi("clocks.sm,power.draw")
                res[arm]["qps"].append(round(n_q / dt, 2))
                res[arm]["sm_mhz"].append(s[0] if s else None)
                res[arm]["power_w"].append(s[1] if s else None)
                embs[arm] = e
        assert torch.equal(embs["cache_on"], embs["cache_off"]), name
        for arm in arms:
            res[arm]["median_qps"] = statistics.median(res[arm]["qps"])
            res[arm]["lm_tokens_per_query"] = round(lm_tokens_per_query(batches, tok, cfg, arms[arm]), 1)
        res["speedup"] = round(res["cache_on"]["median_qps"] / res["cache_off"]["median_qps"], 3)
        out["workloads"][name] = res
        print(json.dumps({name: res}), flush=True)
    out["prefix_stats"] = arms["cache_on"].prefix_stats
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
