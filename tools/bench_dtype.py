"""Device-resident encode throughput of a bf16 engine and an fp16 engine (VisRAGEngine(dtype=...)) on bench.py's workload:
128 synthetic 448x448 pages per step, full-size random weights. Both engines live in one process with the same weights and
the same uploaded batch; their timed windows alternate (bf16, fp16, bf16, ...) so that drift on a shared machine hits both.
Prints pages/s of every window and the median per dtype with the median SM clock and power draw sampled during that
window, the card and its power limit (read in the same run), kernel time per kind for one profiled step of each engine
(a separate pass after the timed windows), and how far the two engines' embeddings are apart (cosine, max |diff|).
  python tools/bench_dtype.py [--pages 128] [--steps 6] [--warmup 2] [--runs 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200.config import VisRAGConfig  # noqa: E402
from visrag_b200.encoder import VisRAGEngine  # noqa: E402
from visrag_b200.host import prepare_batch  # noqa: E402
from visrag_b200.tokenizer_stub import StubTokenizer  # noqa: E402
from visrag_b200.weights import random_state_dict_device  # noqa: E402


def gpu_state(index=0):
    """Card name, power limit, current and maximum SM clock (read-only nvidia-smi query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(index)}


class WindowSampler:
    """Read-only nvidia-smi sampling (SM clock, power draw; every 100 ms) for the duration of one timed window."""

    def __enter__(self):
        self.path = os.path.join(tempfile.gettempdir(), f"vr_bench_dtype_{os.getpid()}.csv")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except OSError:
            self.proc = None
        return self

    def __exit__(self, *exc):
        self.sm_mhz = self.power_w = None
        if self.proc is None:
            return False
        self.proc.terminate()
        try:
            self.proc.wait(5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            self.proc.wait()
        rows = []
        for line in open(self.path):
            try:
                rows.append([float(x) for x in line.split(",")[:2]])
            except ValueError:
                pass
        os.unlink(self.path)
        if rows:
            self.sm_mhz, self.power_w = (float(np.median([r[i] for r in rows])) for i in (0, 1))
        return False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=128)
    ap.add_argument("--page-px", type=int, default=448)
    ap.add_argument("--steps", type=int, default=6, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3, help="timed windows per dtype (alternating)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dtype.py measures on a CUDA device; none is available")
    from PIL import Image

    dev = "cuda:0"
    cfg = VisRAGConfig.full()
    tok = StubTokenizer(cfg.vocab)
    sd = random_state_dict_device(cfg, 2024, dev)
    engines = {"bf16": VisRAGEngine(cfg, sd, dev, dtype=torch.bfloat16), "fp16": VisRAGEngine(cfg, sd, dev, dtype=torch.float16)}
    del sd
    torch.cuda.empty_cache()
    rs = np.random.RandomState(1000)
    pages = [Image.fromarray(x) for x in rs.randint(0, 256, (a.pages, a.page_px, a.page_px, 3), dtype=np.uint8)]
    pb = prepare_batch([""] * a.pages, pages, tok, cfg, 2048)
    max_len = int(pb.seq_lens.max())
    steps, reps = {}, {}
    for name, eng in engines.items():
        groups, src, pos, cu = eng.upload(pb)
        steps[name] = (lambda e=eng, g=groups, s=src, p=pos, c=cu: e.encode_device(g, pb.group_row0, pb.n_slices, s, p, c, max_len))
        for _ in range(a.warmup):
            reps[name] = steps[name]()
    torch.cuda.synchronize()
    state_before = gpu_state()
    rates, clocks = {name: [] for name in engines}, {name: [] for name in engines}
    for _ in range(a.runs):
        for name, step in steps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with WindowSampler() as smp:
                e0.record()
                for _ in range(a.steps):
                    step()
                e1.record()
                torch.cuda.synchronize()
            rates[name].append(a.pages * a.steps / (e0.elapsed_time(e1) / 1e3))
            clocks[name].append((smp.sm_mhz, smp.power_w))
    state_after = gpu_state()
    from visrag_b200 import ops

    kinds = {}
    for name, step in steps.items():            # kernel time per kind, one step each, profiler on (not the timed windows)
        ops.profile_begin()
        step()
        prof = ops.profile_end()
        kinds[name] = {}
        for k, (_, ms, _) in prof.items():
            kk = k.split(":")[0]
            kinds[name][kk] = kinds[name].get(kk, 0.0) + ms
    x, y = reps["bf16"].double(), reps["fp16"].double()
    cos = (x * y).sum(1) / (x.norm(dim=1) * y.norm(dim=1))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    spread = {k: float(max(v) - min(v)) for k, v in rates.items()}
    for name in engines:
        print(f"{name}: pages/s per window {', '.join(f'{r:.1f}' for r in rates[name])}; median {med[name]:.1f}, "
              f"spread {spread[name]:.1f}; SM MHz / W per window {', '.join(f'{c} / {w}' for c, w in clocks[name])}")
        print(f"{name}: kernel ms per kind in one profiled step: " + ", ".join(f"{k} {v:.1f}" for k, v in sorted(kinds[name].items())))
    print(f"fp16 / bf16 = {med['fp16'] / med['bf16']:.4f}; embeddings bf16 vs fp16: min cos {float(cos.min()):.7f}, "
          f"max |diff| {float((x - y).abs().max()):.3e}")
    print(f"card {state_before.get('name')}, power limit {state_before.get('power.limit')}, SM clock "
          f"{state_before.get('clocks.sm')} before / {state_after.get('clocks.sm')} after the timed windows "
          f"(max {state_before.get('clocks.max.sm')})")
    print(json.dumps({"pages_per_s": med, "spread": spread, "windows": rates, "sm_mhz_power_w": clocks, "kernel_ms": kinds,
                      "pages": a.pages, "steps": a.steps,
                      "min_cos_bf16_fp16": float(cos.min()), "max_abs_diff_bf16_fp16": float((x - y).abs().max()),
                      "gpu_before": state_before, "gpu_after": state_after}))


if __name__ == "__main__":
    main()
