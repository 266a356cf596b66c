"""Times vr_attention at the three attention shapes of the bench step (128 pages of 448x448), in one process, over
several rounds: CUDA events around --launches back-to-back launches per round, median and spread (min..max) of the
per-launch time over the rounds, and useful TFLOP/s (4 d per visible (query, key) pair: QK^T plus PV at the head dim,
not the padded head stride). F.scaled_dot_product_attention at the ViT shape is timed the same way for context.
One JSON line per shape.

The library is loaded through visrag_b200._lib, so VR_LIB=<path to libvisrag_b200.so> times another build (for example
one of the parent commit) with the same script.
  python tools/bench_attention.py [--rounds 5] [--launches 10] [--shapes vit,lm,resampler]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from visrag_b200 import _lib as L  # noqa: E402
from visrag_b200 import ops  # noqa: E402

DEV = "cuda"


def gpu_info():
    """Card name, power limit and SM clocks (read-only query)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        line = r.stdout.strip().splitlines()[torch.cuda.current_device()]
        return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "nvidia_smi": f"unavailable ({e})"}


def time_rounds(fn, rounds, launches):
    fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        per.append(e0.elapsed_time(e1) / launches)
    return per


def report(name, per, flops, extra=None):
    med = statistics.median(per)
    rec = {"shape": name, "ms_median": round(med, 4), "ms_min": round(min(per), 4), "ms_max": round(max(per), 4),
           "spread_pct": round(100 * (max(per) - min(per)) / med, 2), "tflops_useful": round(flops / med / 1e9, 1)}
    rec.update(extra or {})
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--pages", type=int, default=128)
    ap.add_argument("--no-sdpa", action="store_true")
    ap.add_argument("--shapes", type=lambda x: set(x.split(",")), default={"vit", "lm", "resampler"},
                    help="a later shape runs on a card that the earlier ones have heated")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_attention needs a CUDA device"
    torch.manual_seed(0)
    print(json.dumps({"gpu": gpu_info(), "lib": os.path.relpath(L.LIB_PATH), "rounds": a.rounds, "launches": a.launches}), flush=True)

    if "vit" in a.shapes:
        vit_shape(a)
    if "lm" in a.shapes:
        lm_shape(a)
    if "resampler" in a.shapes:
        resampler_shape(a)


def vit_shape(a):
    S = a.pages
    # ViT: S slices x 1024 tokens, 16 heads of 72 stored at stride 80 (zero pad columns), non-causal
    nh, hd, hs, n = 16, 72, 80, 1024
    T = S * n
    qkv = torch.zeros(T, 3, nh, hs, dtype=torch.bfloat16, device=DEV)
    qkv[..., :hd] = torch.randn(T, 3, nh, hd, device=DEV).bfloat16()
    qkv = qkv.view(T, 3 * nh * hs)
    cu = torch.arange(0, T + 1, n, dtype=torch.int32, device=DEV)
    out = torch.empty(T, nh * hd, dtype=torch.bfloat16, device=DEV)

    def vit():
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                      batch=S, cu_k=cu, max_k=n, cu_q=cu, max_q=n, causal=False, scale=hd ** -0.5, out=out)

    vit_flops = 4.0 * S * nh * n * n * hd
    report("vit", time_rounds(vit, a.rounds, a.launches), vit_flops, {"dims": f"{S}x{nh}h x {n} tok, d {hd}/{hs}"})
    if not a.no_sdpa:
        qh = qkv.view(S, n, 3, nh, hs)[..., :hd].permute(2, 0, 3, 1, 4).contiguous()  # [3, S, nh, n, hd]

        def sdpa():
            F.scaled_dot_product_attention(qh[0], qh[1], qh[2])

        report("vit_sdpa", time_rounds(sdpa, a.rounds, a.launches), vit_flops, {"dims": f"{S}x{nh}h x {n} tok, d {hd}"})
        del qh


def lm_shape(a):
    S = a.pages
    # LM: S sequences x 68 tokens, 36 heads of 64, causal var-len (packed)
    nh, hd, n = 36, 64, 68
    H = nh * hd
    T = S * n
    qkv = torch.randn(T, 3 * H, device=DEV).bfloat16()
    cu = torch.arange(0, T + 1, n, dtype=torch.int32, device=DEV)
    out = torch.empty(T, H, dtype=torch.bfloat16, device=DEV)

    def lm():
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=H, v_col0=2 * H, head_stride=hd, head_dim=hd, heads=nh, batch=S,
                      cu_k=cu, max_k=n, cu_q=cu, max_q=n, causal=True, scale=hd ** -0.5, out=out)

    report("lm", time_rounds(lm, a.rounds, a.launches), 4.0 * S * nh * hd * n * (n + 1) / 2, {"dims": f"{S}x{nh}h x {n} tok causal, d {hd}"})


def resampler_shape(a):
    S = a.pages
    # Resampler: 64 shared learned queries x 1024 keys per slice, 18 heads of 128
    nh, hd, n = 18, 128, 1024
    E = nh * hd
    q = torch.randn(64, E, device=DEV).bfloat16()
    k = torch.randn(S * n, E, device=DEV).bfloat16()
    v = torch.randn(S * n, E, device=DEV).bfloat16()
    cu = torch.arange(0, S * n + 1, n, dtype=torch.int32, device=DEV)
    out = torch.empty(S * 64, E, dtype=torch.bfloat16, device=DEV)

    def rs():
        ops.attention(q, k, v, q_col0=0, k_col0=0, v_col0=0, head_stride=hd, head_dim=hd, heads=nh, batch=S, cu_k=cu,
                      max_k=n, cu_q=None, max_q=64, causal=False, scale=hd ** -0.5, out=out)

    report("resampler", time_rounds(rs, a.rounds, a.launches), 4.0 * S * nh * 64 * n * hd, {"dims": f"{S}x{nh}h 64 q x {n} keys, d {hd}"})


if __name__ == "__main__":
    main()
