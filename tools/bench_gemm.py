"""Time every GEMM launch class of the bench.py step (128 pages of 448 x 448: ViT at M = 131072 tokens, LM at M = 8704)
at its exact shape and epilogue. The arms alternate in one process over several rounds:
  old       the cooperative kernel at the tile width vr_gemm picked before the ping-pong kernel (explicit block_n)
  auto      what vr_gemm picks now (block_n = 0): what the step runs
  pp_nfast  ping-pong kernel, plain n-fastest tile order (block_n = 5)
  pp        ping-pong kernel, L2-sliced tile order (block_n = 2): pp_nfast -> pp is the tile-order step
  pp_mc     ping-pong kernel in CTA pairs with the B tile multicast (block_n = 4): pp -> pp_mc is the multicast step
with plain cuBLAS (torch.matmul, bf16 out, no epilogue) beside them for context.

    python tools/bench_gemm.py [--rounds 5] [--only lm] [--match KEY] [--arms auto]

Prints the card name, power limit and SM clocks (read-only nvidia-smi query) first, then one JSON line per class:
median ms and TFLOP/s of each arm, their spread over rounds ((max - min) / median), and max |arm - old| on the same
inputs; a last line sums launches x ms over the step for each arm.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (class key as bench.py's roofline pass names it, launches per step, epilogue arguments)
CLASSES = [
    ("131072x4352x1152:gelubf16", 26, {"bias": True, "gelu": True}),          # ViT fc1 (MLP width 4304 padded to 4352)
    ("131072x1152x4352:+residf32", 26, {"bias": True, "resid": True}),        # ViT fc2
    ("131072x4304x1152:gelubf16", 0, {"bias": True, "gelu": True}),           # the unpadded fc1 / fc2, for comparison:
    ("131072x1152x4304:+residf32", 0, {"bias": True, "resid": True}),         #   not in the step
    ("131072x3840x1152:bf16", 26, {"bias": True}),                            # ViT qkv
    ("131072x1152x1152:+residf32", 26, {"bias": True, "resid": True}),        # ViT proj
    ("8704x11520x2304:swiglu", 40, {"swiglu": True}),                         # LM gate|up
    ("8704x6912x2304:rope", 40, {"rope": True}),                              # LM qkv
    ("8704x2304x5760:+residf32", 40, {"resid": True, "scale": 0.2}),          # LM down
    ("8704x2304x2304:+residf32", 40, {"resid": True, "scale": 0.2}),          # LM o
    ("131072x2304x2304:bf16", 2, {"bias": True}),                             # resampler k, v
    ("131072x1152x640:f32", 1, {"bias": True, "rowadd": True, "f32": True}),  # patch embed (K 588 padded to 640)
    ("131072x2304x1152:f32", 1, {"f32": True}),                               # resampler kv
    ("8192x2304x2304:f32", 2, {"bias": True, "f32": True}),                   # resampler o / proj
]


PP_ARMS = {"pp_nfast": 5, "pp": 2, "pp_mc": 4}


def cooperative_width(M, N):
    """The tile width vr_gemm chose for the cooperative kernel before the ping-pong kernel existed."""
    if M <= 128:
        return 64
    if N < 256:
        return 128
    return 192 if N % 192 == 0 and N % 256 != 0 else 256


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"query": q, "value": r.stdout.strip() or r.stderr.strip()}


def make_case(M, N, K, kw, seed):
    import torch
    from visrag_b200 import ops, _lib as L

    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).bfloat16()
    args = {}
    if kw.get("bias"):
        args["bias"] = torch.randn(N, device="cuda", generator=g)
    if kw.get("gelu"):
        args["gelu"] = True
    if kw.get("rowadd"):
        args["rowadd"] = torch.randn(1024, N, device="cuda", generator=g)
    if "scale" in kw:
        args["scale"] = kw["scale"]
    if kw.get("f32"):
        args["out_dtype"] = torch.float32
    if kw.get("rope"):
        inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, device="cuda").float() / 64))
        fr = torch.outer(torch.arange(2048, device="cuda").float(), inv)
        args.update(mode=L.VR_EPI_ROPE, positions=torch.randint(0, 2048, (M,), device="cuda", dtype=torch.int32, generator=g),
                    rope_cos=fr.cos().contiguous(), rope_sin=fr.sin().contiguous(), rope_cols=2 * N // 3)
    if kw.get("swiglu"):
        args["mode"] = L.VR_EPI_SWIGLU
    x0 = torch.randn(M, N, device="cuda", generator=g) if kw.get("resid") else None

    def run(bn, x=None):
        if x0 is None:
            return ops.gemm(a, w, block_n=bn, **args)
        x = x0 if x is None else x  # timing accumulates into x0 in place, as the step does into its residual stream
        return ops.gemm(a, w, resid=x, out=x, out_dtype=torch.float32, block_n=bn, **args)

    def fresh(bn):
        return run(bn, None if x0 is None else x0.clone())

    return a, w, run, fresh


def time_ms(fn, iters):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window-ms", type=float, default=40.0, help="least time per timed window")
    ap.add_argument("--only", choices=["vit", "lm"], default=None, help="ViT-side (M = 131072) or LM (M = 8704) classes")
    ap.add_argument("--match", default=None, help="only the classes whose key contains this string")
    ap.add_argument("--no-cublas", dest="cublas", action="store_false")
    ap.add_argument("--arms", default=None, help="comma-separated subset of old,auto,pp_nfast,pp,pp_mc (old always runs: "
                                                  "it is the reference of max_abs_diff_vs_old)")
    a = ap.parse_args()

    import torch

    print(json.dumps({"gpu": gpu_info(), "torch": torch.__version__, "lib": os.environ.get("VR_LIB", "in-tree")}), flush=True)
    tot = {}
    for ci, (key, per_step, kw) in enumerate(CLASSES):
        M, N, K = (int(v) for v in key.split(":")[0].split("x"))
        if a.only == "lm" and M != 8704 or a.only == "vit" and M == 8704 or a.match and a.match not in key:
            continue
        old_bn = cooperative_width(M, N)
        A, W, run, fresh = make_case(M, N, K, kw, 100 + ci)
        arm_bn = {"old": old_bn, "auto": 0}
        arm_bn.update(PP_ARMS)
        if a.arms:
            arm_bn = {k: v for k, v in arm_bn.items() if k == "old" or k in a.arms.split(",")}
        ref = fresh(old_bn)
        diff = {}
        for k, bn in arm_bn.items():
            if k != "old":
                out = fresh(bn)
                diff[k] = (out.float() - ref.float()).abs().max().item()
                del out
        del ref
        arms = {k: (lambda bn=bn: run(bn)) for k, bn in arm_bn.items()}
        if a.cublas:
            arms["cublas_plain"] = lambda: torch.matmul(A, W.t())
        iters = max(3, int(a.window_ms / max(time_ms(arms["old"], 2), 1e-3)))
        samples = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                samples[k].append(time_ms(fn, iters))
        flops = 2.0 * M * N * K
        res = {"class": key, "launches_per_step": per_step, "iters": iters, "rounds": a.rounds}
        for k, v in samples.items():
            v = sorted(v)
            med = v[len(v) // 2]
            res[k] = {"ms": round(med, 4), "tflops": round(flops / med / 1e9, 1), "spread": round((v[-1] - v[0]) / med, 4)}
            if k in arm_bn:
                res[k]["block_n"] = arm_bn[k]
                res[k]["speedup_vs_old"] = round(res["old"]["ms"] / med, 3) if "old" in res else None
                tot[k] = tot.get(k, 0.0) + per_step * med
        res["max_abs_diff_vs_old"] = diff
        print(json.dumps(res), flush=True)
        del A, W, run, fresh
        torch.cuda.empty_cache()
    print(json.dumps({"step_gemm_ms": {k: round(v, 2) for k, v in tot.items()},
                      "speedup_vs_old": {k: round(tot["old"] / v, 3) for k, v in tot.items()}}), flush=True)


if __name__ == "__main__":
    main()
