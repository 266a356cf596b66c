"""GPU check of the wgmma GEMM.

Each case runs in its own subprocess (a device trap poisons the CUDA context), results go to stdout
and check_gemm.log in the system temporary directory. Reference = torch fp32 matmul of the same bf16 inputs.
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def ref_linear(a, w, bias=None, gelu=False, scale=1.0, resid=None, rowadd=None):
    import torch

    y = a.float() @ w.float().t()
    if bias is not None:
        y = y + bias
    if gelu:
        y = torch.nn.functional.gelu(y)
    y = y * scale
    if rowadd is not None:
        idx = torch.arange(y.shape[0], device=y.device) % rowadd.shape[0]
        y = y + rowadd[idx]
    if resid is not None:
        y = y + resid
    return y


def report(name, got, want, tol):
    import torch

    err = (got.float() - want.float()).abs().max().item()
    ref = want.float().abs().max().item()
    bad = not (err <= tol * max(ref, 1.0)) or not torch.isfinite(got.float()).all().item()
    print(f"{'FAIL' if bad else 'ok  '} {name}: max_abs_err={err:.4e} ref_max={ref:.3e}", flush=True)
    return not bad


def case_basic(bn):
    import torch
    from visrag_b200 import ops

    torch.manual_seed(0)
    ok = True
    for (M, N, K) in [(128, 256, 64), (128, 256, 128), (256, 512, 1152), (1000, 1152, 4304), (333, 4304, 1152), (64, 2304, 2304), (4096, 3840, 1152)]:
        if bn == 128 and N < 128:
            continue
        a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        got = ops.gemm(a, w, out_dtype=torch.float32, block_n=bn)
        torch.cuda.synchronize()
        ok &= report(f"plain f32 bn={bn} M={M} N={N} K={K}", got, ref_linear(a, w), 2e-3)
    return ok


def case_epilogues(bn):
    import torch
    from visrag_b200 import ops, _lib as L

    torch.manual_seed(1)
    ok = True
    M, N, K = 777, 1152, 640
    a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda")
    resid = torch.randn(M, N, device="cuda")
    rowadd = torch.randn(37, N, device="cuda")
    got = ops.gemm(a, w, bias=bias, block_n=bn)
    ok &= report("bias bf16", got, ref_linear(a, w, bias), 1e-2)
    got = ops.gemm(a, w, bias=bias, gelu=True, block_n=bn)
    ok &= report("bias gelu bf16", got, ref_linear(a, w, bias, gelu=True), 1e-2)
    got = ops.gemm(a, w, bias=bias, rowadd=rowadd, out_dtype=torch.float32, block_n=bn)
    ok &= report("bias rowadd f32", got, ref_linear(a, w, bias, rowadd=rowadd), 2e-3)
    x = resid.clone()
    got = ops.gemm(a, w, bias=bias, resid=x, out=x, scale=0.25, out_dtype=torch.float32, block_n=bn)
    ok &= report("bias scale resid in-place f32", got, ref_linear(a, w, bias, scale=0.25, resid=resid), 2e-3)
    # N tail not multiple of 32 (fc1: 4304)
    N2 = 4304
    w2 = (torch.randn(N2, K, device="cuda") * 0.05).bfloat16()
    b2 = torch.randn(N2, device="cuda")
    got = ops.gemm(a, w2, bias=b2, gelu=True, block_n=bn)
    ok &= report("fc1-like N=4304 gelu", got, ref_linear(a, w2, b2, gelu=True), 1e-2)
    # row-tail / odd token counts with a bf16 output (the feature-major kernel pairs lanes for its bf16 stores)
    for M3 in (1, 31, 130):
        a4 = a[:M3].contiguous()
        got = ops.gemm(a4, w, bias=bias, block_n=bn)
        ok &= report(f"bias bf16 M={M3}", got, ref_linear(a4, w, bias), 1e-2)
        x = resid[:M3].clone()
        got = ops.gemm(a4, w, resid=x, out=x, out_dtype=torch.float32, block_n=bn)
        ok &= report(f"resid in-place f32 M={M3}", got, ref_linear(a4, w, resid=resid[:M3]), 2e-3)
    if bn == 3:
        return ok  # the feature-major kernel implements LINEAR epilogues only
    # RoPE epilogue
    T, H = 300, 2304
    hd = 64
    a3 = (torch.randn(T, H, device="cuda") * 0.5).bfloat16()
    w3 = (torch.randn(3 * H, H, device="cuda") * 0.03).bfloat16()
    pos = torch.randint(0, 500, (T,), device="cuda", dtype=torch.int32)
    inv = 1.0 / (10000 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
    fr = torch.outer(torch.arange(2048, device="cuda").float(), inv)
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    got = ops.gemm(a3, w3, mode=L.VR_EPI_ROPE, positions=pos, rope_cos=cos, rope_sin=sin, rope_cols=2 * H, block_n=bn)
    y = (a3.float() @ w3.float().t()).view(T, 3, H // hd, hd)
    c = cos[pos.long()][:, None, None, :]
    s = sin[pos.long()][:, None, None, :]
    qk = y[:, :2]
    lo, hi = qk[..., :32], qk[..., 32:]
    rot = torch.cat([lo * c - hi * s, hi * c + lo * s], dim=-1)
    want = torch.cat([rot, y[:, 2:]], dim=1).reshape(T, 3 * H)
    ok &= report("rope qkv", got, want, 1e-2)
    # SwiGLU epilogue (interleaved gate/up rows)
    I = 5760
    wg = (torch.randn(I, H, device="cuda") * 0.03).bfloat16()
    wu = (torch.randn(I, H, device="cuda") * 0.03).bfloat16()
    wi = torch.stack([wg.view(I // 32, 32, H), wu.view(I // 32, 32, H)], dim=1).reshape(2 * I, H).contiguous()
    got = ops.gemm(a3, wi, mode=L.VR_EPI_SWIGLU, block_n=bn)
    g = a3.float() @ wg.float().t()
    u = a3.float() @ wu.float().t()
    ok &= report("swiglu", got, torch.nn.functional.silu(g) * u, 1e-2)
    return ok


ANATOMY = [  # the epilogue-heavy ViT / LM shapes with the epilogue peeled off piece by piece
    (131072, 1152, 4304, {}), (131072, 1152, 4304, {"f32": True}), (131072, 1152, 4304, {"resid": True}),
    (131072, 1152, 1152, {}), (131072, 1152, 1152, {"f32": True}), (131072, 1152, 1152, {"resid": True}),
    (131072, 4304, 1152, {}), (131072, 4304, 1152, {"gelu": True, "bias": True}),
    (8704, 2304, 5760, {}), (8704, 2304, 5760, {"resid": True}), (8704, 2304, 2304, {}), (8704, 2304, 2304, {"resid": True}),
]


def case_anatomy(bn):
    return case_perf(bn, ANATOMY, cublas=False)


def case_perf(bn, shapes=None, cublas=True):
    import torch
    from visrag_b200 import ops

    torch.manual_seed(2)
    ok = True
    for (M, N, K, kw) in shapes or [
        (65536, 3840, 1152, {}),
        (65536, 4304, 1152, {"gelu": True, "bias": True}),
        (65536, 1152, 4304, {"resid": True, "bias": True}),
        (65536, 1152, 1152, {"resid": True, "bias": True}),
        (16384, 11520, 2304, {}),
        (16384, 2304, 5760, {"resid": True}),
        (8192, 8192, 8192, {}),
    ]:
        a = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        bias = torch.randn(N, device="cuda") if kw.get("bias") else None
        x = torch.randn(M, N, device="cuda") if kw.get("resid") else None
        args = dict(bias=bias, gelu=kw.get("gelu", False), block_n=bn)
        if x is not None:
            args.update(resid=x, out=x, out_dtype=torch.float32)
        elif kw.get("f32"):
            args.update(out_dtype=torch.float32)
        for _ in range(3):
            ops.gemm(a, w, **args)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 10
        ev0.record()
        for _ in range(n):
            ops.gemm(a, w, **args)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / n
        tf = 2.0 * M * N * K / ms / 1e9
        if not cublas:
            print(f"perf bn={bn} M={M} N={N} K={K} {kw}: {ms:.3f} ms {tf:.1f} TFLOP/s", flush=True)
            continue
        # cuBLAS for context
        for _ in range(3):
            torch.matmul(a, w.t())
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(n):
            torch.matmul(a, w.t())
        ev1.record()
        torch.cuda.synchronize()
        ms2 = ev0.elapsed_time(ev1) / n
        print(f"perf bn={bn} M={M} N={N} K={K} {kw}: {ms:.3f} ms {tf:.1f} TFLOP/s | cublas(plain) {ms2:.3f} ms {2.0*M*N*K/ms2/1e9:.1f} TFLOP/s", flush=True)
    return ok


CASES = {"basic": case_basic, "epilogues": case_epilogues, "perf": case_perf, "anatomy": case_anatomy}

if __name__ == "__main__":
    if len(sys.argv) >= 3:
        ok = CASES[sys.argv[1]](int(sys.argv[2]))
        sys.exit(0 if ok else 1)
    import tempfile

    log = open(os.path.join(tempfile.gettempdir(), "check_gemm.log"), "w")
    rc_all = 0
    for case in ("basic", "epilogues", "perf"):
        for bn in (256, 128, 3):
            t0 = time.time()
            p = subprocess.run([sys.executable, __file__, case, str(bn)], capture_output=True, text=True, timeout=600)
            msg = f"=== {case} bn={bn} rc={p.returncode} ({time.time()-t0:.1f}s)\n{p.stdout}{p.stderr[-3000:]}\n"
            print(msg, flush=True)
            log.write(msg)
            log.flush()
            rc_all |= p.returncode
    sys.exit(rc_all)
