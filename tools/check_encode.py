"""GPU check of the encode path, stage by stage.
Each stage runs in its own subprocess; results -> stdout and check_encode.log in the system temporary directory."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def report(name, got, want, tol):
    import torch

    got, want = got.float().cpu(), want.float().cpu()
    err = (got - want).abs().max().item()
    ref = want.abs().max().item()
    bad = not (err <= tol * max(ref, 1e-3)) or not torch.isfinite(got).all().item()
    print(f"{'FAIL' if bad else 'ok  '} {name}: max_abs_err={err:.4e} ref_max={ref:.3e}", flush=True)
    return not bad


def stage_elementwise():
    import torch
    import torch.nn.functional as F
    from visrag_b200 import ops

    torch.manual_seed(0)
    ok = True
    dev = "cuda"
    # (slices, h, w): 4-byte-only aligned strips (odd grid width), 16-byte aligned strips, a wide slice, every byte value
    for (S, hh_, ww_) in ((3, 28, 42), (2, 448, 448), (1, 28, 1414), (5, 14, 70)):
        px = torch.randint(0, 256, (S, hh_, ww_, 3), dtype=torch.uint8, device=dev)
        px.view(-1)[:256] = torch.arange(256, dtype=torch.uint8, device=dev)
        got = ops.im2col_norm(px, 14, 640)
        # reference arithmetic on the CPU like torchvision's ToTensor/Normalize (true division; CUDA torch divides by reciprocal)
        x = ((px.cpu().float() / 255 - 0.5) / 0.5).permute(0, 3, 1, 2)  # [S,3,h,w]
        want = F.unfold(x, kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588).to(dev)
        ok &= report(f"im2col {S}x{hh_}x{ww_}", got[:, :588], want.bfloat16(), 0.0)   # bit-exact bf16
        ok &= report("im2col pad", got[:, 588:], torch.zeros_like(got[:, 588:]), 0.0)
    px = torch.randint(0, 256, (4, 32, 48, 3), dtype=torch.uint8, device=dev)       # another patch size / row pitch
    got = ops.im2col_norm(px, 16, 768)
    x = ((px.cpu().float() / 255 - 0.5) / 0.5).permute(0, 3, 1, 2)
    ok &= report("im2col patch16", got, F.unfold(x, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768).to(dev).bfloat16(), 0.0)
    for D in (288, 1152, 2304):
        x = torch.randn(1000, D, device=dev) * 3 + 1
        g, b = torch.randn(D, device=dev), torch.randn(D, device=dev)
        add = torch.randn(37, D, device=dev)
        o1, o2 = ops.layernorm(x, g, b, 1e-6, add=add)
        ref = F.layer_norm(x, (D,), g, b, 1e-6)
        ok &= report(f"layernorm D={D}", o1, ref, 1e-2)
        ok &= report(f"layernorm+add D={D}", o2, ref + add[torch.arange(1000, device=dev) % 37], 1e-2)
        o = ops.rmsnorm(x, g, 1e-5)
        ok &= report(f"rmsnorm D={D}", o, x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * g, 1e-2)
    D = 256
    emb = torch.randn(512, D, device=dev).bfloat16()
    vis = torch.randn(128, D, device=dev)
    src = torch.tensor([-1 - 5, 0, 1, 127, -1 - 511, -1 - 0], dtype=torch.int32, device=dev)
    h = ops.build_lm_input(src, emb, 12.0, vis)
    want = torch.stack([emb[5].float() * 12, vis[0], vis[1], vis[127], emb[511].float() * 12, emb[0].float() * 12])
    ok &= report("build_lm_input", h, want, 1e-6)
    # pool_norm is checked against its fp64 bound in tests/test_gpu_kernel_bounds.py
    return ok


def _attn_ref(q, k, v, scale, causal):
    import torch

    s = (q.float() @ k.float().transpose(-1, -2)) * scale
    if causal:
        Lq, Lk = s.shape[-2], s.shape[-1]
        m = torch.ones(Lq, Lk, dtype=torch.bool, device=s.device).tril(Lk - Lq)
        s = s.masked_fill(~m, float("-inf"))
    return torch.softmax(s, -1) @ v.float()


def stage_attention(force_v1=False):
    import torch
    from visrag_b200 import ops, _lib as L

    L.lib().vr_attention_force_v1(1 if force_v1 else 0)
    try:
        return _stage_attention_body(torch, ops)
    finally:
        L.lib().vr_attention_force_v1(0)


def stage_attention_v1():
    return stage_attention(True)


def _stage_attention_body(torch, ops):
    torch.manual_seed(1)
    ok = True
    dev = "cuda"
    # --- ViT style: heads x 72 padded to 80, non-causal, fixed N per slice
    # ((40, 784, 16) has partial last query and key tiles in every sequence; ones=True: V carries a ones column in its
    #  padding and VR_ATTN_V_ONES_COLUMN is set - the kernels must ignore the column)
    for (S, N, nh, ones) in [(1, 128, 1, False), (1, 256, 2, False), (3, 1024, 4, True), (2, 1036, 16, False), (5, 130, 3, True),
                             (40, 784, 16, True), (7, 300, 5, False), (33, 1024, 16, True)]:
        hd, hs = 72, 80
        qkv = torch.zeros(S * N, 3, nh, hs, device=dev)
        qkv[..., :hd] = torch.randn(S * N, 3, nh, hd, device=dev)
        if ones:
            qkv[:, 2, :, hd] = 1.0
        qkv = qkv.reshape(S * N, 3 * nh * hs).bfloat16()
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=dev)
        out = torch.zeros(S * N, nh * hd, dtype=torch.bfloat16, device=dev)
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                      batch=S, cu_k=cu, max_k=N, cu_q=cu, max_q=N, causal=False, scale=hd ** -0.5, out=out, v_ones_column=ones)
        torch.cuda.synchronize()
        x = qkv.view(S, N, 3, nh, hs)[..., :hd].permute(2, 0, 3, 1, 4)  # [3,S,nh,N,hd]
        want = _attn_ref(x[0], x[1], x[2], hd ** -0.5, False).permute(0, 2, 1, 3).reshape(S * N, nh * hd)
        ok &= report(f"attn vit S={S} N={N} heads={nh} ones={ones}", out, want, 2e-2)
    # --- non-causal var-len with head dim 64 (no padding column): ragged sequences, some shorter than one tile pair
    for lens in ([300, 129, 1000, 128, 257, 512],):
        nh, hd = 3, 64
        H = nh * hd
        T = sum(lens)
        qkv = torch.randn(T, 3 * H, device=dev).bfloat16()
        cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
        out = torch.zeros(T, H, dtype=torch.bfloat16, device=dev)
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=H, v_col0=2 * H, head_stride=64, head_dim=64, heads=nh, batch=len(lens),
                      cu_k=cu, max_k=max(lens), cu_q=cu, max_q=max(lens), causal=False, scale=hd ** -0.5, out=out)
        torch.cuda.synchronize()
        wants = []
        for i, n in enumerate(lens):
            x = qkv[cu[i]:cu[i + 1]].view(n, 3, nh, hd).permute(1, 2, 0, 3)
            wants.append(_attn_ref(x[0], x[1], x[2], hd ** -0.5, False).permute(1, 0, 2).reshape(n, H))
        ok &= report(f"attn non-causal var-len lens={lens}", out, torch.cat(wants), 2e-2)
    # --- growing row maxima: later key tiles carry much larger scores, which forces the O rescale
    for (S, N, nh) in [(2, 512, 2), (1, 1024, 3)]:
        hd, hs = 72, 80
        qkv = torch.zeros(S * N, 3, nh, hs, device=dev)
        qkv[..., :hd] = torch.randn(S * N, 3, nh, hd, device=dev)
        ramp = torch.linspace(0.2, 6.0, N, device=dev).repeat(S)[:, None, None]   # key scale grows with position
        qkv[:, 1, :, :hd] *= ramp
        qkv[:, 2, :, hd] = 1.0 if S == 2 else 0.0
        qkv = qkv.reshape(S * N, 3 * nh * hs).bfloat16()
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=dev)
        out = torch.zeros(S * N, nh * hd, dtype=torch.bfloat16, device=dev)
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                      batch=S, cu_k=cu, max_k=N, cu_q=cu, max_q=N, causal=False, scale=hd ** -0.5, out=out, v_ones_column=(S == 2))
        torch.cuda.synchronize()
        x = qkv.view(S, N, 3, nh, hs)[..., :hd].permute(2, 0, 3, 1, 4)
        want = _attn_ref(x[0], x[1], x[2], hd ** -0.5, False).permute(0, 2, 1, 3).reshape(S * N, nh * hd)
        ok &= report(f"attn vit growing-max S={S} N={N} heads={nh}", out, want, 2e-2)
    # --- LM style: causal var-len, hd 64
    for lens in ([68], [1, 5, 68, 127, 128, 129, 300], [670, 33]):
        nh, hd = 4, 64
        H = nh * hd
        T = sum(lens)
        qkv = torch.randn(T, 3 * H, device=dev).bfloat16()
        cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
        out = torch.zeros(T, H, dtype=torch.bfloat16, device=dev)
        ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=H, v_col0=2 * H, head_stride=64, head_dim=64, heads=nh, batch=len(lens),
                      cu_k=cu, max_k=max(lens), cu_q=cu, max_q=max(lens), causal=True, scale=hd ** -0.5, out=out)
        torch.cuda.synchronize()
        wants = []
        for i, n in enumerate(lens):
            x = qkv[cu[i]:cu[i + 1]].view(n, 3, nh, hd).permute(1, 2, 0, 3)
            wants.append(_attn_ref(x[0], x[1], x[2], hd ** -0.5, True).permute(1, 0, 2).reshape(n, H))
        ok &= report(f"attn lm causal lens={lens}", out, torch.cat(wants), 2e-2)
    # --- resampler style: 64 shared queries, hd 128
    for (S, N, nh) in [(1, 1024, 2), (3, 1036, 18), (2, 100, 2)]:
        E = nh * 128
        q = torch.zeros(128, E, device=dev)
        q[:64] = torch.randn(64, E, device=dev)
        q = q.bfloat16()
        k = torch.randn(S * N, E, device=dev).bfloat16()
        v = torch.randn(S * N, E, device=dev).bfloat16()
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=dev)
        out = torch.zeros(S * 64, E, dtype=torch.bfloat16, device=dev)
        ops.attention(q, k, v, q_col0=0, k_col0=0, v_col0=0, head_stride=128, head_dim=128, heads=nh, batch=S, cu_k=cu,
                      max_k=N, cu_q=None, max_q=64, causal=False, scale=128 ** -0.5, out=out)
        torch.cuda.synchronize()
        Q = q[:64].view(64, nh, 128).permute(1, 0, 2)[None]
        K = k.view(S, N, nh, 128).permute(0, 2, 1, 3)
        V = v.view(S, N, nh, 128).permute(0, 2, 1, 3)
        want = _attn_ref(Q, K, V, 128 ** -0.5, False).permute(0, 2, 1, 3).reshape(S * 64, E)
        ok &= report(f"attn resampler S={S} N={N} heads={nh}", out, want, 2e-2)
    return ok


def stage_attention_perf():
    """ViT attention at bench shape (128 slices x 16 heads x 1024 tokens x 72) timed alone: TFLOP/s of 4*N^2*D."""
    import torch
    from visrag_b200 import ops, _lib as L

    S, N, nh, hd, hs = 128, 1024, 16, 72, 80
    qkv = torch.zeros(S * N, 3, nh, hs, device="cuda")
    qkv[..., :hd] = torch.randn(S * N, 3, nh, hd, device="cuda")
    qkv = qkv.reshape(S * N, 3 * nh * hs).bfloat16()
    cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device="cuda")
    out = torch.zeros(S * N, nh * hd, dtype=torch.bfloat16, device="cuda")
    qkv1 = qkv.clone().view(S * N, 3, nh, hs)
    qkv1[:, 2, :, hd] = 1.0
    qkv1 = qkv1.view(S * N, 3 * nh * hs)
    for force, ones in ((0, True), (0, False), (1, False)):
        L.lib().vr_attention_force_v1(force)
        src = qkv1 if ones else qkv

        def run():
            ops.attention(src, src, src, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                          batch=S, cu_k=cu, max_k=N, cu_q=cu, max_q=N, causal=False, scale=hd ** -0.5, out=out, v_ones_column=ones)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        print(f"attention variant {force} ones_column={ones}: {ms:.3f} ms  {4.0 * N * N * nh * hd * S / ms / 1e9:.1f} TFLOP/s (useful)", flush=True)
    L.lib().vr_attention_force_v1(0)
    return True


STAGES = {"elementwise": stage_elementwise, "attention": stage_attention, "attention_v1": stage_attention_v1,
          "attention_perf": stage_attention_perf}

if __name__ == "__main__":
    if len(sys.argv) == 2:
        sys.exit(0 if STAGES[sys.argv[1]]() else 1)
    import tempfile

    log = open(os.path.join(tempfile.gettempdir(), "check_encode.log"), "w")
    rc_all = 0
    for st in STAGES:
        t0 = time.time()
        p = subprocess.run([sys.executable, __file__, st], capture_output=True, text=True, timeout=900, cwd=ROOT)
        msg = f"=== {st} rc={p.returncode} ({time.time()-t0:.1f}s)\n{p.stdout}{p.stderr[-4000:]}\n"
        print(msg, flush=True)
        log.write(msg)
        log.flush()
        rc_all |= p.returncode
    sys.exit(rc_all)
