"""fp16 error bounds and checker for the kernels of an fp16 engine (VisRAGEngine(dtype=torch.float16)), next to the bf16
ones of tests/kernel_bounds.py, which they reuse wherever the arithmetic is the same.

  * Stored fp16 values: unit roundoff U16 = 2^-11 for normal values (11 significant bits). `check` handles the rounding of
    an fp16 output exactly, by the rule kernel_bounds.check applies to bf16: the stored value must be the round-to-nearest
    image of SOME y with |y - ref| <= bound, i.e. ref must lie within `bound` of the fp16 cell of the stored value
    (subnormals included). So no bound below adds the output rounding.
  * GEMM: an fp16 x fp16 product has 22 significant bits, exact in fp32 as the bf16 one is, so the accumulation model and
    the epilogue terms of kernel_bounds hold unchanged: gemm_linear_ref / gemm_rope_ref / gemm_swiglu_ref are the fp16
    bounds too.
  * Norms, build_lm_input: the fp32 arithmetic does not depend on the output type (an fp16 table entry widens to fp32
    exactly): norm_ref / layernorm_ref / rmsnorm_ref / build_lm_input_ref as they are.
  * Attention: P is rounded to fp16 for the PV MMA, round to nearest with no flush. Normal p (>= 2^-14):
    |fp16(p) - p| <= 2^-11 p. Subnormal p: the spacing is 2^-24, so |fp16(p) - p| <= 2^-25. Both together:
        |fp16(p) - p| <= 2^-11 p + 2^-25.
    The p of a key tile are in units of the running max at that tile; O is later rescaled by alpha <= 1 into the final
    max's units, where the row's l >= 1 (the maximal key contributes p = ex2(rounding of m c) = 1 up to 2^-22). So the
    absolute part adds at most 2^-25 sum_j |v_jd| to |out_d| (taken with l = 1), and the relative part replaces
    kernel_bounds.BF16_P c_id by F16_P c_id. A kernel that flushed p < 2^-14 to zero would be off by up to 2^-14 per key.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import kernel_bounds as KB

U16 = 2.0 ** -11
F16_P = 2.0 ** -11
F16_P_ABS = 2.0 ** -25


def attention_head_ref_f16(q, k, v, scale, causal, hs):
    """kernel_bounds.attention_head_ref with P rounded to fp16 instead of bf16 (see above). Returns (ref, e) [Lq, hd]."""
    Q, K, V = q.double(), k.double(), v.double()
    Lq, Lk = Q.shape[0], K.shape[0]
    s = (Q @ K.T) * scale
    ds = (Q.abs() @ K.abs().T) * (KB.k_steps(hs) * KB.ULP * scale)
    vis = torch.ones(Lq, Lk, dtype=torch.bool, device=s.device)
    if causal:
        vis = vis.tril(Lk - Lq)
        s = s.masked_fill(~vis, float("-inf"))
        ds = ds.masked_fill(~vis, 0.0)
    P = torch.softmax(s, -1)
    ref = P @ V
    c = P @ V.abs()
    nkt = -(-Lk // KB.ATT_BN)
    eps_s = 2 * ds.amax(-1, keepdim=True) + KB.EPS_EXP
    e = (F16_P + eps_s + (KB.k_steps(Lk) + nkt) * KB.ULP) * c + (eps_s + (36 + 2 * nkt) * KB.U) * ref.abs()
    return ref, e + F16_P_ABS * (vis.double() @ V.abs())


def attention_ref_f16(q, k, v, *, q_col0, k_col0, v_col0, head_stride, head_dim, heads, cu_k, cu_q, max_q, causal, scale):
    """kernel_bounds.attention_ref with the fp16 bound of attention_head_ref_f16."""
    batch = cu_k.numel() - 1
    rows = int(cu_q[-1]) if cu_q is not None else batch * max_q
    ref = torch.zeros(rows, heads * head_dim, dtype=torch.float64, device=q.device)
    err = torch.zeros_like(ref)
    cu_k = cu_k.tolist()
    cu_q = cu_q.tolist() if cu_q is not None else None
    for b in range(batch):
        k0, k1 = cu_k[b], cu_k[b + 1]
        q0, q1 = (cu_q[b], cu_q[b + 1]) if cu_q is not None else (0, max_q)
        o0 = q0 if cu_q is not None else b * max_q
        if k1 <= k0 or q1 <= q0:
            continue
        for h in range(heads):
            qh = q[q0:q1, q_col0 + h * head_stride:q_col0 + h * head_stride + head_dim]
            kh = k[k0:k1, k_col0 + h * head_stride:k_col0 + h * head_stride + head_dim]
            vh = v[k0:k1, v_col0 + h * head_stride:v_col0 + h * head_stride + head_dim]
            r, e = attention_head_ref_f16(qh, kh, vh, scale, causal, head_stride)
            ref[o0:o0 + (q1 - q0), h * head_dim:(h + 1) * head_dim] = r
            err[o0:o0 + (q1 - q0), h * head_dim:(h + 1) * head_dim] = e
    return ref, err


def f16_cell(got):
    """[lo, hi] of the reals that round to each fp16 value `got` (round to nearest): spacing 2^(e - 10) for a normal value
    of exponent e, halved below a power of two above 2^-14; 2^-24 for the subnormals (and across 2^-14); zero's cell is
    [-2^-25, 2^-25]. float64 in, float64 out."""
    g = got.double()
    a = g.abs()
    ex = torch.clamp(torch.frexp(a).exponent - 1, min=-14).double()
    ulp = torch.exp2(ex - 10)
    pow2 = (a == torch.exp2(ex)) & (a > 2.0 ** -14)
    down = torch.where(pow2, ulp / 2, ulp) / 2
    up = ulp / 2
    tiny = torch.full_like(a, 2.0 ** -25)
    down = torch.where(a > 0, down, tiny)
    up = torch.where(a > 0, up, tiny)
    lo = torch.where(g >= 0, g - down, g - up)
    hi = torch.where(g >= 0, g + up, g + down)
    return lo, hi


def check(name, got, ref, bound, *, cr_min=None, rms_rel=None, verbose=True):
    """kernel_bounds.check extended to fp16 outputs: an fp16 `got` must be fp16_rn(y) for some |y - ref| <= bound (the
    bf16 rule with fp16's cells); cr is then the fraction equal to fp16_rn(ref). Any other dtype goes to
    kernel_bounds.check unchanged. Returns the same dict (frac, rms_rel, cr)."""
    if got.dtype != torch.float16:
        return KB.check(name, got, ref, bound, cr_min=cr_min, rms_rel=rms_rel, verbose=verbose)
    ref = ref.double()
    bound = bound.double().expand_as(ref)
    if not torch.isfinite(got.float()).all():
        raise AssertionError(f"{name}: non-finite output")
    lo, hi = f16_cell(got)
    need = torch.clamp(torch.maximum(lo - ref, ref - hi), min=0.0)   # distance from ref to got's rounding cell
    frac_all = need / bound.clamp_min(1e-300)
    frac_all = torch.where(need == 0, torch.zeros_like(frac_all), frac_all)
    worst = int(torch.argmax(frac_all))
    frac = float(frac_all.reshape(-1)[worst])
    err = got.double() - ref
    out = {"frac": frac,
           "rms_rel": float(err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-300)),
           "cr": float((got == ref.half()).double().mean())}
    idx = np.unravel_index(worst, tuple(ref.shape))
    msg = (f"{name}: worst at {tuple(int(i) for i in idx)}: got {float(got.reshape(-1)[worst]):.8g} ref "
           f"{float(ref.reshape(-1)[worst]):.8g} bound {float(bound.reshape(-1)[worst]):.3g} -> {frac:.3g} of the bound; "
           f"rms_rel {out['rms_rel']:.3g}, correctly rounded {out['cr']:.4f}")
    if verbose:
        print(msg, flush=True)
    assert frac <= 1.0, msg
    if cr_min is not None:
        assert out["cr"] >= cr_min, f"{msg}: correctly rounded fraction below {cr_min}"
    if rms_rel is not None:
        assert out["rms_rel"] <= rms_rel, f"{msg}: rms error above {rms_rel:.3g} of rms(ref)"
    return out
