"""An IEEE-aware checker for kernel outputs that may hold inf or NaN, next to the finite checkers of tests/kernel_bounds.py
and tests/kernel_bounds_f16.py, whose rounding cells and bounds it reuses.

The rule, per element, with `ref` the float64 reference and `bound` its per-element bound (the same as in those modules):
  * ref NaN:   the output must be NaN;
  * ref +-inf: the output must be the same-signed inf;
  * ref finite: the output must be the rounding of some y with |y - ref| <= bound. For a 16-bit output the rounding cells
    run on past the largest finite value: fp16 +inf is the image of [65520, inf) and 65504 of [65488, 65520) (bf16: +inf
    of [2^128 - 2^119, inf)); the negative side mirrors this. So an output of inf passes exactly when ref + bound reaches
    65520, a finite 65504 only when ref - bound < 65520, and a NaN never. An fp32 output passes when |got - ref| <= bound.

The references are the float64 formulas the reference model uses, evaluated with IEEE semantics: GELU(-inf) =
0.5 (-inf) (1 + erf(-inf)) and SiLU(-inf) = -inf sigmoid(-inf) are NaN, as they are in torch, and every product in a
matrix product is formed, so 0 * inf is NaN whatever the BLAS does with zeros (`ieee_matmul`).
"""
from __future__ import annotations

import numpy as np
import torch

from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF

# the smallest real that rounds to +inf (round to nearest): the largest finite value plus half its spacing
OVERFLOW = {torch.float16: 65504.0 + 16.0, torch.bfloat16: 2.0 ** 128 - 2.0 ** 119}
F16_MAX = 65504.0


def ieee_matmul(x, y):
    """x @ y in float64 where every product x_ik y_kj is formed, so a non-finite entry reaches every output it feeds
    (inf * 0 = NaN, inf + -inf = NaN) independently of how the matmul treats zeros."""
    X, Y = x.double(), y.double()
    out = X @ Y
    # the outputs a non-finite entry feeds: its row of x, or its column of y. Those are summed product by product.
    rows = (~torch.isfinite(X)).any(1).nonzero().flatten()
    cols = (~torch.isfinite(Y)).any(0).nonzero().flatten()
    for r0 in range(0, rows.numel(), 64):
        r = rows[r0:r0 + 64]
        out[r] = (X[r][:, :, None] * Y[None]).sum(1)
    if cols.numel():
        out[:, cols] = (X[:, :, None] * Y[:, cols][None]).sum(1)
    return out


def _abs_mm(x, y):
    return ieee_matmul(x.double().abs(), y.double().abs())


def gemm_linear_ref(a, w, *, bias=None, gelu=False, scale=1.0, rowadd=None, resid=None):
    """kernel_bounds.gemm_linear_ref with the accumulation in ieee_matmul (the same epilogue formula and bound)."""
    x = ieee_matmul(a, w.double().T)
    S = _abs_mm(a, w.double().T)
    e = KB.k_steps(a.shape[1]) * KB.ULP * S
    if bias is not None:
        b = bias.double()
        x = x + b
        e = e + KB.U * (S + b.abs())
    if gelu:
        e = KB.GELU_DERIV * e + KB.GELU_REL * x.abs()
        x = KB.gelu64(x)
    if scale != 1.0:
        x = x * scale
        e = abs(scale) * e + KB.U * x.abs()
    if rowadd is not None:
        idx = torch.arange(x.shape[0], device=x.device) % rowadd.shape[0]
        x = x + rowadd.double()[idx]
        e = e + KB.U * x.abs()
    if resid is not None:
        x = x + resid.double()
        e = e + KB.U * x.abs()
    return x, e + KB.U * x.abs()


def gemm_rope_ref(a, w, positions, cos, sin, rope_cols):
    """kernel_bounds.gemm_rope_ref on finite operands (its accumulation is an ordinary matmul)."""
    return KB.gemm_rope_ref(a, w, positions, cos, sin, rope_cols)


def gemm_swiglu_ref(a, w):
    return KB.gemm_swiglu_ref(a, w)


def attention_head_ref(q, k, v, scale, causal, hs, f16):
    """One head with IEEE semantics: kernel_bounds(_f16).attention_head_ref's formula and bound, where a key whose score
    is -inf has p = 0 and adds nothing to the bound, p = 0 times a non-finite v is NaN, and a +inf or NaN score makes
    the row NaN (torch.softmax). Returns (ref, e) [Lq, hd] float64."""
    Q, K, V = q.double(), k.double(), v.double()
    Lq, Lk = Q.shape[0], K.shape[0]
    s = ieee_matmul(Q, K.T) * scale
    ds = _abs_mm(Q, K.T) * (KB.k_steps(hs) * KB.ULP * scale)
    vis = torch.ones(Lq, Lk, dtype=torch.bool, device=s.device)
    if causal:
        vis = vis.tril(Lk - Lq)
        s = s.masked_fill(~vis, float("-inf"))
    ds = ds.masked_fill(~vis | (s == float("-inf")), 0.0)
    P = torch.softmax(s, -1)
    ref = ieee_matmul(P, V)
    Vf = torch.where(torch.isfinite(V), V, 0.0)     # the bound of a finite output sees finite v only
    c = P.nan_to_num(0.0) @ Vf.abs()
    nkt = -(-Lk // KB.ATT_BN)
    eps_s = 2 * ds.amax(-1, keepdim=True) + KB.EPS_EXP
    p_rel = KF.F16_P if f16 else KB.BF16_P
    e = (p_rel + eps_s + (KB.k_steps(Lk) + nkt) * KB.ULP) * c + (eps_s + (36 + 2 * nkt) * KB.U) * ref.abs().nan_to_num(0.0)
    if f16:
        e = e + KF.F16_P_ABS * (vis.double() @ Vf.abs())
    return ref, e


def norm_ref(x, gamma, beta, eps, rms, add=None):
    """kernel_bounds.layernorm_ref / rmsnorm_ref, whose row formulas carry NaN and inf per IEEE already. With `add`,
    returns the second output (LN(x) + add[row % P]) only. A row with a non-finite input gets the bound 0: a LayerNorm
    row is then NaN throughout (its mean is not finite), and an RMSNorm row with an inf has rsqrt(inf) = 0, so its
    finite inputs give exact zeros (the inf gives NaN)."""
    if rms:
        y, e = KB.rmsnorm_ref(x, gamma, eps)
    elif add is None:
        y, e = KB.layernorm_ref(x, gamma, beta, eps)
    else:
        y, e = KB.layernorm_ref(x, gamma, beta, eps, add=add)[1]
    return y, torch.where(torch.isfinite(x).all(1, keepdim=True), e, torch.zeros_like(e))


def _cells(got):
    """[lo, hi] of the reals that round to each value of `got`, with the overflow cells of a 16-bit type: +inf is
    [OVERFLOW, inf], -inf is [-inf, -OVERFLOW]. NaN outputs get an empty cell (lo = inf, hi = -inf)."""
    g = got.double()
    if got.dtype in OVERFLOW:
        fin = torch.isfinite(g)
        lo, hi = (KF.f16_cell if got.dtype == torch.float16 else KB.bf16_cell)(torch.where(fin, got, torch.zeros_like(got)))
        top = OVERFLOW[got.dtype]
        inf = torch.full_like(g, float("inf"))
        lo = torch.where(fin, lo, torch.where(g == inf, torch.full_like(g, top), -inf))
        hi = torch.where(fin, hi, torch.where(g == -inf, torch.full_like(g, -top), inf))
        # the top finite cells end at the overflow threshold (f16_cell already gives 65504 the cell [65488, 65520])
        hi = torch.where(fin, torch.clamp(hi, max=top), hi)
        lo = torch.where(fin, torch.clamp(lo, min=-top), lo)
    else:
        lo, hi = g, g
    nan = torch.isnan(g)
    return torch.where(nan, float("inf"), lo), torch.where(nan, float("-inf"), hi)


def check(name, got, ref, bound, *, verbose=True):
    """Assert the rule of the module doc, per element. Returns a dict: frac (the worst finite-reference element's
    required error as a fraction of its bound), and the counts of NaN / inf references."""
    ref = ref.double()
    bound = bound.double().expand_as(ref)
    g = got.double()
    nan_ref, inf_ref = torch.isnan(ref), torch.isinf(ref)
    fin_ref = ~(nan_ref | inf_ref)
    bad = (nan_ref & ~torch.isnan(g)) | (inf_ref & (g != ref))
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        idx = tuple(int(t) for t in np.unravel_index(i, tuple(ref.shape)))
        raise AssertionError(f"{name}: at {idx}: got {float(g.reshape(-1)[i])} where the reference is "
                             f"{float(ref.reshape(-1)[i])} ({int(bad.sum())} such elements)")
    if not torch.isfinite(bound[fin_ref]).all():
        raise AssertionError(f"{name}: the bound of a finite reference is not finite")
    lo, hi = _cells(got)
    need = torch.clamp(torch.maximum(lo - ref, ref - hi), min=0.0)
    need = torch.where(fin_ref, need, torch.zeros_like(need))
    frac_all = torch.where(need == 0, torch.zeros_like(need), need / bound.clamp_min(1e-300))
    worst = int(torch.argmax(frac_all))
    frac = float(frac_all.reshape(-1)[worst])
    idx = tuple(int(t) for t in np.unravel_index(worst, tuple(ref.shape)))
    msg = (f"{name}: worst at {idx}: got {float(g.reshape(-1)[worst]):.8g} ref {float(ref.reshape(-1)[worst]):.8g} "
           f"bound {float(bound.reshape(-1)[worst]):.3g} -> {frac:.3g} of the bound; "
           f"{int(nan_ref.sum())} NaN and {int(inf_ref.sum())} inf references")
    if verbose:
        print(msg, flush=True)
    assert frac <= 1.0, msg
    return {"frac": frac, "nan": int(nan_ref.sum()), "inf": int(inf_ref.sum())}
