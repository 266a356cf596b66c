"""fp64 references, per-element error bounds and one checker for the GEMM, attention and norm kernels.

Every reference is computed in float64 from the exact bf16 / fp32 tensors the kernel received, on whatever device they
live on (the GPU tests keep everything on the device, the host tests run the same functions on the CPU). Next to each
reference sits a per-element bound `e`, derived below from the kernel's arithmetic, never from observed output:

    |y - ref| <= e      y = the kernel's value before its final rounding to the output type

For an fp32 output the final rounding is part of `e`. For a bf16 output `check` asks for the bf16 value the kernel
stored to be the round-to-nearest image of SOME y with |y - ref| <= e: wherever the interval [ref - e, ref + e] holds
no rounding midpoint, the output must equal bf16_rn(ref) exactly. Rounding is monotone, so this is exact, and it is far
sharper than adding half a bf16 ulp to `e` when `e` is small against the bf16 spacing (GEMMs, norms).

Notation: U = 2^-24 is the unit roundoff of fp32 round-to-nearest; one fp32 ulp relative to a value is at most 2^-23
(the error of a truncating, round-toward-zero operation).
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24          # fp32 round-to-nearest: |fl(x) - x| <= U |x|
ULP = 2.0 ** -23        # fp32 round-toward-zero: |fl(x) - x| <= ULP |x|

# ----------------------------------------------------------------------------------------------------------------------
# GEMM accumulation model.  ASSUMPTION, not a measured property of the H100: a bf16 x bf16 product is exact in fp32
# (8 + 8 significant bits), and each wgmma k16 step adds its 16 products to the fp32 accumulator with one error of at most
# one fp32 ulp of the magnitudes involved, whether the tensor core rounds or truncates:
#     |step error| <= 2^-23 (|acc| + sum_16 |a_k w_k|) <= 2^-23 S,     S = sum_k |a_ik| |w_jk|
# Summed over ceil(K/16) steps (a partly filled last step is zero-padded):  e_acc = ceil(K/16) 2^-23 S.
# The epilogue's fp32 operations (bias add, scale, row add, residual add, store) each add one rounding, U |intermediate|.
# ----------------------------------------------------------------------------------------------------------------------


def k_steps(K: int) -> int:
    return -(-K // 16)


# The rms of the accumulation error, for zero-mean independent operands (what the tests feed; only used without GELU,
# which changes rms(ref)). Over a matrix, the error of step t has rms <= 2^-23 (rms(acc_t) + rms(sum_16 |a w|)), with
# rms(acc_t) = sqrt(t/T) rms(a w^T) (T = ceil(K/16) steps) and sum_16 |a w| <= 16 rms(a w) = (4 / sqrt(T)) rms(a w^T).
# By the triangle inequality in L2, summed over the steps:
#     rms(err) <= 2^-23 (sum_t sqrt(t/T) + 4 sqrt(T)) rms(a w^T) <= 2^-23 (2T/3 + 1 + 4 sqrt(T)) rms(a w^T).
# The bound below takes T for 2T/3 + 1 and adds 4 for the epilogue's roundings and sampling noise in rms(acc_t).
def gemm_rms_rel(K: int) -> float:
    T = k_steps(K)
    return (T + 4 * math.sqrt(T) + 4) * ULP


# ----------------------------------------------------------------------------------------------------------------------
# GELU. gemm.cuh evaluates erf(z), z = clamp(x / sqrt2, +-3.2), as z P(u) with a degree-10 polynomial in fp32 FMAs, and
# GELU(x) = 0.5 x (1 + erf(z)). Its error is  0.5 |x| |erf(z_true) - erf_poly(z)| + the fp32 roundings (z, erf, the last
# FMA: 3 U |x| at most). In range the fit's erf error is <= 3.2e-6 (gemm.cuh); past the clamp erf_poly(3.2) stands in
# for erf(z) -> 1, off by at most 1 - erf_poly(3.2) = 2.9e-6 (fp32 emulation below). So
#     |GELU error| <= 0.5 ERF_ERR |x| + 3 U |x|,   ERF_ERR = max(in-range fit error, 1 - erf_poly(3.2))
# which grows with |x| (1.6e-6 |x|): an absolute bound such as 1.2e-5 holds only for |x| below about 7.
# test_kernel_bounds_host.py checks the whole GELU term against the emulation on a dense grid out to |x| = 120.
# ----------------------------------------------------------------------------------------------------------------------
GELU_ZMAX = 3.2
GELU_COEF = (2.982273671e-03, -7.046153472e-03, 7.957076705e-03, -1.521942819e-02, 3.318292224e-02, -5.471928813e-02,
             8.062700147e-02, -1.136467381e-01, 1.543549678e-01, -2.173077339e-01, 4.413341836e-01)


def _fma32(a, b, c):
    """fp32 fused multiply-add: a*b is exact in fp64 (24 + 24 bits); the sum rounds once in fp64 and once to fp32 (the
    double rounding can differ from a true fp32 FMA only on exact fp32 ties, which these magnitudes do not reach)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def erf_poly_f32(z):
    """erf of gemm.cuh's gelu_erf2, op by op in fp32 (z already clamped)."""
    z = np.asarray(z, np.float32)
    A = np.float32(2.0 / (GELU_ZMAX * GELU_ZMAX))
    w = _fma32(z, z, 0.0)
    u = _fma32(w, A, -1.0)
    p = _fma32(u, GELU_COEF[0], GELU_COEF[1])
    for c in GELU_COEF[2:]:
        p = _fma32(p, u, c)
    return _fma32(p, z, 0.0)


def gelu_poly_f32(x):
    """gemm.cuh's gelu_erf2, op by op in fp32."""
    x = np.asarray(x, np.float32)
    zmax = np.float32(GELU_ZMAX)
    z = np.minimum(np.maximum((x * np.float32(0.70710678118654752)).astype(np.float32), -zmax), zmax)
    r = erf_poly_f32(z)
    h = (np.float32(0.5) * x).astype(np.float32)
    return _fma32(h, r, h)


ERF_TAIL = float(1.0 - erf_poly_f32(np.float32(GELU_ZMAX)))   # 2.9e-6: erf past the clamp
ERF_FIT = 3.2e-6            # the fit's in-range erf error stated in gemm.cuh (checked in test_kernel_bounds_host.py)
ERF_ERR = max(ERF_FIT, ERF_TAIL)
GELU_REL = 0.5 * ERF_ERR + 3 * U
GELU_DERIV = 1.13           # max |d/dx x Phi(x)| = Phi(sqrt2) + sqrt2 phi(sqrt2) = 1.1289: input errors pass through GELU


def gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x * (0.5 ** 0.5)))


def silu64(x):
    return x * torch.sigmoid(x)


# SiLU in gemm.cuh: g * rcp.approx(1 + ex2.approx(-g log2e)). PTX documents ex2.approx.ftz.f32 and rcp.approx.f32 with
# a maximum relative error of 2^-22 each (taken at that, the looser of the two); the argument's rounding U |g log2 e|
# becomes a relative error U |g| of the exponential; 1 + e, the product g r and the product with `up` round once each.
SILU_REL_CONST = 2.0 * 2.0 ** -22 + 3 * U
SILU_DERIV = 1.1            # max |silu'(x)| = 1.0998


# ----------------------------------------------------------------------------------------------------------------------
# GEMM references
# ----------------------------------------------------------------------------------------------------------------------


def _acc64(a, w):
    A, W = a.double(), w.double()
    return A @ W.T, A.abs() @ W.abs().T


def gemm_linear_ref(a, w, *, bias=None, gelu=False, scale=1.0, rowadd=None, resid=None):
    """LINEAR epilogue, in the kernel's order: [resid +] scale * gelu?(a w^T + bias) [+ rowadd[row % P]].
    Returns (ref, e) in float64; e is the bound before any bf16 rounding of the output (fp32 store included)."""
    x, S = _acc64(a, w)
    e = k_steps(a.shape[1]) * ULP * S
    if bias is not None:
        b = bias.double()
        x = x + b
        e = e + U * (S + b.abs())
    if gelu:
        e = GELU_DERIV * e + GELU_REL * x.abs()
        x = gelu64(x)
    if scale != 1.0:
        x = x * scale
        e = abs(scale) * e + U * x.abs()
    if rowadd is not None:
        idx = torch.arange(x.shape[0], device=x.device) % rowadd.shape[0]
        x = x + rowadd.double()[idx]
        e = e + U * x.abs()
    if resid is not None:
        x = x + resid.double()
        e = e + U * x.abs()
    return x, e + U * x.abs()       # + the fp32 rounding of the last operation (or of the store)


def gemm_rope_ref(a, w, positions, cos, sin, rope_cols):
    """ROPE epilogue: 64-column heads [lo 32 | hi 32]; heads below rope_cols rotate by (cos, sin)[pos], the rest (v)
    pass through. lo' = lo c - hi s, hi' = hi c + lo s: two products and a sum, 3 U of the magnitudes at most."""
    x, S = _acc64(a, w)
    e = k_steps(a.shape[1]) * ULP * S + U * x.abs()
    M, N = x.shape
    c = cos.double()[positions.long()]          # [M, 32]
    s = sin.double()[positions.long()]
    xr, er = x.view(M, N // 64, 2, 32), e.view(M, N // 64, 2, 32)
    lo, hi, elo, ehi = xr[:, :, 0], xr[:, :, 1], er[:, :, 0], er[:, :, 1]
    C, Sn = c[:, None, :], s[:, None, :]
    rot = torch.stack([lo * C - hi * Sn, hi * C + lo * Sn], 2)
    mag = torch.stack([(lo * C).abs() + (hi * Sn).abs(), (hi * C).abs() + (lo * Sn).abs()], 2)
    erot = torch.stack([elo * C.abs() + ehi * Sn.abs(), ehi * C.abs() + elo * Sn.abs()], 2) + 3 * U * mag
    heads = torch.arange(N // 64, device=x.device)[None, :, None, None] * 64 < rope_cols
    ref = torch.where(heads, rot, xr).reshape(M, N)
    return ref, torch.where(heads, erot, er).reshape(M, N)


def swiglu_ref(gate, up, eg, eu):
    """silu(gate) * up from fp64 accumulators and their bounds."""
    sg = silu64(gate)
    ref = sg * up
    e = up.abs() * (SILU_DERIV * eg + (SILU_REL_CONST + U * gate.abs()) * sg.abs()) + sg.abs() * eu + U * ref.abs()
    return ref, e


def gemm_swiglu_ref(a, w):
    """SWIGLU epilogue: w holds interleaved 32-row [gate | up] blocks; output column j of block b = silu(g) * u."""
    x, S = _acc64(a, w)
    e = k_steps(a.shape[1]) * ULP * S + U * x.abs()
    M, N = x.shape
    xr, er = x.view(M, N // 64, 2, 32), e.view(M, N // 64, 2, 32)
    ref, eb = swiglu_ref(xr[:, :, 0], xr[:, :, 1], er[:, :, 0], er[:, :, 1])
    return ref.reshape(M, N // 2), eb.reshape(M, N // 2)


# ----------------------------------------------------------------------------------------------------------------------
# Attention.  out_i = sum_j bf16(p_ij) v_j / l_i with p_ij = exp2((s_ij - m_i) scale log2e) in fp32, l_i = sum_j p_ij from the
# fp32 p (attention.cuh). Error terms, with c_id = sum_j P_ij |v_jd| (P = the exact softmax):
#   * P rounded to bf16 for the PV MMA: |bf16(p) - p| <= 2^-8 p, so <= 2^-8 c_id.
#   * scores: s_ij accumulates ceil(HS/16) k16 steps (model above): |ds| <= ceil(HS/16) 2^-23 sum_d |q_d||k_jd|; the
#     softmax ratio p_ij / l_i moves by at most exp(2 scale max_j|ds|) - 1 ~ 2 scale max_j |ds| relative;
#     ex2.approx (2^-22 relative, PTX) in p and in alpha, and the argument's rounding (U |arg| relative, and
#     |arg| 2^-arg <= 0.54): EPS_EXP = 2 (2^-22 + U).  Both scale c_id and |out|.
#   * PV: one k16 step per 16 keys plus the alpha rescale per key tile: (ceil(N/16) + nkt) 2^-23 c_id.
#   * l: each thread sums its 32 p of a tile serially, then l = l alpha + lt per tile, then two shuffles:
#     (32 + 2 nkt + 2) U relative; 1/l and the product O/l round once each: 2 U |out|.
# ----------------------------------------------------------------------------------------------------------------------
EPS_EXP = 2 * (2.0 ** -22 + U)
BF16_P = 2.0 ** -8
ATT_BN = 128


def attention_head_ref(q, k, v, scale, causal, hs):
    """One head: q [Lq, hd], k / v [Lk, hd] (any dtype) -> (ref, e) [Lq, hd] float64. Causal: query i sees keys
    <= i + (Lk - Lq)."""
    Q, K, V = q.double(), k.double(), v.double()
    Lq, Lk = Q.shape[0], K.shape[0]
    s = (Q @ K.T) * scale
    ds = (Q.abs() @ K.abs().T) * (k_steps(hs) * ULP * scale)
    if causal:
        mask = torch.ones(Lq, Lk, dtype=torch.bool, device=s.device).tril(Lk - Lq)
        s = s.masked_fill(~mask, float("-inf"))
        ds = ds.masked_fill(~mask, 0.0)
    P = torch.softmax(s, -1)
    ref = P @ V
    c = P @ V.abs()
    nkt = -(-Lk // ATT_BN)
    eps_s = 2 * ds.amax(-1, keepdim=True) + EPS_EXP
    e = (BF16_P + eps_s + (k_steps(Lk) + nkt) * ULP) * c + (eps_s + (36 + 2 * nkt) * U) * ref.abs()
    return ref, e


def attention_ref(q, k, v, *, q_col0, k_col0, v_col0, head_stride, head_dim, heads, cu_k, cu_q, max_q, causal, scale):
    """The full var-len / cross-attention call of ops.attention, sequence by sequence and head by head (no score
    matrix larger than one sequence x one head). Returns (ref, e) with the kernel's output layout."""
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
            r, e = attention_head_ref(qh, kh, vh, scale, causal, head_stride)
            ref[o0:o0 + (q1 - q0), h * head_dim:(h + 1) * head_dim] = r
            err[o0:o0 + (q1 - q0), h * head_dim:(h + 1) * head_dim] = e
    return ref, err


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm / RMSNorm (elementwise.cu: one warp per row, two passes). The sums run per lane over D/128 float4 (each
# summed as (x+y)+(z+w)), then over the 32 lanes by a 5-level shuffle tree: depth D/128 + 7, so a sum of D terms is off
# by at most (D/128 + 7) U sum|terms|; the division by D adds U.
#   mean:      dm <= G U mean|x|,   G = D/128 + 8
#   variance:  v^ = mean((x - m^)^2) = var + dm^2 (sum(x - m) = 0) plus (G + 3) U v^ from the subtraction, the square
#              and the sum:  dv <= dm^2 + (G + 3) U (var + dm^2)
#   rstd:      rsqrtf (2^-22 relative, PTX rsqrt.approx) of v^ + eps (one more U): dr/r <= dv / (2 (var + eps)) + 2^-22 + U
#   output:    (x - m^) r g [+ b]: |g| r (|x - m| dr/r + dm + U |x - m|) + 3 U (|(x - m) r g| + |b|)
# ----------------------------------------------------------------------------------------------------------------------


def norm_ref(x, gamma, beta, eps, rms):
    X = x.double()
    D = X.shape[1]
    G = D / 128 + 8
    m = torch.zeros_like(X[:, :1]) if rms else X.mean(-1, keepdim=True)
    dm = torch.zeros_like(m) if rms else G * U * X.abs().mean(-1, keepdim=True)
    var = ((X - m) ** 2).mean(-1, keepdim=True)
    dv = dm ** 2 + (G + 3) * U * (var + dm ** 2)
    r = torch.rsqrt(var + eps)
    dr = dv / (2 * (var + eps)) + 2.0 ** -22 + U
    g = gamma.double()
    y = (X - m) * r * g
    mag = y.abs()
    e = g.abs() * r * ((X - m).abs() * dr + dm + U * (X - m).abs())
    if beta is not None:
        y = y + beta.double()
        mag = mag + beta.double().abs()
    return y, e + 3 * U * mag


def layernorm_ref(x, gamma, beta, eps, add=None):
    """(LN(x), e) and, with `add` [P, D], (LN(x) + add[row % P], e + U |.|): the kernel adds in fp32 before rounding."""
    y, e = norm_ref(x, gamma, beta, eps, rms=False)
    if add is None:
        return y, e
    idx = torch.arange(x.shape[0], device=x.device) % add.shape[0]
    y2 = y + add.double()[idx]
    return (y, e), (y2, e + U * y2.abs())


def rmsnorm_ref(x, gamma, eps):
    return norm_ref(x, gamma, None, eps, rms=True)


def build_lm_input_ref(src, embed, scale_emb, vision):
    """src >= 0: vision row src (copied); src < 0: embed row -(src+1) (bf16, exact in fp32) * scale_emb (one rounding)."""
    s = src.long()
    out = torch.empty(s.numel(), embed.shape[1], dtype=torch.float64, device=embed.device)
    txt = s < 0
    out[txt] = embed.double()[-(s[txt] + 1)] * float(np.float32(scale_emb))
    if vision is not None:
        out[~txt] = vision.double()[s[~txt]]
    return out, U * out.abs()


# ----------------------------------------------------------------------------------------------------------------------
# Final RMSNorm + pooling + L2 normalise (elementwise.cu pool_norm_kernel), per sequence over its weighted rows t:
#   ss_t:   sum of squares as in the norms: a lane sums ceil(D/128) float4 groups (x^2 + y^2) + (z^2 + w^2) serially, then
#           the 5-level shuffle tree: depth ceil(D/128) + 8 with the products, so ss^ = ss (1 + d), |d| <= G U.
#   r_t:    rsqrtf(ss / D + eps): the division and the add round once each, rsqrt.approx adds 2^-22 (PTX). With
#           rho = (ss/D) / (ss/D + eps) only the ss part of the argument carries d:
#           dr/r <= rho (G + 1) U / 2 + U / 2 + 2^-22  (half the argument's relative error, plus rsqrt's own).
#   sc_t:   w_t r_t, w_t = t + 1 (wmean) or 1, an integer exact in fp32: one more U.
#   A:      sum_t sc_t x_t. A warp adds its rows serially (one product and one add per row, or one FMA), ceil(n/32) rows
#           at most; then 3 adds over the CTA's 4 warps and 8 over the virtual ranks (0 + the first is exact):
#           |dA_c| <= sum_t |sc_t x_tc| (dsc_t + U) + (ceil(n/32) + 11) U sum_t |sc_t x_tc|,  dsc_t = dr_t/r_t + U.
#   p:      A_c gamma_c / W: a product and an IEEE division (2 U |p|). W = sum w_t is exact in fp32 for n <= 5792
#           (n (n + 1) < 2^25 and even).
#   norm:   sq = sum_c p_c^2 per thread over ceil(D/512) float4 groups, the shuffle tree and 4 warps serially: depth
#           ceil(D/512) + 11 (G2 U relative), plus 2 sum_c |p_c| |dp_c| from p's error; sqrtf and 1 / max(., 1e-12) are
#           IEEE (U each), so 1/N^ is off by sum|p||dp| / N^2 + (G2 / 2 + 2) U relative; the product p / N rounds once more.
#           y = p / N moves by |dp_c| / N + |y_c| (relative error of 1/N). Second-order terms are covered by 1e-3 of slack.
#   An empty sequence is written as zeros, and an all-zero one pools to p = 0 and y = 0 (the max(N, 1e-12) guard).
# ----------------------------------------------------------------------------------------------------------------------
POOL_VRANKS = 8


def pool_norm_ref(h, gamma, eps, cu, pooling, normalize):
    """ops.pool_norm in float64: h [T, D] fp32 (any row pitch), gamma [D], cu [B + 1]. Returns (ref, e) [B, D]."""
    D = gamma.numel()
    g = gamma.double()
    eps32 = float(np.float32(eps))
    G = -(-D // 128) + 8
    G2 = -(-D // 512) + 11
    cu = [int(c) for c in cu.tolist()]
    B = len(cu) - 1
    ref = torch.zeros(B, D, dtype=torch.float64, device=h.device)
    err = torch.zeros_like(ref)
    for b in range(B):
        n = cu[b + 1] - cu[b]
        if n <= 0:
            continue
        t_lo, t_hi = {"lasttoken": (n - 1, n), "cls": (0, 1)}.get(pooling, (0, n))
        X = h[cu[b] + t_lo:cu[b] + t_hi, :D].double()
        m = t_hi - t_lo
        w = torch.arange(t_lo + 1, t_hi + 1, dtype=torch.float64, device=h.device) if pooling == "wmean" else \
            torch.ones(m, dtype=torch.float64, device=h.device)
        ms = (X * X).sum(1) / D
        r = torch.rsqrt(ms + eps32)
        rho = ms / (ms + eps32)
        dsc = rho * (G + 1) * U / 2 + U / 2 + 2.0 ** -22 + U          # + U: the product w r
        Y = (w * r)[:, None] * X
        aY = Y.abs()
        eA = (aY * (dsc + U)[:, None]).sum(0) + (-(-m // 32) + 11) * U * aY.sum(0)
        W = float(w.sum())
        p = Y.sum(0) * g / W
        ep = g.abs() * eA / W + 2 * U * p.abs()
        if not normalize:
            ref[b], err[b] = p, ep * (1 + 1e-3)
            continue
        N = float(p.norm())
        if N == 0.0:
            continue
        y = p / max(N, 1e-12)
        dinv = float((p.abs() * ep).sum()) / N ** 2 + (G2 / 2 + 2) * U
        ref[b] = y
        err[b] = (ep / N + y.abs() * (dinv + U)) * (1 + 1e-3)
    return ref, err


# ----------------------------------------------------------------------------------------------------------------------
# The checker
# ----------------------------------------------------------------------------------------------------------------------


def bf16_cell(got):
    """[lo, hi] of the reals that round to each bf16 value `got` (round to nearest; the spacing halves below a power of
    two). float64 in, float64 out."""
    g = got.double()
    a = g.abs()
    ex = (torch.frexp(a).exponent - 1).double()     # floor(log2 a), exactly (a log2 on the device may miss it)
    ulp = torch.exp2(ex - 7)
    pow2 = (a == torch.exp2(ex)) & (a > 0)
    down = torch.where(pow2, ulp / 2, ulp) / 2          # toward zero
    up = ulp / 2                                          # away from zero
    tiny = torch.full_like(a, 2.0 ** -134)
    down = torch.where(a > 0, down, tiny)
    up = torch.where(a > 0, up, tiny)
    lo = torch.where(g >= 0, g - down, g - up)
    hi = torch.where(g >= 0, g + up, g + down)
    return lo, hi


def check(name, got, ref, bound, *, cr_min=None, rms_rel=None, verbose=True):
    """Assert that the kernel output `got` is within `bound` of the float64 `ref`, per element.

    fp32 `got`: |got - ref| <= bound. bf16 `got`: got = bf16_rn(y) for some |y - ref| <= bound (see the module doc).
    cr_min: the fraction of bf16 outputs equal to bf16_rn(ref) must be at least this.
    rms_rel: rms(got - ref) / rms(ref) must be at most this.
    Returns a dict: frac (the worst element's required error as a fraction of its bound: pass <= 1), cr, rms_rel."""
    ref = ref.double()
    bound = bound.double().expand_as(ref)
    if not torch.isfinite(got.float()).all():
        raise AssertionError(f"{name}: non-finite output")
    if got.dtype == torch.bfloat16:
        lo, hi = bf16_cell(got)
        need = torch.clamp(torch.maximum(lo - ref, ref - hi), min=0.0)   # distance from ref to got's rounding cell
    else:
        need = (got.double() - ref).abs()
    frac_all = need / bound.clamp_min(1e-300)
    frac_all = torch.where(need == 0, torch.zeros_like(frac_all), frac_all)
    worst = int(torch.argmax(frac_all))
    frac = float(frac_all.reshape(-1)[worst])
    out = {"frac": frac}
    err = got.double() - ref
    out["rms_rel"] = float(err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-300))
    if got.dtype == torch.bfloat16:
        out["cr"] = float((got == ref.float().bfloat16()).double().mean())
    idx = np.unravel_index(worst, tuple(ref.shape))
    msg = (f"{name}: worst at {tuple(int(i) for i in idx)}: got {float(got.reshape(-1)[worst]):.8g} ref "
           f"{float(ref.reshape(-1)[worst]):.8g} bound {float(bound.reshape(-1)[worst]):.3g} -> {frac:.3g} of the bound; "
           f"rms_rel {out['rms_rel']:.3g}" + (f", correctly rounded {out['cr']:.4f}" if "cr" in out else ""))
    if verbose:
        print(msg, flush=True)
    assert frac <= 1.0, msg
    if cr_min is not None:
        assert out["cr"] >= cr_min, f"{msg}: correctly rounded fraction below {cr_min}"
    if rms_rel is not None:
        assert out["rms_rel"] <= rms_rel, f"{msg}: rms error above {rms_rel:.3g} of rms(ref)"
    return out
