"""float64 references of the operations the encode path's kernel launches stand for, built from the checkpoint (the state
dict in its original layout), the reference model's formulas and constants and `oracle/restated.py`, never from the
arguments the engine passes. Each check takes the launch's actual 16-bit or fp32 input (teacher forcing: no error
carries over from earlier launches) and applies the per-element bounds of tests/kernel_bounds.py, so a wiring mistake
(a table, a layout, a constant, a position) fails at the launch where it happens instead of hiding in 26 + 40 layers of
accumulated rounding. tests/test_gpu_launch_parity.py runs them on every launch of real encodes;
tests/test_launch_parity_host.py shows on the CPU that they accept faithful outputs and reject plausible mistakes.

Every check returns kernel_bounds.check's dict (frac = worst element's error as a fraction of its bound) and raises
AssertionError on a violation. Weights are the state-dict tensors rounded to the engine's 16-bit type; for fp16 that
rounding is the dtype choice, not wiring.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import restated as O
from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF

U = KB.U
# Tables computed in fp32 (the engine's and the reference model's): the ViT position table by a two-pass separable
# bicubic filter of up to ~20 taps per pass with |weights| summing to < 1.3, so it is off the float64 table by at most
# (2 x 20 + slack) U max|pos_embed|; RoPE cos / sin round once each (a few U).
POS_TABLE_U = 64
ROPE_TABLE_U = 4


def check(name, got, ref, e, verbose=False):
    return KF.check(name, got, ref, e, verbose=verbose)


def assert_pos_zero(name, t):
    """Pad columns must be +0 bit for bit (the next GEMM reads them)."""
    bits = t.contiguous().view(torch.int16)
    if not (bits == 0).all():
        raise AssertionError(f"{name}: {int((bits != 0).sum())} pad values are not +0")


def w16(t, dtype):
    """A state-dict weight rounded to the engine's 16-bit type."""
    return t.to(dtype)


# ---------------------------------------------------------------------------------------------------------- tables


def vit_pos_table64(pos_embed, gh, gw):
    """timm's resample_abs_pos_embed (`pos_embed.py:17-57`, no prefix tokens) in float64: bicubic with antialias from the
    native square grid to (gh, gw); the identity at the native grid. pos_embed [1, S*S, D] -> [gh*gw, D] (on its device)."""
    S = math.isqrt(pos_embed.shape[1])
    D = pos_embed.shape[-1]
    p = pos_embed.detach().double().cpu().reshape(1, S, S, D)
    if (gh, gw) != (S, S):
        p = F.interpolate(p.permute(0, 3, 1, 2), size=(gh, gw), mode="bicubic", antialias=True).permute(0, 2, 3, 1)
    return p.reshape(gh * gw, D).to(pos_embed.device)


def sincos64(E, gh, gw, device):
    """The resampler's 2-D sincos table as `oracle/restated.py` restates it (`resampler.py:38-90`), in float64."""
    return torch.from_numpy(O.sincos_2d(E, gh, gw)).to(device=device, dtype=torch.float64)


def rope_tables(head_dim, theta, n, device):
    """`MiniCPMRotaryEmbedding` (`modeling_minicpm.py:142-182`) as the reference computes it, in fp32: cos / sin of
    positions 0..n-1, the first head_dim / 2 columns (the second half repeats them)."""
    c, s = O.rope_tables(head_dim, theta, n)
    return c[:, :head_dim // 2].contiguous().to(device), s[:, :head_dim // 2].contiguous().to(device)


def normalized_pixels(px_u8, dtype):
    """uint8 [S,h,w,3] -> ToTensor + Normalize(0.5, 0.5) (`modeling_minicpmv.py:84-92`) in fp32, rounded to `dtype`,
    [S,3,h,w]; computed on the CPU in the oracle's order of operations."""
    x = px_u8.cpu().permute(0, 3, 1, 2).float() / 255.0
    return ((x - 0.5) / 0.5).to(dtype).to(px_u8.device)


# ---------------------------------------------------------------------------------------------------------- checks


def check_im2col(name, got, px16, K):
    """got [S*gh*gw, ld] must be F.unfold of the normalised pixels bit for bit, pad columns +0."""
    S, C, h, w = px16.shape
    P = int(round(math.sqrt(K // C)))
    want = F.unfold(px16.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, K).to(px16.dtype)
    same = got[:, :K].view(torch.int16) == want.view(torch.int16)
    if not same.all():
        r, c = (~same).nonzero()[0].tolist()
        raise AssertionError(f"{name}: row {r} col {c}: got {float(got[r, c])} want {float(want[r, c])}")
    assert_pos_zero(name + " pad", got[:, K:])
    return {"frac": 0.0}


def patch_embed_ref(px16, weight, bias, pos_embed, dtype):
    """Patch embedding + position table, [S*gh*gw, D] float64: F.conv2d of the normalised pixels with the conv weight in
    its [D, 3, P, P] layout (stride P) plus the conv bias, plus vit_pos_table64 for this grid. The bound is
    kernel_bounds.gemm_linear_ref's for bias + row add, plus the fp32 table's deviation (POS_TABLE_U)."""
    W = w16(weight, dtype).double()
    X = px16.double()
    P = W.shape[-1]
    D = W.shape[0]
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(-1, D)   # NCHW -> rows in (slice, patch row, patch col) order  # noqa: E731
    x = F.conv2d(X, W, stride=P)
    gh, gw = x.shape[2], x.shape[3]
    x, Sa = flat(x), flat(F.conv2d(X.abs(), W.abs(), stride=P))
    e = KB.k_steps(W[0].numel()) * KB.ULP * Sa
    b = bias.double()
    x = x + b
    e = e + U * (Sa + b.abs())
    pos = vit_pos_table64(pos_embed, gh, gw)
    x = x + pos[torch.arange(x.shape[0], device=x.device) % (gh * gw)]
    e = e + U * x.abs() + POS_TABLE_U * U * float(pos_embed.double().abs().max())
    return x, e + U * x.abs()


def check_patch(name, got, px16, weight, bias, pos_embed):
    return check(name, got, *patch_embed_ref(px16, weight, bias, pos_embed, px16.dtype))


def check_layernorm(name, got, x, gamma, beta, eps, add=None, got_add=None):
    """LN(x) (and LN(x) + add[row % P]) with the checkpoint's gain / bias and the reference's eps."""
    if add is None:
        return check(name, got, *KB.layernorm_ref(x, gamma.float(), beta.float(), eps))
    (y, e), (y2, e2) = KB.layernorm_ref(x, gamma.float(), beta.float(), eps, add=add)
    r = check(name, got, y, e)
    r2 = check(name + " + add", got_add, y2, e2)
    return r if r["frac"] >= r2["frac"] else r2


def check_rmsnorm(name, got, x, gamma, eps):
    return check(name, got, *KB.rmsnorm_ref(x, gamma.float(), eps))


def check_linear(name, got, a, weight, bias=None, *, gelu=False, scale=1.0, resid=None):
    """y = [resid +] scale * gelu?(a weight^T + bias) with the checkpoint's [N, K] weight (N, K = got's / a's widths)."""
    return check(name, got, *KB.gemm_linear_ref(a, w16(weight, a.dtype), bias=None if bias is None else bias.float(),
                                                 gelu=gelu, scale=scale, resid=resid))


def vit_qkv_canonical(got, heads, head_dim):
    """[M, 3 * heads * stride] (per-head padded layout) -> ([M, 3 * heads * head_dim], the pad columns)."""
    g = got.view(got.shape[0], 3, heads, -1)
    return g[..., :head_dim].reshape(got.shape[0], 3 * heads * head_dim), g[..., head_dim:]


def check_vit_qkv(name, got, a, weight, bias, heads, head_dim):
    """The ViT's qkv GEMM in its padded layout against the checkpoint's [3 * heads * head_dim, D] weight; pad columns +0."""
    canon, pad = vit_qkv_canonical(got, heads, head_dim)
    assert_pos_zero(name + " pad", pad)
    return check_linear(name, canon, a, weight, bias)


def check_fc1(name, got, a, weight, bias):
    """GELU(a W1^T + b1) over the checkpoint's width; the padded columns beyond it +0."""
    n = weight.shape[0]
    assert_pos_zero(name + " pad", got[:, n:])
    return check_linear(name, got[:, :n], a, weight, bias, gelu=True)


def check_fc2(name, got, a, weight, bias, resid):
    """resid + (a W2^T + b2) over the checkpoint's width; the operand's padded columns must be +0."""
    n = weight.shape[1]
    assert_pos_zero(name + " operand pad", a[:, n:])
    return check_linear(name, got, a[:, :n].contiguous(), weight, bias, resid=resid)


def check_rope_qkv(name, got, a, wq, wk, wv, positions, cos, sin):
    """q|k|v = a [Wq; Wk; Wv]^T with q and k rotated by (cos, sin)[position] (64-column heads: lo' = lo c - hi s,
    hi' = hi c + lo s, the HF rotate_half form); v passes through. cos / sin are the fp32 tables of rope_tables."""
    W = torch.cat([w16(wq, a.dtype), w16(wk, a.dtype), w16(wv, a.dtype)], 0)
    H = wq.shape[0]
    ref, e = KB.gemm_rope_ref(a, W, positions, cos, sin, 2 * H)
    x = a.double() @ W.double().T
    M, N = x.shape
    xr = x.view(M, N // 64, 2, 32)
    mag = (xr[:, :, 0].abs() + xr[:, :, 1].abs())[:, :, None, :].expand(-1, -1, 2, -1)
    heads = torch.arange(N // 64, device=x.device)[None, :, None, None] * 64 < 2 * H
    e = e + torch.where(heads, ROPE_TABLE_U * U * mag, torch.zeros_like(mag)).reshape(M, N)
    return check(name, got, ref, e)


def check_swiglu(name, got, a, wg, wu):
    """silu(a Wg^T) * (a Wu^T) from the separate gate and up weights."""
    g, Sg = KB._acc64(a, w16(wg, a.dtype))
    u, Su = KB._acc64(a, w16(wu, a.dtype))
    K = a.shape[1]
    ref, e = KB.swiglu_ref(g, u, KB.k_steps(K) * KB.ULP * Sg + U * g.abs(), KB.k_steps(K) * KB.ULP * Su + U * u.abs())
    return check(name, got, ref, e)


def check_attention(name, got, q, k, v, *, heads, head_dim, cu_k, cu_q, max_q, causal, scale):
    """softmax(q k^T scale) v per sequence and head; q / k / v in the canonical [rows, heads * head_dim] layout."""
    ref_fn = KF.attention_ref_f16 if got.dtype == torch.float16 else KB.attention_ref
    ref, e = ref_fn(q, k, v, q_col0=0, k_col0=0, v_col0=0, head_stride=head_dim, head_dim=head_dim, heads=heads,
                    cu_k=cu_k, cu_q=cu_q, max_q=max_q, causal=causal, scale=scale)
    return check(name, got, ref, e)


def lm_input_ref(embed, dtype, scale_emb, ids, bounds, vision_rows):
    """`get_vllm_embedding` (oracle.restated.lm_inputs): per item, embed[ids] * scale_emb with the item's resampler rows
    written over its image_bound spans (span j <- vision_rows[item][j], [64, E]). Items packed in order. float64 + bound
    (the fp32 product rounds once; the copies are exact)."""
    out = []
    for b, (ids_b, bound_b) in enumerate(zip(ids, bounds)):
        rows = embed[torch.as_tensor(np.asarray(ids_b), device=embed.device, dtype=torch.long)]
        x = w16(rows, dtype).double() * float(np.float32(scale_emb))
        for j, (s, t) in enumerate(bound_b):
            x[int(s):int(t)] = vision_rows[b][j][: int(t) - int(s)].double()
        out.append(x)
    ref = torch.cat(out)
    return ref, U * ref.abs()


def check_lm_input(name, got, embed, scale_emb, ids, bounds, vision_rows, dtype):
    return check(name, got, *lm_input_ref(embed, dtype, scale_emb, ids, bounds, vision_rows))


def check_pool(name, got, h, gamma, eps, lengths, pooling, normalize=True):
    """Final RMSNorm + pooling (+ L2 normalisation) over the items' lengths, with the pooling the caller asked for."""
    cu = torch.tensor([0] + list(np.cumsum(lengths)), dtype=torch.int32)
    return check(name, got, *KB.pool_norm_ref(h, gamma.float(), eps, cu, pooling, normalize))
