"""Python launch wrappers over the C ABI. Each function validates shapes/dtypes, allocates the output with
torch (memory plumbing only) and enqueues ONE library call on the current CUDA stream."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib as L

_PROF = None  # list of (kind, start_event, end_event, flops) while profiling is on


def profile_begin() -> None:
    """Start recording one CUDA-event pair around every kernel launch (bench.py's roofline pass)."""
    global _PROF
    _PROF = []


def profiling() -> bool:
    """True while per-launch event profiling is on (the engine then avoids CUDA-graph capture and replay)."""
    return _PROF is not None


def profile_end():
    """Stop recording; returns {kind: (launches, total_ms, total_flops)} (synchronises the device)."""
    global _PROF
    rec, _PROF = _PROF, None
    torch.cuda.synchronize()
    out = {}
    for kind, e0, e1, flops in rec or []:
        n, ms, fl = out.get(kind, (0, 0.0, 0.0))
        out[kind] = (n + 1, ms + e0.elapsed_time(e1), fl + flops)
    return out


def _launch(kind: str, flops: float, fn, *args) -> None:
    if _PROF is None:
        L.check(fn(*args))
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    L.check(fn(*args))
    e1.record()
    _PROF.append((kind, e0, e1, flops))


HALF_DTYPES = (torch.bfloat16, torch.float16)  # the 16-bit types of the kernels' operands and activations
_VR_DTYPE = {torch.bfloat16: L.VR_BF16, torch.float16: L.VR_F16, torch.float32: L.VR_F32}


def _half_operands(**named: torch.Tensor) -> torch.dtype:
    """The named tensors are all bf16 or all fp16 CUDA matrices with unit inner stride; returns their dtype. The dtype
    checks run first, over all of them, before anything looks at a device."""
    dtype = next(iter(named.values())).dtype
    for name, t in named.items():
        if t.dtype not in HALF_DTYPES:
            raise ValueError(f"{name}: expected a bf16 or fp16 matrix, got {t.dtype} {tuple(t.shape)}")
        if t.dtype != dtype:
            raise ValueError(f"{name}: is {t.dtype} but the other operands are {dtype}: bf16 and fp16 operands do not mix")
    for name, t in named.items():
        if t.dim() != 2 or t.stride(1) != 1 or not t.is_cuda:
            raise ValueError(f"{name}: expected a CUDA {t.dtype} matrix with unit inner stride, got {tuple(t.shape)}")
        L.check_device(t)
    return dtype


def _operand(fn: str, name: str, t: torch.Tensor, dtypes, shape, align: int, like: torch.Tensor,
             contiguous: bool = False) -> None:
    """Refuse, naming the argument, a tensor the kernels cannot read as given: a dtype not in `dtypes`, a shape other than
    `shape` (None: any size), a non-unit inner stride (or, with `contiguous`, any gap: the kernels index it with its
    logical width), a base address that is not a multiple of `align` bytes (the widest vector access the kernels make to
    it), or a device other than `like`'s. Every check runs before anything reaches the library."""
    if t.dtype not in dtypes:
        want = " or ".join(str(d).replace("torch.", "") for d in dtypes)
        raise ValueError(f"{fn}: {name} must be {want}, got {t.dtype}")
    if t.dim() != len(shape) or any(n is not None and n != m for n, m in zip(shape, t.shape)):
        want = "[" + ", ".join("*" if n is None else str(n) for n in shape) + "]"
        raise ValueError(f"{fn}: {name} must have shape {want}, got {tuple(t.shape)}")
    if contiguous and not t.is_contiguous() or not contiguous and t.dim() and t.shape[-1] > 1 and t.stride(-1) != 1:
        raise ValueError(f"{fn}: {name} must be {'contiguous' if contiguous else 'unit-stride in its last dimension'}, "
                         f"got strides {t.stride()}")
    if not t.is_cuda:
        raise ValueError(f"{fn}: {name} must be a CUDA tensor, got one on {t.device}")
    if t.device != like.device:
        raise ValueError(f"{fn}: {name} is on {t.device} but the operands are on {like.device}")
    if t.data_ptr() % align:
        raise ValueError(f"{fn}: {name} must be {align}-byte aligned (its storage offset is {t.storage_offset()} elements)")


_F32, _I32 = (torch.float32,), (torch.int32,)


def _half_dtype(dtype: torch.dtype, name: str) -> int:
    if dtype not in HALF_DTYPES:
        raise ValueError(f"{name}: the 16-bit output type must be bf16 or fp16, got {dtype}")
    return _VR_DTYPE[dtype]


def gemm(
    a: torch.Tensor,
    w: torch.Tensor,
    *,
    bias: Optional[torch.Tensor] = None,
    gelu: bool = False,
    scale: float = 1.0,
    resid: Optional[torch.Tensor] = None,
    rowadd: Optional[torch.Tensor] = None,
    out: Optional[torch.Tensor] = None,
    out_dtype: Optional[torch.dtype] = None,
    mode: int = L.VR_EPI_LINEAR,
    positions: Optional[torch.Tensor] = None,
    rope_cos: Optional[torch.Tensor] = None,
    rope_sin: Optional[torch.Tensor] = None,
    rope_cols: int = 0,
    block_n: int = 0,
) -> torch.Tensor:
    """``out = epilogue(a @ w.T)`` on wgmma. ``a`` [M,K], ``w`` [N,K] (nn.Linear layout), both bf16 or both fp16.

    LINEAR: ``out = [resid +] scale * gelu?(a@w.T + bias) [+ rowadd[row % period]]``; out in the operands' type (the
    default) or fp32. ROPE / SWIGLU write the operands' type; see include/visrag_b200.h.
    """
    _half_operands(a=a, w=w)
    M, K = a.shape
    N, K2 = w.shape
    if K != K2:
        raise ValueError(f"gemm: K mismatch {K} vs {K2}")
    out_cols = N // 2 if mode == L.VR_EPI_SWIGLU else N
    if mode != L.VR_EPI_LINEAR or out_dtype is None:
        out_dtype = a.dtype
    if out_dtype not in (a.dtype, torch.float32):
        raise ValueError(f"gemm: {a.dtype} operands write {a.dtype} or float32, not {out_dtype}")
    # A and W are TMA sources (16-byte bases); the epilogue reads bias, rowadd, resid and the RoPE tables as float2 and
    # positions as int32; a LINEAR out takes 16-byte stores, ROPE / SWIGLU outputs 4-byte ones (include/visrag_b200.h)
    _operand("gemm", "a", a, HALF_DTYPES, (M, K), 16, a)
    _operand("gemm", "w", w, HALF_DTYPES, (N, K), 16, a)
    if out is None:
        out = torch.empty((M, out_cols), dtype=out_dtype, device=a.device)
    _operand("gemm", "out", out, (out_dtype,), (M, out_cols), 16 if mode == L.VR_EPI_LINEAR else 4, a)
    if bias is not None:
        _operand("gemm", "bias", bias, _F32, (N,), 8, a, contiguous=True)
    if rowadd is not None:
        _operand("gemm", "rowadd", rowadd, _F32, (None, N), 8, a, contiguous=True)
    if resid is not None:
        _operand("gemm", "resid", resid, _F32, (M, out_cols), 8, a)
        if resid.stride(0) != out.stride(0):
            raise ValueError("gemm: resid must have out's row pitch")
    if positions is not None:
        _operand("gemm", "positions", positions, _I32, (M,), 4, a, contiguous=True)
    for t, n in ((rope_cos, "rope_cos"), (rope_sin, "rope_sin")):
        if t is not None:
            _operand("gemm", n, t, _F32, (None, 32), 8, a, contiguous=True)
    e = L.GemmEpilogue()
    e.mode = mode
    e.out_dtype = _VR_DTYPE[out_dtype]
    e.act_gelu = int(gelu)
    e.scale = float(scale)
    e.bias = L.ptr(bias)
    e.resid = L.ptr(resid)
    e.rowadd = L.ptr(rowadd)
    e.rowadd_period = 0 if rowadd is None else rowadd.shape[0]
    e.positions = L.ptr(positions)
    e.rope_cos = L.ptr(rope_cos)
    e.rope_sin = L.ptr(rope_sin)
    e.rope_cols = rope_cols
    e.out = out.data_ptr()
    e.ldo = out.stride(0)
    kind = "gemm" if _PROF is None else f"gemm:{M}x{N}x{K}:" + ("rope" if mode == L.VR_EPI_ROPE else "swiglu" if mode == L.VR_EPI_SWIGLU
                                                               else ("gelu" if gelu else "") + ("+resid" if resid is not None else "") +
                                                               ("f32" if out_dtype == torch.float32 else "bf16" if out_dtype == torch.bfloat16 else "f16"))
    _launch(kind, 2.0 * M * N * K, L.lib().vr_gemm_tuned, a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), _VR_DTYPE[a.dtype],
            M, N, K, C.byref(e), block_n, L.stream_ptr())
    return out


def attention(
    q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, q_col0: int, k_col0: int, v_col0: int, head_stride: int,
    head_dim: int, heads: int, batch: int, cu_k: torch.Tensor, max_k: int, cu_q: Optional[torch.Tensor], max_q: int,
    causal: bool, scale: float, out: torch.Tensor, v_ones_column: bool = False,
) -> torch.Tensor:
    """softmax(QK^T*scale)V on wgmma; q/k/v/out are bf16 or fp16 token matrices, all of one type (see
    include/visrag_b200.h)."""
    _half_operands(q=q, k=k, v=v, out=out)
    for name, t in (("q", q), ("k", k), ("v", v)):  # TMA sources
        _operand("attention", name, t, HALF_DTYPES, (None, None), 16, q)
    _operand("attention", "out", out, HALF_DTYPES, (None, None), 4, q)
    _operand("attention", "cu_k", cu_k, _I32, (batch + 1,), 4, q, contiguous=True)
    if cu_q is not None:
        _operand("attention", "cu_q", cu_q, _I32, (batch + 1,), 4, q, contiguous=True)
    p = L.AttnParams()
    p.q, p.ldq, p.q_rows = q.data_ptr(), q.stride(0), q.shape[0]
    p.k, p.ldk = k.data_ptr(), k.stride(0)
    p.v, p.ldv, p.kv_rows = v.data_ptr(), v.stride(0), k.shape[0]
    p.q_col0, p.k_col0, p.v_col0 = q_col0, k_col0, v_col0
    p.head_stride, p.head_dim, p.heads, p.batch = head_stride, head_dim, heads, batch
    p.cu_q, p.cu_k = L.ptr(cu_q), cu_k.data_ptr()
    p.max_q, p.max_k = max_q, max_k
    p.causal, p.scale = int(causal), float(scale)
    p.out, p.ldo = out.data_ptr(), out.stride(0)
    p.flags = (L.VR_ATTN_V_ONES_COLUMN if v_ones_column else 0) | (L.VR_ATTN_F16 if q.dtype == torch.float16 else 0)
    _launch("attention", 0.0, L.lib().vr_attention, C.byref(p), L.stream_ptr())
    return out


def im2col_norm(pixels: torch.Tensor, patch: int, ld_out: int, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """uint8 [S,h,w,3] -> bf16 / fp16 patch matrix [S*(h/p)*(w/p), ld_out] (normalised, zero padded columns)."""
    vr_dtype = _half_dtype(dtype, "im2col_norm")
    if pixels.dtype != torch.uint8 or pixels.dim() != 4 or pixels.shape[3] != 3 or not pixels.is_contiguous():
        raise ValueError("im2col_norm: expected contiguous uint8 [S,h,w,3]")
    L.check_device(pixels)
    S, h, w, _ = pixels.shape
    out = torch.empty((S * (h // patch) * (w // patch), ld_out), dtype=dtype, device=pixels.device)
    _launch("im2col", 0.0, L.lib().vr_im2col_norm_ex, pixels.data_ptr(), S, h, w, patch, out.data_ptr(), ld_out, vr_dtype,
            L.stream_ptr())
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, *, add: Optional[torch.Tensor] = None,
              dtype: torch.dtype = torch.bfloat16):
    """fp32 [M,D] -> LN(x) in `dtype` (bf16 or fp16); with ``add`` [P,D] also returns LN(x)+add[row % P] (same dtype)."""
    vr_dtype = _half_dtype(dtype, "layernorm")
    _operand("layernorm", "x", x, _F32, (None, None), 16, x)
    M, D = x.shape
    _operand("layernorm", "gamma", gamma, _F32, (D,), 16, x, contiguous=True)
    _operand("layernorm", "beta", beta, _F32, (D,), 16, x, contiguous=True)
    if add is not None:
        _operand("layernorm", "add", add, _F32, (None, D), 16, x, contiguous=True)
    L.check_device(x)
    out = torch.empty((M, D), dtype=dtype, device=x.device)
    out2 = torch.empty_like(out) if add is not None else None
    _launch("norm", 0.0, L.lib().vr_layernorm_ex, x.data_ptr(), x.stride(0), gamma.data_ptr(), beta.data_ptr(), eps, M, D,
            out.data_ptr(), out.stride(0), L.ptr(out2), L.ptr(add), 0 if add is None else add.shape[0], vr_dtype, L.stream_ptr())
    return out if add is None else (out, out2)


def rmsnorm(x: torch.Tensor, gamma: torch.Tensor, eps: float, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """fp32 [M,D] -> RMSNorm(x) in `dtype` (bf16 or fp16)."""
    vr_dtype = _half_dtype(dtype, "rmsnorm")
    _operand("rmsnorm", "x", x, _F32, (None, None), 16, x)
    M, D = x.shape
    _operand("rmsnorm", "gamma", gamma, _F32, (D,), 16, x, contiguous=True)
    L.check_device(x)
    out = torch.empty((M, D), dtype=dtype, device=x.device)
    _launch("norm", 0.0, L.lib().vr_rmsnorm_ex, x.data_ptr(), x.stride(0), gamma.data_ptr(), eps, M, D, out.data_ptr(),
            out.stride(0), vr_dtype, L.stream_ptr())
    return out


def build_lm_input(src: torch.Tensor, embed: torch.Tensor, scale_emb: float, vision: Optional[torch.Tensor]) -> torch.Tensor:
    """Packed LM input rows (fp32) from the vision rows and a bf16 or fp16 embedding table."""
    vr_dtype = _half_dtype(embed.dtype, "build_lm_input")
    _operand("build_lm_input", "embed", embed, HALF_DTYPES, (None, None), 8, embed, contiguous=True)
    T, D = src.shape[0], embed.shape[1]
    _operand("build_lm_input", "src", src, _I32, (T,), 4, embed, contiguous=True)
    if vision is not None:
        _operand("build_lm_input", "vision", vision, _F32, (None, D), 16, embed)
    L.check_device(embed)
    h = torch.empty((T, D), dtype=torch.float32, device=embed.device)
    _launch("other", 0.0, L.lib().vr_build_lm_input_ex, src.data_ptr(), T, D, embed.data_ptr(), vr_dtype, scale_emb, L.ptr(vision),
            0 if vision is None else vision.stride(0), h.data_ptr(), h.stride(0), L.stream_ptr())
    return h


POOLING = {"wmean": 0, "mean": 1, "lasttoken": 2, "cls": 3}


def pool_norm(h: torch.Tensor, gamma: torch.Tensor, eps: float, cu: torch.Tensor, pooling: str, normalize: bool) -> torch.Tensor:
    """fp32 h [T, D] (any row pitch) -> reps [B, D] fp32: final RMSNorm, pooling over rows cu[b]..cu[b+1], L2 normalise."""
    _operand("pool_norm", "h", h, _F32, (None, None), 16, h)
    _operand("pool_norm", "gamma", gamma, _F32, (h.shape[1],), 16, h, contiguous=True)
    _operand("pool_norm", "cu", cu, _I32, (None,), 4, h, contiguous=True)
    if pooling not in POOLING:
        raise ValueError(f"pool_norm: pooling must be one of {sorted(POOLING)}, got {pooling!r}")
    B = cu.shape[0] - 1
    L.check_device(h)
    reps = torch.empty((B, h.shape[1]), dtype=torch.float32, device=h.device)
    _launch("other", 0.0, L.lib().vr_pool_norm, h.data_ptr(), h.stride(0), gamma.data_ptr(), eps, cu.data_ptr(), B, h.shape[1],
            POOLING[pooling], int(normalize), reps.data_ptr(), L.stream_ptr())
    return reps


def prefix_rows(prefix: torch.Tensor, rows: torch.Tensor, out: torch.Tensor, cu_rows: torch.Tensor, cu_out: torch.Tensor) -> torch.Tensor:
    """Sequence b of `out` (rows cu_out[b]..cu_out[b+1]) = [all rows of `prefix` ; rows cu_rows[b]..cu_rows[b+1] of `rows`].
    The three are matrices of one dtype (16-bit or fp32) with unit inner stride and the same column count; they may be
    column blocks of wider rows (include/visrag_b200.h)."""
    for name, t in (("prefix", prefix), ("rows", rows), ("out", out)):
        if t.dtype != out.dtype or t.dim() != 2 or t.stride(1) != 1 or t.shape[1] != out.shape[1] or not t.is_cuda:
            raise ValueError(f"prefix_rows: {name} must be a CUDA {out.dtype} matrix of {out.shape[1]} unit-stride columns, "
                             f"got {t.dtype} {tuple(t.shape)}")
        L.check_device(t)
    if cu_rows.dtype != torch.int32 or cu_out.dtype != torch.int32 or cu_rows.shape != cu_out.shape:
        raise ValueError("prefix_rows: cu_rows and cu_out must be int32 of the same length")
    _launch("other", 0.0, L.lib().vr_prefix_rows, prefix.data_ptr(), prefix.stride(0), rows.data_ptr(), rows.stride(0),
            out.data_ptr(), out.stride(0), cu_rows.data_ptr(), cu_out.data_ptr(), cu_out.shape[0] - 1, prefix.shape[0],
            out.shape[0], out.shape[1], out.element_size(), L.stream_ptr())
    return out
