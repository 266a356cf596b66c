"""Every kernel on strided, offset and edge-tile operands, against the float64 references and per-element bounds of
tests/kernel_bounds.py (kernel_bounds_f16.py for fp16 outputs).

Each case runs on views: A and W are column blocks of wider matrices (lda, ldb > K), `out` and the in-place residual are
column blocks of wider buffers, bias / rowadd / the RoPE tables start 16 bytes into their storage. Everything around a
view holds finite poison, so a stray read is a wrong value (not a NaN a comparison could miss), and everything around an
output view must keep its bits. The same case then runs again on contiguous copies of the same operands and must give
the same bits, and every block_n selector that accepts a case must give the same bits too (DESIGN §5).

GEMM covering set (EDGE_CASES): for each (dtype, epilogue form) case i takes M = M_CLASSES[i], the N class
(i + a) % 5 and the K class (i + b) % 6 of its form, with offsets a, b fixed per form; every selector runs the same
cases. So every (selector, dtype, form) meets every M, N and K class, and the offsets vary which classes meet. PAIRS
adds the interacting edges: partial M x partial N and an unpaired CTA-pair tile (odd row-tile count) x partial N.
  M: 1, 64, 65, 128, 129, 255, 257, 385 - the auto switch at 128, partial row tiles, CTA pairs whose 2nd tile is past M
  N (LINEAR): 8, 72, 136, 200, 1160 - partial 8-column groups of 64/128/192/256-wide tiles
  N (ROPE / SWIGLU): 64, 192, 320, 448, 704 - N = 64 or 128 mod 192 and 256 and 64 mod 128: a last tile holding one
      or two 64-column blocks, and a multicast half wholly past N
  K: 8, 56 (one partial k-block), 64, 72, 1152 (the ping-pong epilogue's short K), 1160 (a partial block after 18)
  rope_cols: 0, 64, an odd multiple of 64 inside a tile, N
"""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF, F16, F32 = torch.bfloat16, torch.float16, torch.float32
POISON = 1000.0         # finite, exact in bf16 / fp16: a poisoned element read into a result moves it far past its bound
SELECTORS = [0, 2, 3, 4, 5, 64, 128, 192, 256]
M_CLASSES = [1, 64, 65, 128, 129, 255, 257, 385]
N_LINEAR = [8, 72, 136, 200, 1160]
N_BLOCKS = [64, 192, 320, 448, 704]
K_CLASSES = [8, 56, 64, 72, 1152, 1160]
MAX_POS = 512
# epilogue form -> (LINEAR?, offsets of the N and K classes in the covering set)
FORMS = {
    "f32": (True, 0, 0),
    "f32 bias scale rowadd resid": (True, 1, 2),
    "16 bias (lean)": (True, 2, 4),
    "16 bias gelu (lean)": (True, 3, 1),
    "16 plain": (True, 4, 3),
    "16 bias scale": (True, 0, 5),
    "rope": (False, 1, 1),
    "swiglu": (False, 2, 3),
}
PAIRS = [(129, 72, 56), (255, 200, 1160), (257, 136, 72), (385, 1160, 8), (65, 8, 1152)]
PAIRS_BLOCKS = [(129, 192, 56), (257, 320, 72), (385, 64, 1160), (65, 704, 1152)]


def EDGE_CASES(form):
    linear, a, b = FORMS[form]
    ns = N_LINEAR if linear else N_BLOCKS
    cases = [(m, ns[(i + a) % len(ns)], K_CLASSES[(i + b) % len(K_CLASSES)]) for i, m in enumerate(M_CLASSES)]
    return cases + (PAIRS if linear else PAIRS_BLOCKS)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0, mean=0.0):
    return torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale + mean


def _bits(t):
    """Integer view of a tensor's bits (so -0 / +0 and NaN payloads compare exactly)."""
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same_bits(x, y):
    return x.shape == y.shape and x.dtype == y.dtype and torch.equal(_bits(x), _bits(y))


def _block(x, left, right, fill=POISON):
    """x as columns [left, left + cols) of a wider buffer whose other columns hold `fill`: returns (buffer, view)."""
    buf = torch.full((x.shape[0], left + x.shape[1] + right), fill, dtype=x.dtype, device=DEV)
    view = buf[:, left:left + x.shape[1]]
    view.copy_(x)
    return buf, view


def _shifted(x, elems=4, fill=POISON):
    """x at a storage offset of `elems` elements (16 bytes of fp32), poison in front."""
    buf = torch.full((elems + x.numel(),), fill, dtype=x.dtype, device=DEV)
    view = buf[elems:].view(x.shape)
    view.copy_(x)
    return view


def _outside_unchanged(name, buf, before, left, cols):
    """Every column of `buf` outside [left, left + cols) keeps the bits it had in `before`."""
    keep = torch.ones(buf.shape[1], dtype=torch.bool, device=DEV)
    keep[left:left + cols] = False
    assert torch.equal(_bits(buf[:, keep]), _bits(before[:, keep])), f"{name}: a store landed outside the output view"


def _check(name, got, ref, e):
    return KF.check(name, got, ref, e, verbose=False)


# ---------------------------------------------------------------------------------------------------------------- GEMM


def _positions(M, seed):
    """Not monotone, with repeats, 0 and MAX_POS - 1."""
    p = torch.randint(0, MAX_POS, (M,), device=DEV, dtype=torch.int32, generator=_gen(seed))
    p[0] = MAX_POS - 1
    if M > 1:
        p[1] = 0
    if M > 3:
        p[3] = p[2]
    return p


def _rope_tables():
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, device=DEV).float() / 64))
    fr = torch.outer(torch.arange(MAX_POS, device=DEV).float(), inv)
    return fr.cos().contiguous(), fr.sin().contiguous()


def _rope_cols(N, i):
    """0, 64, an odd multiple of 64 inside a 128/192/256-wide tile, N - in turn over the cases."""
    odd = 320 if N > 320 else 64      # 320: inside a tile of every width from 128 to 256
    return [0, 64, odd, N][i % 4]


def _gemm_inputs(form, dtype, M, N, K, i):
    """Contiguous operands and the ops.gemm keywords of one case (the same for every selector)."""
    from visrag_b200 import _lib as L

    seed = (M * 7919 + N * 104729 + K * 13 + i) % (2 ** 31)
    a = _randn(M, K, seed=seed, scale=0.5).to(dtype)
    w = _randn(N, K, seed=seed + 1, scale=0.05).to(dtype)
    kw, out_dtype = {}, dtype
    if form.startswith("f32"):
        out_dtype = F32
    if "bias" in form:
        kw["bias"] = _randn(N, seed=seed + 2)
    if "gelu" in form:
        kw["gelu"] = True
    if form == "f32 bias scale rowadd resid":
        kw.update(scale=-0.75, rowadd=_randn(37, N, seed=seed + 3), resid=_randn(M, N, seed=seed + 4))
    if form == "16 bias scale":
        kw["scale"] = 0.5
    if form == "rope":
        cos, sin = _rope_tables()
        kw.update(mode=L.VR_EPI_ROPE, positions=_positions(M, seed + 5), rope_cos=cos, rope_sin=sin, rope_cols=_rope_cols(N, i))
    if form == "swiglu":
        kw["mode"] = L.VR_EPI_SWIGLU
    return a, w, kw, out_dtype


def _gemm_ref(form, a, w, kw):
    if form == "rope":
        return KB.gemm_rope_ref(a, w, kw["positions"], kw["rope_cos"], kw["rope_sin"], kw["rope_cols"])
    if form == "swiglu":
        return KB.gemm_swiglu_ref(a, w)
    return KB.gemm_linear_ref(a, w, **{n: kw[n] for n in ("bias", "gelu", "scale", "rowadd", "resid") if n in kw})


def _gemm_run(a, w, kw, out_dtype, bn, views):
    """One launch; with `views`, every operand is a view with poison around it (returns the output as a contiguous copy
    after checking that nothing outside the output view changed)."""
    from visrag_b200 import _lib as L
    from visrag_b200 import ops

    M, N = a.shape[0], w.shape[0]
    cols = N // 2 if kw.get("mode") == L.VR_EPI_SWIGLU else N
    args = dict(kw)
    if not views:
        out = args.pop("resid").clone() if "resid" in args else torch.empty(M, cols, dtype=out_dtype, device=DEV)
        if "resid" in kw:
            args["resid"] = out
        return ops.gemm(a, w, out=out, out_dtype=out_dtype, block_n=bn, **args).clone()
    _, av = _block(a, 8, 16)                      # lda = ldb = K + 24: TMA must read zeros, not columns K.., past K
    _, wv = _block(w, 8, 16)
    for n in ("bias", "rowadd", "rope_cos", "rope_sin"):
        if n in args:
            args[n] = _shifted(args[n])
    left = 8                                      # 16 bytes (16-bit) / 32 bytes (fp32) into the row: every row stays aligned
    if "resid" in args:
        buf, ov = _block(args.pop("resid"), left, 8)
        args["resid"] = ov
    else:
        buf, ov = _block(torch.empty(M, cols, dtype=out_dtype, device=DEV).fill_(-POISON), left, 8, -7.0)
    before = buf.clone()
    got = ops.gemm(av, wv, out=ov, out_dtype=out_dtype, block_n=bn, **args)
    assert got.data_ptr() == ov.data_ptr()
    _outside_unchanged("gemm", buf, before, left, cols)
    return got.clone()


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("form", list(FORMS))
def test_gemm_edge_tiles_and_views(form, dtype):
    """The covering set of the module doc: within bounds on views, the same bits on contiguous copies, the same bits from
    every selector."""
    linear = FORMS[form][0]
    selectors = [b for b in SELECTORS if linear or b != 3]   # block_n = 3 runs LINEAR epilogues only
    for i, (M, N, K) in enumerate(EDGE_CASES(form)):
        a, w, kw, out_dtype = _gemm_inputs(form, dtype, M, N, K, i)
        ref, e = _gemm_ref(form, a, w, kw)
        first = None
        for bn in selectors:
            name = f"{form} {dtype} {M}x{N}x{K} bn={bn}" + (f" rope_cols={kw['rope_cols']}" if form == "rope" else "")
            got = _gemm_run(a, w, kw, out_dtype, bn, views=True)
            _check(name, got, ref, e)
            assert _same_bits(got, _gemm_run(a, w, kw, out_dtype, bn, views=False)), f"{name}: views and contiguous copies differ"
            if first is None:
                first = (bn, got)
            assert _same_bits(got, first[1]), f"{name}: differs from block_n={first[0]}"


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_gemm_negative_zero_accumulator_survives_the_16bit_store(dtype):
    """16-bit LINEAR with no bias keeps the generic epilogue: an accumulator of -0 (a row of -0 times positive weights)
    is stored as -0, the sign the fp32 output of the same GEMM shows. A bias (the lean path) adds +0 on purpose."""
    from visrag_b200 import ops

    for M, N, K in [(129, 136, 64), (1, 72, 1152), (257, 200, 1152)]:
        a = _randn(M, K, seed=M + K, scale=0.5).to(dtype)
        a[0] = -0.0
        w = _randn(N, K, seed=N + K, scale=0.05).abs().to(dtype)
        for bn in SELECTORS:
            f32 = ops.gemm(a, w, out_dtype=F32, block_n=bn)
            h16 = ops.gemm(a, w, block_n=bn)
            z = f32 == 0
            assert z[0].any(), "the -0 row did not give a zero accumulator"
            assert torch.equal(torch.signbit(h16[z]), torch.signbit(f32[z])), f"{M}x{N}x{K} bn={bn}: sign of zero lost"


# ---------------------------------------------------------------------------------------------------------------- norms


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("D", [288, 1152, 2304])
def test_norms_on_column_blocks(D, dtype):
    from visrag_b200 import ops

    g, b, add = _randn(D, seed=D), _randn(D, seed=D + 1), _randn(37, D, seed=D + 2)
    for M in (1, 13, 300):
        x = _randn(M, D, seed=M + D, scale=3.0, mean=1.0)
        buf, xv = _block(x, 4, 12)                                  # ldx = D + 16, 16 bytes into the row
        before = buf.clone()
        gv, bv, av = _shifted(g), _shifted(b), _shifted(add)
        o1, o2 = ops.layernorm(xv, gv, bv, 1e-6, add=av, dtype=dtype)
        (r1, e1), (r2, e2) = KB.layernorm_ref(x, g, b, 1e-6, add=add)
        _check(f"layernorm D={D} M={M}", o1, r1, e1)
        _check(f"layernorm+add D={D} M={M}", o2, r2, e2)
        c1, c2 = ops.layernorm(x, g, b, 1e-6, add=add, dtype=dtype)
        assert _same_bits(o1, c1) and _same_bits(o2, c2), f"layernorm D={D} M={M}: views and contiguous copies differ"
        o3 = ops.layernorm(xv, gv, bv, 1e-6, dtype=dtype)
        assert _same_bits(o3, c1), f"layernorm D={D} M={M}: without add differs"
        r = ops.rmsnorm(xv, gv, 1e-5, dtype)
        _check(f"rmsnorm D={D} M={M}", r, *KB.rmsnorm_ref(x, g, 1e-5))
        assert _same_bits(r, ops.rmsnorm(x, g, 1e-5, dtype)), f"rmsnorm D={D} M={M}: views and contiguous copies differ"
        assert torch.equal(_bits(buf), _bits(before)), "a norm wrote into its input"


# ---------------------------------------------------------------------------------------------------- LM input, pooling


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_build_lm_input_with_vision_column_block(dtype):
    from visrag_b200 import ops

    D = 2304
    emb = _randn(512, D, seed=60).to(dtype)
    vis = _randn(128, D, seed=61)
    _, vv = _block(vis, 4, 28)
    src = torch.tensor([-6, 0, 1, 127, -512, -1, 5, -300, 127, 0], dtype=torch.int32, device=DEV)
    got = ops.build_lm_input(src, emb, 12.0, vv)
    _check("build_lm_input vision view", got, *KB.build_lm_input_ref(src, emb, 12.0, vis))
    assert _same_bits(got, ops.build_lm_input(src, emb, 12.0, vis))


@pytest.mark.parametrize("pooling", ["wmean", "mean", "lasttoken", "cls"])
def test_pool_norm_with_hidden_column_block(pooling):
    """Both cluster sizes: 8 CTAs per sequence while batch * 8 fits 5 per SM, else 4 (batch 200)."""
    from visrag_b200 import ops

    for D in (288, 2304):
        gamma = _randn(D, seed=D)
        for lens in ([1, 7, 300, 64], [3, 40, 1] * 67):
            cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)
            h = _randn(int(cu[-1]), D, seed=len(lens) + D, scale=2.0)
            buf, hv = _block(h, 4, 12)
            before = buf.clone()
            got = ops.pool_norm(hv, _shifted(gamma), 1e-5, cu, pooling, True)
            _check(f"pool_norm {pooling} D={D} B={len(lens)}", got, *KB.pool_norm_ref(h, gamma, 1e-5, cu, pooling, True))
            assert _same_bits(got, ops.pool_norm(h, gamma, 1e-5, cu, pooling, True))
            assert torch.equal(_bits(buf), _bits(before))


# ---------------------------------------------------------------------------------------------------------------- attention


@pytest.fixture(params=[0, 1], ids=["auto", "one_warpgroup"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


def _attn_case(dtype, lens, nh, hd, hs, causal, seed, resampler=False):
    """q / k / v as heads at non-zero column offsets inside wider rows whose other columns hold poison (pad columns
    inside a head are zero, as the header requires); returns the wide matrix, the column offsets, contiguous copies of
    q / k / v and the ops.attention keywords."""
    T = sum(lens)
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)
    heads = torch.zeros(T, 3, nh, hs, device=DEV)
    heads[..., :hd] = _randn(T, 3, nh, hd, seed=seed)
    q, k, v = (heads[:, j].reshape(T, nh * hs).to(dtype) for j in range(3))
    c0 = [16, 16 + nh * hs + 8, 16 + 2 * nh * hs + 16]                 # a gap of poison between the blocks
    wide = torch.full((T, c0[2] + nh * hs + 24), POISON, dtype=dtype, device=DEV)
    for c, t in zip(c0, (q, k, v)):
        wide[:, c:c + nh * hs] = t
    common = dict(head_stride=hs, head_dim=hd, heads=nh, causal=causal, scale=hd ** -0.5, batch=len(lens), cu_k=cu,
                  max_k=max(lens))
    if resampler:
        common.update(cu_q=None, max_q=64)
    else:
        common.update(cu_q=cu, max_q=max(lens))
    return wide, c0, (q, k, v), common


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", ["vit", "lm-causal", "resampler"])
def test_attention_heads_at_column_offsets(shape, dtype, attn_variant):
    from visrag_b200 import ops

    nh, hd, hs, causal, lens = {"vit": (4, 72, 80, False, [1036, 300, 1, 65]),
                                "lm-causal": (6, 64, 64, True, [1, 2, 129, 300, 64]),
                                "resampler": (3, 128, 128, False, [100, 1036])}[shape]
    wide, c0, (q, k, v), kw = _attn_case(dtype, lens, nh, hd, hs, causal, 77 + len(lens), resampler=shape == "resampler")
    rows = kw["batch"] * 64 if shape == "resampler" else sum(lens)
    buf, ov = _block(torch.zeros(rows, nh * hd, dtype=dtype, device=DEV), 8, 24, -POISON)
    before = buf.clone()
    if shape == "resampler":   # 64 learned queries, the same for every item, in their own matrix
        qc = _randn(64, nh * hs, seed=5).to(dtype)
        qa, q_col0 = _block(qc, 16, 8)[0], 16
    else:
        qa, q_col0, qc = wide, c0[0], q
    ops.attention(qa, wide, wide, q_col0=q_col0, k_col0=c0[1], v_col0=c0[2], out=ov, **kw)
    _outside_unchanged("attention", buf, before, 8, nh * hd)
    refkw = {n: kw[n] for n in ("head_stride", "head_dim", "heads", "cu_k", "cu_q", "max_q", "causal", "scale")}
    ref_fn = KF.attention_ref_f16 if dtype == F16 else KB.attention_ref
    ref, e = ref_fn(qc, k, v, q_col0=0, k_col0=0, v_col0=0, **refkw)
    _check(f"attention {shape} {dtype}", ov, ref, e)
    want = torch.empty(rows, nh * hd, dtype=dtype, device=DEV)
    ops.attention(qc, k, v, q_col0=0, k_col0=0, v_col0=0, out=want, **kw)
    assert _same_bits(ov, want), f"attention {shape}: views and contiguous copies differ"


# ------------------------------------------------------------------------------------------- refusals, with no launch


class _NoLibrary:
    """Stands in for the C library: any use of it fails the test, so a missing check shows as "reached the library"."""

    def __getattr__(self, name):
        raise AssertionError(f"reached the library ({name}): the operand was not refused")


@pytest.fixture
def no_library(monkeypatch):
    from visrag_b200 import _lib as L

    monkeypatch.setattr(L, "lib", lambda: _NoLibrary())


def _refusals():
    """(wrapper, argument, call) for every tensor argument of every wrapper: wrong dtype, non-unit inner stride, wrong
    length or width, a storage offset below the argument's alignment."""
    from visrag_b200 import _lib as L
    from visrag_b200 import ops

    M, N, K, D = 256, 128, 64, 1152
    a, w = torch.zeros(M, K, dtype=BF, device=DEV), torch.zeros(N, K, dtype=BF, device=DEV)
    f = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)  # noqa: E731
    cos = f(MAX_POS, 32)
    rope = dict(mode=L.VR_EPI_ROPE, positions=i32(M), rope_cos=cos, rope_sin=cos, rope_cols=64)
    shift = lambda t, n=1: _shifted(t, n, 0)  # noqa: E731
    cases = [
        ("gemm", "a", lambda: ops.gemm(shift(a), w)),
        ("gemm", "a", lambda: ops.gemm(f(K, M).bfloat16().t(), w)),
        ("gemm", "w", lambda: ops.gemm(a, shift(w))),
        ("gemm", "out", lambda: ops.gemm(a, w, out=shift(torch.zeros(M, N, dtype=BF, device=DEV), 2))),
        ("gemm", "out", lambda: ops.gemm(a, w, out=torch.zeros(M, N + 8, dtype=BF, device=DEV))),
        ("gemm", "out", lambda: ops.gemm(a, w, out=torch.zeros(N, M, dtype=BF, device=DEV).t())),
        ("gemm", "bias", lambda: ops.gemm(a, w, bias=f(N + 1)[1:])),
        ("gemm", "bias", lambda: ops.gemm(a, w, bias=f(N - 8))),
        ("gemm", "bias", lambda: ops.gemm(a, w, bias=f(N).half())),
        ("gemm", "bias", lambda: ops.gemm(a, w, bias=f(2 * N)[::2])),
        ("gemm", "rowadd", lambda: ops.gemm(a, w, rowadd=f(37, N - 8))),
        ("gemm", "rowadd", lambda: ops.gemm(a, w, rowadd=f(N + 1)[1:].view(1, N))),
        ("gemm", "rowadd", lambda: ops.gemm(a, w, rowadd=f(N, 37).t())),
        ("gemm", "resid", lambda: ops.gemm(a, w, out_dtype=F32, resid=f(M, N).bfloat16())),
        ("gemm", "resid", lambda: ops.gemm(a, w, out_dtype=F32, resid=f(M, N - 8))),
        ("gemm", "resid", lambda: ops.gemm(a, w, out_dtype=F32, resid=shift(f(M, N)))),
        ("gemm", "positions", lambda: ops.gemm(a, w, **dict(rope, positions=i32(M).long()))),
        ("gemm", "positions", lambda: ops.gemm(a, w, **dict(rope, positions=i32(M - 1)))),
        ("gemm", "positions", lambda: ops.gemm(a, w, **dict(rope, positions=i32(2 * M)[::2]))),
        ("gemm", "rope_cos", lambda: ops.gemm(a, w, **dict(rope, rope_cos=f(MAX_POS, 64)))),
        ("gemm", "rope_cos", lambda: ops.gemm(a, w, **dict(rope, rope_cos=shift(cos)))),
        ("gemm", "rope_sin", lambda: ops.gemm(a, w, **dict(rope, rope_sin=f(32, MAX_POS).t()))),
        ("gemm", "rope_sin", lambda: ops.gemm(a, w, **dict(rope, rope_sin=cos.double()))),
        ("layernorm", "x", lambda: ops.layernorm(f(M, D).bfloat16(), f(D), f(D), 1e-6)),
        ("layernorm", "x", lambda: ops.layernorm(f(D, M).t(), f(M), f(M), 1e-6)),
        ("layernorm", "x", lambda: ops.layernorm(shift(f(M, D)), f(D), f(D), 1e-6)),
        ("layernorm", "gamma", lambda: ops.layernorm(f(M, D), f(D - 4), f(D), 1e-6)),
        ("layernorm", "gamma", lambda: ops.layernorm(f(M, D), shift(f(D)), f(D), 1e-6)),
        ("layernorm", "gamma", lambda: ops.layernorm(f(M, D), f(D).bfloat16(), f(D), 1e-6)),
        ("layernorm", "beta", lambda: ops.layernorm(f(M, D), f(D), f(2 * D)[::2], 1e-6)),
        ("layernorm", "beta", lambda: ops.layernorm(f(M, D), f(D), f(D - 4), 1e-6)),
        ("layernorm", "add", lambda: ops.layernorm(f(M, D), f(D), f(D), 1e-6, add=f(37, D - 4))),
        ("layernorm", "add", lambda: ops.layernorm(f(M, D), f(D), f(D), 1e-6, add=shift(f(37, D)))),
        ("rmsnorm", "x", lambda: ops.rmsnorm(f(M, D).half(), f(D), 1e-5)),
        ("rmsnorm", "x", lambda: ops.rmsnorm(f(D, M).t(), f(M), 1e-5)),
        ("rmsnorm", "gamma", lambda: ops.rmsnorm(f(M, D), f(D - 4), 1e-5)),
        ("rmsnorm", "gamma", lambda: ops.rmsnorm(f(M, D), shift(f(D)), 1e-5)),
        ("build_lm_input", "src", lambda: ops.build_lm_input(i32(8).long(), f(64, D).bfloat16(), 1.0, None)),
        ("build_lm_input", "src", lambda: ops.build_lm_input(i32(16)[::2], f(64, D).bfloat16(), 1.0, None)),
        ("build_lm_input", "embed", lambda: ops.build_lm_input(i32(8), shift(f(64, D).bfloat16()), 1.0, None)),
        ("build_lm_input", "vision", lambda: ops.build_lm_input(i32(8), f(64, D).bfloat16(), 1.0, f(16, D).bfloat16())),
        ("build_lm_input", "vision", lambda: ops.build_lm_input(i32(8), f(64, D).bfloat16(), 1.0, f(D, 16).t())),
        ("build_lm_input", "vision", lambda: ops.build_lm_input(i32(8), f(64, D).bfloat16(), 1.0, f(16, D - 4))),
        ("build_lm_input", "vision", lambda: ops.build_lm_input(i32(8), f(64, D).bfloat16(), 1.0, shift(f(16, D)))),
        ("pool_norm", "h", lambda: ops.pool_norm(f(M, D).bfloat16(), f(D), 1e-5, i32(3), "mean", True)),
        ("pool_norm", "h", lambda: ops.pool_norm(f(D, M).t(), f(M), 1e-5, i32(3), "mean", True)),
        ("pool_norm", "h", lambda: ops.pool_norm(shift(f(M, D)), f(D), 1e-5, i32(3), "mean", True)),
        ("pool_norm", "gamma", lambda: ops.pool_norm(f(M, D), f(D - 4), 1e-5, i32(3), "mean", True)),
        ("pool_norm", "gamma", lambda: ops.pool_norm(f(M, D), shift(f(D)), 1e-5, i32(3), "mean", True)),
        ("pool_norm", "cu", lambda: ops.pool_norm(f(M, D), f(D), 1e-5, i32(3).long(), "mean", True)),
        ("pool_norm", "cu", lambda: ops.pool_norm(f(M, D), f(D), 1e-5, i32(6)[::2], "mean", True)),
    ]
    qkv = torch.zeros(M, 3 * 64, dtype=BF, device=DEV)
    akw = dict(q_col0=0, k_col0=64, v_col0=128, head_stride=64, head_dim=64, heads=1, batch=1, max_k=M, max_q=M,
               causal=True, scale=0.125)
    cu = torch.tensor([0, M], dtype=torch.int32, device=DEV)
    out = torch.zeros(M, 64, dtype=BF, device=DEV)
    att = lambda **o: ops.attention(**dict(dict(q=qkv, k=qkv, v=qkv, cu_k=cu, cu_q=cu, out=out, **akw), **o))  # noqa: E731
    cases += [
        ("attention", "q", lambda: att(q=shift(qkv))),
        ("attention", "k", lambda: att(k=shift(qkv))),
        ("attention", "v", lambda: att(v=shift(qkv))),
        ("attention", "out", lambda: att(out=shift(out))),
        ("attention", "cu_k", lambda: att(cu_k=cu.long())),
        ("attention", "cu_k", lambda: att(cu_k=torch.tensor([0, M // 2, M], dtype=torch.int32, device=DEV))),
        ("attention", "cu_q", lambda: att(cu_q=torch.tensor([[0, M]], dtype=torch.int32, device=DEV).t())),
        ("attention", "cu_q", lambda: att(cu_q=cu.long())),
    ]
    if torch.cuda.device_count() > 1:
        o = torch.device("cuda", 1)
        cases += [
            ("gemm", "bias", lambda: ops.gemm(a, w, bias=torch.zeros(N, device=o))),
            ("layernorm", "gamma", lambda: ops.layernorm(f(M, D), torch.zeros(D, device=o), f(D), 1e-6)),
            ("pool_norm", "cu", lambda: ops.pool_norm(f(M, D), f(D), 1e-5, torch.zeros(3, dtype=torch.int32, device=o), "mean", True)),
            ("attention", "cu_k", lambda: att(cu_k=cu.to(o))),
        ]
    return cases


def test_bad_operands_are_refused_before_the_library(no_library):
    cases = _refusals()
    for i, (fn, arg, call) in enumerate(cases):
        with pytest.raises(ValueError) as ei:
            call()
        msg = str(ei.value)
        assert msg.startswith((f"{fn}: {arg} ", f"{arg}: ")), f"case {i} ({fn} {arg}): {msg}"
