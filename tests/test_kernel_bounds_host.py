"""The bounds of tests/kernel_bounds.py have power: on the CPU, a faithful emulation of each kernel's arithmetic passes
its check and every mutant of a catalogue of plausible precision and indexing bugs fails it.

The emulations follow the kernels op by op where it matters: GEMM accumulates k16 steps into fp32 with truncation
(the pessimistic end of the accumulation model), runs the fp32 epilogue in the kernel's order (bias, GELU, scale, row
add, residual) with gemm.cuh's polynomial GELU; attention walks 128-key tiles with a running maximum, rounds P to bf16
for the PV product and sums the denominator from the fp32 p (attention.cuh); the norms use the two-pass fp32 mean and
variance of elementwise.cu."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB

def _randn(*shape, scale=1.0, mean=0.0, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float32) * scale + mean


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


def _check(name, got, ref, e, **kw):
    return KB.check(name, got, ref, e, verbose=False, **kw)


# ---------------------------------------------------------------------------------------------------------------- GEMM


def _f32_trunc(x64):
    """float64 -> the fp32 value next to it toward zero (round-toward-zero)."""
    f = x64.float()
    over = f.double().abs() > x64.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def emu_acc(a, w, *, bf16_kblocks=False, k_drop=0):
    """wgmma accumulation: fp32 accumulator, one k16 step at a time (16 exact products summed), truncated to fp32."""
    A, W = a.double(), w.double()
    K = A.shape[1] - k_drop
    acc = torch.zeros(A.shape[0], W.shape[0], dtype=torch.float32)
    for k0 in range(0, K, 16):
        k1 = min(K, k0 + 16)
        acc = _f32_trunc(acc.double() + A[:, k0:k1] @ W[:, k0:k1].T)
        if bf16_kblocks and k1 % 64 == 0:
            acc = acc.bfloat16().float()
    return acc


def gelu_f32(x):
    return torch.from_numpy(KB.gelu_poly_f32(x.numpy()))


def gelu_tanh_f32(x):
    return torch.nn.functional.gelu(x, approximate="tanh")


def emu_linear(a, w, *, bias=None, gelu=False, scale=1.0, rowadd=None, resid=None, out_dtype=torch.float32, mut=None):
    """The LINEAR epilogue in fp32, in the kernel's order. `mut` names one mutant."""
    x = emu_acc(a, w, bf16_kblocks=mut == "bf16 accumulation between k blocks", k_drop=8 if mut == "last 8 of K dropped" else 0)
    if mut in ("accumulator rounded to bf16", "bf16 out: acc -> bf16, + bias -> bf16"):
        x = x.bfloat16().float()
    if bias is not None:
        x = x + (bias.bfloat16().float() if mut == "bias rounded to bf16" else bias)
    if mut == "gelu after scale":
        x = gelu_f32(x * scale)
    else:
        if gelu:
            x = gelu_tanh_f32(x) if mut == "tanh GELU" else gelu_f32(x)
        x = x * scale
    if rowadd is not None:
        P = rowadd.shape[0] + (1 if mut == "row add period P + 1" else 0)
        x = x + rowadd[torch.arange(x.shape[0]) % P % rowadd.shape[0]]
    if resid is not None:
        x = x + (resid.bfloat16().float() if mut == "residual read as bf16" else resid)
    if mut == "fp32 output rounded through bf16":
        x = x.bfloat16().float()
    return x.to(out_dtype)


M, N, K = 777, 1152, 640
A = _randn(M, K, scale=0.5, seed=1).bfloat16()
W = _randn(N, K, scale=0.05, seed=2).bfloat16()
BIAS = _randn(N, seed=3)
RESID = _randn(M, N, seed=4)
ROWADD = _randn(37, N, seed=5)

# name -> (epilogue arguments, output dtype); the configurations of the GPU test's case shapes
CONFIGS = {
    "bias scale resid f32": (dict(bias=BIAS, scale=0.25, resid=RESID), torch.float32),
    "bias rowadd f32": (dict(bias=BIAS, rowadd=ROWADD), torch.float32),
    "bias bf16": (dict(bias=BIAS), torch.bfloat16),
    "bias gelu bf16": (dict(bias=BIAS, gelu=True), torch.bfloat16),
    "bias gelu scale bf16": (dict(bias=BIAS, gelu=True, scale=0.25), torch.bfloat16),
}

GEMM_MUTANTS = [
    ("bias rounded to bf16", "bias scale resid f32"),
    ("accumulator rounded to bf16", "bias scale resid f32"),
    ("bf16 accumulation between k blocks", "bias scale resid f32"),
    ("bf16 out: acc -> bf16, + bias -> bf16", "bias bf16"),
    ("tanh GELU", "bias gelu bf16"),
    ("residual read as bf16", "bias scale resid f32"),
    ("fp32 output rounded through bf16", "bias scale resid f32"),
    ("last 8 of K dropped", "bias scale resid f32"),
    ("row add period P + 1", "bias rowadd f32"),
    ("gelu after scale", "bias gelu scale bf16"),
]


def _gemm_case(config, mut=None):
    kw, dt = CONFIGS[config]
    got = emu_linear(A, W, out_dtype=dt, mut=mut, **kw)
    ref, e = KB.gemm_linear_ref(A, W, **kw)
    rms = KB.gemm_rms_rel(K) if dt == torch.float32 and not kw.get("gelu") else None
    return got, ref, e, rms


@pytest.mark.parametrize("config", list(CONFIGS))
def test_gemm_faithful_emulation_passes(config):
    got, ref, e, rms = _gemm_case(config)
    _check(config, got, ref, e, rms_rel=rms)


@pytest.mark.parametrize("mut,config", GEMM_MUTANTS, ids=[m for m, _ in GEMM_MUTANTS])
def test_gemm_mutant_fails(mut, config):
    got, ref, e, rms = _gemm_case(config, mut)
    _fails(lambda: _check(f"{config} / {mut}", got, ref, e, rms_rel=rms))


def test_gemm_faithful_passes_at_the_edges():
    """The loosest accumulation (K = 5760 with scale and residual), a single partly filled k step, and GELU tails (pre-
    activations spanning about +-40) where the erf clamp's error grows with |x|."""
    a, w = _randn(64, 5760, scale=0.5, seed=6).bfloat16(), _randn(256, 5760, scale=0.02, seed=7).bfloat16()
    kw = dict(scale=1.4 / 40 ** 0.5, resid=_randn(64, 256, seed=8))
    _check("K=5760", emu_linear(a, w, **kw), *KB.gemm_linear_ref(a, w, **kw), rms_rel=KB.gemm_rms_rel(5760))
    a, w = _randn(129, 8, seed=9).bfloat16(), _randn(72, 8, seed=10).bfloat16()
    _check("K=8", emu_linear(a, w, bias=BIAS[:72]), *KB.gemm_linear_ref(a, w, bias=BIAS[:72]), rms_rel=KB.gemm_rms_rel(8))
    a, w = _randn(300, 1152, seed=11).bfloat16(), _randn(512, 1152, scale=0.4, seed=12).bfloat16()
    b = (torch.rand(512, generator=torch.Generator().manual_seed(13)) * 2 - 1) * 25
    ref, e = KB.gemm_linear_ref(a, w, bias=b, gelu=True)
    assert ref.abs().max() > 35
    _check("gelu tails", emu_linear(a, w, bias=b, gelu=True, out_dtype=torch.bfloat16), ref, e)


def test_gelu_bound_covers_the_polynomial_everywhere():
    """The GELU term of the bound against gemm.cuh's polynomial, evaluated op by op in fp32, on a dense grid out to
    |x| = 120, where the clamp's error (1.6e-6 |x|) far exceeds an absolute 1.2e-5."""
    from scipy.special import erf

    x = np.linspace(-120, 120, 2_400_001).astype(np.float32)
    X = x.astype(np.float64)
    err = np.abs(KB.gelu_poly_f32(x).astype(np.float64) - 0.5 * X * (1 + erf(X / np.sqrt(2))))
    assert (err <= KB.GELU_REL * np.abs(X) + 1e-30).all()
    assert err[np.abs(X) > 60].max() > 1.2e-5            # the absolute form of the contract does not hold
    z = np.linspace(0, KB.GELU_ZMAX, 1_000_001).astype(np.float32)
    assert np.abs(KB.erf_poly_f32(z).astype(np.float64) - erf(z.astype(np.float64))).max() <= KB.ERF_FIT


# RoPE / SwiGLU
T, H = 64, 256
AR = _randn(T, H, scale=0.5, seed=20).bfloat16()
WR = _randn(3 * H, H, scale=0.05, seed=21).bfloat16()
POS = torch.randint(0, 2048, (T,), generator=torch.Generator().manual_seed(22), dtype=torch.int32)
_inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
_fr = torch.outer(torch.arange(2049).float(), _inv)
COS, SIN = _fr.cos().contiguous(), _fr.sin().contiguous()


def emu_rope(mut=None):
    x = emu_acc(AR, WR).view(T, 3 * H // 64, 2, 32)
    p = POS.long() + (1 if mut == "RoPE position + 1" else 0)
    c, s = COS[p][:, None, :], SIN[p][:, None, :]
    lo, hi = x[:, :, 0], x[:, :, 1]
    rot = torch.stack([lo * c - hi * s, hi * c + lo * s], 2)
    cols = 2 * H + (64 if mut == "RoPE on the v columns too" else 0)
    heads = torch.arange(3 * H // 64)[None, :, None, None] * 64 < cols
    return torch.where(heads, rot, x).reshape(T, 3 * H).bfloat16()


def emu_swiglu(w, mut=None):
    x = emu_acc(AR, w).view(T, -1, 2, 32)
    g, u = (x[:, :, 1], x[:, :, 0]) if mut == "SwiGLU gate and up swapped" else (x[:, :, 0], x[:, :, 1])
    return (torch.nn.functional.silu(g) * u).reshape(T, -1).bfloat16()


WS = _randn(2 * 512, H, scale=0.05, seed=23).bfloat16()


@pytest.mark.parametrize("mut", [None, "RoPE position + 1", "RoPE on the v columns too"])
def test_rope(mut):
    ref, e = KB.gemm_rope_ref(AR, WR, POS, COS, SIN, 2 * H)
    run = lambda: _check(f"rope {mut}", emu_rope(mut), ref, e)   # noqa: E731
    run() if mut is None else _fails(run)


@pytest.mark.parametrize("mut", [None, "SwiGLU gate and up swapped"])
def test_swiglu(mut):
    ref, e = KB.gemm_swiglu_ref(AR, WS)
    run = lambda: _check(f"swiglu {mut}", emu_swiglu(WS, mut), ref, e)   # noqa: E731
    run() if mut is None else _fails(run)


# ------------------------------------------------------------------------------------------------------------ attention


def emu_attention_head(q, k, v, scale, causal, hs, mut=None):
    """attention.cuh for one head and sequence: q [Lq, hd], k / v [Lk, hd] bf16 -> bf16 [Lq, hd]."""
    Lq, Lk = q.shape[0], k.shape[0]
    s_all = (q.double() @ k.double().T).float()
    if mut == "scale head_stride^-0.5":
        scale = hs ** -0.5
    sl2 = np.float32(scale * 1.4426950408889634)
    rows = torch.arange(Lq)[:, None]
    m = torch.full((Lq, 1), -float("inf"))
    l = torch.zeros(Lq, 1)
    o = torch.zeros(Lq, q.shape[1])
    nkt = -(-Lk // KB.ATT_BN)
    if causal:
        nkt = min(nkt, (Lq - 1 + Lk - Lq) // KB.ATT_BN + 1)
    for kt in range(nkt):
        key0 = kt * KB.ATT_BN
        keys = key0 + torch.arange(KB.ATT_BN)[None, :]
        lim = torch.full((Lq, 1), Lk)
        if mut == "last partial key tile dropped":
            lim = torch.full((Lq, 1), (Lk // KB.ATT_BN) * KB.ATT_BN)
        if causal:
            vis = rows + (Lk - Lq) + 1
            if mut == "causal mask admits key i + 1 for rows >= 128":
                vis = vis + (rows >= 128).long()
            lim = torch.minimum(lim, vis)
        ok = keys < lim
        if causal and mut == "diagonal key excluded for rows >= 64":
            ok &= ~((keys == rows + (Lk - Lq)) & (rows >= 64))
        if mut == "rows 64-127 of a tile skip the first key tile" and kt == 0:
            ok &= ~((rows % 128) >= 64)
        s = torch.zeros(Lq, KB.ATT_BN)
        s[:, :min(KB.ATT_BN, Lk - key0)] = s_all[:, key0:key0 + KB.ATT_BN]
        mt = torch.where(ok, s, torch.tensor(-float("inf"))).amax(1, keepdim=True)
        mn = torch.maximum(m, mt)
        mu = torch.where(mn == -float("inf"), torch.zeros_like(mn), mn)
        alpha = torch.exp2((m - mu) * sl2)
        m = mn
        p = torch.where(ok, torch.exp2((s - mu) * sl2), torch.zeros_like(s))
        l = l * alpha + p.sum(1, keepdim=True)
        al = alpha.expand(-1, o.shape[1]).clone()
        if mut == "O rescale missing on the 16-wide chunk":
            al[:, 64:] = 1.0
        vt = torch.zeros(KB.ATT_BN, v.shape[1])
        vt[:min(KB.ATT_BN, Lk - key0)] = v[key0:key0 + KB.ATT_BN].float()
        o = (o.double() * al.double() + p.bfloat16().double() @ vt.double()).float()
        if mut == "O accumulator rounded to bf16 between key tiles":
            o = o.bfloat16().float()
    return (o * (1.0 / l)).bfloat16()


def _attn_case(lens, nh, hd, hs, causal, seed, ramp=False, v_mean=0.0, mut=None):
    T = sum(lens)
    x = _randn(T, 3, nh, hd, seed=seed)
    if ramp:
        x[:, 1] *= torch.cat([torch.linspace(0.2, 6.0, n) for n in lens])[:, None, None]
    x[:, 2] += v_mean
    qkv = torch.zeros(T, 3, nh, hs)
    qkv[..., :hd] = x
    qkv = qkv.reshape(T, 3 * nh * hs).bfloat16()
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)
    args = dict(q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh, cu_k=cu, cu_q=cu,
                max_q=max(lens), causal=causal, scale=hd ** -0.5)
    ref, e = KB.attention_ref(qkv, qkv, qkv, **args)
    got = torch.zeros(T, nh * hd, dtype=torch.bfloat16)
    for b in range(len(lens)):
        r0, r1 = int(cu[b]), int(cu[b + 1])
        for h in range(nh):
            sl = lambda c0: qkv[r0:r1, c0 + h * hs:c0 + h * hs + hd]   # noqa: E731
            got[r0:r1, h * hd:(h + 1) * hd] = emu_attention_head(sl(0), sl(nh * hs), sl(2 * nh * hs), hd ** -0.5, causal,
                                                                  hs, mut)
    return got, ref, e


ATT_CASES = {   # name -> (lens, heads, head dim, head stride, causal, extra)
    "vit N=1036": ([1036], 2, 72, 80, False, {}),
    "vit growing max": ([1024], 2, 72, 80, False, {"ramp": True}),
    "vit positive-mean V": ([1024], 2, 72, 80, False, {"v_mean": 1.0}),
    "lm causal": ([300, 129], 2, 64, 64, True, {}),
}
ATT_MUTANTS = [
    ("causal mask admits key i + 1 for rows >= 128", "lm causal"),
    ("diagonal key excluded for rows >= 64", "lm causal"),
    ("scale head_stride^-0.5", "vit N=1036"),
    ("last partial key tile dropped", "vit N=1036"),
    ("rows 64-127 of a tile skip the first key tile", "vit N=1036"),
    ("O rescale missing on the 16-wide chunk", "vit growing max"),
    ("O accumulator rounded to bf16 between key tiles", "vit positive-mean V"),
]


def _att(case, mut=None):
    lens, nh, hd, hs, causal, extra = ATT_CASES[case]
    return _attn_case(lens, nh, hd, hs, causal, seed=len(case), mut=mut, **extra)


@pytest.mark.parametrize("case", list(ATT_CASES))
def test_attention_faithful_emulation_passes(case):
    _check(case, *_att(case))


@pytest.mark.parametrize("mut,case", ATT_MUTANTS, ids=[m for m, _ in ATT_MUTANTS])
def test_attention_mutant_fails(mut, case):
    got, ref, e = _att(case, mut)
    _fails(lambda: _check(f"{case} / {mut}", got, ref, e))


# ---------------------------------------------------------------------------------------------------------------- norms


def emu_norm(x, g, b, eps, mut=None):
    mean = x.sum(1, keepdim=True) / x.shape[1]
    if mut == "one-pass variance":
        var = (x * x).sum(1, keepdim=True) / x.shape[1] - mean * mean
    else:
        var = ((x - mean) ** 2).sum(1, keepdim=True) / x.shape[1]
    r = 1.0 / (var.clamp_min(0).sqrt() + eps) if mut == "eps outside the square root" else torch.rsqrt(var + eps)
    gg = torch.roll(g, 4) if mut == "gamma read 4 columns off" else g
    y = (x - mean) * r * gg
    if mut != "beta omitted":
        y = y + b
    return y.bfloat16()


def _norm_data(D):
    x = _randn(64, D, scale=3.0, mean=1.0, seed=D)
    x[1:9] = _randn(8, D, seed=D + 1) + 1e3          # |mean| >> std
    x[9] = 0.75                                       # constant rows: the output is beta
    x[10] = -2.5
    x[11:19] = _randn(8, D, scale=1e-3, seed=D + 2)   # variance ~ eps
    return x, _randn(D, seed=D + 3), _randn(D, seed=D + 4)


NORM_MUTANTS = ["one-pass variance", "eps outside the square root", "beta omitted", "gamma read 4 columns off"]


@pytest.mark.parametrize("D", [288, 1152, 2304])
@pytest.mark.parametrize("mut", [None] + NORM_MUTANTS)
def test_layernorm(D, mut):
    x, g, b = _norm_data(D)
    ref, e = KB.layernorm_ref(x, g, b, 1e-6)
    run = lambda: _check(f"layernorm D={D} {mut}", emu_norm(x, g, b, 1e-6, mut), ref, e)   # noqa: E731
    run() if mut is None else _fails(run)


def test_rmsnorm_and_build_lm_input_faithful():
    x, g, _ = _norm_data(2304)
    y = (x * torch.rsqrt((x * x).sum(1, keepdim=True) / 2304 + 1e-5) * g).bfloat16()
    _check("rmsnorm", y, *KB.rmsnorm_ref(x, g, 1e-5))
    _fails(lambda: _check("rmsnorm, mean subtracted", emu_norm(x, g, torch.zeros(2304), 1e-5), *KB.rmsnorm_ref(x, g, 1e-5)))
    emb = _randn(50, 256, seed=30).bfloat16()
    vis = _randn(7, 256, seed=31)
    src = torch.tensor([-1, 0, 6, -50, 3], dtype=torch.int32)
    h = torch.stack([emb[0].float() * 12, vis[0], vis[6], emb[49].float() * 12, vis[3]])
    _check("build_lm_input", h, *KB.build_lm_input_ref(src, emb, 12.0, vis))


def test_bf16_cell_is_the_rounding_interval():
    """`check`'s bf16 rule: a value rounds to g exactly when it lies in bf16_cell(g) (ties aside)."""
    g = torch.tensor([1.0, 1.0078125, -1.0, 0.99609375, 3.0e-3, -7.5, 2.0 ** -100], dtype=torch.bfloat16)
    lo, hi = KB.bf16_cell(g)
    eps = g.double().abs() * 2.0 ** -20          # above fp32 resolution: the nudged values are exact in fp32
    assert torch.equal((lo + eps).float().bfloat16(), g) and torch.equal((hi - eps).float().bfloat16(), g)
    assert ((lo - eps).float().bfloat16() != g).all() and ((hi + eps).float().bfloat16() != g).all()


# ---------------------------------------------------------------------------------------------------------- pool_norm


def _butterfly(v):
    """warp_sum over the last axis (32 lanes): xor-shuffle tree, fp32."""
    lanes = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ off]).astype(np.float32)
    return v[..., 0]


def _sum_sq_f32(x, per_lane):
    """Sum of squares of the rows of x [m, D] as the kernel's lanes take it: float4 f = lane + 32 * per_lane_index
    (pool rows: 32 lanes; the final norm: 128 threads = 4 warps), each float4 as (x^2 + y^2) + (z^2 + w^2), serially."""
    m, D = x.shape
    threads = 32 * per_lane
    steps = -(-D // (4 * threads))
    xp = np.zeros((m, steps * threads * 4), np.float32)
    xp[:, :D] = x
    q = (xp * xp).reshape(m, steps, threads, 4)
    grp = ((q[..., 0] + q[..., 1]).astype(np.float32) + (q[..., 2] + q[..., 3]).astype(np.float32)).astype(np.float32)
    acc = np.zeros((m, threads), np.float32)
    for i in range(steps):
        acc = (acc + grp[:, i]).astype(np.float32)
    return acc.reshape(m, per_lane, 32)


def emu_pool_norm(h, gamma, eps, cu, pooling, normalize, mut=None):
    """pool_norm_kernel in fp32, in its order: 8 virtual ranks of 4 warps, warp slot 4v + w takes rows t_lo + 4v + w + 32k."""
    h, g = h.numpy().astype(np.float32), gamma.numpy().astype(np.float32)
    D = g.size
    eps32 = np.float32(eps)
    out = np.zeros((len(cu) - 1, D), np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):     # the mutants' 1/0 and 0/0 become inf / NaN, as on the GPU
        for b in range(len(cu) - 1):
            out[b] = _emu_pool_seq(h, g, eps32, int(cu[b]), int(cu[b + 1]), pooling, normalize, mut)
    return torch.from_numpy(out)


def _emu_pool_seq(h, g, eps32, r0, r1, pooling, normalize, mut):
    D = g.size
    n = r1 - r0
    if n <= 0:
        return np.zeros(D, np.float32)
    t_lo, t_hi = {"lasttoken": (n - 1, n), "cls": (0, 1)}.get(pooling, (0, n))
    if mut == "lasttoken reads row len - 2" and pooling == "lasttoken":
        t_lo, t_hi = n - 2, n - 1
    X = h[r0 + t_lo:r0 + t_hi, :D]
    m = X.shape[0]
    ss = _butterfly(_sum_sq_f32(X, 1)[:, 0])
    ms = (ss / np.float32(D)).astype(np.float32)
    if mut != "eps omitted":
        ms = (ms + eps32).astype(np.float32)
    r = (1.0 / np.sqrt(ms.astype(np.float64))).astype(np.float32)
    t = np.arange(t_lo, t_hi)
    w = (t + (0 if mut == "weights t instead of t + 1" else 1)).astype(np.float32) if pooling == "wmean" else np.ones(m, np.float32)
    sc = (w * r).astype(np.float32)
    Y = np.zeros((-(-m // 32) * 32, D), np.float32)
    Y[:m] = (sc[:, None] * X).astype(np.float32)
    acc = np.zeros((32, D), np.float32)
    for k in range(Y.shape[0] // 32):
        acc = (acc + Y[32 * k:32 * k + 32]).astype(np.float32)
        if mut == "accumulator rounded to bf16":
            acc = torch.from_numpy(acc).bfloat16().float().numpy()
    total = np.zeros(D, np.float32)
    for v in range(KB.POOL_VRANKS):
        part = acc[4 * v]
        for wv in range(1, 4):
            part = (part + acc[4 * v + wv]).astype(np.float32)
        if not (mut == "one virtual rank's partial dropped" and v == KB.POOL_VRANKS - 1):
            total = (total + part).astype(np.float32)
    nf = np.float32(m)
    W = (np.float32(0.5) * nf * (nf + np.float32(1))).astype(np.float32) if pooling == "wmean" else nf
    if mut == "sum of weights off by one":
        W = np.float32(W + 1)
    p = ((total * g).astype(np.float32) / W).astype(np.float32)
    inv = np.float32(1)
    if normalize:
        warps = _butterfly(_sum_sq_f32(p[None], 4)[0])
        sq = np.float32(0)
        for s in warps:
            sq = np.float32(sq + s)
        nrm = np.float32(np.sqrt(sq))
        inv = np.float32(1) / (nrm if mut == "norm guard removed" else max(nrm, np.float32(1e-12)))
    return (p * inv).astype(np.float32)


POOL_EPS = 1e-5
POOL_LENS = [0, 1, 2, 17, 33, 300, 40]


def _pool_data(D):
    """Rows of the LM's last residual stream: O(1) rows, rows with mean square ~ eps next to them (so a missing or doubled
    eps changes their weight against the others; a uniform scale error would cancel in the L2 normalisation), |h| ~ 1e3
    rows, and one all-zero sequence (the last)."""
    T = sum(POOL_LENS)
    x = _randn(T, D, seed=D)
    x[1::3] *= POOL_EPS ** 0.5
    x[2::7] = _randn(len(range(2, T, 7)), D, scale=1e3, seed=D + 1)
    x[T - POOL_LENS[-1]:] = 0.0
    cu = torch.tensor([0] + list(np.cumsum(POOL_LENS)), dtype=torch.int32)
    return x, _randn(D, seed=D + 2), cu


POOL_MUTANTS = [
    ("eps omitted", "wmean", True),
    ("weights t instead of t + 1", "wmean", True),
    ("sum of weights off by one", "mean", False),
    ("lasttoken reads row len - 2", "lasttoken", True),
    ("one virtual rank's partial dropped", "mean", True),
    ("accumulator rounded to bf16", "wmean", True),
    ("norm guard removed", "wmean", True),
]


@pytest.mark.parametrize("D", [64, 576, 2304])
@pytest.mark.parametrize("normalize", [True, False], ids=["l2", "raw"])
@pytest.mark.parametrize("pooling", ["wmean", "mean", "lasttoken", "cls"])
def test_pool_norm_faithful_emulation_passes(pooling, normalize, D):
    x, g, cu = _pool_data(D)
    _check(f"pool_norm {pooling} {normalize} D={D}", emu_pool_norm(x, g, POOL_EPS, cu, pooling, normalize),
           *KB.pool_norm_ref(x, g, POOL_EPS, cu, pooling, normalize))


@pytest.mark.parametrize("D", [64, 2304])
@pytest.mark.parametrize("mut,pooling,normalize", POOL_MUTANTS, ids=[m for m, _, _ in POOL_MUTANTS])
def test_pool_norm_mutant_fails(mut, pooling, normalize, D):
    x, g, cu = _pool_data(D)
    got = emu_pool_norm(x, g, POOL_EPS, cu, pooling, normalize, mut)
    ref, e = KB.pool_norm_ref(x, g, POOL_EPS, cu, pooling, normalize)
    fin = torch.isfinite(got).all(1)
    need = (got.double() - ref)[fin].abs()
    frac = float(torch.where(need == 0, torch.zeros_like(need), need / e[fin].clamp_min(1e-300)).max())
    print(f"pool_norm mutant '{mut}' D={D}: {frac:.3g} x the bound on finite rows, {int((~fin).sum())} non-finite rows")
    _fails(lambda: _check(f"pool_norm {mut}", got, ref, e))
