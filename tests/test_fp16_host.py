"""fp16 engines without a GPU: the fp16 error bounds of tests/kernel_bounds_f16.py have power, the pixel normalisation carries
over to fp16 bit for bit, `dtype="float16"` reaches the engine through the drop-in classes, and the C ABI refuses type
mix-ups before any CUDA call.

The emulations follow the kernels as tests/test_kernel_bounds_host.py does (fp32 accumulation of exact 16-bit products in
k16 steps, truncated; the fp32 epilogue in the kernel's order; attention over 128-key tiles with a running maximum), with
fp16 where the bf16 engine stores bf16: the operands, P (round to nearest, no flush: subnormal p survive) and the output.
Each mutant is a plausible way to get fp16 wrong; every one must fail its check, and the test prints by how much."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF
from tests.test_kernel_bounds_host import emu_acc, gelu_f32
from visrag_b200 import _lib as L


def _randn(*shape, scale=1.0, mean=0.0, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float32) * scale + mean


def _passes(name, got, ref, e, **kw):
    return KF.check(name, got, ref, e, verbose=False, **kw)


def _rejects(name, got, ref, e, **kw):
    """The check must fail; prints the failure (the worst element's error as a multiple of its bound)."""
    with pytest.raises(AssertionError) as ei:
        KF.check(name, got, ref, e, verbose=False, **kw)
    print(f"rejected: {str(ei.value).splitlines()[0]}")


def test_f16_cell_is_the_rounding_interval():
    """`check`'s fp16 rule: a value rounds to g exactly when it lies in f16_cell(g), for normal values, powers of two,
    the smallest normal (2^-14), subnormals, zero and the largest finite value."""
    g = torch.tensor([1.0, 1.0009765625, -1.0, 0.99951171875, 3.0e-3, -7.5, 2.0 ** -14, 3 * 2.0 ** -24, 2.0 ** -24,
                      -5 * 2.0 ** -24, 65504.0, 0.0], dtype=torch.float16)
    lo, hi = KF.f16_cell(g)
    eps = torch.maximum(g.double().abs(), torch.full_like(lo, 2.0 ** -24)) * 2.0 ** -16
    assert torch.equal((lo + eps).half(), g) and torch.equal((hi - eps).half(), g)
    outside_lo, outside_hi = (lo - eps).half(), (hi + eps).half()
    assert (outside_lo != g).all() and (outside_hi != g).all()


# ---------------------------------------------------------------------------------------------------------------- GEMM

M, N, K = 777, 1152, 640
A = _randn(M, K, scale=0.5, seed=1).half()
W = _randn(N, K, scale=0.05, seed=2).half()
BIAS = _randn(N, seed=3)
RESID = _randn(M, N, seed=4)
ROWADD = _randn(37, N, seed=5)

CONFIGS = {   # name -> (epilogue arguments, output dtype)
    "bias scale resid f32": (dict(bias=BIAS, scale=0.25, resid=RESID), torch.float32),
    "bias rowadd f32": (dict(bias=BIAS, rowadd=ROWADD), torch.float32),
    "bias f16": (dict(bias=BIAS), torch.float16),
    "bias gelu f16": (dict(bias=BIAS, gelu=True), torch.float16),
    "bias gelu scale rowadd f16": (dict(bias=BIAS, gelu=True, scale=-0.5, rowadd=ROWADD), torch.float16),
}

GEMM_MUTANTS = [
    ("output rounded to bf16 instead of fp16", "bias f16"),
    ("output rounded to bf16 instead of fp16", "bias gelu f16"),
    ("operands rounded through bf16", "bias scale resid f32"),
    ("bias rounded to fp16", "bias scale resid f32"),
]


def emu_linear16(a, w, *, bias=None, gelu=False, scale=1.0, rowadd=None, resid=None, out_dtype=torch.float32, mut=None):
    """The LINEAR epilogue with fp16 operands, in the kernel's order; `mut` names one mutant."""
    if mut == "operands rounded through bf16":
        a, w = a.bfloat16(), w.bfloat16()
    x = emu_acc(a, w)
    if bias is not None:
        x = x + (bias.half().float() if mut == "bias rounded to fp16" else bias)
    if gelu:
        x = gelu_f32(x)
    x = x * scale
    if rowadd is not None:
        x = x + rowadd[torch.arange(x.shape[0]) % rowadd.shape[0]]
    if resid is not None:
        x = x + resid
    if mut == "output rounded to bf16 instead of fp16":
        return x.bfloat16().to(out_dtype)
    return x.to(out_dtype)


def _gemm_case(config, mut=None):
    kw, dt = CONFIGS[config]
    got = emu_linear16(A, W, out_dtype=dt, mut=mut, **kw)
    ref, e = KB.gemm_linear_ref(A, W, **kw)
    rms = KB.gemm_rms_rel(K) if dt == torch.float32 and not kw.get("gelu") else None
    return got, ref, e, rms


@pytest.mark.parametrize("config", list(CONFIGS))
def test_gemm_f16_faithful_emulation_passes(config):
    got, ref, e, rms = _gemm_case(config)
    assert got.dtype in (torch.float16, torch.float32)
    _passes(config, got, ref, e, rms_rel=rms)


@pytest.mark.parametrize("mut,config", GEMM_MUTANTS, ids=[f"{m} / {c}" for m, c in GEMM_MUTANTS])
def test_gemm_f16_mutant_fails(mut, config):
    got, ref, e, rms = _gemm_case(config, mut)
    _rejects(f"{config} / {mut}", got, ref, e, rms_rel=rms)


T, H = 64, 256
AR = _randn(T, H, scale=0.5, seed=20).half()
WR = _randn(3 * H, H, scale=0.05, seed=21).half()
WS = _randn(2 * 512, H, scale=0.05, seed=23).half()
POS = torch.randint(0, 2048, (T,), generator=torch.Generator().manual_seed(22), dtype=torch.int32)
_inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
_fr = torch.outer(torch.arange(2049).float(), _inv)
COS, SIN = _fr.cos().contiguous(), _fr.sin().contiguous()


@pytest.mark.parametrize("mut", [None, "output rounded to bf16 instead of fp16"])
def test_rope_and_swiglu_f16(mut):
    out = (lambda t: t.bfloat16().half()) if mut else (lambda t: t.half())
    x = emu_acc(AR, WR).view(T, 3 * H // 64, 2, 32)
    c, s = COS[POS.long()][:, None, :], SIN[POS.long()][:, None, :]
    lo, hi = x[:, :, 0], x[:, :, 1]
    rope = out(torch.stack([lo * c - hi * s, hi * c + lo * s], 2).reshape(T, 3 * H))   # rope_cols = 3H: every head
    xs = emu_acc(AR, WS).view(T, -1, 2, 32)
    swiglu = out((torch.nn.functional.silu(xs[:, :, 0]) * xs[:, :, 1]).reshape(T, -1))
    checks = [("rope f16", rope, *KB.gemm_rope_ref(AR, WR, POS, COS, SIN, 3 * H)), ("swiglu f16", swiglu, *KB.gemm_swiglu_ref(AR, WS))]
    for name, got, ref, e in checks:
        (_passes if mut is None else _rejects)(f"{name} {mut}", got, ref, e)


# ------------------------------------------------------------------------------------------------------------ attention


def emu_attention_f16(q, k, v, scale, causal, mut=None):
    """attention.cuh with F16 for one head and sequence: q [Lq, hd], k / v [Lk, hd] fp16 -> fp16 [Lq, hd]."""
    Lq, Lk = q.shape[0], k.shape[0]
    s_all = (q.double() @ k.double().T).float()
    sl2 = np.float32(scale * 1.4426950408889634)
    rows = torch.arange(Lq)[:, None]
    m = torch.full((Lq, 1), -float("inf"))
    l = torch.zeros(Lq, 1)
    o = torch.zeros(Lq, q.shape[1])
    nkt = -(-Lk // KB.ATT_BN)
    for kt in range(nkt):
        key0 = kt * KB.ATT_BN
        keys = key0 + torch.arange(KB.ATT_BN)[None, :]
        lim = torch.full((Lq, 1), Lk)
        if causal:
            lim = torch.minimum(lim, rows + (Lk - Lq) + 1)
        ok = keys < lim
        s = torch.zeros(Lq, KB.ATT_BN)
        s[:, :min(KB.ATT_BN, Lk - key0)] = s_all[:, key0:key0 + KB.ATT_BN]
        mt = torch.where(ok, s, torch.tensor(-float("inf"))).amax(1, keepdim=True)
        mn = torch.maximum(m, mt)
        mu = torch.where(mn == -float("inf"), torch.zeros_like(mn), mn)
        alpha = torch.exp2((m - mu) * sl2)
        m = mn
        p = torch.where(ok, torch.exp2((s - mu) * sl2), torch.zeros_like(s))
        l = l * alpha + p.sum(1, keepdim=True)
        if mut == "P rounded to bf16":
            p16 = p.bfloat16().double()
        elif mut == "P flushed to zero below 2^-14":
            p16 = torch.where(p < 2.0 ** -14, torch.zeros_like(p), p).half().double()
        else:
            p16 = p.half().double()          # round to nearest, subnormals kept
        vt = torch.zeros(KB.ATT_BN, v.shape[1])
        vt[:min(KB.ATT_BN, Lk - key0)] = v[key0:key0 + KB.ATT_BN].float()
        o = (o.double() * alpha.double() + p16 @ vt.double()).float()
    y = o * (1.0 / l)
    return y.bfloat16().half() if mut == "output rounded to bf16 instead of fp16" else y.half()


ATT_CASES = {   # name -> (lens, heads, head dim, head stride, causal, q/k scale, V mean)
    "vit N=1036": ([1036], 2, 72, 80, False, 1.0, 0.0),
    "lm causal (rows with 1 and 2 keys)": ([300, 129], 2, 64, 64, True, 1.0, 0.0),
    "resampler-like stride 128": ([200], 2, 128, 128, False, 1.0, 0.0),
    "small P (most p below 2^-14)": ([1036], 2, 64, 64, False, 2.0, 1.0),
}
ATT_MUTANTS = [
    ("P rounded to bf16", "lm causal (rows with 1 and 2 keys)"),
    ("P flushed to zero below 2^-14", "small P (most p below 2^-14)"),
    ("output rounded to bf16 instead of fp16", "vit N=1036"),
]


def _att(case, mut=None):
    lens, nh, hd, hs, causal, qk_scale, v_mean = ATT_CASES[case]
    Tn = sum(lens)
    x = _randn(Tn, 3, nh, hd, seed=len(case))
    x[:, :2] *= qk_scale
    x[:, 2] += v_mean
    qkv = torch.zeros(Tn, 3, nh, hs)
    qkv[..., :hd] = x
    qkv = qkv.reshape(Tn, 3 * nh * hs).half()
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)
    args = dict(q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh, cu_k=cu, cu_q=cu,
                max_q=max(lens), causal=causal, scale=hd ** -0.5)
    ref, e = KF.attention_ref_f16(qkv, qkv, qkv, **args)
    got = torch.zeros(Tn, nh * hd, dtype=torch.float16)
    small = 0.0
    for b in range(len(lens)):
        r0, r1 = int(cu[b]), int(cu[b + 1])
        for h in range(nh):
            sl = lambda c0: qkv[r0:r1, c0 + h * hs:c0 + h * hs + hd]   # noqa: E731
            got[r0:r1, h * hd:(h + 1) * hd] = emu_attention_f16(sl(0), sl(nh * hs), sl(2 * nh * hs), hd ** -0.5, causal, mut)
            if not causal:
                P = torch.softmax((sl(0).double() @ sl(nh * hs).double().T) * hd ** -0.5, -1)
                small = max(small, float((P < 2.0 ** -14).double().mean()))
    return got, ref, e, small


@pytest.mark.parametrize("case", list(ATT_CASES))
def test_attention_f16_faithful_emulation_passes(case):
    got, ref, e, small = _att(case)
    if case.startswith("small P"):
        assert small > 0.5, small          # the case exercises subnormal P
    _passes(case, got, ref, e)


@pytest.mark.parametrize("mut,case", ATT_MUTANTS, ids=[m for m, _ in ATT_MUTANTS])
def test_attention_f16_mutant_fails(mut, case):
    got, ref, e, _ = _att(case, mut)
    _rejects(f"{case} / {mut}", got, ref, e)


# ---------------------------------------------------------------------------------------------------------------- norms


def _norm_data(D):
    x = _randn(64, D, scale=3.0, mean=1.0, seed=D)
    x[1:9] = _randn(8, D, seed=D + 1) + 1e3          # |mean| >> std
    x[9] = 0.75                                       # constant rows: the output is beta
    x[11:19] = _randn(8, D, scale=1e-3, seed=D + 2)   # variance ~ eps
    return x, _randn(D, seed=D + 3), _randn(D, seed=D + 4)


@pytest.mark.parametrize("D", [288, 1152, 2304])
def test_norms_f16(D):
    x, g, b = _norm_data(D)
    mean = x.sum(1, keepdim=True) / D
    y = (x - mean) * torch.rsqrt(((x - mean) ** 2).sum(1, keepdim=True) / D + 1e-6) * g + b
    add = _randn(37, D, seed=D + 5)
    (r1, e1), (r2, e2) = KB.layernorm_ref(x, g, b, 1e-6, add=add)
    _passes(f"layernorm f16 D={D}", y.half(), r1, e1)
    _passes(f"layernorm+add f16 D={D}", (y + add[torch.arange(64) % 37]).half(), r2, e2)
    _rejects(f"layernorm D={D} / output rounded to bf16 instead of fp16", y.bfloat16().half(), r1, e1)
    r = x * torch.rsqrt((x * x).sum(1, keepdim=True) / D + 1e-5) * g
    _passes(f"rmsnorm f16 D={D}", r.half(), *KB.rmsnorm_ref(x, g, 1e-5))
    _rejects(f"rmsnorm D={D} / output rounded to bf16 instead of fp16", r.bfloat16().half(), *KB.rmsnorm_ref(x, g, 1e-5))


def test_build_lm_input_f16():
    emb = _randn(50, 256, seed=30).half()
    vis = _randn(7, 256, seed=31)
    src = torch.tensor([-1, 0, 6, -50, 3], dtype=torch.int32)
    h = torch.stack([emb[0].float() * 12, vis[0], vis[6], emb[49].float() * 12, vis[3]])
    _passes("build_lm_input f16", h, *KB.build_lm_input_ref(src, emb, 12.0, vis))
    _rejects("build_lm_input / table read through bf16", torch.stack([emb[0].bfloat16().float() * 12, vis[0], vis[6],
                                                                      emb[49].bfloat16().float() * 12, vis[3]]),
             *KB.build_lm_input_ref(src, emb, 12.0, vis))


# ------------------------------------------------------------------------------------------------------------- pixels


def test_pixel_normalisation_is_exact_in_fp16():
    """The im2col kernels compute fma(u, 2/255, -1) in fp32 and round it once to the 16-bit type. For every byte u this
    equals the reference's ToTensor + Normalize(0.5, 0.5) in fp32, ((u / 255) - 0.5) / 0.5, rounded to fp16 (and to
    bf16). The FMA is emulated in float64, where u * fp32(2/255) - 1 is exact (a multiple of 2^-30 below 2 in
    magnitude), so one rounding to fp32 gives the fused result."""
    u = np.arange(256, dtype=np.float32)
    c = np.float32(2.0 / 255.0)
    fused = (u.astype(np.float64) * np.float64(c) - 1.0).astype(np.float32)
    ref = ((u / np.float32(255.0)).astype(np.float32) - np.float32(0.5)).astype(np.float32) / np.float32(0.5)
    ref = ref.astype(np.float32)
    assert np.array_equal(fused.astype(np.float16).view(np.uint16), ref.astype(np.float16).view(np.uint16))
    assert torch.equal(torch.from_numpy(fused).bfloat16(), torch.from_numpy(ref).bfloat16())
    assert not np.array_equal(fused, ref)          # the fp32 values do differ: the identity is a property of the rounding


# --------------------------------------------------------------------------------------------- dtype through the classes


@pytest.fixture
def checkpoint_dir(tmp_path):
    d = tmp_path / "ckpt"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({}))
    torch.save({"w": torch.zeros(2)}, str(d / "pytorch_model.bin"))
    return str(d)


def _stub_backbone(calls):
    from visrag_b200 import modeling as M

    class StubBackbone(M.VisRAGRetB200):
        def __init__(self, *args, **kwargs):
            calls.append((args, kwargs))
            self.config = args[0]
            self.dtype = kwargs.get("dtype", torch.bfloat16)

    return StubBackbone


@pytest.mark.parametrize("dtype", [None, "bfloat16", "float32", "float16"])
def test_build_maps_dtype_to_the_engine(checkpoint_dir, monkeypatch, dtype):
    """DRModelForInference.build(model_args): "float16" constructs the backbone with dtype=torch.float16; "bfloat16",
    "float32" and no dtype attribute construct it exactly as before, with the three positional arguments (cfg, state_dict,
    device) - a subclass with that three-argument constructor keeps working."""
    from visrag_b200 import modeling as M

    calls = []
    monkeypatch.setattr(M, "VisRAGRetB200", _stub_backbone(calls))
    margs = SimpleNamespace(model_name_or_path=checkpoint_dir, pooling="wmean", normalize=True)
    if dtype is not None:
        margs.dtype = dtype
    model = M.DRModelForInference.build(margs)
    (args, kwargs), = calls
    assert len(args) == 3 and args[2] == "cuda:0"
    if dtype == "float16":
        assert kwargs == {"dtype": torch.float16} and model.lm_q.dtype == torch.float16
    else:
        assert kwargs == {}


@pytest.mark.parametrize("torch_dtype", [None, torch.bfloat16, torch.float32, torch.float16])
def test_from_pretrained_maps_torch_dtype(checkpoint_dir, torch_dtype):
    from visrag_b200 import modeling as M

    calls = []

    class ThreeArgs(M.VisRAGRetB200):        # the constructor the reference-driver test's subclass has
        def __init__(self, cfg, state_dict, device="cuda:0"):
            calls.append((cfg, state_dict, device))

    if torch_dtype is torch.float16:
        calls16 = []
        M_ = _stub_backbone(calls16)
        M_.from_pretrained(checkpoint_dir, torch_dtype=torch_dtype)
        assert calls16[0][1] == {"dtype": torch.float16}
    else:
        ThreeArgs.from_pretrained(checkpoint_dir, torch_dtype=torch_dtype)
        assert len(calls) == 1 and calls[0][2] == "cuda:0"


# --------------------------------------------------------------------------------------------------------------- ABI

NEW_SYMBOLS = ("vr_im2col_norm_ex", "vr_layernorm_ex", "vr_rmsnorm_ex", "vr_build_lm_input_ex")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


def test_fp16_entry_points_are_exported(lib):
    syms = G.exported_symbols()
    for s in NEW_SYMBOLS:
        assert s in syms and getattr(lib, s) is not None
    assert lib.vr_abi_version() == 2 and L.VR_ATTN_F16 == 2


def _gemm_rc(lib, ab_dtype, out_dtype, mode=L.VR_EPI_LINEAR, gelu=0, block_n=0):
    e = L.GemmEpilogue()
    e.mode, e.out_dtype, e.act_gelu, e.scale = mode, out_dtype, gelu, 1.0
    e.positions = e.rope_cos = e.rope_sin = 16
    e.out, e.ldo = 16, 128
    rc = lib.vr_gemm_tuned(16, 64, 16, 64, ab_dtype, 256, 128, 64, C.byref(e), block_n, None)
    return rc, lib.vr_last_error().decode()


@pytest.mark.parametrize("block_n", [0, 2, 3, 4, 5, 64, 128, 192, 256])
def test_gemm_type_validation_runs_before_any_cuda_call(lib, block_n):
    """Pointers here are not device memory: these calls must be refused by argument validation alone."""
    rc, msg = _gemm_rc(lib, L.VR_BF16, L.VR_F16, block_n=block_n)        # fp16 output from bf16 operands
    assert rc == 2 and "out_dtype must be VR_BF16 or VR_F32" in msg, msg
    rc, msg = _gemm_rc(lib, L.VR_F16, L.VR_BF16, block_n=block_n)        # bf16 output from fp16 operands
    assert rc == 2 and "fp16 operands out_dtype must be VR_F16 or VR_F32" in msg, msg
    rc, msg = _gemm_rc(lib, L.VR_F16, L.VR_F32, gelu=1, block_n=block_n)
    assert rc == 2 and "GELU epilogue writes fp16 only" in msg, msg
    rc, msg = _gemm_rc(lib, L.VR_F32, L.VR_F32, block_n=block_n)
    assert rc == 2 and "operands must be bf16 or fp16" in msg, msg
    if block_n != 3:
        rc, msg = _gemm_rc(lib, L.VR_F16, L.VR_BF16, mode=L.VR_EPI_ROPE, block_n=block_n)
        assert rc == 2 and "ROPE / SWIGLU write fp16" in msg, msg


def test_elementwise_type_validation(lib):
    assert lib.vr_layernorm_ex(16, 64, 16, 16, 1e-6, 4, 64, 16, 64, None, None, 0, L.VR_F32, None) == 2
    assert b"out_dtype must be VR_BF16 or VR_F16" in lib.vr_last_error()
    assert lib.vr_rmsnorm_ex(16, 64, 16, 1e-6, 4, 64, 16, 64, L.VR_F32, None) == 2
    assert b"out_dtype must be VR_BF16 or VR_F16" in lib.vr_last_error()
    assert lib.vr_im2col_norm_ex(16, 1, 14, 14, 14, 16, 640, L.VR_F32, None) == 2
    assert b"out_dtype must be VR_BF16 or VR_F16" in lib.vr_last_error()
    assert lib.vr_build_lm_input_ex(16, 4, 64, 16, L.VR_F32, 1.0, None, 0, 16, 64, None) == 2
    assert b"embed_dtype must be VR_BF16 or VR_F16" in lib.vr_last_error()


def test_mixed_operands_are_refused_before_any_device_access():
    """bf16 with fp16 in one call is refused by the op wrappers from the dtypes alone (CPU tensors: nothing else runs)."""
    from visrag_b200 import ops

    a16, b16 = torch.zeros(128, 64, dtype=torch.float16), torch.zeros(64, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="do not mix"):
        ops.gemm(a16, b16)
    with pytest.raises(ValueError, match="do not mix"):
        ops.gemm(b16, a16[:64])
    q = torch.zeros(128, 192, dtype=torch.float16)
    with pytest.raises(ValueError, match="do not mix"):
        ops.attention(q, q, q.bfloat16(), q_col0=0, k_col0=64, v_col0=128, head_stride=64, head_dim=64, heads=1, batch=1,
                      cu_k=torch.tensor([0, 128], dtype=torch.int32), max_k=128, cu_q=None, max_q=128, causal=False,
                      scale=0.125, out=torch.zeros(128, 64, dtype=torch.float16))
    with pytest.raises(ValueError, match="bf16 or fp16"):
        ops.gemm(a16.float(), a16.float())
