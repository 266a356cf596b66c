"""The IEEE-aware checker of tests/nonfinite_bounds.py has teeth: on the CPU, faithful emulations of an fp16 store that
overflows to inf, of NaN and inf flowing through a norm row, and of tiled attention over packed sequences that keeps
each sequence to its own keys pass it, and each mutant fails it with a printed reason: a saturating store, a variance
clamped with fmaxf, a NaN where the reference is finite, an inf of the wrong sign, and attention whose last partial key
tile lets p = 0 multiply the next sequence's V rows."""
import numpy as np
import pytest
import torch

from tests import nonfinite_bounds as NF

INF, NAN = float("inf"), float("nan")


def _randn(*shape, scale=1.0, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


def _rejects(fn):
    with pytest.raises(AssertionError) as ei:
        fn()
    print("rejected:", ei.value)


def _check(name, got, ref, e):
    return NF.check(name, got, ref, e, verbose=False)


# ------------------------------------------------------------------------------------------------------- fp16 stores

# references around the overflow threshold 65520 with a bound of 8 (so [ref - 8, ref + 8] straddles it for the middle
# ones), the fp16 subnormals, and infinities and NaN passed through
STORE_REF = torch.tensor([65000.0, 65487.0, 65504.0, 65511.0, 65515.0, 65519.0, 65520.0, 65525.0, 65530.0, 70000.0, 1e30,
                          -65515.0, -65525.0, -1e9, 3e-6, -1e-7, 2.0 ** -24, 6e-8, 1.0, INF, -INF, NAN],
                         dtype=torch.float64)
STORE_E = torch.full_like(STORE_REF, 8.0)
STORE_E[14:18] = 2.0 ** -30


def _store(y, mut=None):
    """An fp32 value y stored as fp16: round to nearest, inf past 65520 (cvt.rn.f16.f32). `sat`: cvt.rn.satfinite,
    which clamps to +-65504; `ftz`: subnormals flushed to zero."""
    y = y.float()
    if mut == "sat":
        y = torch.where(torch.isnan(y), y, y.clamp(-NF.F16_MAX, NF.F16_MAX))
    out = y.half()
    if mut == "ftz":
        out = torch.where(out.abs() < 2.0 ** -14, torch.zeros_like(out), out)
    return out


@pytest.mark.parametrize("shift", [-1.0, 0.0, 1.0])
def test_fp16_store_with_overflow_to_inf_passes(shift):
    """y = ref + a shift within the bound, stored as fp16: every value, inf included, passes."""
    y = STORE_REF + shift * torch.where(STORE_REF.abs() > 1.0, STORE_E, torch.zeros_like(STORE_E))
    out = _check("fp16 store", _store(y), STORE_REF, STORE_E)
    assert out["nan"] == 1 and out["inf"] == 2


def test_inf_output_needs_the_reference_to_reach_the_threshold():
    """inf passes exactly when ref + bound reaches 65520; 65504 only when ref - bound < 65520."""
    e = torch.tensor([8.0])
    for ref, got, ok in [(65512.0, INF, True), (65511.9, INF, False), (65527.9, 65504.0, True), (65528.5, 65504.0, False),
                         (-65512.0, -INF, True), (-65511.0, -INF, False)]:
        fn = lambda: _check("threshold", torch.tensor([got]).half(), torch.tensor([ref], dtype=torch.float64), e)
        if ok:
            fn()
        else:
            _rejects(fn)


@pytest.mark.parametrize("mut", ["sat", "ftz"])
def test_fp16_store_mutant_fails(mut):
    fin = torch.isfinite(STORE_REF)       # finite references only: the cells alone must reject the mutant
    _rejects(lambda: _check(f"fp16 store {mut}", _store(STORE_REF[fin], mut), STORE_REF[fin], STORE_E[fin]))


def test_nan_where_the_reference_is_finite_fails():
    got = _store(STORE_REF)
    got[0] = NAN
    _rejects(lambda: _check("nan for finite", got, STORE_REF, STORE_E))


def test_inf_of_the_wrong_sign_fails():
    got = _store(STORE_REF)
    got[20] = INF                 # the reference is -inf
    _rejects(lambda: _check("wrong-signed inf", got, STORE_REF, STORE_E))
    got = _store(STORE_REF)
    got[19] = NAN                 # NaN for +inf
    _rejects(lambda: _check("nan for inf", got, STORE_REF, STORE_E))


def test_fp32_output_rule():
    ref = torch.tensor([1.0, INF, -INF, NAN], dtype=torch.float64)
    e = torch.full_like(ref, 1e-6)
    _check("fp32", torch.tensor([1.0, INF, -INF, NAN]), ref, e)
    _rejects(lambda: _check("fp32 nan", torch.tensor([1.0, INF, -INF, 0.0]), ref, e))
    _rejects(lambda: _check("fp32 inf", torch.tensor([INF, INF, -INF, NAN]), ref, e))


# ------------------------------------------------------------------------------------------------------------- norms


def emu_norm(x, g, b, eps, rms, out_dtype=torch.float16, mut=None):
    """elementwise.cu's two-pass norm in fp32: mean, then the mean square of x - mean, rsqrt(var + eps). `clamp`:
    var = fmaxf(var, 0), which returns 0 for a NaN variance (fmaxf drops a NaN operand)."""
    X = x.float().numpy()
    m = np.zeros((X.shape[0], 1), np.float32) if rms else X.mean(1, keepdims=True, dtype=np.float32)
    d = (X - m).astype(np.float32)
    var = (d * d).mean(1, keepdims=True, dtype=np.float32)
    if mut == "clamp":
        var = np.fmax(var, np.float32(0))
    r = (1.0 / np.sqrt(var + np.float32(eps))).astype(np.float32)
    y = d * r * g.float().numpy()
    if b is not None:
        y = y + b.float().numpy()
    return torch.from_numpy(y.astype(np.float32)).to(out_dtype)


def _norm_rows(D):
    x = _randn(6, D, seed=D).float()
    x[1, 7] = NAN
    x[2, 0] = INF
    x[3, 5] = -INF
    x[4] *= 1e3                   # with gamma below: outputs past 65504 -> inf in fp16
    return x


@pytest.mark.parametrize("rms", [False, True], ids=["layernorm", "rmsnorm"])
def test_norm_nan_propagation_faithful_passes(rms):
    D = 256
    x = _norm_rows(D)
    g = (_randn(D, seed=1).abs() * 2e4 + 1.0).float()
    b = None if rms else _randn(D, seed=2).float()
    ref, e = NF.norm_ref(x, g, b, 1e-6, rms)
    got = emu_norm(x, g, b, 1e-6, rms)
    out = _check("norm", got, ref, e)
    assert out["nan"] >= 1 and out["inf"] == 0 and torch.isinf(got.float()).any()   # fp16 overflow of finite refs
    assert torch.isnan(got[1]).all()


@pytest.mark.parametrize("rms", [False, True], ids=["layernorm", "rmsnorm"])
def test_norm_variance_clamp_mutant_fails(rms):
    D = 256
    x = _norm_rows(D)
    g = _randn(D, seed=1).float()
    b = None if rms else _randn(D, seed=2).float()
    ref, e = NF.norm_ref(x, g, b, 1e-6, rms)
    _rejects(lambda: _check("norm var clamp", emu_norm(x, g, b, 1e-6, rms, mut="clamp"), ref, e))


# --------------------------------------------------------------------------------------------------------- attention


def emu_packed_attention(q, k, v, cu, scale, zero_tail):
    """attention.cuh's walk over one packed buffer in fp32: each sequence reads 128-key tiles starting at its first row,
    so its last partial tile holds rows of the next sequence (rows past the buffer read as zero, as TMA does). Scores of
    keys past the sequence are -inf (p = 0); P V multiplies every p by its tile row, so 0 * NaN is NaN unless those V
    rows are zeroed first (`zero_tail`, the fixed kernel). Non-causal, one head. Returns float32 [T, d]."""
    q, k, v = q.float(), k.float(), v.float()
    T, d = q.shape
    kpad = torch.cat([k, torch.zeros(128, d)])
    vpad = torch.cat([v, torch.zeros(128, d)])
    out = torch.zeros(T, d)
    for b in range(len(cu) - 1):
        k0, n = cu[b], cu[b + 1] - cu[b]
        Q = q[k0:k0 + n]
        m = torch.full((n, 1), -INF)
        l = torch.zeros(n, 1)
        o = torch.zeros(n, d)
        for key0 in range(0, n, 128):
            K = kpad[k0 + key0:k0 + key0 + 128]
            V = vpad[k0 + key0:k0 + key0 + 128].clone()
            s = Q @ K.T * scale
            inside = torch.arange(128) < n - key0
            s = torch.where(inside[None, :], s, torch.full_like(s, -INF))
            if zero_tail:
                V[~inside] = 0.0
            mt = torch.maximum(m, s.amax(1, keepdim=True))
            alpha = torch.exp(m - mt)
            p = torch.exp(s - mt)
            l = l * alpha + p.sum(1, keepdim=True)
            o = o * alpha + (p[:, :, None] * V[None, :, :]).sum(1)     # every product formed, as the MMA does
            m = mt
        out[k0:k0 + n] = o / l
    return out


@pytest.mark.parametrize("zero_tail", [False, True], ids=["p0_times_next_v", "zeroed_tail"])
def test_packed_attention_isolation(zero_tail):
    """Sequences A (130 keys: its second tile holds 2 of its keys and 126 of B's) and B, NaN in B's first V row: A must
    match its float64 reference and equal A run alone; today's p = 0 times B's V makes A NaN."""
    lens, d = [130, 200], 64
    cu = [0, 130, 330]
    q, k, v = (_randn(330, d, seed=s).float().bfloat16() for s in (1, 2, 3))
    v[130, 0] = NAN
    scale = d ** -0.5
    got = emu_packed_attention(q, k, v, cu, scale, zero_tail).bfloat16()
    alone = emu_packed_attention(q[:130], k[:130], v[:130], [0, 130], scale, zero_tail).bfloat16()
    ref, e = NF.attention_head_ref(q[:130], k[:130], v[:130], scale, False, 64, f16=False)
    refb, eb = NF.attention_head_ref(q[130:], k[130:], v[130:], scale, False, 64, f16=False)

    def isolated():
        _check("sequence A", got[:130], ref, e)
        assert torch.equal(got[:130], alone), "sequence A differs from A alone"
        _check("sequence B", got[130:], refb, eb)

    if zero_tail:
        isolated()
        assert torch.isnan(got[130:, 0]).all() and torch.isfinite(got[130:, 1:]).all()
    else:
        _rejects(isolated)


def test_attention_ref_ieee_rules():
    """A -inf score drops its key (finite v), +inf or NaN in a key's score makes the row NaN, an inf v at a visible key
    makes its column inf, and in a causal row that cannot see it, p = 0 times inf is NaN, as a masked softmax followed by a
    matmul gives."""
    d = 8
    q, k, v = (_randn(4, d, seed=s) for s in (4, 5, 6))
    q[:, 0] = q[:, 0].abs() + 0.5
    k2 = k.clone()
    k2[2, 0] = -INF
    ref, e = NF.attention_head_ref(q, k2, v, 1.0, False, 64, f16=True)
    ref0, _ = NF.attention_head_ref(q, k2[[0, 1, 3]], v[[0, 1, 3]], 1.0, False, 64, f16=True)
    assert torch.allclose(ref, ref0) and torch.isfinite(e).all()
    k2[2, 0] = INF
    assert torch.isnan(NF.attention_head_ref(q, k2, v, 1.0, False, 64, f16=True)[0]).all()
    v2 = v.clone()
    v2[2, 3] = INF
    ref, _ = NF.attention_head_ref(q, k, v2, 1.0, True, 64, f16=True)
    assert (ref[2:, 3] == INF).all() and torch.isfinite(ref[:, :3]).all() and torch.isfinite(ref[:, 4:]).all()
    assert torch.isnan(ref[:2, 3]).all()      # rows that cannot see key 2: p = 0 times inf, as the masked softmax gives


def test_ieee_matmul_forms_every_product():
    x = torch.tensor([[0.0, 1.0], [2.0, 3.0]], dtype=torch.float64)
    y = torch.tensor([[INF, 1.0], [1.0, 1.0]], dtype=torch.float64)
    out = NF.ieee_matmul(x, y)
    assert torch.isnan(out[0, 0]) and out[1, 0] == INF and out[0, 1] == 1.0 and out[1, 1] == 5.0
    out = NF.ieee_matmul(y.T, x)          # the non-finite entry on the left
    assert torch.isnan(out[0, 0]) and out[0, 1] == INF
