"""The GEMM, attention, norm and LM-input kernels against float64 references with the per-element error bounds of
tests/kernel_bounds.py (derived from each kernel's arithmetic; test_kernel_bounds_host.py shows on the CPU that the
bounds pass a faithful emulation and reject a catalogue of plausible bugs). Every case runs once; the references are
float64 matmuls on the device. Plus the retrieval filter path at k > 16, where the result rests on the proof flag and
the fp32 fallback."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0, mean=0.0):
    return torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale + mean


# ---------------------------------------------------------------------------------------------------------------- GEMM


def _check_linear(name, a, w, out_dtype=torch.float32, block_n=0, **kw):
    from visrag_b200 import ops

    resid = kw.get("resid")
    args = dict(kw)
    if resid is not None:               # in place, as the engine's residual GEMMs run
        x = resid.clone()
        args.update(resid=x, out=x)
    got = ops.gemm(a, w, out_dtype=out_dtype, block_n=block_n, **args)
    ref, e = KB.gemm_linear_ref(a, w, **kw)
    rms = KB.gemm_rms_rel(a.shape[1]) if out_dtype == torch.float32 and not kw.get("gelu") else None
    return KB.check(f"{name} bn={block_n}", got, ref, e, rms_rel=rms)


def _operands(M, N, K, seed, a_scale=0.5, w_scale=0.05):
    a = _randn(M, K, seed=seed, scale=a_scale).bfloat16()
    w = _randn(N, K, seed=seed + 1, scale=w_scale).bfloat16()
    return a, w


SELECTORS = [0, 2, 3, 4, 5, 64, 128, 192, 256]   # 0 auto, 2/4/5 ping-pong (4 = CTA pairs), 3 feature-major, widths


@pytest.mark.parametrize("bn", SELECTORS)
def test_gemm_linear_epilogues_within_bounds(bn):
    M, N, K = 777, 1152, 640
    a, w = _operands(M, N, K, 10)
    bias = _randn(N, seed=12)
    resid = _randn(M, N, seed=13)
    rowadd = _randn(37, N, seed=14)
    for (Mb, Nb, Kb) in [(128, 256, 64), (256, 512, 1152), (1000, 1152, 4304), (333, 4304, 1152), (64, 2304, 2304)]:
        a2, w2 = _operands(Mb, Nb, Kb, 20 + Mb)
        _check_linear(f"plain {Mb}x{Nb}x{Kb}", a2, w2, block_n=bn)
    _check_linear("bias bf16", a, w, torch.bfloat16, bn, bias=bias)
    _check_linear("bias gelu bf16", a, w, torch.bfloat16, bn, bias=bias, gelu=True)
    _check_linear("bias rowadd f32", a, w, torch.float32, bn, bias=bias, rowadd=rowadd)
    _check_linear("bias scale resid f32", a, w, torch.float32, bn, bias=bias, scale=0.25, resid=resid)
    _check_linear("bias gelu scale rowadd bf16", a, w, torch.bfloat16, bn, bias=bias, gelu=True, scale=-0.5, rowadd=rowadd)
    a1, w1 = _operands(M, 4304, K, 15)
    _check_linear("fc1-like N=4304 gelu", a1, w1, torch.bfloat16, bn, bias=_randn(4304, seed=16), gelu=True)
    for M3 in (1, 31, 130):
        _check_linear(f"bias bf16 M={M3}", a[:M3].contiguous(), w, torch.bfloat16, bn, bias=bias)
        _check_linear(f"resid f32 M={M3}", a[:M3].contiguous(), w, torch.float32, bn, resid=resid[:M3])


@pytest.mark.parametrize("bn", [b for b in SELECTORS if b != 3])   # the feature-major kernel is LINEAR only
def test_gemm_rope_and_swiglu_within_bounds(bn):
    from visrag_b200 import ops, _lib as L

    T, H, hd = 300, 2304, 64
    a = _randn(T, H, seed=30, scale=0.5).bfloat16()
    w = _randn(3 * H, H, seed=31, scale=0.03).bfloat16()
    pos = torch.randint(0, 2048, (T,), device=DEV, dtype=torch.int32, generator=_gen(32))
    inv = 1.0 / (10000 ** (torch.arange(0, hd, 2, device=DEV).float() / hd))
    fr = torch.outer(torch.arange(2048, device=DEV).float(), inv)
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    got = ops.gemm(a, w, mode=L.VR_EPI_ROPE, positions=pos, rope_cos=cos, rope_sin=sin, rope_cols=2 * H, block_n=bn)
    KB.check(f"rope qkv bn={bn}", got, *KB.gemm_rope_ref(a, w, pos, cos, sin, 2 * H))
    I = 5760
    wi = _randn(2 * I, H, seed=33, scale=0.03).bfloat16()    # interleaved 32-row gate / up blocks
    got = ops.gemm(a, wi, mode=L.VR_EPI_SWIGLU, block_n=bn)
    KB.check(f"swiglu bn={bn}", got, *KB.gemm_swiglu_ref(a, wi))


def test_gemm_cta_pair_path_edges_within_bounds():
    """block_n = 0 with M > 128 runs the ping-pong kernel in CTA pairs: B tiles whose multicast half lies wholly or
    partly past N (N = 8, 72, 136), a single partly filled k block (K = 8, 16, 56), M one past a tile, one short of two
    tiles, one past two tiles (an unpaired partner tile)."""
    for M in (129, 255, 257):
        for N in (8, 72, 136):
            for K in (8, 16, 56):
                a, w = _operands(M, N, K, M * 1000 + N * 10 + K, a_scale=1.0, w_scale=1.0)
                bias = _randn(N, seed=K)
                _check_linear(f"pairs {M}x{N}x{K} bias resid f32", a, w, torch.float32, 0, bias=bias,
                              resid=_randn(M, N, seed=N))
                _check_linear(f"pairs {M}x{N}x{K} bias gelu bf16", a, w, torch.bfloat16, 0, bias=bias, gelu=True)


def test_gemm_gelu_tails_within_bounds():
    """fc1-like pre-activations spanning about +-40 (shifted by the bias): the erf clamp's error grows with |x|."""
    M, N, K = 777, 1152, 1152
    a, w = _operands(M, N, K, 40, a_scale=1.0, w_scale=0.4)          # acc std ~ 13.6
    bias = (torch.rand(N, device=DEV, generator=_gen(41)) * 2 - 1) * 25
    for bn in (0, 3, 256):     # the GELU epilogue writes bf16 only
        _check_linear("gelu tails", a, w, torch.bfloat16, bn, bias=bias, gelu=True)


def test_gemm_patch_embed_and_lm_residuals_within_bounds():
    """Patch embedding (row add period = tokens per slice, an odd slice count) and the LM's residual GEMMs with the
    depth scale and the residual updated in place, at K = 5760 (down) and 2304 (o_proj): the loosest accumulation."""
    S, NT, D, Kp = 3, 256, 1152, 640
    a, w = _operands(S * NT, D, Kp, 50, a_scale=1.0, w_scale=0.04)
    _check_linear("patch embed", a, w, torch.float32, 0, bias=_randn(D, seed=51), rowadd=_randn(NT, D, seed=52))
    for K in (5760, 2304):
        a, w = _operands(300, 2304, K, 53 + K, a_scale=0.5, w_scale=0.02)
        _check_linear(f"lm residual K={K}", a, w, torch.float32, 0, scale=1.4 / 40 ** 0.5, resid=_randn(300, 2304, seed=K))


# ------------------------------------------------------------------------------------------------------------ attention


@pytest.fixture(params=[0, 1], ids=["auto", "single_tile"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


def _attend(q, k, v, *, name, cu_k, cu_q, max_q, **kw):
    from visrag_b200 import ops

    rows = int(cu_q[-1]) if cu_q is not None else (cu_k.numel() - 1) * max_q
    out = torch.zeros(rows, kw["heads"] * kw["head_dim"], dtype=torch.bfloat16, device=DEV)
    max_k = int((cu_k[1:] - cu_k[:-1]).max())
    ops.attention(q, k, v, batch=cu_k.numel() - 1, cu_k=cu_k, max_k=max_k, cu_q=cu_q, max_q=max_q, out=out, **kw)
    ref, e = KB.attention_ref(q, k, v, cu_k=cu_k, cu_q=cu_q, max_q=max_q, **{n: kw[n] for n in (
        "q_col0", "k_col0", "v_col0", "head_stride", "head_dim", "heads", "causal", "scale")})
    return KB.check(name, out, ref, e)


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


def _vit(lens, nh, seed, ramp=False, v_mean=0.0, ones=False):
    hd, hs = 72, 80
    T = sum(lens)
    qkv = torch.zeros(T, 3, nh, hs, device=DEV)
    qkv[..., :hd] = _randn(T, 3, nh, hd, seed=seed)
    if ramp:   # key scale grows with position: later key tiles raise the row maximum, which forces the O rescale
        qkv[:, 1, :, :hd] *= torch.cat([torch.linspace(0.2, 6.0, n, device=DEV) for n in lens])[:, None, None]
    qkv[:, 2, :, :hd] += v_mean
    if ones:
        qkv[:, 2, :, hd] = 1.0
    qkv = qkv.reshape(T, 3 * nh * hs).bfloat16()
    cu = _cu(lens)
    return dict(q=qkv, k=qkv, v=qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                cu_k=cu, cu_q=cu, max_q=max(lens), causal=False, scale=hd ** -0.5, v_ones_column=ones)


def test_attention_vit_within_bounds(attn_variant):
    for (lens, nh, kw) in [([128], 1, {}), ([256], 2, {}), ([1024] * 3, 4, {"ones": True}), ([1036] * 2, 16, {}),
                           ([130] * 5, 3, {"ones": True}), ([784] * 6, 16, {}), ([300] * 7, 5, {}),
                           ([1024, 300, 784, 130, 1, 64, 65], 16, {}),    # unequal N per sequence in one launch
                           ([512] * 2, 2, {"ramp": True}), ([1024], 3, {"ramp": True}),
                           ([1024, 1036], 4, {"v_mean": 1.0})]:           # |out| ~ c: the output rounding dominates
        _attend(name=f"vit lens={lens[:4]} heads={nh} {kw}", **_vit(lens, nh, len(lens) * 100 + nh, **kw))


def test_attention_lm_causal_within_bounds(attn_variant):
    """Causal var-len at the LM's 36 heads, up to the engine's max_inp_length of 2048."""
    nh, hd = 36, 64
    H = nh * hd
    for lens in ([2048], [1025, 1023, 1, 64, 65], [1, 5, 68, 127, 128, 129, 300], [670, 33]):
        qkv = _randn(sum(lens), 3 * H, seed=sum(lens)).bfloat16()
        cu = _cu(lens)
        _attend(qkv, qkv, qkv, name=f"lm causal lens={lens}", q_col0=0, k_col0=H, v_col0=2 * H, head_stride=64,
                head_dim=64, heads=nh, cu_k=cu, cu_q=cu, max_q=max(lens), causal=True, scale=hd ** -0.5)


def test_attention_resampler_within_bounds(attn_variant):
    """64 learned queries shared by every slice (cross-attention), 18 heads of 128."""
    nh = 18
    E = nh * 128
    for N in (100, 1024, 1036):
        S = 2
        q = torch.zeros(128, E, device=DEV)
        q[:64] = _randn(64, E, seed=N)
        q = q.bfloat16()
        k = _randn(S * N, E, seed=N + 1).bfloat16()
        v = _randn(S * N, E, seed=N + 2).bfloat16()
        cu = torch.arange(0, (S + 1) * N, N, dtype=torch.int32, device=DEV)
        _attend(q, k, v, name=f"resampler S={S} N={N}", q_col0=0, k_col0=0, v_col0=0, head_stride=128, head_dim=128,
                heads=nh, cu_k=cu, cu_q=None, max_q=64, causal=False, scale=128 ** -0.5)


# ---------------------------------------------------------------------------------------------------------------- norms


def _norm_rows(M, D, seed):
    """Random rows, rows with |mean| >> std, constant rows (variance 0: the output is beta up to the mean's rounding),
    and rows whose variance is near eps (so eps placement matters)."""
    x = _randn(M, D, seed=seed, scale=3.0, mean=1.0)
    if M >= 8:
        x[1] = _randn(D, seed=seed + 1) + 1e3
        x[2] = _randn(D, seed=seed + 2) - 1e3
        x[3] = 0.75
        x[4] = -2.5
        x[5] = _randn(D, seed=seed + 3, scale=1e-3)
        x[6] = _randn(D, seed=seed + 4, scale=1e-3, mean=5.0)
    return x


@pytest.mark.parametrize("D", [288, 1152, 2304])     # generic kernel, register-resident 9 and 18 float4 per lane
def test_norms_within_bounds(D):
    from visrag_b200 import ops

    g, b = _randn(D, seed=D), _randn(D, seed=D + 1)
    add = _randn(37, D, seed=D + 2)
    for M in (1000, 1, 13):          # 13: not a multiple of the 8 warps per block
        x = _norm_rows(M, D, M + D)
        o1, o2 = ops.layernorm(x, g, b, 1e-6, add=add)
        (r1, e1), (r2, e2) = KB.layernorm_ref(x, g, b, 1e-6, add=add)
        KB.check(f"layernorm D={D} M={M}", o1, r1, e1)
        KB.check(f"layernorm+add D={D} M={M}", o2, r2, e2)
        KB.check(f"layernorm (no add) D={D} M={M}", ops.layernorm(x, g, b, 1e-5), *KB.layernorm_ref(x, g, b, 1e-5))
        KB.check(f"rmsnorm D={D} M={M}", ops.rmsnorm(x, g, 1e-5), *KB.rmsnorm_ref(x, g, 1e-5))


def test_build_lm_input_within_bounds():
    from visrag_b200 import ops

    D = 2304
    emb = _randn(512, D, seed=60).bfloat16()
    vis = _randn(128, D, seed=61)
    src = torch.tensor([-6, 0, 1, 127, -512, -1, 5, -300], dtype=torch.int32, device=DEV)
    KB.check("build_lm_input", ops.build_lm_input(src, emb, 12.0, vis), *KB.build_lm_input_ref(src, emb, 12.0, vis))
    KB.check("build_lm_input text only", ops.build_lm_input(src[src < 0], emb, 1.5, None),
             *KB.build_lm_input_ref(src[src < 0], emb, 1.5, None))


# ------------------------------------------------------------------------------------------------------------ retrieval


@pytest.mark.parametrize("k", [17, 32, 100, 129, 300])
def test_score_topk_filter_path_large_k(k):
    """A filter list holds 16 candidates and keep = min(2k, lists * 16, 256) are rescored: k > 16 relies on the proof
    flag and the fp32 fallback, k > 128 keeps fewer candidates than 2k. Ids equal the fp32 scan's; where two reference
    scores lie within fp32 summation-order noise (2e-6) of each other their order may differ, so those positions are
    compared by score."""
    from oracle import restated as O
    from visrag_b200 import retriever as R

    rs = np.random.RandomState(k)
    Q = rs.randn(300, 128).astype(np.float32)
    D = rs.randn(20000, 128).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    stats = {}
    s, i = R.score_topk(torch.from_numpy(Q).cuda(), R.build_index(D), k, stats=stats)
    s, i = s.cpu().numpy(), i.cpu().numpy()
    s_ref, i_ref = O.score_topk(Q, D, k)
    assert stats["path"] == "filter+rescore"
    assert np.abs(s - s_ref).max() <= 2e-6
    exact = Q.astype(np.float64) @ D.astype(np.float64).T
    assert np.abs(np.take_along_axis(exact, i, 1) - s).max() <= 2e-6        # each score belongs to its id
    assert all(len(set(row)) == k for row in i)
    drop = -np.diff(O.score_topk(Q, D, k + 1)[0], axis=1)          # [nq, k]: score drop after each of the top k
    above = np.concatenate([np.full((len(Q), 1), np.inf), drop[:, :-1]], axis=1)
    clear = (above > 2e-6) & (drop > 2e-6)                           # no near-tie on either side
    assert clear.mean() > 0.9 and np.array_equal(i[clear], i_ref[clear])
    assert (np.take_along_axis(exact, i, 1) >= s_ref[:, -1:] - 2e-6).all()
