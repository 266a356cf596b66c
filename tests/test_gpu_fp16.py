"""fp16 engines on the H100: every kernel of the encode path in its fp16 form against the float64 bounds of
tests/kernel_bounds_f16.py (test_fp16_host.py shows on the CPU that the fp16 bounds pass a faithful emulation and reject fp16
mistakes), the batch-invariance contract in fp16, the golden end-to-end contract for an fp16 engine next to a bf16 one, and
the reference driver's `dtype="float16"` through DRModelForInference.build."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB
from tests import kernel_bounds_f16 as KF
from tests.helpers import cosine_rows, load_case, synth_pages

pytestmark = pytest.mark.gpu

DEV = "cuda"
F16 = torch.float16
COS_MIN, ABS_MAX = 0.9999, 1e-3


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0, mean=0.0):
    return torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale + mean


def _check(worst, name, got, ref, e, **kw):
    r = KF.check(name, got, ref, e, **kw)
    worst[name.split(" ")[0]] = max(worst.get(name.split(" ")[0], 0.0), r["frac"])
    return r


def _report(title, worst):
    print(f"{title}: worst fraction of the fp16 bound per case family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


# ---------------------------------------------------------------------------------------------------------------- GEMM


def _operands(M, N, K, seed, a_scale=0.5, w_scale=0.05):
    return _randn(M, K, seed=seed, scale=a_scale).half(), _randn(N, K, seed=seed + 1, scale=w_scale).half()


def _linear(worst, name, a, w, out_dtype=F16, block_n=0, **kw):
    from visrag_b200 import ops

    args = dict(kw)
    if kw.get("resid") is not None:        # in place, as the engine's residual GEMMs run
        x = kw["resid"].clone()
        args.update(resid=x, out=x)
    got = ops.gemm(a, w, out_dtype=out_dtype, block_n=block_n, **args)
    assert got.dtype == out_dtype
    ref, e = KB.gemm_linear_ref(a, w, **kw)
    rms = KB.gemm_rms_rel(a.shape[1]) if out_dtype == torch.float32 and not kw.get("gelu") else None
    return _check(worst, f"{name} bn={block_n}", got, ref, e, rms_rel=rms)


SELECTORS = [0, 2, 3, 4, 5, 64, 128, 192, 256]


@pytest.mark.parametrize("bn", SELECTORS)
def test_gemm_f16_linear_epilogues_within_bounds(bn):
    M, N, K = 777, 1152, 640
    a, w = _operands(M, N, K, 10)
    bias, resid, rowadd = _randn(N, seed=12), _randn(M, N, seed=13), _randn(37, N, seed=14)
    worst = {}
    for (Mb, Nb, Kb) in [(128, 256, 64), (256, 512, 1152), (1000, 1152, 4304), (64, 2304, 2304)]:
        _linear(worst, f"plain-{Mb}x{Nb}x{Kb}", *_operands(Mb, Nb, Kb, 20 + Mb), block_n=bn)
    _linear(worst, "bias-f16", a, w, F16, bn, bias=bias)
    _linear(worst, "bias-gelu-f16", a, w, F16, bn, bias=bias, gelu=True)
    _linear(worst, "bias-rowadd-f32", a, w, torch.float32, bn, bias=bias, rowadd=rowadd)
    _linear(worst, "bias-scale-resid-f32", a, w, torch.float32, bn, bias=bias, scale=0.25, resid=resid)
    _linear(worst, "bias-gelu-scale-rowadd-f16", a, w, F16, bn, bias=bias, gelu=True, scale=-0.5, rowadd=rowadd)
    a1, w1 = _operands(M, 4304, K, 15)
    _linear(worst, "fc1-like-N=4304-gelu", a1, w1, F16, bn, bias=_randn(4304, seed=16), gelu=True)
    for M3 in (1, 31, 130):
        _linear(worst, f"bias-f16-M={M3}", a[:M3].contiguous(), w, F16, bn, bias=bias)
        _linear(worst, f"resid-f32-M={M3}", a[:M3].contiguous(), w, torch.float32, bn, resid=resid[:M3])
    _report(f"gemm linear bn={bn}", worst)


@pytest.mark.parametrize("bn", [b for b in SELECTORS if b != 3])
def test_gemm_f16_rope_and_swiglu_within_bounds(bn):
    from visrag_b200 import _lib as L
    from visrag_b200 import ops

    T, H, hd = 300, 2304, 64
    a = _randn(T, H, seed=30, scale=0.5).half()
    w = _randn(3 * H, H, seed=31, scale=0.03).half()
    pos = torch.randint(0, 2048, (T,), device=DEV, dtype=torch.int32, generator=_gen(32))
    fr = torch.outer(torch.arange(2048, device=DEV).float(), 1.0 / (10000 ** (torch.arange(0, hd, 2, device=DEV).float() / hd)))
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    worst = {}
    got = ops.gemm(a, w, mode=L.VR_EPI_ROPE, positions=pos, rope_cos=cos, rope_sin=sin, rope_cols=2 * H, block_n=bn)
    assert got.dtype == F16
    _check(worst, f"rope bn={bn}", got, *KB.gemm_rope_ref(a, w, pos, cos, sin, 2 * H))
    wi = _randn(2 * 5760, H, seed=33, scale=0.03).half()
    got = ops.gemm(a, wi, mode=L.VR_EPI_SWIGLU, block_n=bn)
    assert got.dtype == F16
    _check(worst, f"swiglu bn={bn}", got, *KB.gemm_swiglu_ref(a, wi))
    _report(f"gemm rope/swiglu bn={bn}", worst)


def test_gemm_f16_cta_pair_edges_and_gelu_tails_within_bounds():
    """CTA-pair edges of the automatic choice (M 129 / 255 / 257, N 8 / 72 / 136, K 8 / 16 / 56) and GELU tails
    (pre-activations spanning about +-40) on the kernels the fp16 engine's GELU GEMMs can take."""
    worst = {}
    for M in (129, 255, 257):
        for N in (8, 72, 136):
            for K in (8, 16, 56):
                a, w = _operands(M, N, K, M * 1000 + N * 10 + K, a_scale=1.0, w_scale=1.0)
                bias = _randn(N, seed=K)
                _linear(worst, f"pairs-{M}x{N}x{K}-bias-resid-f32", a, w, torch.float32, 0, bias=bias, resid=_randn(M, N, seed=N))
                _linear(worst, f"pairs-{M}x{N}x{K}-bias-gelu-f16", a, w, F16, 0, bias=bias, gelu=True)
    a, w = _operands(777, 1152, 1152, 40, a_scale=1.0, w_scale=0.4)
    bias = (torch.rand(1152, device=DEV, generator=_gen(41)) * 2 - 1) * 25
    for bn in (0, 3, 4, 256):
        _linear(worst, "gelu-tails", a, w, F16, bn, bias=bias, gelu=True)
    _report("gemm edges", {k.split("-")[0] + ("-gelu" if "gelu" in k else ""): v for k, v in worst.items()})


# ------------------------------------------------------------------------------------------------------------ attention


@pytest.fixture(params=[0, 1], ids=["auto", "single_tile"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


def _attend(q, k, v, *, cu_k, cu_q, max_q, out_fill=0.0, **kw):
    from visrag_b200 import ops

    rows = int(cu_q[-1]) if cu_q is not None else (cu_k.numel() - 1) * max_q
    out = torch.full((rows, kw["heads"] * kw["head_dim"]), out_fill, dtype=F16, device=DEV)
    max_k = int((cu_k[1:] - cu_k[:-1]).max())
    ops.attention(q, k, v, batch=cu_k.numel() - 1, cu_k=cu_k, max_k=max_k, cu_q=cu_q, max_q=max_q, out=out, **kw)
    return out


def _attend_checked(worst, name, q, k, v, *, cu_k, cu_q, max_q, **kw):
    out = _attend(q, k, v, cu_k=cu_k, cu_q=cu_q, max_q=max_q, **kw)
    ref, e = KF.attention_ref_f16(q, k, v, cu_k=cu_k, cu_q=cu_q, max_q=max_q, **{n: kw[n] for n in (
        "q_col0", "k_col0", "v_col0", "head_stride", "head_dim", "heads", "causal", "scale")})
    return _check(worst, name, out, ref, e)


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


def _qkv(lens, nh, hd, hs, seed, qk_scale=1.0, v_mean=0.0, ramp=False):
    T = sum(lens)
    qkv = torch.zeros(T, 3, nh, hs, device=DEV)
    qkv[..., :hd] = _randn(T, 3, nh, hd, seed=seed)
    qkv[:, :2] *= qk_scale
    if ramp:
        qkv[:, 1, :, :hd] *= torch.cat([torch.linspace(0.2, 6.0, n, device=DEV) for n in lens])[:, None, None]
    qkv[:, 2, :, :hd] += v_mean
    qkv = qkv.reshape(T, 3 * nh * hs).half()
    cu = _cu(lens)
    return dict(q=qkv, k=qkv, v=qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                cu_k=cu, cu_q=cu, max_q=max(lens), scale=hd ** -0.5)


def test_attention_f16_within_bounds(attn_variant):
    """Both forms at head strides 80 (ViT), 64 (LM, causal, incl. rows that see 1 and 2 keys) and 128 (resampler), plus
    rows where most p fall below 2^-14 (fp16 subnormals in the P V MMA)."""
    worst = {}
    for lens, nh, kw in [([1036] * 2, 16, {}), ([1024, 300, 784, 130, 1, 64, 65], 16, {}), ([1024], 3, {"ramp": True}),
                         ([1024, 1036], 4, {"v_mean": 1.0})]:
        _attend_checked(worst, f"vit lens={lens[:4]} {kw}", causal=False, **_qkv(lens, nh, 72, 80, len(lens) * 100 + nh, **kw))
    for lens in ([2048], [1025, 1023, 1, 64, 65], [1, 2, 5, 68, 127, 128, 129, 300]):
        _attend_checked(worst, f"lm-causal lens={lens}", causal=True, **_qkv(lens, 36, 64, 64, sum(lens)))
    _attend_checked(worst, "small-P", causal=False, **_qkv([1036, 700], 4, 64, 64, 77, qk_scale=2.0, v_mean=1.0))
    _attend_checked(worst, "small-P-causal", causal=True, **_qkv([1036, 700], 4, 64, 64, 78, qk_scale=2.0, v_mean=1.0))
    E = 18 * 128
    for N in (100, 1036):
        q = torch.zeros(128, E, device=DEV)
        q[:64] = _randn(64, E, seed=N)
        k, v = _randn(2 * N, E, seed=N + 1).half(), _randn(2 * N, E, seed=N + 2).half()
        cu = torch.arange(0, 3 * N, N, dtype=torch.int32, device=DEV)
        _attend_checked(worst, f"resampler N={N}", q.half(), k, v, q_col0=0, k_col0=0, v_col0=0, head_stride=128, head_dim=128,
                        heads=18, cu_k=cu, cu_q=None, max_q=64, causal=False, scale=128 ** -0.5)
    _report(f"attention variant={attn_variant}", worst)


# ---------------------------------------------------------------------------------------------------------------- norms


@pytest.mark.parametrize("D", [288, 1152, 2304])
def test_norms_f16_within_bounds(D):
    from visrag_b200 import ops

    g, b, add = _randn(D, seed=D), _randn(D, seed=D + 1), _randn(37, D, seed=D + 2)
    worst = {}
    for M in (1000, 1, 13):
        x = _randn(M, D, seed=M + D, scale=3.0, mean=1.0)
        if M >= 8:
            x[1] = _randn(D, seed=M + D + 1) + 1e3
            x[3] = 0.75
            x[5] = _randn(D, seed=M + D + 3, scale=1e-3)
        o1, o2 = ops.layernorm(x, g, b, 1e-6, add=add, dtype=F16)
        assert o1.dtype == o2.dtype == F16
        (r1, e1), (r2, e2) = KB.layernorm_ref(x, g, b, 1e-6, add=add)
        _check(worst, f"layernorm D={D} M={M}", o1, r1, e1)
        _check(worst, f"layernorm+add D={D} M={M}", o2, r2, e2)
        _check(worst, f"rmsnorm D={D} M={M}", ops.rmsnorm(x, g, 1e-5, F16), *KB.rmsnorm_ref(x, g, 1e-5))
    _report(f"norms D={D}", worst)


def test_build_lm_input_and_im2col_f16():
    from visrag_b200 import ops

    D = 2304
    emb = _randn(512, D, seed=60).half()
    vis = _randn(128, D, seed=61)
    src = torch.tensor([-6, 0, 1, 127, -512, -1, 5, -300], dtype=torch.int32, device=DEV)
    worst = {}
    _check(worst, "build_lm_input", ops.build_lm_input(src, emb, 12.0, vis), *KB.build_lm_input_ref(src, emb, 12.0, vis))
    _check(worst, "build_lm_input-text-only", ops.build_lm_input(src[src < 0], emb, 1.5, None),
           *KB.build_lm_input_ref(src[src < 0], emb, 1.5, None))
    _report("build_lm_input", worst)
    # im2col: the fp16 patch matrix holds fp16(((u / 255) - 0.5) / 0.5) of the pixel, column c*p*p + ky*p + kx
    for h, w in ((448, 448), (14 * 5, 14 * 7)):
        px = torch.randint(0, 256, (2, h, w, 3), dtype=torch.uint8, device=DEV, generator=_gen(h + w))
        got = ops.im2col_norm(px, 14, 640, F16)
        want = ((px.float() / 255.0 - 0.5) / 0.5).reshape(2, h // 14, 14, w // 14, 14, 3).permute(0, 1, 3, 5, 2, 4)
        want = want.reshape(-1, 588).half()
        assert got.dtype == F16 and torch.equal(got[:, :588], want) and (got[:, 588:] == 0).all()


# ---------------------------------------------------------------------------------------------------- batch invariance


@pytest.mark.parametrize("hs,hd,causal", [(64, 64, True), (80, 72, False)], ids=["lm-causal", "vit-noncausal"])
def test_attention_f16_alone_equals_in_a_long_batch(hs, hd, causal):
    for L in (1, 2, 17, 63, 64):
        lens = [200, L, 100]
        kw = _qkv(lens, 4, hd, hs, seed=L + hs)
        batch = _attend(causal=causal, out_fill=float("nan"), **kw)
        qkv = kw["q"]
        alone_kw = dict(kw, q=qkv[200:200 + L].contiguous(), k=qkv[200:200 + L].contiguous(), v=qkv[200:200 + L].contiguous(),
                        cu_k=_cu([L]), cu_q=_cu([L]), max_q=L)
        alone = _attend(causal=causal, out_fill=float("nan"), **alone_kw)
        assert torch.equal(alone, batch[200:200 + L]), (L, (alone.float() - batch[200:200 + L].float()).abs().max())


@pytest.mark.parametrize("causal", [False, True], ids=["noncausal", "causal"])
@pytest.mark.parametrize("hs,hd", [(64, 64), (80, 72), (128, 128)])
def test_attention_f16_one_warpgroup_kernel_equals_default_dispatch(hs, hd, causal):
    from visrag_b200 import _lib as L

    for lens in ([300, 129, 0, 65, 17, 1036, 1, 64], [2, 63, 64], [128, 5, 257]):
        kw = _qkv(lens, 3, hd, hs, seed=sum(lens) + hs + causal)
        want = _attend(causal=causal, **kw)
        L.lib().vr_attention_force_v1(1)
        try:
            got = _attend(causal=causal, **kw)
        finally:
            L.lib().vr_attention_force_v1(0)
        assert torch.equal(got, want), (lens, (got.float() - want.float()).abs().max())


@pytest.mark.parametrize("M", [1, 64, 128, 129, 300, 8192])
def test_gemm_f16_rows_do_not_depend_on_m(M):
    from visrag_b200 import _lib as L
    from visrag_b200 import ops

    R, K, N = 8192, 320, 384
    a = _randn(R, K, seed=1, scale=0.5).half()
    w = _randn(N, K, seed=2, scale=0.05).half()
    bias, rowadd, resid = _randn(N, seed=3), _randn(37, N, seed=4), _randn(R, N, seed=5)
    pos = torch.randint(0, 2048, (R,), device=DEV, dtype=torch.int32, generator=_gen(6))
    fr = torch.outer(torch.arange(2048, device=DEV).float(), 1.0 / (10000 ** (torch.arange(0, 64, 2, device=DEV).float() / 64)))
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()

    def resid_gemm(rows):
        x = resid[:rows].clone()
        return ops.gemm(a[:rows], w, scale=0.3, resid=x, out=x, out_dtype=torch.float32, bias=bias)

    runs = {
        "bias f16": lambda rows: ops.gemm(a[:rows], w, bias=bias),
        "bias gelu f16": lambda rows: ops.gemm(a[:rows], w, bias=bias, gelu=True),
        "bias rowadd f32": lambda rows: ops.gemm(a[:rows], w, bias=bias, rowadd=rowadd, out_dtype=torch.float32),
        "in-place resid f32, scale": resid_gemm,
        "rope": lambda rows: ops.gemm(a[:rows], w, mode=L.VR_EPI_ROPE, positions=pos[:rows], rope_cos=cos, rope_sin=sin, rope_cols=128),
        "swiglu": lambda rows: ops.gemm(a[:rows], w, mode=L.VR_EPI_SWIGLU),
    }
    for name, run in runs.items():
        full, part = run(R), run(M)
        assert torch.equal(part, full[:M]), (name, (part.float() - full[:M].float()).abs().max().item())


def test_cuda_graph_equals_eager_f16():
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 5)
    eager = VisRAGEngine(cfg, sd, cuda_graphs=False, dtype=F16)
    graphed = VisRAGEngine(cfg, sd, cuda_graphs=True, dtype=F16)
    assert graphed.patch_w.dtype == F16 and graphed.rs_q.dtype == F16 and graphed.embed.dtype == F16
    tok = StubTokenizer(cfg.vocab)
    sizes = [(448, 448), (700, 900), (448, 448)]
    for seed in (1, 2, 3):
        pages = synth_pages(sizes, seed)
        assert torch.equal(graphed.encode([""] * 3, pages, tok), eager.encode([""] * 3, pages, tok)), seed
    for q in (["revenue table 2020"], ["cat", "a much longer question about the climate chart"]):
        for _ in range(3):
            assert torch.equal(graphed.encode(q, [None] * len(q), tok), eager.encode(q, [None] * len(q), tok)), q
    assert graphed.graph_stats["replayed"] > 0 and graphed.graph_stats["captured"] > 0


# ---------------------------------------------------------------------------------------------------------- end to end


def _golden_errors(name, dtype):
    """Encode the golden case with a `dtype` engine: the golden contract, and (max |diff|, max (1 - cos)) over pages and
    queries against the reference's fp32 embeddings."""
    from oracle import restated as O
    from visrag_b200 import retriever as R
    from visrag_b200.modeling import DRModelForInference, VisRAGRetB200
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg, wseed, pages, queries, z = load_case(name)
    model = DRModelForInference(lm_q=VisRAGRetB200(cfg, random_state_dict(cfg, wseed), "cuda:0", dtype=dtype), pooling="wmean",
                                normalize=True)
    assert model.lm_q.dtype == dtype
    tok = StubTokenizer(cfg.vocab)
    items = lambda texts, imgs, p: {"id": [f"{p}{i}" for i in range(len(texts))], "text": list(texts), "image": list(imgs)}  # noqa: E731
    out = model(query=items(queries, [None] * len(queries), "q"), passage=items([""] * len(pages), pages, "d"), tokenizer=tok,
                max_inp_length=2048)
    assert out.p_reps.dtype == torch.float32
    p, q = out.p_reps.cpu().numpy(), out.q_reps.cpu().numpy()
    cp, cq = cosine_rows(p, z["page_reps"]), cosine_rows(q, z["query_reps"])
    diff = max(np.abs(p - z["page_reps"]).max(), np.abs(q - z["query_reps"]).max())
    one_minus_cos = float(max(1 - cp.min(), 1 - cq.min()))
    assert cp.min() >= COS_MIN and cq.min() >= COS_MIN, (dtype, cp, cq)
    assert diff <= ABS_MAX, (dtype, diff)
    k = z["topk_indices"].shape[1]
    ref_top = z["topk_indices"]
    s_run, i_run = R.score_topk(out.q_reps, R.build_index(out.p_reps), k)
    i_run = i_run.cpu().numpy()
    assert np.array_equal(i_run, ref_top), (dtype, i_run, ref_top)
    relevant = [{int(ref_top[qi, 0])} for qi in range(len(queries))]
    if "page_spec" in z.files:
        spec = [e.get("name") for e in __import__("json").loads(str(z["page_spec"]))]
        for r, nm in enumerate(("parquet0", "parquet1")):
            relevant[len(queries) - 2 + r].add(spec.index(nm))
    for kk in (1, 5):
        assert O.recall_at_k(i_run, relevant, kk) == O.recall_at_k(ref_top, relevant, kk)
    del model, out
    torch.cuda.empty_cache()
    return float(diff), one_minus_cos


@pytest.mark.parametrize("name", ["tiny_v2", "full_v2"])
def test_golden_f16_engine_meets_the_contract_and_beats_bf16(name):
    """The fp16 engine meets the golden contract (cos >= 0.9999, max |diff| <= 1e-3, ordered top-k ids equal to the
    reference's, Recall@1/5 equal) and sits strictly closer to the reference's fp32 embeddings than the bf16 engine on
    the same case: fp16 rounds every stored activation 8x finer, and everything else is the same arithmetic."""
    d16, c16 = _golden_errors(name, torch.float16)
    d_bf, c_bf = _golden_errors(name, torch.bfloat16)
    print(f"{name}: max |diff| fp16 {d16:.3e} vs bf16 {d_bf:.3e} ({d_bf / d16:.2f}x); max (1 - cos) fp16 {c16:.3e} vs bf16 "
          f"{c_bf:.3e} ({c_bf / max(c16, 1e-300):.2f}x)")
    assert d16 < d_bf and c16 < c_bf


def test_build_with_dtype_float16(tmp_path):
    """DRModelForInference.build(model_args) with model_args.dtype = "float16" (the reference evaluation's --dtype float16)
    on a synthetic checkpoint directory: an fp16 backbone, fp16 B1 hidden states, fp32 unit embeddings that match the oracle."""
    from types import SimpleNamespace

    from oracle import restated as O
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.modeling import DRModelForInference
    from visrag_b200.synth import synth_doc_pages
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict, save_checkpoint

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, 77)
    ckpt = str(tmp_path / "VisRAG-Ret-synthetic")
    save_checkpoint(ckpt, cfg, sd)
    model = DRModelForInference.build(SimpleNamespace(model_name_or_path=ckpt, pooling="wmean", normalize=True, dtype="float16"))
    assert model.lm_q.dtype == F16 and model.lm_q.engine.dtype == F16 and model.lm_q.engine.layers[0]["qkv_w"].dtype == F16
    tok = StubTokenizer(cfg.vocab)
    pages = synth_doc_pages([(448, 448), (700, 900), (640, 300)], 31)
    out = model.lm_q(text=["", "", "a caption"], image=pages, tokenizer=tok, max_inp_length=2048)
    assert out.last_hidden_state.dtype == F16
    reps = model(passage={"id": ["d0", "d1", "d2"], "text": [""] * 3, "image": pages}, tokenizer=tok, max_inp_length=2048).p_reps
    assert reps.dtype == torch.float32
    assert np.allclose(np.linalg.norm(reps.cpu().numpy(), axis=1), 1.0, atol=1e-5)
    assert cosine_rows(reps.cpu().numpy(), O.encode(sd, cfg, tok, [""] * 3, pages)).min() >= COS_MIN
