"""NaN, inf and fp16 overflow through every encode kernel, against the IEEE-aware checker of tests/nonfinite_bounds.py:
  a. fp16 stores past 65504 become inf (and subnormals stay subnormal) at every 16-bit store: each GEMM kernel's LINEAR,
     ROPE and SWIGLU epilogues under every block_n selector, and the three norm kernels;
  b. a NaN or inf in one row of a GEMM, norm, pool_norm or build_lm_input launch gives the float64 reference's value in
     the outputs it feeds and leaves every other output bit-identical to a clean run;
  c. attention: a non-finite K or V row of one sequence never reaches another sequence of the launch, whatever the
     neighbour's length mod 128 (a sequence's last key tile reads rows of the next one);
  d. the engine: one item whose embedding overflows leaves the other items of its batch bit-identical, eager, under CUDA
     graphs and through the prefix cache, and the inference loop stops on it with the reference's NaN assertion.
Every case runs once."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB
from tests import nonfinite_bounds as NF

pytestmark = pytest.mark.gpu

DEV = "cuda"
INF, NAN = float("inf"), float("nan")
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
SELECTORS = [0, 2, 3, 4, 5, 64, 128, 192, 256]   # 0 auto, 2/4/5 ping-pong (4 = CTA pairs), 3 feature-major, widths
POISON = [NAN, INF, -INF]


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


@pytest.fixture(params=[0, 1], ids=["auto", "single_tile"])
def attn_variant(request):
    from visrag_b200 import _lib as L

    L.lib().vr_attention_force_v1(request.param)
    yield request.param
    L.lib().vr_attention_force_v1(0)


# ------------------------------------------------------------------------------------------- a. fp16 overflow at stores


def _overflow_operands(M, N, K, seed):
    """fp16 operands whose float64 products reach about +-4e4 (std), so the outputs straddle +-65520, and a bias that
    puts row 0 within +-2 of 65520 (and row 1 of -65520): inside the bound of the threshold."""
    a = _randn(M, K, seed=seed).half()
    w = _randn(N, K, seed=seed + 1, scale=2500.0).half()
    acc = a.double() @ w.double().T
    bias = _randn(N, seed=seed + 2, scale=3e4)
    delta = torch.linspace(-2.0, 2.0, N, device=DEV, dtype=torch.float64)
    bias[: N // 2] = (65520.0 + delta[: N // 2] - acc[0, : N // 2]).float()
    bias[N // 2:] = (-65520.0 + delta[N // 2:] - acc[1, N // 2:]).float()
    return a, w, bias


def _check_linear_nf(name, a, w, out_dtype, bn, **kw):
    from visrag_b200 import ops

    args = dict(kw)
    if kw.get("resid") is not None:                  # in place, as the engine's residual GEMMs run
        x = kw["resid"].clone()
        args.update(resid=x, out=x)
    got = ops.gemm(a, w, out_dtype=out_dtype, block_n=bn, **args)
    NF.check(f"{name} bn={bn}", got, *NF.gemm_linear_ref(a, w, **kw))
    return got


@pytest.mark.parametrize("bn", SELECTORS)
def test_gemm_linear_fp16_overflow_and_subnormals(bn):
    M, N, K = 300, 512, 256
    a, w, bias = _overflow_operands(M, N, K, 10)
    rowadd = _randn(37, N, seed=13, scale=2e4)
    got = _check_linear_nf("plain", a, w, torch.float16, bn)
    assert torch.isinf(got).any() and torch.isfinite(got).any()
    got = _check_linear_nf("bias", a, w, torch.float16, bn, bias=bias)
    assert torch.isinf(got[:2]).any() and (got[:2].abs() == 65504).any()      # both sides of the threshold
    _check_linear_nf("bias gelu", a, w, torch.float16, bn, bias=bias, gelu=True)
    _check_linear_nf("bias scale", a, w, torch.float16, bn, bias=bias, scale=-1.25)
    _check_linear_nf("bias gelu scale rowadd", a, w, torch.float16, bn, bias=bias, gelu=True, scale=0.75, rowadd=rowadd)
    got = _check_linear_nf("subnormal", a, w, torch.float16, bn, scale=2.0 ** -30)      # |out| ~ 4e-5 < 2^-14
    sub = (got != 0) & (got.abs() < 2.0 ** -14)
    assert sub.float().mean() > 0.3


@pytest.mark.parametrize("bn", [b for b in SELECTORS if b != 3])   # the feature-major kernel is LINEAR only
def test_gemm_rope_and_swiglu_fp16_overflow(bn):
    from visrag_b200 import ops, _lib as L

    T, H, K = 300, 256, 256
    a = _randn(T, K, seed=30).half()
    w = _randn(3 * H, K, seed=31, scale=2500.0).half()
    pos = torch.randint(0, 2048, (T,), device=DEV, dtype=torch.int32, generator=_gen(32))
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, device=DEV).float() / 64))
    fr = torch.outer(torch.arange(2048, device=DEV).float(), inv)
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    got = ops.gemm(a, w, mode=L.VR_EPI_ROPE, positions=pos, rope_cos=cos, rope_sin=sin, rope_cols=2 * H, block_n=bn)
    NF.check(f"rope fp16 bn={bn}", got, *NF.gemm_rope_ref(a, w, pos, cos, sin, 2 * H))
    assert torch.isinf(got).any() and torch.isfinite(got).any()
    wi = _randn(2 * H, K, seed=33, scale=18.0).half()      # gate and up ~ 290: silu(g) u ~ 8e4
    got = ops.gemm(a, wi, mode=L.VR_EPI_SWIGLU, block_n=bn)
    NF.check(f"swiglu fp16 bn={bn}", got, *NF.gemm_swiglu_ref(a, wi))
    assert torch.isinf(got).any() and torch.isfinite(got).any()


def _wide_gamma(D, seed):
    """Gains from 1e-7 to 5e4 in magnitude: outputs past 65504 and in the fp16 subnormals in one row."""
    mag = 10.0 ** (torch.rand(D, device=DEV, generator=_gen(seed)) * 11.7 - 7.0)
    return mag * torch.sign(_randn(D, seed=seed + 1))


@pytest.mark.parametrize("D", [288, 1152, 2304])     # generic kernel, register-resident 9 and 18 float4 per lane
def test_norms_fp16_overflow_and_subnormals(D):
    from visrag_b200 import ops

    x = _randn(200, D, seed=D, scale=2.0)
    g, b = _wide_gamma(D, D), _wide_gamma(D, D + 7)
    add = _randn(37, D, seed=D + 3, scale=3e4)
    o1, o2 = ops.layernorm(x, g, b, 1e-6, add=add, dtype=torch.float16)
    NF.check(f"layernorm D={D}", o1, *NF.norm_ref(x, g, b, 1e-6, rms=False))
    NF.check(f"layernorm+add D={D}", o2, *NF.norm_ref(x, g, b, 1e-6, rms=False, add=add))
    o3 = ops.layernorm(x, g, b, 1e-6, dtype=torch.float16)
    NF.check(f"layernorm (no add) D={D}", o3, *NF.norm_ref(x, g, b, 1e-6, rms=False))
    o4 = ops.rmsnorm(x, g, 1e-5, dtype=torch.float16)
    NF.check(f"rmsnorm D={D}", o4, *NF.norm_ref(x, g, None, 1e-5, rms=True))
    for o in (o1, o2, o4):
        assert torch.isinf(o).any() and torch.isfinite(o).any()
    for o in (o1, o4):
        assert ((o != 0) & (o.abs() < 2.0 ** -14)).any()


# ---------------------------------------------------------------------------------- b. NaN and inf stay in their rows


def _poison_rows(t, rows, cols):
    t = t.clone()
    for i, (r, c) in enumerate(zip(rows, cols)):
        t[r, c] = POISON[i % 3]
    return t


def _same_except(got, want, rows=None, cols=None):
    keep_r = torch.ones(got.shape[0], dtype=torch.bool, device=got.device)
    keep_c = torch.ones(got.shape[1], dtype=torch.bool, device=got.device)
    if rows is not None:
        keep_r[list(rows)] = False
    if cols is not None:
        keep_c[list(cols)] = False
    g, w = got[keep_r][:, keep_c], want[keep_r][:, keep_c]
    assert torch.equal(g, w), (g.float() - w.float()).abs().max()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("M", [1, 129, 255, 257, 300])       # M tails and the CTA-pair edges
def test_gemm_nonfinite_rows_stay_in_their_rows(dtype, M):
    N, K = 200, 320
    a = _randn(M, K, seed=M, scale=0.5).to(dtype)
    w = _randn(N, K, seed=M + 1, scale=0.05).to(dtype)
    bias = _randn(N, seed=M + 2)
    resid = _randn(M, N, seed=M + 3)
    rows = sorted({0, M // 2, min(127, M - 1), min(128, M - 1), M - 1})
    ap = _poison_rows(a, rows, [(7 * i) % K for i in range(len(rows))])
    rp = _poison_rows(resid, rows[::-1], [(5 * i) % N for i in range(len(rows))])
    bp = bias.clone()
    bp[[3, 77, N - 1]] = torch.tensor(POISON, device=DEV)
    for bn in SELECTORS:
        cases = [("bias", dtype, dict(bias=bias), None),
                 ("bias gelu", dtype, dict(bias=bias, gelu=True), None),
                 ("bias scale rowadd f32", torch.float32, dict(bias=bias, scale=-0.5, rowadd=resid[:37]), None),
                 ("in-place resid f32", torch.float32, dict(resid=resid, scale=0.3), dict(resid=rp, scale=0.3))]
        for name, odt, clean_kw, poison_kw in cases:
            want = _check_linear_nf(f"clean {name} M={M}", a, w, odt, bn, **clean_kw)
            got = _check_linear_nf(f"poisoned A {name} M={M}", ap, w, odt, bn, **clean_kw)
            _same_except(got, want, rows=rows)
            if poison_kw is not None:
                got = _check_linear_nf(f"poisoned resid {name} M={M}", a, w, odt, bn, **poison_kw)
                _same_except(got, want, rows=rows)
        got = _check_linear_nf(f"poisoned bias M={M}", a, w, dtype, bn, bias=bp, gelu=True)
        want = _check_linear_nf(f"clean bias M={M}", a, w, dtype, bn, bias=bias, gelu=True)
        _same_except(got, want, cols=[3, 77, N - 1])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [288, 1152, 2304])
def test_norm_nonfinite_rows_stay_in_their_rows(dtype, D):
    from visrag_b200 import ops

    x = _randn(300, D, seed=D, scale=2.0)
    g, b = _randn(D, seed=D + 1), _randn(D, seed=D + 2)
    add = _randn(37, D, seed=D + 3)
    rows = [0, 7, 8, 150, 299]
    xp = _poison_rows(x, rows, [1, D - 1, 64, 0, 5])
    xp[150] = INF                                     # a whole row of inf as well
    for inp, tag in ((x, "clean"), (xp, "poisoned")):
        o1, o2 = ops.layernorm(inp, g, b, 1e-6, add=add, dtype=dtype)
        NF.check(f"{tag} layernorm D={D}", o1, *NF.norm_ref(inp, g, b, 1e-6, rms=False))
        NF.check(f"{tag} layernorm+add D={D}", o2, *NF.norm_ref(inp, g, b, 1e-6, rms=False, add=add))
        o3 = ops.rmsnorm(inp, g, 1e-5, dtype=dtype)
        NF.check(f"{tag} rmsnorm D={D}", o3, *NF.norm_ref(inp, g, None, 1e-5, rms=True))
        if tag == "clean":
            clean = (o1, o2, o3)
    for got, want in zip((o1, o2, o3), clean):
        _same_except(got, want, rows=rows)
        assert not torch.isfinite(got[rows]).all(1).any()


@pytest.mark.parametrize("D", [64, 2304])
def test_pool_norm_poisoned_sequence_stays_in_its_sequence(D):
    """Batch sizes on both sides of the 8-CTA / 4-CTA cluster switch (see test_gpu_batch_invariance.py)."""
    from visrag_b200 import ops

    switch = 5 * torch.cuda.get_device_properties(0).multi_processor_count // 8
    g = _randn(D, seed=D)
    for N in (3, switch, switch + 1):
        rs = np.random.RandomState(N)
        lens = [int(n) for n in rs.randint(1, 70, N)]
        h = _randn(sum(lens), D, seed=N)
        cu = _cu(lens)
        for bad in sorted({0, N // 2, N - 1}):
            hp = h.clone()
            r0, r1 = int(cu[bad]), int(cu[bad + 1])
            hp[r0, 3] = POISON[bad % 3]                 # the cls row and the last row: every pooling reads one
            hp[r1 - 1, D - 1] = POISON[(bad + 1) % 3]
            for pooling in ("wmean", "mean", "lasttoken", "cls"):
                for normalize in (True, False):
                    want = ops.pool_norm(h, g, 1e-5, cu, pooling, normalize)
                    got = ops.pool_norm(hp, g, 1e-5, cu, pooling, normalize)
                    _same_except(got, want, rows=[bad])
                    assert not torch.isfinite(got[bad]).all(), (N, bad, pooling, normalize)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_build_lm_input_nonfinite_rows(dtype):
    from visrag_b200 import ops

    D = 2304
    emb = _randn(512, D, seed=60).to(dtype)
    vis = _randn(128, D, seed=61)
    src = torch.tensor([-6, 0, 1, 127, -512, -1, 5, -300], dtype=torch.int32, device=DEV)
    want = ops.build_lm_input(src, emb, 12.0, vis)
    emb_p, vis_p = emb.clone(), vis.clone()
    emb_p[5, 10] = INF                                   # src -6
    emb_p[299, :] = NAN                                  # src -300
    vis_p[1, 0] = -INF
    got = ops.build_lm_input(src, emb_p, 12.0, vis_p)
    NF.check(f"build_lm_input {dtype}", got, *KB.build_lm_input_ref(src, emb_p, 12.0, vis_p))
    _same_except(got, want, rows=[0, 2, 7])
    assert torch.isinf(got[0, 10]) and torch.isnan(got[7]).all() and got[2, 0] == -INF


# ---------------------------------------------------------------------------------------------- c. attention isolation

# (head stride, head dim, causal, cross): ViT, LM, resampler (64 shared queries, cu_q = None), and the prefix-cache
# layout (causal, each sequence's queries are its last rows: len_q < len_k)
ATT_SHAPES = {"vit": (80, 72, False, False), "lm": (64, 64, True, False), "resampler": (128, 128, False, True),
              "prefix": (64, 64, True, False)}


def _att_inputs(kind, lens, dtype, seed):
    hs, hd, causal, cross = ATT_SHAPES[kind]
    nh, T = 2, sum(lens)
    k = torch.zeros(T, nh, hs, device=DEV)
    v = torch.zeros(T, nh, hs, device=DEV)
    k[..., :hd] = _randn(T, nh, hd, seed=seed, scale=1.5)
    v[..., :hd] = _randn(T, nh, hd, seed=seed + 1)
    k, v = k.reshape(T, nh * hs).to(dtype), v.reshape(T, nh * hs).to(dtype)
    cu_k = _cu(lens)
    if cross:
        q = torch.zeros(128, nh * hs, device=DEV)
        q[:64] = _randn(64, nh * hs, seed=seed + 2)
        return dict(q=q.to(dtype), k=k, v=v, cu_k=cu_k, cu_q=None, max_q=64, lq=[64] * len(lens))
    if kind == "prefix":
        lq = [min(n, 50) for n in lens]
    else:
        lq = list(lens)
    rows = torch.cat([torch.arange(int(cu_k[b + 1]) - lq[b], int(cu_k[b + 1]), device=DEV) for b in range(len(lens))])
    q = torch.zeros(T, nh, hs, device=DEV)
    q[..., :hd] = _randn(T, nh, hd, seed=seed + 2)
    q = q.reshape(T, nh * hs).to(dtype)[rows].contiguous()
    return dict(q=q, k=k, v=v, cu_k=cu_k, cu_q=_cu(lq), max_q=max(lq), lq=lq)


def _att_run(kind, inp, dtype):
    from visrag_b200 import ops

    hs, hd, causal, _ = ATT_SHAPES[kind]
    nh = inp["k"].shape[1] // hs
    lens = (inp["cu_k"][1:] - inp["cu_k"][:-1]).tolist()
    rows = int(inp["cu_q"][-1]) if inp["cu_q"] is not None else len(lens) * inp["max_q"]
    out = torch.zeros(rows, nh * hd, dtype=dtype, device=DEV)
    ops.attention(inp["q"], inp["k"], inp["v"], q_col0=0, k_col0=0, v_col0=0, head_stride=hs, head_dim=hd, heads=nh,
                  batch=len(lens), cu_k=inp["cu_k"], max_k=max(lens), cu_q=inp["cu_q"], max_q=inp["max_q"],
                  causal=causal, scale=hd ** -0.5, out=out)
    return out


def _out_rows(inp, b):
    if inp["cu_q"] is None:
        return b * inp["max_q"], (b + 1) * inp["max_q"]
    return int(inp["cu_q"][b]), int(inp["cu_q"][b + 1])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind", list(ATT_SHAPES))
def test_attention_nonfinite_keys_stay_in_their_sequence(kind, dtype, attn_variant):
    """Sequence 1 of [128 + r, 300, 200] (r = 1, 64, 127, 0: the first sequence's last key tile holds 127, 64, 1 and no
    rows of sequence 1) gets NaN, +inf or -inf in one K and one V row: its first row, rows 63 and 127 (the rows the
    first sequence's last tile reads), or its last two rows (read by no other sequence; sequence 1's own last tile
    reads 84 rows of sequence 2). Sequences 0 and 2 must equal the launch without the poison bit for bit; sequence 1's
    rows that can see the poisoned key match the float64 reference under the checker."""
    hs, hd, causal, cross = ATT_SHAPES[kind]
    f16 = dtype == torch.float16
    for r in (1, 64, 127, 0):
        lens = [128 + r, 300, 200]
        inp = _att_inputs(kind, lens, dtype, seed=r + 10 * len(kind))
        clean = _att_run(kind, inp, dtype)
        k0 = int(inp["cu_k"][1])
        o0, o1 = _out_rows(inp, 1)
        for j in (0, 63, 127, 298, 299):
            for val in POISON:
                p = dict(inp)
                p["k"], p["v"] = inp["k"].clone(), inp["v"].clone()
                for h in range(inp["k"].shape[1] // hs):
                    p["k"][k0 + j, h * hs + (j % hd)] = val
                    p["v"][k0 + j, h * hs + ((j + 5) % hd)] = val
                got = _att_run(kind, p, dtype)
                tag = f"{kind} {dtype} r={r} key {j} = {val}"
                assert torch.equal(got[:o0], clean[:o0]), f"{tag}: the sequence before changed"
                assert torch.equal(got[o1:], clean[o1:]), f"{tag}: the sequence after changed"
                # the poisoned sequence: rows that see key j (causal: query i sees keys <= i + len_k - len_q)
                lq = inp["lq"][1]
                first = max(0, j - (300 - lq)) if causal else 0
                if first >= lq:
                    continue
                nh = inp["k"].shape[1] // hs
                qrows = inp["q"][o0:o1] if not cross else inp["q"][:64]
                for h in range(nh):
                    c = slice(h * hs, h * hs + hd)
                    ref, e = NF.attention_head_ref(qrows[:, c], p["k"][k0:k0 + 300, c], p["v"][k0:k0 + 300, c],
                                                   hd ** -0.5, causal, hs, f16)
                    NF.check(tag, got[o0 + first:o1, h * hd:(h + 1) * hd], ref[first:], e[first:], verbose=False)


# ------------------------------------------------------------------------------------------------------- d. the engine

POISON_CHAR = "§"


def _poisoned_engine_inputs(dtype, seed=7):
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.tokenizer_stub import StubTokenizer
    from visrag_b200.weights import random_state_dict

    cfg = VisRAGConfig.tiny()
    sd = random_state_dict(cfg, seed)
    tok = StubTokenizer(cfg.vocab)
    tid = tok.encode(POISON_CHAR)[-1]
    # bf16: inf in the table. fp16: 1e5 is finite in fp32 and becomes inf where the engine stores its fp16 table.
    sd["llm.model.embed_tokens.weight"][tid] = INF if dtype == torch.bfloat16 else 1e5
    return cfg, sd, tok, tid


def _texts(tok, prefix=""):
    """A: a length that is not a multiple of 128, so its last key tile holds B's first rows; B: the poisoned character
    right after its prefix, inside A's last tile; C: clean."""
    a = prefix + "alpha beta gamma delta " * 7
    while len(tok.encode(a)) % 128 not in range(8, 40):
        a += "x"
    b = prefix + POISON_CHAR + " is the poisoned character"
    c = prefix + "a clean item after the poisoned one"
    assert POISON_CHAR not in a + c
    return a, b, c


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_engine_poisoned_item_leaves_its_batch_alone(dtype):
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.synth import QUERY_PREFIX

    cfg, sd, tok, _ = _poisoned_engine_inputs(dtype)
    for graphs, prefix_cache, prefix in ((False, False, ""), (True, False, ""), (False, True, QUERY_PREFIX),
                                         (True, True, QUERY_PREFIX)):
        eng = VisRAGEngine(cfg, sd, cuda_graphs=graphs, dtype=dtype, prefix_cache=prefix_cache)
        a, b, c = _texts(tok, prefix)
        for rep in range(3):                              # with graphs: eager, capture, replay
            got = eng.encode([a, b, c], [None] * 3, tok)
            want = eng.encode([a, c], [None] * 2, tok)
            tag = (dtype, graphs, prefix_cache, rep)
            assert torch.isfinite(want).all(), tag
            assert not torch.isfinite(got[1]).all(), tag
            assert torch.equal(got[0], want[0]) and torch.equal(got[2], want[1]), tag
        if prefix_cache:
            assert eng.prefix_stats["hits"] > 0, eng.prefix_stats
        if graphs:
            assert eng.graph_stats["replayed"] > 0, eng.graph_stats


def test_inference_loop_stops_on_the_poisoned_item(tmp_path):
    from types import SimpleNamespace

    from visrag_b200 import inference as I
    from visrag_b200.modeling import DRModelForInference, VisRAGRetB200

    cfg, sd, tok, _ = _poisoned_engine_inputs(torch.bfloat16)
    model = DRModelForInference(lm_q=VisRAGRetB200(cfg, sd, "cuda:0"), pooling="wmean", normalize=True)
    args = SimpleNamespace(output_dir=str(tmp_path), per_device_eval_batch_size=3, max_inmem_docs=12, world_size=1,
                           process_index=0, device="cuda:0")
    qset = [{"id": f"q{i}", "text": t, "image": None} for i, t in enumerate(_texts(tok))]
    with pytest.raises(AssertionError, match="model output has nan"):
        I.distributed_parallel_embedding_inference(qset, model, args, "query", False,
                                                   {"tokenizer": tok, "max_inp_length": 2048})
