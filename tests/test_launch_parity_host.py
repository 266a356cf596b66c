"""The per-launch checks of tests/launch_parity.py have power: on the CPU, on small random operands, an output that is
the float64 reference rounded to the engine's type at the engine's storage points passes, and an output built with one
plausible wiring mistake of the encode path fails:
  1. the resampler's sincos table built with gh and gw swapped,
  2. the ViT position table resampled bilinear instead of bicubic,
  3. RoPE tables from theta x 1.5,
  4. the ViT LayerNorm eps 1e-5 instead of 1e-6,
  5. mean pooling where wmean was asked for,
  6. the resampler's k and v swapped,
  7. cached-prefix suffix positions not offset by the prefix length,
  8. GELU written with tanh.
Each of these moves the end-to-end embeddings by less than the suite's end-to-end tolerances (cos >= 0.9999 and
max |d| <= 1e-3 on the tiny model); here each fails the check of the one launch it touches."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import kernel_bounds as KB
from tests import launch_parity as LP
from visrag_b200.weights import sincos_2d

DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "f16"]


def _randn(*shape, scale=1.0, mean=0.0, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float32) * scale + mean


def _bf16_exact(t):
    """State-dict values (the synthetic checkpoints hold bf16-exact fp32)."""
    return t.bfloat16().float()


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


# -------------------------------------------------------------------------------------------------- patch embedding


def _pos_table32(pos, gh, gw, mode):
    """The engine's table: resampled in fp32 (encoder._pos_table), bicubic + antialias; `mode` = the mistake's filter."""
    S = math.isqrt(pos.shape[1])
    p = pos.float().reshape(1, S, S, -1).permute(0, 3, 1, 2)
    p = F.interpolate(p, size=(gh, gw), mode=mode, antialias=True)
    return p.permute(0, 2, 3, 1).reshape(gh * gw, -1)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("mode", ["bicubic", "bilinear"])
def test_patch_embedding(mode, dtype):
    """Two slices of a 3 x 7 patch grid (patch 14, 32 channels) from a 9 x 9 position grid: conv2d + bias + the fp32 table
    rounded to fp32 passes; the bilinear table fails."""
    D, P, gh, gw = 32, 14, 3, 7
    px = torch.randint(0, 256, (2, gh * P, gw * P, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    px16 = LP.normalized_pixels(px, dtype)
    w = _bf16_exact(_randn(D, 3, P, P, scale=0.02, seed=2))
    b = _bf16_exact(_randn(D, scale=0.02, seed=3))
    pos = _bf16_exact(_randn(1, 81, D, scale=0.02, seed=4))
    conv = F.conv2d(px16.double(), w.to(dtype).double(), stride=P).permute(0, 2, 3, 1).reshape(-1, D)
    table = _pos_table32(pos, gh, gw, mode).double()
    got = (conv + b.double() + table.repeat(2, 1)).float()
    run = lambda: LP.check_patch(f"patch {mode}", got, px16, w, b, pos)   # noqa: E731
    run() if mode == "bicubic" else _fails(run)


def test_im2col_reference_is_unfold():
    px = torch.randint(0, 256, (2, 28, 42, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    px16 = LP.normalized_pixels(px, torch.bfloat16)
    cols = F.unfold(px16.float(), kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588)
    got = torch.zeros(cols.shape[0], 640, dtype=torch.bfloat16)
    got[:, :588] = cols.bfloat16()
    LP.check_im2col("im2col", got, px16, 588)
    bad = got.clone()
    bad[:, :588] = cols.view(-1, 3, 196).transpose(1, 2).reshape(-1, 588).bfloat16()   # channel-last column order
    _fails(lambda: LP.check_im2col("im2col HWC columns", bad, px16, 588))
    bad = got.clone()
    bad[:, 600] = -0.0
    _fails(lambda: LP.check_im2col("im2col pad -0", bad, px16, 588))


# ------------------------------------------------------------------------------------------------------------- norms


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
def test_vit_layernorm_eps(eps, dtype):
    """ViT residual rows of variance ~0.1 (a patch embedding's): LN with eps 1e-5 moves them by ~5e-5 relative, against
    a bound near 1e-6."""
    D = 288
    x = _randn(64, D, scale=0.3, mean=0.05, seed=6)
    g, b = _bf16_exact(1 + 0.1 * _randn(D, seed=7)), _bf16_exact(0.02 * _randn(D, seed=8))
    X = x.double()
    m = X.mean(1, keepdim=True)
    got = (((X - m) * torch.rsqrt(((X - m) ** 2).mean(1, keepdim=True) + eps)) * g.double() + b.double()).to(dtype)
    run = lambda: LP.check_layernorm(f"ln eps {eps}", got, x, g, b, 1e-6)   # noqa: E731
    run() if eps == 1e-6 else _fails(run)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("swapped", [False, True], ids=["faithful", "gh_gw_swapped"])
def test_resampler_ln_kv_plus_sincos(swapped, dtype):
    """LN_kv(x) and LN_kv(x) + sincos(gh, gw) on a 3 x 5 grid: the engine's table (visrag_b200.weights.sincos_2d) passes
    against the oracle's restatement, the table of a 5 x 3 grid fails."""
    E, gh, gw = 256, 3, 5
    x = _randn(2 * gh * gw, E, scale=0.5, seed=9)
    g, b = _bf16_exact(1 + 0.1 * _randn(E, seed=10)), _bf16_exact(0.02 * _randn(E, seed=11))
    y = F.layer_norm(x.double(), (E,), g.double(), b.double(), 1e-6)
    table = torch.from_numpy(sincos_2d(E, gw, gh) if swapped else sincos_2d(E, gh, gw)).double()
    got2 = (y + table.repeat(2, 1)).to(dtype)
    add = LP.sincos64(E, gh, gw, "cpu")
    run = lambda: LP.check_layernorm("ln_kv", y.to(dtype), x, g, b, 1e-6, add=add, got_add=got2)   # noqa: E731
    run() if not swapped else _fails(run)


# ------------------------------------------------------------------------------------------------------------- GEMMs


def _engine_rope(theta, n):
    """The engine's tables (encoder._load), fp32."""
    inv = 1.0 / (theta ** (torch.arange(0, 64, 2).float() / 64))
    fr = torch.outer(torch.arange(n).float(), inv)
    return fr.cos(), fr.sin()


ROPE_MUTANTS = [None, "theta x 1.5", "suffix positions not offset by P"]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("mut", ROPE_MUTANTS)
def test_rope_qkv(mut, dtype):
    """Two cached-prefix suffixes (P = 58, 7 and 12 own tokens) and one full 40-token sequence, H = 256."""
    H, P = 256, 58
    a = _randn(59, H, seed=12).to(dtype)
    wq, wk, wv = (_bf16_exact(_randn(H, H, scale=0.05, seed=13 + i)) for i in range(3))
    pos = torch.cat([torch.arange(P, P + 7), torch.arange(P, P + 12), torch.arange(40)])
    cos, sin = LP.rope_tables(64, 10000.0, 2048, "cpu")
    ec, es = _engine_rope(15000.0 if mut == "theta x 1.5" else 10000.0, 2048)
    epos = pos.clone()
    if mut == "suffix positions not offset by P":
        epos[:19] -= P
    x = (a.double() @ torch.cat([wq, wk, wv]).to(dtype).double().T).view(59, 12, 2, 32)
    c, s = ec.double()[epos][:, None], es.double()[epos][:, None]
    lo, hi = x[:, :, 0], x[:, :, 1]
    rot = torch.stack([lo * c - hi * s, hi * c + lo * s], 2)
    got = torch.where(torch.arange(12)[None, :, None, None] < 8, rot, x).reshape(59, 3 * H).to(dtype)
    run = lambda: LP.check_rope_qkv(f"rope {mut}", got, a, wq, wk, wv, pos, cos, sin)   # noqa: E731
    run() if mut is None else _fails(run)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("gelu", ["erf", "tanh"])
def test_fc1_gelu_and_pad(gelu, dtype):
    """fc1 + exact-erf GELU on a padded width (the tiny model's 1008 -> 1024, here 112 -> 128): pre-activations of a few
    units, where the tanh form is off by up to 2e-4 relative."""
    D, n, pad = 96, 112, 16
    a = _randn(64, D, seed=20).to(dtype)
    w = _bf16_exact(_randn(n, D, scale=0.25, seed=21))
    b = _bf16_exact(_randn(n, scale=0.5, seed=22))
    pre = a.double() @ w.to(dtype).double().T + b.double()
    y = F.gelu(pre, approximate="tanh" if gelu == "tanh" else "none")
    got = torch.cat([y.to(dtype), torch.zeros(64, pad, dtype=dtype)], 1)
    run = lambda: LP.check_fc1(f"fc1 {gelu}", got, a, w, b)   # noqa: E731
    run() if gelu == "erf" else _fails(run)
    if gelu == "erf":
        bad = got.clone()
        bad[3, n + 2] = 1.0
        _fails(lambda: LP.check_fc1("fc1 pad", bad, a, w, b))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("swapped", [False, True], ids=["faithful", "gate_up_swapped"])
def test_swiglu_from_separate_weights(swapped, dtype):
    H, I = 128, 96
    a = _randn(40, H, seed=30).to(dtype)
    wg, wu = _bf16_exact(_randn(I, H, scale=0.1, seed=31)), _bf16_exact(_randn(I, H, scale=0.1, seed=32))
    g, u = (a.double() @ t.to(dtype).double().T for t in ((wu, wg) if swapped else (wg, wu)))
    got = (F.silu(g) * u).to(dtype)
    run = lambda: LP.check_swiglu("swiglu", got, a, wg, wu)   # noqa: E731
    run() if not swapped else _fails(run)


# --------------------------------------------------------------------------------------------------------- attention


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("swapped", [False, True], ids=["faithful", "k_v_swapped"])
def test_resampler_attention_k_v(swapped, dtype):
    """64 queries over two slices of 45 keys, 2 heads of 128: the output with k and v exchanged fails."""
    E, N = 256, 45
    q = _randn(64, E, seed=40).to(dtype)
    k, v = _randn(2 * N, E, seed=41).to(dtype), _randn(2 * N, E, seed=42).to(dtype)
    cu = torch.tensor([0, N, 2 * N], dtype=torch.int32)
    kw = dict(heads=2, head_dim=128, cu_k=cu, cu_q=None, max_q=64, causal=False, scale=128 ** -0.5)
    kk, vv = (v, k) if swapped else (k, v)
    ref, _ = KB.attention_ref(q, kk, vv, q_col0=0, k_col0=0, v_col0=0, head_stride=128, **kw)
    run = lambda: LP.check_attention("rs attention", ref.to(dtype), q, k, v, **kw)   # noqa: E731
    run() if not swapped else _fails(run)


# ----------------------------------------------------------------------------------------------------------- pooling


@pytest.mark.parametrize("pooling", ["wmean", "mean"])
def test_pool_wmean(pooling):
    """Three items of 5, 17 and 60 rows, wmean asked for: the mean-pooled output fails."""
    lens = [5, 17, 60]
    h = _randn(sum(lens), 256, seed=50)
    g = _bf16_exact(1 + 0.1 * _randn(256, seed=51))
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)
    got = KB.pool_norm_ref(h, g, 1e-5, cu, pooling, True)[0].float()
    run = lambda: LP.check_pool("pool", got, h, g, 1e-5, lens, "wmean")   # noqa: E731
    run() if pooling == "wmean" else _fails(run)


def test_lm_input_scatters_vision_rows_at_the_image_bound():
    emb = _bf16_exact(_randn(50, 32, seed=60))
    vis = [[_randn(4, 32, seed=61), _randn(4, 32, seed=62)], []]
    ids = [np.array([1, 3, 0, 0, 0, 0, 4, 3, 0, 0, 0, 0, 4, 9]), np.array([1, 7, 8])]
    bounds = [np.array([[2, 6], [8, 12]]), np.zeros((0, 2), np.int64)]
    E = emb.bfloat16().double()
    rows = [E[ids[0]] * 12, E[ids[1]] * 12]
    rows[0][2:6], rows[0][8:12] = vis[0][0].double(), vis[0][1].double()
    got = torch.cat(rows).float()
    LP.check_lm_input("lm input", got, emb, 12.0, ids, bounds, vis, torch.bfloat16)
    swapped = [[vis[0][1], vis[0][0]], []]                            # slices scattered in the wrong order
    _fails(lambda: LP.check_lm_input("lm input, slices swapped", got, emb, 12.0, ids, bounds, swapped, torch.bfloat16))
