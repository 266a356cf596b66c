"""An item's result must not depend on what else shares its launch. The engine relies on it: the streaming loop, the CUDA
graph path and query sharding all batch items differently, and an embedding must come out with the same bits either way.
The kernels pick their form from the batch (attention from the longest sequence, pool_norm's cluster size from the batch
size, the GEMM's tile kernel from M), so each check here puts one item alone and inside batches on both sides of every
such switch and asks for torch.equal. pool_norm is also checked against the float64 bound of tests/kernel_bounds.py."""
import numpy as np
import pytest
import torch

from tests import kernel_bounds as KB

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=DEV)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------------------- attention


def _attend(qkv, lens, nh, hd, hs, causal):
    from visrag_b200 import ops

    cu = _cu(lens)
    out = torch.full((qkv.shape[0], nh * hd), float("nan"), dtype=torch.bfloat16, device=DEV)
    ops.attention(qkv, qkv, qkv, q_col0=0, k_col0=nh * hs, v_col0=2 * nh * hs, head_stride=hs, head_dim=hd, heads=nh,
                  batch=len(lens), cu_k=cu, max_k=max(lens), cu_q=cu, max_q=max(lens), causal=causal, scale=hd ** -0.5,
                  out=out)
    return out


def _qkv(T, nh, hd, hs, seed):
    qkv = torch.zeros(T, 3, nh, hs, device=DEV)
    qkv[..., :hd] = _randn(T, 3, nh, hd, seed=seed, scale=2.0)
    return qkv.reshape(T, 3 * nh * hs).bfloat16()


@pytest.mark.parametrize("hs,hd,causal", [(64, 64, True), (80, 72, False)], ids=["lm-causal", "vit-noncausal"])
@pytest.mark.parametrize("L", [1, 2, 17, 63, 64])
def test_attention_short_sequence_alone_equals_in_a_long_batch(hs, hd, causal, L):
    """Alone (max_q <= 64: the one-warpgroup kernel) and between a 200- and a 100-token sequence (max_q > 64: the
    pipelined two-warpgroup kernel): the same bits."""
    nh = 4
    lens = [200, L, 100]
    qkv = _qkv(sum(lens), nh, hd, hs, seed=L + hs)
    batch = _attend(qkv, lens, nh, hd, hs, causal)
    alone = _attend(qkv[200:200 + L].contiguous(), [L], nh, hd, hs, causal)
    assert torch.equal(alone, batch[200:200 + L]), (alone.float() - batch[200:200 + L].float()).abs().max()


@pytest.mark.parametrize("causal", [False, True], ids=["noncausal", "causal"])
@pytest.mark.parametrize("hs,hd", [(64, 64), (80, 72), (128, 128)])
def test_attention_one_warpgroup_kernel_equals_default_dispatch(hs, hd, causal):
    """vr_attention_force_v1(1) runs every shape on the one-warpgroup kernel; the default runs batches with a sequence
    longer than 64 on the two-warpgroup form (pipelined at head stride 64 / 80, sequential at 128). Ragged batches with
    empty, short and long sequences must come out the same from both."""
    from visrag_b200 import _lib as L

    nh = 3
    for lens in ([300, 129, 0, 65, 17, 1036, 1, 64], [2, 63, 64], [128, 5, 257]):
        qkv = _qkv(sum(lens), nh, hd, hs, seed=sum(lens) + hs + causal)
        want = _attend(qkv, lens, nh, hd, hs, causal)
        L.lib().vr_attention_force_v1(1)
        try:
            got = _attend(qkv, lens, nh, hd, hs, causal)
        finally:
            L.lib().vr_attention_force_v1(0)
        assert torch.equal(got, want), (lens, (got.float() - want.float()).abs().max())


# ----------------------------------------------------------------------------------------------------------- pool_norm

POOL_LENS = [0, 1, 5, 16, 17, 33, 68, 300, 700, 2048]
POOL_DIMS = [64, 576, 2304, 4096]          # every instantiation: <= 512, <= 2048, 2304, <= 4096
POOLINGS = ["wmean", "mean", "lasttoken", "cls"]
EPS = 1e-5


def _pool_rows(n, D, seed):
    """LM-like final hidden rows: O(1), mean square ~ eps, |h| ~ 1e3."""
    x = _randn(n, D, seed=seed)
    x[1::3] *= EPS ** 0.5
    x[2::7] *= 1e3
    return x


def _batch_sizes():
    switch = 5 * _sms() // 8              # the largest batch that pool_norm runs with 8-CTA clusters
    return [1, 6, switch, switch + 1, 128, 700]


def _pool_batches(D, N, seed):
    """Batches of N sequences holding the fixed sequences of POOL_LENS (as many per batch as fit, spread between short
    filler sequences): yields (h with a row pitch above D, cu, {fixed index: batch position})."""
    fixed = [_pool_rows(n, D, seed=1000 + i) for i, n in enumerate(POOL_LENS)]
    rs = np.random.RandomState(N + D)
    per = min(N, len(fixed))
    for g0 in range(0, len(fixed), per):
        group = list(range(g0, min(g0 + per, len(fixed))))
        slots = sorted(rs.choice(N, len(group), replace=False).tolist())
        seqs, where, k = [], {}, 0
        for pos in range(N):
            if k < len(group) and pos == slots[k]:
                seqs.append(fixed[group[k]])
                where[group[k]] = pos
                k += 1
            else:
                seqs.append(_randn(int(rs.randint(0, 40)), D, seed=seed + pos))
        lens = [s.shape[0] for s in seqs]
        buf = torch.full((max(sum(lens), 1), D + 12), float("nan"), device=DEV)   # row pitch D + 12: the pad is never read
        h = buf[:, :D]
        h[:sum(lens)] = torch.cat(seqs)
        yield h, _cu(lens), where


@pytest.mark.parametrize("D", POOL_DIMS)
def test_pool_norm_is_independent_of_the_batch(D):
    """The fixed sequences pooled alone and inside batches of 6, the largest batch of 8-CTA clusters, one more (4-CTA
    clusters), 128 (the benchmark's page batch) and 700 (several waves of clusters): the same bits, every pooling,
    normalised or not."""
    from visrag_b200 import ops

    g = _randn(D, seed=D)
    want = {}
    for N in _batch_sizes():
        for h, cu, where in _pool_batches(D, N, seed=N):
            for pooling in POOLINGS:
                for normalize in (True, False):
                    out = ops.pool_norm(h, g, EPS, cu, pooling, normalize)
                    for i, pos in where.items():
                        key = (i, pooling, normalize)
                        if key not in want:
                            want[key] = out[pos].clone()
                        assert torch.equal(out[pos], want[key]), (N, POOL_LENS[i], pooling, normalize,
                                                                  (out[pos] - want[key]).abs().max().item())
    assert len(want) == len(POOL_LENS) * len(POOLINGS) * 2


@pytest.mark.parametrize("D", POOL_DIMS)
def test_pool_norm_within_bounds(D):
    """Against the float64 reference and bound of tests/kernel_bounds.py, with a row pitch above D, at batch sizes on both
    sides of the cluster-size switch."""
    from visrag_b200 import ops

    g = _randn(D, seed=D + 1)
    sw = 5 * _sms() // 8
    for N in (len(POOL_LENS), sw + 1, 700):
        for h, cu, where in _pool_batches(D, N, seed=7 * N):
            for pooling in POOLINGS:
                for normalize in (True, False):
                    out = ops.pool_norm(h, g, EPS, cu, pooling, normalize)
                    pos = sorted(where.values())
                    ref, e = _pool_ref_at(h, g, cu, pos, pooling, normalize)
                    KB.check(f"pool_norm D={D} N={N} {pooling} normalize={normalize}", out[pos], ref, e)


def _pool_ref_at(h, g, cu, pos, pooling, normalize):
    """pool_norm_ref of the batch positions `pos` only (each sequence on its own: the reference has no batch effects)."""
    refs, errs = [], []
    for p in pos:
        r0, r1 = int(cu[p]), int(cu[p + 1])
        ref, e = KB.pool_norm_ref(h[r0:r1], g, EPS, torch.tensor([0, r1 - r0]), pooling, normalize)
        refs.append(ref[0])
        errs.append(e[0])
    return torch.stack(refs), torch.stack(errs)


# ---------------------------------------------------------------------------------------------------------------- GEMM


@pytest.mark.parametrize("M", [1, 64, 128, 129, 300, 8192])
def test_gemm_rows_do_not_depend_on_m(M):
    """Row i of gemm(a[:M]) equals row i of gemm(a) for 8192 rows, for every epilogue the engine uses. The automatic
    choice runs M <= 128 on the single-tile kernels and larger M on the ping-pong CTA pairs."""
    from visrag_b200 import ops, _lib as L

    R, K, N = 8192, 320, 384
    a = _randn(R, K, seed=1, scale=0.5).bfloat16()
    w = _randn(N, K, seed=2, scale=0.05).bfloat16()
    bias = _randn(N, seed=3)
    rowadd = _randn(37, N, seed=4)
    resid = _randn(R, N, seed=5)
    pos = torch.randint(0, 2048, (R,), device=DEV, dtype=torch.int32, generator=_gen(6))
    fr = torch.outer(torch.arange(2048, device=DEV).float(), 1.0 / (10000 ** (torch.arange(0, 64, 2, device=DEV).float() / 64)))
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()

    def resid_gemm(rows):
        x = resid[:rows].clone()
        return ops.gemm(a[:rows], w, scale=0.3, resid=x, out=x, out_dtype=torch.float32, bias=bias)

    runs = {
        "bias bf16": lambda rows: ops.gemm(a[:rows], w, bias=bias),
        "bias gelu bf16": lambda rows: ops.gemm(a[:rows], w, bias=bias, gelu=True),
        "bias rowadd f32": lambda rows: ops.gemm(a[:rows], w, bias=bias, rowadd=rowadd, out_dtype=torch.float32),
        "in-place resid f32, scale": resid_gemm,
        "rope": lambda rows: ops.gemm(a[:rows], w, mode=L.VR_EPI_ROPE, positions=pos[:rows], rope_cos=cos, rope_sin=sin,
                                      rope_cols=128),
        "swiglu": lambda rows: ops.gemm(a[:rows], w, mode=L.VR_EPI_SWIGLU),
    }
    for name, run in runs.items():
        full = run(R)
        part = run(M)
        assert torch.equal(part, full[:M]), (name, (part.float() - full[:M].float()).abs().max().item())
