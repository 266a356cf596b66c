"""The ping-pong GEMM kernel (block_n = 2; 4 = in CTA pairs with the B tile multicast; 5 = plain n-fastest tile order): parity against PyTorch fp32 references, its scheduling edge cases, and bit
identity with the cooperative kernel it replaces on the same inputs (both accumulate the same k16 steps in the same
order; only the tile width and the schedule differ)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tools import check_gemm as CG  # noqa: E402

PP = 2  # block_n selector of the ping-pong kernel
PP_MC = 4  # ... in 2-CTA clusters with the B tile multicast
PP_NFAST = 5  # ... with plain n-fastest tile order
ALL_PP = [PP, PP_MC, PP_NFAST]


@pytest.mark.parametrize("bn", ALL_PP)
def test_pingpong_plain_shapes(bn):
    assert CG.case_basic(bn)


@pytest.mark.parametrize("bn", ALL_PP)
def test_pingpong_fused_epilogues(bn):
    assert CG.case_epilogues(bn)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(bn, M, N, K, seed, **kw):
    from visrag_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    got = ops.gemm(a, w, bias=bias, out_dtype=torch.float32, block_n=bn, **kw)
    torch.cuda.synchronize()
    return CG.report(f"pingpong bn={bn} M={M} N={N} K={K}", got, CG.ref_linear(a, w, bias), 2e-3)


@pytest.mark.parametrize("bn", [PP, PP_MC])
def test_pingpong_scheduling_edges(bn):
    """Tile counts around the persistent grid: each CTA takes tiles blockIdx, blockIdx + grid, ... and hands them to
    its two consumer warpgroups in turn, so a CTA may have one tile (the second warpgroup idles), an odd number (the
    first warpgroup takes the last) or an even number. 128 x 128 tiles. With CTA pairs (bn = 4) a pair takes two M
    tiles of one N tile, so an odd number of M tiles leaves the last pair's second tile entirely past M."""
    sms = _sms()
    ok = True
    ok &= _check(bn, 128, 128, 64, 0)                 # one tile: one CTA, one warpgroup works
    ok &= _check(bn, 384, 256, 128, 1)                # 6 tiles, fewer than the SMs; odd tiles_m (3)
    ok &= _check(bn, 129, 512, 256, 2)                # M = 129: the second row tile holds one valid row
    ok &= _check(bn, 256, 1152, 200, 3)               # K = 200: the last k-block is zero-filled past K
    ok &= _check(bn, 128 * (sms + 1), 128, 128, 4)    # grid + 1 tiles: CTA 0 takes 2 (even), the others 1
    ok &= _check(bn, 128 * (2 * sms + 1), 128, 192, 5)  # 2 grid + 1 tiles: CTA 0 takes 3 (odd), the others 2
    ok &= _check(bn, 128 * 7, 128 * 60, 320, 6)       # 420 tiles, tiles_m odd: 3 or 4 per CTA on 132 SMs
    assert ok


@pytest.mark.parametrize("bn", [PP, PP_MC])
def test_pingpong_l2_slices(bn):
    """Weights larger than the L2 slice budget are cut into N slices (here K = 5760: 14 tiles per slice, so 2304
    columns = 18 tiles make 2 slices of 9, 4608 columns 3 slices of 12, and 2432 columns = 19 tiles 2 slices of
    10 of which the last is one tile narrower)."""
    ok = True
    ok &= _check(bn, 1000, 2304, 5760, 7)
    ok &= _check(bn, 300, 4608, 5760, 8)
    ok &= _check(bn, 700, 2432, 5760, 9)
    assert ok


def _pair(bn_new, M, N, K, old_bn, seed, bias=False, gelu=False, resid=False):
    """(ping-pong output, cooperative-kernel output) on identical inputs; `resid` adds into an fp32 matrix in place."""
    from visrag_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).bfloat16()
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    x0 = torch.randn(M, N, device="cuda", generator=g) if resid else None
    outs = []
    for bn in (bn_new, old_bn):
        if resid:
            x = x0.clone()
            outs.append(ops.gemm(a, w, bias=b, resid=x, out=x, out_dtype=torch.float32, block_n=bn))
        else:
            outs.append(ops.gemm(a, w, bias=b, gelu=gelu, block_n=bn))
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("bn", [PP, PP_MC])
@pytest.mark.parametrize("name,M,N,K,old_bn,kw", [
    ("vit_qkv", 8192, 3840, 1152, 256, {"bias": True}),
    ("vit_proj", 8192, 1152, 1152, 192, {"bias": True, "resid": True}),
    ("vit_fc1", 8192, 4304, 1152, 256, {"bias": True, "gelu": True}),
    ("vit_fc2", 8192, 1152, 4304, 192, {"bias": True, "resid": True}),
    ("lm_o_resid", 1088, 2304, 2304, 256, {"resid": True}),
    ("lm_down_resid", 1088, 2304, 5760, 256, {"resid": True}),
])
def test_pingpong_bit_identical_to_cooperative_linear(name, M, N, K, old_bn, kw, bn):
    new, old = _pair(bn, M, N, K, old_bn, 11, **kw)
    assert torch.equal(new, old), f"{name}: max |diff| {(new.float() - old.float()).abs().max().item():.3e}"


@pytest.mark.parametrize("bn", [PP, PP_MC])
def test_pingpong_bit_identical_to_cooperative_rope_swiglu(bn):
    from visrag_b200 import ops, _lib as L

    g = torch.Generator(device="cuda").manual_seed(12)
    T, H = 1088, 2304
    a = (torch.randn(T, H, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(3 * H, H, device="cuda", generator=g) * 0.03).bfloat16()
    pos = torch.randint(0, 2048, (T,), device="cuda", dtype=torch.int32, generator=g)
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2, device="cuda").float() / 64))
    fr = torch.outer(torch.arange(2048, device="cuda").float(), inv)
    cos, sin = fr.cos().contiguous(), fr.sin().contiguous()
    rope = [ops.gemm(a, w, mode=L.VR_EPI_ROPE, positions=pos, rope_cos=cos, rope_sin=sin, rope_cols=2 * H, block_n=b)
            for b in (bn, 256)]
    wi = (torch.randn(11520, H, device="cuda", generator=g) * 0.03).bfloat16()
    swiglu = [ops.gemm(a, wi, mode=L.VR_EPI_SWIGLU, block_n=b) for b in (bn, 256)]
    torch.cuda.synchronize()
    assert torch.equal(rope[0], rope[1]), (rope[0].float() - rope[1].float()).abs().max().item()
    assert torch.equal(swiglu[0], swiglu[1]), (swiglu[0].float() - swiglu[1].float()).abs().max().item()


def test_auto_selection_uses_pingpong_pairs_above_one_row_tile():
    """block_n=0 picks the ping-pong kernel in CTA pairs (block_n=4) for M > 128, SwiGLU included, and the 64-wide
    cooperative kernel for M <= 128: the automatic result equals the named kernel's bit for bit. (The kernels agree
    bit for bit among themselves too, so this pins the result of the automatic path, not the kernel's identity.)"""
    from visrag_b200 import ops, _lib as L

    g = torch.Generator(device="cuda").manual_seed(13)
    for M, other in ((300, PP_MC), (100, 64)):
        a = (torch.randn(M, 1152, device="cuda", generator=g) * 0.5).bfloat16()
        w = (torch.randn(2304, 1152, device="cuda", generator=g) * 0.03).bfloat16()
        for kw in ({}, {"mode": L.VR_EPI_SWIGLU}):
            auto = ops.gemm(a, w, block_n=0, **kw)
            want = ops.gemm(a, w, block_n=other, **kw)
            torch.cuda.synchronize()
            assert torch.equal(auto, want), (M, kw)
