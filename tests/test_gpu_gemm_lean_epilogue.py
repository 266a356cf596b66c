"""The ping-pong kernel's lean 16-bit LINEAR epilogue (bias [+ GELU], scale 1, no row add, no residual: ViT qkv and fc1,
the resampler's k / v). It must give the bits of the cooperative kernel's generic epilogue on interior and edge tiles, in
bf16 and fp16, and vr_gemm must pick it only for that epilogue: a NULL bias, a scale, a row add or a residual keep the
generic one. Outputs are compared as raw 16-bit patterns, so -0 and +0 count as different."""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

PP, PP_MC, PP_NFAST = 2, 4, 5  # ping-pong block_n selectors; 4 (CTA pairs) is what vr_gemm picks for M > 128
COOP = 128  # the cooperative kernel, 128 x 128 tiles

SHAPES = [
    (1000, 4352, 1152),  # ViT fc1 at reduced M (M not a multiple of 128: the last row tile is partial)
    (768, 3840, 1152),   # ViT qkv
    (640, 2304, 2304),   # resampler k / v
    (300, 136, 200),     # N = 136: the last N tile holds one 8-column group; K = 200: a partial k-block
]


def _bits(t):
    return t.view(torch.int16)


def _case(M, N, K, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    return a, w, bias


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_lean_epilogue_bit_identical_to_cooperative(M, N, K, gelu, dtype):
    from visrag_b200 import ops

    a, w, bias = _case(M, N, K, dtype, M + N + K)
    ref = ops.gemm(a, w, bias=bias, gelu=gelu, block_n=COOP)
    for bn in (PP_MC, PP, PP_NFAST, 0):
        got = ops.gemm(a, w, bias=bias, gelu=gelu, block_n=bn)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(ref)), \
            f"block_n={bn}: max |diff| {(got.float() - ref.float()).abs().max().item():.3e}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("gelu", [False, True])
def test_zero_accumulators_and_signed_zero_bias(gelu, dtype):
    """Rows of A that are zero give zero accumulators (against a negative weight every product is -0; the H100's
    tensor cores return their sum as +0), and a bias of -0 or +0 on some columns: the sign of each zero output must
    be the generic epilogue's."""
    from visrag_b200 import ops

    M, N, K = 384, 256, 128
    a, w, bias = _case(M, N, K, dtype, 7)
    a[::3] = 0
    w = -w.abs() - 0.01
    bias[::4] = -0.0
    bias[1::4] = 0.0
    for b in (bias, None):
        ref = ops.gemm(a, w, bias=b, gelu=gelu, block_n=COOP)
        got = ops.gemm(a, w, bias=b, gelu=gelu, block_n=PP_MC)
        torch.cuda.synchronize()
        assert (got[::3, ::4] == 0).all() and (got[::3, 1::4] == 0).all()
        assert torch.equal(_bits(got), _bits(ref))


def _pingpong_lean_flags(fn):
    """Run fn under the profiler and return, for each ping-pong launch, whether it was the lean instantiation (the last
    template argument of gemm_pingpong_kernel)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    flags = []
    for ev in prof.events():
        name = ev.name
        if "gemm_pingpong_kernel" not in name:
            continue
        m = re.search(r"gemm_pingpong_kernel<([^>]*)>", name)
        if m:
            flags.append(m.group(1).split(",")[-1].strip() == "true")
        else:  # mangled: ..._kernelILb0ELi0ELb0ELb1ELi2ELb1EEEv...
            m = re.search(r"gemm_pingpong_kernelI(.*?)EEv", name)
            flags.append(m.group(1).endswith("Lb1E"))
    return flags


def test_only_the_bias_epilogue_takes_the_lean_path():
    from visrag_b200 import ops

    M, N, K = 512, 384, 256
    a, w, bias = _case(M, N, K, torch.bfloat16, 9)
    resid = torch.randn(M, N, device="cuda")
    rowadd = torch.randn(16, N, device="cuda")
    lean = [dict(bias=bias), dict(bias=bias, gelu=True)]
    generic = [dict(), dict(gelu=True), dict(bias=bias, scale=0.5), dict(bias=bias, gelu=True, scale=2.0),
               dict(bias=bias, rowadd=rowadd), dict(bias=bias, resid=resid)]
    for kw, want in [(kw, True) for kw in lean] + [(kw, False) for kw in generic]:
        outs = {}

        def run():
            for bn in (PP_MC, COOP):
                outs[bn] = ops.gemm(a, w, block_n=bn, **kw)

        assert _pingpong_lean_flags(run) == [want], kw
        assert torch.equal(_bits(outs[PP_MC]), _bits(outs[COOP])), kw
