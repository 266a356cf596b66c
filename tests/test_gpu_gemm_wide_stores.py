"""The ping-pong GEMM stores a 16-bit LINEAR output 16 bytes per thread after a transpose across each quad of lanes:
bit identity with the cooperative kernel (which stores each column pair by itself) at widths whose last tile is
partial, and nothing written past N or past M when `out` is a view inside a wider buffer."""
import pytest
import torch

pytestmark = pytest.mark.gpu

PP, PP_MC, PP_NFAST, COOP = 2, 4, 5, 128
M_ODD = 4 * 128 + 37  # 5 row tiles: the last CTA pair's second tile lies past M


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("N", [200, 4304, 4352])
@pytest.mark.parametrize("gelu", [False, True])
def test_16bit_output_equals_cooperative_kernel_in_a_padded_view(dtype, N, gelu):
    from visrag_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(N)
    a = (torch.randn(M_ODD, 256, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(N, 256, device="cuda", generator=g) * 0.05).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    ldo, rows, poison = N + 24, M_ODD + 40, -7.0
    outs = {}
    for bn in (COOP, PP, PP_MC, PP_NFAST):
        buf = torch.full((rows, ldo), poison, dtype=dtype, device="cuda")
        ops.gemm(a, w, bias=bias, gelu=gelu, scale=0.75, out=buf[:M_ODD, :N], block_n=bn)
        outs[bn] = buf
    torch.cuda.synchronize()
    ref = outs[COOP]
    for bn in (PP, PP_MC, PP_NFAST):
        got = outs[bn]
        assert torch.equal(got[:M_ODD, :N], ref[:M_ODD, :N]), (bn, (got[:M_ODD, :N].float() - ref[:M_ODD, :N].float()).abs().max().item())
        assert (got[:, N:] == poison).all() and (got[M_ODD:, :] == poison).all(), bn
