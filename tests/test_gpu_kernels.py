"""Kernel-level parity on the H100 (through the C ABI) against plain PyTorch fp32 references of the same op.
Tolerances: fp32-output paths 2e-3 relative to max|ref| (bf16 operands, fp32 accumulate); bf16-output paths 1e-2
(one bf16 rounding of the result)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tools import check_encode as CE  # noqa: E402
from tools import check_gemm as CG  # noqa: E402


@pytest.mark.parametrize("bn", [256, 128, 64, 192, 3, 0])  # tile width; 3 = feature-major accumulator kernel, 0 = what vr_gemm picks
def test_gemm_plain_shapes(bn):
    assert CG.case_basic(bn)


@pytest.mark.parametrize("bn", [256, 128, 64, 192, 3, 0])
def test_gemm_fused_epilogues(bn):
    assert CG.case_epilogues(bn)


def test_elementwise_kernels():
    assert CE.stage_elementwise()


def test_attention_three_shapes():
    assert CE.stage_attention()          # two-warpgroup (128 queries per CTA) kernel wherever max_q > 64


def test_attention_three_shapes_single_tile_kernel():
    assert CE.stage_attention(force_v1=True)


def test_gemm_rejects_bad_arguments():
    from visrag_b200 import ops

    a = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(100, 64, device="cuda", dtype=torch.bfloat16)  # N not a multiple of 8
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.gemm(a, w)
    with pytest.raises(ValueError):
        ops.gemm(a.float(), w)
