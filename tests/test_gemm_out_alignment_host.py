"""vr_gemm refuses a LINEAR output whose base is not 16-byte aligned (the ping-pong kernel stores 16-bit outputs 16 bytes
at a time) by argument validation alone, before any CUDA call; the pointers here are not device memory."""
import ctypes as C
import os

import pytest

import __graft_entry__ as G
from visrag_b200 import _lib as L


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


@pytest.mark.parametrize("block_n", [0, 2, 4, 5, 128])
@pytest.mark.parametrize("out", [8, 4, 16 + 1024 + 2])
def test_misaligned_linear_output_is_refused(lib, block_n, out):
    e = L.GemmEpilogue()
    e.mode, e.out_dtype, e.scale = L.VR_EPI_LINEAR, L.VR_BF16, 1.0
    e.out, e.ldo = out, 128
    rc = lib.vr_gemm_tuned(16, 64, 16, 64, L.VR_BF16, 256, 128, 64, C.byref(e), block_n, None)
    msg = lib.vr_last_error().decode()
    assert rc == 2 and "LINEAR out must be 16-byte aligned" in msg, msg
