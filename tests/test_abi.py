"""The C-ABI library loads on a CPU-only box and exports every symbol include/visrag_b200.h declares; argument
validation (which happens before any CUDA call) reports errors through the status code + vr_last_error()."""
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


def test_every_declared_symbol_is_exported(lib):
    syms = G.exported_symbols()
    assert len(syms) >= 15 and "vr_gemm" in syms and "vr_attention" in syms and "vr_score_filter" in syms
    for s in syms:
        assert getattr(lib, s) is not None
    assert lib.vr_abi_version() == 2


def test_errors_are_status_codes_with_messages(lib):
    e = L.GemmEpilogue()
    rc = lib.vr_gemm(None, 0, None, 0, L.VR_BF16, 128, 128, 64, C.byref(e), None)
    assert rc != 0 and b"null pointer" in lib.vr_last_error()
    rc = lib.vr_im2col_norm(1, 1, 15, 14, 14, 1, 640, None)   # h not a multiple of the patch size
    assert rc != 0 and b"bad geometry" in lib.vr_last_error()
    rc = lib.vr_pool_norm(1, 8, 1, 1e-5, 1, 1, 8, 9, 1, 1, None)  # pooling id out of range
    assert rc != 0 and b"pooling" in lib.vr_last_error()
    assert lib.vr_score_list_len() == 16


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(L, "_lib", None)
    monkeypatch.setattr(L, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no fallback"):
        L.lib()


def test_score_plan_is_host_logic_and_bounded():
    """vr_score_ranges (the candidate-buffer sizing the caller needs before vr_score_filter) is pure host arithmetic: it must
    answer without a GPU (the 132 SMs of an H100 SXM assumed) and stay within the rescoring kernel's list limit for any problem size."""
    import ctypes as C

    from visrag_b200 import _lib as L

    lib = L.lib()
    lib.vr_score_ranges.restype = C.c_int32
    lib.vr_score_ranges.argtypes = [C.c_int32, C.c_int64]
    assert lib.vr_score_list_len() == 16
    for nq, nd in ((1, 256), (1, 1_000_000), (5, 1_000_000), (129, 4097), (1000, 10_000), (10_000, 125_000), (100_000, 10_000_000)):
        r = lib.vr_score_ranges(nq, nd)
        assert 1 <= r <= 33, (nq, nd, r)
    assert lib.vr_score_ranges(10_000, 125_000) <= 8          # few lists per query where the rescoring cost matters
    # the work decomposition itself: every (query block, doc tile) is covered exactly once, the launch never exceeds the pairs
    # of a 132-SM device, and the candidate buffers have a spare slot beyond the R real lists (the running threshold)
    import numpy as np

    for nq, nd in ((1, 256), (700, 33_333), (257, 70_001), (2600, 9000), (10_000, 125_000), (3, 300_000)):
        out = (C.c_int32 * 6)()
        assert lib.vr_score_plan(nq, nd, out) == 0
        T, R, QB, items, pairs, lists = list(out)
        assert T == -(-nd // 256) and QB == -(-nq // 256) and 1 <= R <= min(T, 64) and items == R * QB
        assert 1 <= pairs <= min(items, 66) and lists == 2 * lib.vr_score_ranges(nq, nd) and lists >= R + 1
        cover = np.zeros((QB, T), dtype=np.int32)
        for i in range(items):
            b, r = i % QB, i // QB
            cover[b, T * r // R: T * (r + 1) // R] += 1
        assert (cover == 1).all()
