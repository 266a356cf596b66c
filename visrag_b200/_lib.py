"""ctypes binding of the C-ABI library ``libvisrag_b200.so`` (include/visrag_b200.h).

PyTorch is plumbing here: it owns device memory and streams; every kernel is launched through the C ABI
with raw device pointers. There is NO fallback: if the shared library is missing, loading raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VR_LIB", os.path.join(_HERE, "libvisrag_b200.so"))  # VR_LIB: debug builds only

VR_BF16, VR_F16, VR_F32 = 0, 1, 2
VR_EPI_LINEAR, VR_EPI_ROPE, VR_EPI_SWIGLU = 0, 1, 2


class GemmEpilogue(C.Structure):
    """Mirror of ``vr_gemm_epilogue``."""

    _fields_ = [
        ("mode", C.c_int32),
        ("out_dtype", C.c_int32),
        ("act_gelu", C.c_int32),
        ("scale", C.c_float),
        ("bias", C.c_void_p),
        ("resid", C.c_void_p),
        ("rowadd", C.c_void_p),
        ("rowadd_period", C.c_int32),
        ("positions", C.c_void_p),
        ("rope_cos", C.c_void_p),
        ("rope_sin", C.c_void_p),
        ("rope_cols", C.c_int32),
        ("out", C.c_void_p),
        ("ldo", C.c_int64),
    ]


class AttnParams(C.Structure):
    """Mirror of ``vr_attn_params``."""

    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_int64), ("q_rows", C.c_int64),
        ("k", C.c_void_p), ("ldk", C.c_int64),
        ("v", C.c_void_p), ("ldv", C.c_int64), ("kv_rows", C.c_int64),
        ("q_col0", C.c_int32), ("k_col0", C.c_int32), ("v_col0", C.c_int32),
        ("head_stride", C.c_int32), ("head_dim", C.c_int32),
        ("heads", C.c_int32), ("batch", C.c_int32),
        ("cu_q", C.c_void_p), ("cu_k", C.c_void_p),
        ("max_q", C.c_int32), ("max_k", C.c_int32),
        ("causal", C.c_int32), ("scale", C.c_float),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("flags", C.c_int32),
    ]


class DocMasks(C.Structure):
    """Mirror of ``vr_doc_masks``: a mask set, query row r searching mask of_query[r] (NULL: mask 0)."""

    _fields_ = [
        ("words", C.c_void_p),
        ("pitch", C.c_int64),
        ("of_query", C.c_void_p),
        ("count", C.c_int32),
    ]


class DocLists(C.Structure):
    """Mirror of ``vr_doc_lists``: a list set in CSR form, query row r scoring list of_query[r] (NULL: list 0)."""

    _fields_ = [
        ("offsets", C.c_void_p),
        ("ids", C.c_void_p),
        ("count", C.c_int32),
        ("of_query", C.c_void_p),
    ]


VR_ATTN_V_ONES_COLUMN = 1
VR_ATTN_F16 = 2  # q / k / v / out are fp16
VR_FUSE_SUM, VR_FUSE_RRF = 0, 1  # vr_fuse_rows modes

_lib: Optional[C.CDLL] = None


def _declare(lib: C.CDLL) -> None:
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    lib.vr_last_error.restype = C.c_char_p
    lib.vr_last_error.argtypes = []
    lib.vr_abi_version.restype = i32
    lib.vr_abi_version.argtypes = []
    lib.vr_gemm.restype = i32
    lib.vr_gemm.argtypes = [vp, i64, vp, i64, i32, i32, i32, i32, C.POINTER(GemmEpilogue), vp]
    lib.vr_gemm_tuned.restype = i32
    lib.vr_gemm_tuned.argtypes = [vp, i64, vp, i64, i32, i32, i32, i32, C.POINTER(GemmEpilogue), i32, vp]
    lib.vr_attention.restype = i32
    lib.vr_attention.argtypes = [C.POINTER(AttnParams), vp]
    lib.vr_attention_force_v1.restype = None
    lib.vr_attention_force_v1.argtypes = [i32]
    lib.vr_im2col_norm.restype = i32
    lib.vr_im2col_norm.argtypes = [vp, i32, i32, i32, i32, vp, i64, vp]
    lib.vr_im2col_norm_ex.restype = i32
    lib.vr_im2col_norm_ex.argtypes = [vp, i32, i32, i32, i32, vp, i64, i32, vp]
    lib.vr_layernorm.restype = i32
    lib.vr_layernorm.argtypes = [vp, i64, vp, vp, f32, i32, i32, vp, i64, vp, vp, i32, vp]
    lib.vr_layernorm_ex.restype = i32
    lib.vr_layernorm_ex.argtypes = [vp, i64, vp, vp, f32, i32, i32, vp, i64, vp, vp, i32, i32, vp]
    lib.vr_rmsnorm.restype = i32
    lib.vr_rmsnorm.argtypes = [vp, i64, vp, f32, i32, i32, vp, i64, vp]
    lib.vr_rmsnorm_ex.restype = i32
    lib.vr_rmsnorm_ex.argtypes = [vp, i64, vp, f32, i32, i32, vp, i64, i32, vp]
    lib.vr_build_lm_input.restype = i32
    lib.vr_build_lm_input.argtypes = [vp, i32, i32, vp, f32, vp, i64, vp, i64, vp]
    lib.vr_build_lm_input_ex.restype = i32
    lib.vr_build_lm_input_ex.argtypes = [vp, i32, i32, vp, i32, f32, vp, i64, vp, i64, vp]
    lib.vr_score_ranges.restype = i32
    lib.vr_score_ranges.argtypes = [i32, i64]
    lib.vr_score_list_len.restype = i32
    lib.vr_score_list_len.argtypes = []
    lib.vr_score_plan.restype = i32
    lib.vr_score_plan.argtypes = [i32, i64, vp]
    lib.vr_f32_to_f16_rows.restype = i32
    lib.vr_f32_to_f16_rows.argtypes = [vp, i64, i32, vp, vp, vp, vp]
    lib.vr_score_filter.restype = i32
    lib.vr_score_filter.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp]
    lib.vr_score_rescore.restype = i32
    lib.vr_score_rescore.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, i32, i64, vp, vp, vp, vp]
    lib.vr_score_exact.restype = i32
    lib.vr_score_exact.argtypes = [vp, i32, vp, i64, i32, vp, vp]
    lib.vr_resample_u8.restype = i32
    lib.vr_resample_u8.argtypes = [vp, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp]
    lib.vr_topk_rows_chunked.restype = i32
    lib.vr_topk_rows_chunked.argtypes = [vp, i32, i64, i32, i64, i32, vp, vp, vp, vp, vp]
    lib.vr_topk_rows.restype = i32
    lib.vr_topk_rows.argtypes = [vp, vp, i32, i64, i32, i64, vp, vp, vp]
    lib.vr_score_filter_masked.restype = i32
    lib.vr_score_filter_masked.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, vp]
    lib.vr_topk_rows_masked.restype = i32
    lib.vr_topk_rows_masked.argtypes = [vp, vp, i32, i64, i32, i64, vp, vp, vp, vp]
    lib.vr_topk_rows_chunked_masked.restype = i32
    lib.vr_topk_rows_chunked_masked.argtypes = [vp, i32, i64, i32, i64, i32, vp, vp, vp, vp, vp, vp]
    lib.vr_score_filter_groups.restype = i32
    lib.vr_score_filter_groups.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, vp, vp]
    lib.vr_score_rescore_groups.restype = i32
    lib.vr_score_rescore_groups.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, i32, i64, vp, vp, vp,
                                            vp, vp]
    lib.vr_group_topk_ws_bytes.restype = i64
    lib.vr_group_topk_ws_bytes.argtypes = [i32, i32, i32, i32]
    lib.vr_group_topk_rows.restype = i32
    lib.vr_group_topk_rows.argtypes = [vp, i32, i64, vp, i32, vp, i32, i64, i32, vp, i64, vp, vp, vp, vp]
    lib.vr_merge_group_topk.restype = i32
    lib.vr_merge_group_topk.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp]
    dm = C.POINTER(DocMasks)
    lib.vr_score_filter_masks.restype = i32
    lib.vr_score_filter_masks.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, dm, vp]
    lib.vr_score_filter_groups_masks.restype = i32
    lib.vr_score_filter_groups_masks.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, dm, vp]
    lib.vr_score_rescore_groups_masks.restype = i32
    lib.vr_score_rescore_groups_masks.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp, vp, vp, i32, dm, vp, i32, i64, vp,
                                                  vp, vp, vp, vp]
    lib.vr_topk_rows_masks.restype = i32
    lib.vr_topk_rows_masks.argtypes = [vp, vp, i32, i64, i32, i64, vp, vp, dm, vp]
    lib.vr_topk_rows_chunked_masks.restype = i32
    lib.vr_topk_rows_chunked_masks.argtypes = [vp, i32, i64, i32, i64, i32, vp, vp, vp, vp, dm, vp]
    lib.vr_select_rows.restype = i32
    lib.vr_select_rows.argtypes = [vp, vp, i32, i64, i32, i64, vp, vp, vp]
    lib.vr_select_rows_masks.restype = i32
    lib.vr_select_rows_masks.argtypes = [vp, vp, i32, i64, i32, i64, vp, vp, dm, vp]
    lib.vr_select_rows_chunked.restype = i32
    lib.vr_select_rows_chunked.argtypes = [vp, i32, i64, i32, i64, i32, vp, vp, vp, vp, vp]
    lib.vr_select_rows_chunked_masks.restype = i32
    lib.vr_select_rows_chunked_masks.argtypes = [vp, i32, i64, i32, i64, i32, vp, vp, vp, vp, dm, vp]
    lib.vr_group_topk_rows_masks.restype = i32
    lib.vr_group_topk_rows_masks.argtypes = [vp, i32, i64, vp, i32, dm, i32, i64, i32, vp, i64, vp, vp, vp, vp]
    lib.vr_score_lists.restype = i32
    lib.vr_score_lists.argtypes = [vp, i32, vp, i64, i32, C.POINTER(DocLists), i32, vp, vp, vp, vp, vp, vp]
    lib.vr_score_filter_range.restype = i32
    lib.vr_score_filter_range.argtypes = [vp, i32, vp, i64, i32, vp, vp, vp, dm, i32, vp, vp, vp]
    lib.vr_score_rescore_range.restype = i32
    lib.vr_score_rescore_range.argtypes = [vp, i32, vp, i64, i32, vp, i32, vp, vp, vp, vp, vp, vp]
    lib.vr_range_rows.restype = i32
    lib.vr_range_rows.argtypes = [vp, i32, i64, vp, dm, i64, vp, vp, vp, vp]
    lib.vr_range_sort_ws_bytes.restype = i64
    lib.vr_range_sort_ws_bytes.argtypes = [i32, i32]
    lib.vr_range_sort.restype = i32
    lib.vr_range_sort.argtypes = [vp, vp, i64, vp, i32, vp, vp, i32, i64, vp, i64, vp, vp, vp]
    lib.vr_range_groups_ws_bytes.restype = i64
    lib.vr_range_groups_ws_bytes.argtypes = [i32, i32]
    lib.vr_range_groups.restype = i32
    lib.vr_range_groups.argtypes = [vp, vp, i64, vp, i32, i32, vp, i64, i32, vp, i64, vp, vp, vp, vp]
    lib.vr_mmr_select.restype = i32
    lib.vr_mmr_select.argtypes = [vp, i64, i32, vp, vp, i32, i32, vp, i32, i64, vp, vp, vp]
    lib.vr_group_pages_topm.restype = i32
    lib.vr_group_pages_topm.argtypes = [vp, i32, vp, i64, i32, vp, i32, vp, vp, i32, dm, i32, i32, i32, i64, vp, vp, vp]
    lib.vr_fuse_rows.restype = i32
    lib.vr_fuse_rows.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, i64, i32, f32, i32, i64, vp, vp, vp, vp]
    lib.vr_group_pages_fused.restype = i32
    lib.vr_group_pages_fused.argtypes = [vp, i32, vp, i64, i32, vp, i32, vp, vp, i32, dm, vp, vp, vp, f32, i32, i32, i64, vp, vp,
                                         vp]
    lib.vr_pool_norm.restype = i32
    lib.vr_pool_norm.argtypes = [vp, i64, vp, f32, vp, i32, i32, i32, i32, vp, vp]
    lib.vr_prefix_rows.restype = i32
    lib.vr_prefix_rows.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, i32, i32, i32, i32, i32, vp]


def lib() -> C.CDLL:
    """Load (once) and return the C-ABI library. Raises if it was not built: no CPU/PyTorch fallback exists."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C visrag_b200/csrc`). visrag_b200 has no fallback path."
            )
        _lib = C.CDLL(LIB_PATH)
        _declare(_lib)
    return _lib


LAUNCHES = 0  # number of library kernel launches issued (bench.py reports it as gpu_launches)


def check(rc: int) -> None:
    global LAUNCHES
    LAUNCHES += 1
    if rc != 0:
        raise RuntimeError(f"visrag_b200: {lib().vr_last_error().decode()} (status {rc})")


def ptr(t) -> Optional[int]:
    """Device pointer of a torch tensor (None passes NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr() -> int:
    """The CURRENT device's current stream. Kernels must be launched with the device that owns their buffers current:
    every public entry point (engine, retriever, knowledge base) enters `on_device(...)`, and the op wrappers refuse tensors
    of another device (`check_device`) instead of launching on the wrong GPU."""
    import torch

    return torch.cuda.current_stream().cuda_stream


def norm_device(device):
    """torch.device with an explicit index ('cuda' -> the current device)."""
    import torch

    d = torch.device(device)
    if d.type != "cuda":
        raise ValueError(f"visrag_b200 runs on CUDA devices only (got {d})")
    return d if d.index is not None else torch.device("cuda", torch.cuda.current_device())


class on_device:
    """Context manager: make `device` current (cudaSetDevice) for the launches inside; no-op when it already is."""

    def __init__(self, device):
        self.idx = norm_device(device).index
        self.prev = None

    def __enter__(self):
        import torch

        cur = torch.cuda.current_device()
        if cur != self.idx:
            self.prev = cur
            torch.cuda.set_device(self.idx)
        return self

    def __exit__(self, *exc):
        if self.prev is not None:
            import torch

            torch.cuda.set_device(self.prev)
        return False


def check_device(t) -> None:
    import torch

    if t.is_cuda and t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"visrag_b200: tensor lives on cuda:{t.device.index} but cuda:{torch.cuda.current_device()} is current; "
                           "wrap the call in `with visrag_b200._lib.on_device(tensor.device):` (the engine / retriever entry points do)")
