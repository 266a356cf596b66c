"""Every C entry point refuses a pointer below the alignment of the widest vector access its kernels make to it, by
argument validation alone, before any CUDA call. The pointers here are fake (no device memory behind them): each call
gets valid arguments except for one base set just below its alignment (+4 for 8- and 16-byte accesses, +2 for 4-byte
ones) and must return 2 with a message naming that argument. The module skips when a CUDA device is visible, so that a
refusal that was forgotten can never launch a kernel on a fake pointer.

TABLE lists each entry point's pointers with the alignment its kernels need, derived from the kernel source; it must
agree with the "Alignment (bytes) of ..." lines of include/visrag_b200.h.
"""
import ctypes as C
import os
import re

import pytest
import torch

import __graft_entry__ as G
from visrag_b200 import _lib as L

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: run only where no CUDA device is visible")

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "visrag_b200.h")

# (entry point, pointer, qualifier) -> bytes, with the access that sets it
TABLE = {
    ("vr_gemm", "A", None): 16,                        # TMA source
    ("vr_gemm", "B", None): 16,                        # TMA source
    ("vr_gemm", "bias", None): 8,                      # float2 loads (epi_linear2, pp_epilogue_linear)
    ("vr_gemm", "rowadd", None): 8,                    # float2 loads
    ("vr_gemm", "resid", None): 8,                     # float2 loads
    ("vr_gemm", "rope_cos", None): 8,                  # float2 loads (epi_rope2)
    ("vr_gemm", "rope_sin", None): 8,                  # float2 loads
    ("vr_gemm", "positions", None): 4,                 # int32 loads
    ("vr_gemm", "out", "LINEAR"): 16,                  # uint4 stores of the ping-pong 16-bit epilogues
    ("vr_gemm", "out", "ROPE, SWIGLU"): 4,             # 16-bit pair stores
    ("vr_attention", "q", None): 16,                   # TMA sources
    ("vr_attention", "k", None): 16,
    ("vr_attention", "v", None): 16,
    ("vr_attention", "cu_q", None): 4,                 # int32 loads
    ("vr_attention", "cu_k", None): 4,
    ("vr_attention", "out", None): 4,                  # 16-bit pair stores (att_store)
    ("vr_im2col_norm", "out", None): 16,               # uint4 stores
    ("vr_layernorm", "x", None): 16,                   # float4 loads
    ("vr_layernorm", "gamma", None): 16,
    ("vr_layernorm", "beta", None): 16,
    ("vr_layernorm", "add", None): 16,
    ("vr_layernorm", "out", None): 8,                  # uint2 stores
    ("vr_layernorm", "out2", None): 8,
    ("vr_rmsnorm", "x", None): 16,
    ("vr_rmsnorm", "gamma", None): 16,
    ("vr_rmsnorm", "out", None): 8,
    ("vr_build_lm_input", "src", None): 4,             # int32 loads
    ("vr_build_lm_input", "embed", None): 8,           # uint2 loads
    ("vr_build_lm_input", "vision", None): 16,         # float4 loads
    ("vr_build_lm_input", "h", None): 16,              # float4 stores
    ("vr_pool_norm", "h", None): 16,                   # float4 loads
    ("vr_pool_norm", "gamma", None): 16,
    ("vr_pool_norm", "cu", None): 4,
    ("vr_pool_norm", "reps", None): 16,                # float4 stores
    ("vr_prefix_rows", "prefix", None): 16,            # uint4 copies
    ("vr_prefix_rows", "rows", None): 16,
    ("vr_prefix_rows", "out", None): 16,
    ("vr_prefix_rows", "cu_rows", None): 4,
    ("vr_prefix_rows", "cu_out", None): 4,
    ("vr_f32_to_f16_rows", "src", None): 16,           # float4 loads
    ("vr_f32_to_f16_rows", "dst_f16", None): 8,        # uint2 stores
    ("vr_score_filter", "q_f16", None): 16,            # TMA sources
    ("vr_score_filter", "d_f16", None): 16,
    ("vr_score_filter", "cand_scores", None): 16,      # float4 stores
    ("vr_score_filter", "cand_ids", None): 16,         # int4 stores
    ("vr_score_filter_masked", "q_f16", None): 16,
    ("vr_score_filter_masked", "d_f16", None): 16,
    ("vr_score_filter_masked", "cand_scores", None): 16,
    ("vr_score_filter_masked", "cand_ids", None): 16,
    ("vr_score_filter_masked", "doc_mask", None): 4,   # uint32 words
    ("vr_score_filter_groups", "q_f16", None): 16,
    ("vr_score_filter_groups", "d_f16", None): 16,
    ("vr_score_filter_groups", "cand_scores", None): 16,
    ("vr_score_filter_groups", "cand_ids", None): 16,
    ("vr_score_filter_groups", "doc_groups", None): 4,
    ("vr_score_filter_groups", "doc_mask", None): 4,
    ("vr_score_rescore", "d_f32", None): 16,           # float4 rows (score_row_dot)
    ("vr_score_exact", "d_f32", None): 16,             # float4 rows
    ("vr_score_rescore_groups", "d_f32", None): 16,
    ("vr_score_rescore_groups", "doc_groups", None): 4,
    ("vr_score_rescore_groups", "group_offsets", None): 4,
    ("vr_score_rescore_groups", "group_pages", None): 4,
    ("vr_score_rescore_groups", "doc_mask", None): 4,
}


def header_table():
    """The "Alignment (bytes) of <entry>: name n [(qualifier)], ..." lines of the header."""
    text = open(HEADER).read()
    out = {}
    for m in re.finditer(r"Alignment \(bytes\) of (\w+): (.*)", text):
        entry, body = m.group(1), m.group(2)
        for name, n, qual in re.findall(r"(\w+) (\d+)(?: \(([^)]*)\))?", body):
            out[(entry, name, qual or None)] = int(n)
    return out


def test_alignment_table_matches_header():
    assert header_table() == TABLE


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        G.build()
    return L.lib()


# fake device pointers: distinct, 256-byte aligned, far from zero
_BASE = {}


def _p(name):
    return _BASE.setdefault(name, 0x7F0000000000 + 0x100000 * (len(_BASE) + 1))


def _gemm(lib, ptrs, qual):
    e = L.GemmEpilogue()
    e.mode = L.VR_EPI_ROPE if qual == "ROPE, SWIGLU" else L.VR_EPI_LINEAR
    e.out_dtype, e.scale = L.VR_F32, 1.0
    e.bias, e.rowadd, e.resid, e.rowadd_period = ptrs["bias"], ptrs["rowadd"], ptrs["resid"], 37
    e.positions, e.rope_cos, e.rope_sin, e.rope_cols = ptrs["positions"], ptrs["rope_cos"], ptrs["rope_sin"], 64
    e.out, e.ldo = ptrs["out"], 128
    if e.mode == L.VR_EPI_ROPE:
        e.bias = e.rowadd = e.resid = None
    return lib.vr_gemm_tuned(ptrs["A"], 64, ptrs["B"], 64, L.VR_BF16, 256, 128, 64, C.byref(e), 0, None)


def _attention(lib, ptrs, qual):
    p = L.AttnParams()
    p.q, p.ldq, p.q_rows = ptrs["q"], 192, 128
    p.k, p.ldk = ptrs["k"], 192
    p.v, p.ldv, p.kv_rows = ptrs["v"], 192, 128
    p.q_col0, p.k_col0, p.v_col0 = 0, 64, 128
    p.head_stride, p.head_dim, p.heads, p.batch = 64, 64, 1, 1
    p.cu_q, p.cu_k, p.max_q, p.max_k = ptrs["cu_q"], ptrs["cu_k"], 128, 128
    p.causal, p.scale, p.out, p.ldo, p.flags = 1, 0.125, ptrs["out"], 64, 0
    return lib.vr_attention(C.byref(p), None)


def _score_args(lib, nq=4, nd=1000):
    return nq, nd, 64, lib.vr_score_ranges(nq, nd)


def _filter(lib, ptrs, qual, masked):
    nq, nd, dim, ranges = _score_args(lib)
    if masked:
        return lib.vr_score_filter_masked(ptrs["q_f16"], nq, ptrs["d_f16"], nd, dim, ranges, ptrs["cand_scores"],
                                          ptrs["cand_ids"], ptrs["doc_mask"], None)
    return lib.vr_score_filter(ptrs["q_f16"], nq, ptrs["d_f16"], nd, dim, ranges, ptrs["cand_scores"], ptrs["cand_ids"], None)


def _filter_groups(lib, ptrs, qual):
    nq, nd, dim, ranges = _score_args(lib)
    return lib.vr_score_filter_groups(ptrs["q_f16"], nq, ptrs["d_f16"], nd, dim, ranges, ptrs["cand_scores"], ptrs["cand_ids"],
                                      ptrs["doc_groups"], ptrs["doc_mask"], None)


def _rescore(lib, ptrs, qual):
    nq, nd, dim, ranges = _score_args(lib)
    return lib.vr_score_rescore(_p("q_f32"), nq, ptrs["d_f32"], nd, dim, ranges, _p("cand_scores"), _p("cand_ids"),
                                _p("max_doc_norm"), 10, 0, _p("out_scores"), _p("out_ids"), _p("flags"), None)


def _rescore_groups(lib, ptrs, qual):
    nq, nd, dim, ranges = _score_args(lib)
    return lib.vr_score_rescore_groups(_p("q_f32"), nq, ptrs["d_f32"], nd, dim, ranges, _p("cand_scores"), _p("cand_ids"),
                                       ptrs["doc_groups"], ptrs["group_offsets"], ptrs["group_pages"], 50, ptrs["doc_mask"],
                                       _p("max_doc_norm"), 10, 0, _p("out_scores"), _p("out_pages"), _p("out_groups"),
                                       _p("flags"), None)


CALLS = {
    "vr_gemm": _gemm,
    "vr_attention": _attention,
    "vr_im2col_norm": lambda lib, p, q: lib.vr_im2col_norm_ex(_p("pixels"), 1, 28, 28, 14, p["out"], 640, L.VR_BF16, None),
    "vr_layernorm": lambda lib, p, q: lib.vr_layernorm_ex(p["x"], 1152, p["gamma"], p["beta"], 1e-6, 64, 1152, p["out"], 1152,
                                                          p["out2"], p["add"], 16, L.VR_BF16, None),
    "vr_rmsnorm": lambda lib, p, q: lib.vr_rmsnorm_ex(p["x"], 2304, p["gamma"], 1e-5, 64, 2304, p["out"], 2304, L.VR_BF16, None),
    "vr_build_lm_input": lambda lib, p, q: lib.vr_build_lm_input_ex(p["src"], 64, 2304, p["embed"], L.VR_BF16, 12.0, p["vision"],
                                                                    2304, p["h"], 2304, None),
    "vr_pool_norm": lambda lib, p, q: lib.vr_pool_norm(p["h"], 2304, p["gamma"], 1e-5, p["cu"], 4, 2304, 0, 1, p["reps"], None),
    "vr_prefix_rows": lambda lib, p, q: lib.vr_prefix_rows(p["prefix"], 1536, p["rows"], 1536, p["out"], 1536, p["cu_rows"],
                                                           p["cu_out"], 2, 8, 40, 1536, 2, None),
    "vr_f32_to_f16_rows": lambda lib, p, q: lib.vr_f32_to_f16_rows(p["src"], 100, 2304, p["dst_f16"], None, None, None),
    "vr_score_filter": lambda lib, p, q: _filter(lib, p, q, False),
    "vr_score_filter_masked": lambda lib, p, q: _filter(lib, p, q, True),
    "vr_score_filter_groups": _filter_groups,
    "vr_score_rescore": _rescore,
    "vr_score_exact": lambda lib, p, q: lib.vr_score_exact(_p("q_f32"), 4, p["d_f32"], 1000, 64, _p("scores"), None),
    "vr_score_rescore_groups": _rescore_groups,
}


def _ptrs(entry, qual):
    return {name: _p(name) for (e, name, _) in TABLE if e == entry}


def _call(lib, entry, qual, ptrs):
    rc = CALLS[entry](lib, ptrs, qual)
    return rc, lib.vr_last_error().decode()


@pytest.mark.parametrize("entry,qual", sorted({(e, q) for (e, _, q) in TABLE}, key=str))
def test_aligned_pointers_pass_validation(lib, entry, qual):
    """The same calls with every pointer aligned get past argument validation: each refusal below comes from the one
    misaligned pointer. Without a device they then stop at their first CUDA call (status 1)."""
    rc, msg = _call(lib, entry, qual, _ptrs(entry, qual))
    assert rc != 2, msg


@pytest.mark.parametrize("entry,name,qual", sorted(TABLE, key=str))
def test_misaligned_pointer_is_refused(lib, entry, name, qual):
    n = TABLE[(entry, name, qual)]
    ptrs = _ptrs(entry, qual)
    ptrs[name] += 4 if n >= 8 else 2
    rc, msg = _call(lib, entry, qual, ptrs)
    assert rc == 2, f"{entry}: {name} at +{ptrs[name] % n} was not refused (status {rc}: {msg})"
    assert re.search(rf"\b{name}\b", msg), msg
