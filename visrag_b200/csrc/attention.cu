#include <string.h>
#include "common.h"
#include "attention.cuh"

namespace vr {

static int g_variant = 0;  // see vr_attention_force_v1()

template <int HS, bool CAUSAL, int NWG, bool F16>
static int launch_attention(const vr_attn_params& p, cudaStream_t stream) {
    using Cfg = AttCfg<HS, NWG>;
    AttMaps maps;
    memset(&maps, 0, sizeof(maps));
    // TMA extents: all columns of the token matrices, rows = buffer rows (out-of-range rows read as zero)
    const uint64_t qcols = p.ldq, kcols = p.ldk, vcols = p.ldv;
    if (int rc = make_tmap_2d(&maps.q64, p.q, p.q_rows, qcols, p.ldq, Cfg::BM, 64, 128, !F16)) return rc;
    if (int rc = make_tmap_2d(&maps.k64, p.k, p.kv_rows, kcols, p.ldk, ATT_BN, 64, 128, !F16)) return rc;
    if (int rc = make_tmap_2d(&maps.v64, p.v, p.kv_rows, vcols, p.ldv, ATT_BN, 64, 128, !F16)) return rc;
    if (Cfg::HAS16) {
        if (int rc = make_tmap_2d(&maps.q16, p.q, p.q_rows, qcols, p.ldq, Cfg::BM, 16, 32, !F16)) return rc;
        if (int rc = make_tmap_2d(&maps.k16, p.k, p.kv_rows, kcols, p.ldk, ATT_BN, 16, 32, !F16)) return rc;
        if (int rc = make_tmap_2d(&maps.v16, p.v, p.kv_rows, vcols, p.ldv, ATT_BN, 16, 32, !F16)) return rc;
    }
    AttArgs a;
    a.q_col0 = p.q_col0; a.k_col0 = p.k_col0; a.v_col0 = p.v_col0;
    a.head_dim = p.head_dim; a.heads = p.heads; a.batch = p.batch;
    a.cu_q = p.cu_q; a.cu_k = p.cu_k; a.max_q = p.max_q;
    a.scale_log2 = p.scale * 1.4426950408889634f;
    a.out = p.out;
    a.ldo = p.ldo;
    auto kern = attention_wgmma_kernel<HS, CAUSAL, NWG, F16>;
    static unsigned long long attr_set = 0;
    if (first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    dim3 grid((p.max_q + Cfg::BM - 1) / Cfg::BM, p.heads, p.batch);
    kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(maps, a);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int HS, bool F16>
static int dispatch_attention(const vr_attn_params& p, cudaStream_t s) {
    const bool two = p.max_q > 64 && g_variant != 1;  // more than one 64-query tile per sequence
    if (p.causal) return two ? launch_attention<HS, true, 2, F16>(p, s) : launch_attention<HS, true, 1, F16>(p, s);
    return two ? launch_attention<HS, false, 2, F16>(p, s) : launch_attention<HS, false, 1, F16>(p, s);
}

template <int HS>
static int dispatch_attention(const vr_attn_params& p, cudaStream_t s) {
    return (p.flags & VR_ATTN_F16) ? dispatch_attention<HS, true>(p, s) : dispatch_attention<HS, false>(p, s);
}

}  // namespace vr

// test hook: 0 = default dispatch, 1 = force the one-warpgroup (64 queries per CTA) kernel for every shape
extern "C" void vr_attention_force_v1(int32_t variant) { vr::g_variant = variant; }

extern "C" int vr_attention(const vr_attn_params* p, void* stream) {
    using namespace vr;
    VR_REQUIRE(p && p->q && p->k && p->v && p->out && p->cu_k, "vr_attention: null pointer argument");
    VR_REQUIRE(p->heads > 0 && p->batch > 0 && p->max_q > 0 && p->max_k > 0, "vr_attention: empty problem");
    VR_REQUIRE(p->batch <= 65535 && p->heads <= 65535, "vr_attention: batch/heads exceed grid limits");
    VR_REQUIRE(p->head_dim <= p->head_stride && p->head_dim % 8 == 0, "vr_attention: head_dim %d vs stride %d",
               p->head_dim, p->head_stride);
    VR_REQUIRE(p->ldo % 8 == 0, "vr_attention: ldo must be a multiple of 8");
    VR_REQUIRE(!(p->flags & VR_ATTN_V_ONES_COLUMN) || p->head_dim == p->head_stride - 8,
               "vr_attention: VR_ATTN_V_ONES_COLUMN needs head_dim == head_stride - 8 (got %d / %d)", p->head_dim, p->head_stride);
    // q / k / v are TMA sources; the kernels read cu_q / cu_k as int32 and store out as 16-bit pairs
    VR_REQUIRE_ALIGNED("vr_attention", "q", p->q, 16);
    VR_REQUIRE_ALIGNED("vr_attention", "k", p->k, 16);
    VR_REQUIRE_ALIGNED("vr_attention", "v", p->v, 16);
    VR_REQUIRE_ALIGNED("vr_attention", "cu_q", p->cu_q, 4);
    VR_REQUIRE_ALIGNED("vr_attention", "cu_k", p->cu_k, 4);
    VR_REQUIRE_ALIGNED("vr_attention", "out", p->out, 4);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    switch (p->head_stride) {
        case 64: return dispatch_attention<64>(*p, s);
        case 80: return dispatch_attention<80>(*p, s);
        case 128: return dispatch_attention<128>(*p, s);
        default: set_error("vr_attention: head_stride must be 64, 80 or 128 (got %d)", p->head_stride); return 2;
    }
}
