#include "common.h"
#include "gemm.cuh"

namespace vr {

template <bool F16, int BN, int MODE, bool OUT_F32, bool GELU, bool SWAP = false>
static int launch_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    CUtensorMap ta, tb;
    // the MMA's M operand is staged in 128-row boxes, its N operand in 64-row boxes: SWAP hands the weight to the M side
    // (128 features per tile) and the activations to the N side (BN tokens per tile)
    if (int rc = make_tmap_2d(SWAP ? &tb : &ta, A, g.M, g.K, lda, SWAP ? 64 : GEMM_BM, GEMM_BK, 128, !F16)) return rc;
    if (int rc = make_tmap_2d(SWAP ? &ta : &tb, B, g.N, g.K, ldb, SWAP ? GEMM_BM : 64, GEMM_BK, 128, !F16)) return rc;
    auto kern = gemm_wgmma_kernel<F16, BN, MODE, OUT_F32, GELU, SWAP>;
    static unsigned long long attr_set = 0;  // per template instantiation, one bit per device
    if (first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    const int tiles = SWAP ? ((g.N + GEMM_BM - 1) / GEMM_BM) * ((g.M + BN - 1) / BN)
                           : ((g.M + GEMM_BM - 1) / GEMM_BM) * ((g.N + BN - 1) / BN);
    const int grid = tiles < num_sms() ? tiles : num_sms();
    kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, g);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <bool F16, int MODE, bool OUT_F32, bool GELU, int CLUSTER, bool LEAN>
static int launch_pingpong(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, bool l2_slices,
                           cudaStream_t stream) {
    CUtensorMap ta, tb;
    if (int rc = make_tmap_2d(&ta, A, g.M, g.K, lda, GEMM_BM, GEMM_BK, 128, !F16)) return rc;
    if (int rc = make_tmap_2d(&tb, B, g.N, g.K, ldb, 64, GEMM_BK, 128, !F16)) return rc;
    auto kern = gemm_pingpong_kernel<F16, MODE, OUT_F32, GELU, CLUSTER, LEAN>;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = GEMM_PP_SMEM_BYTES;
    cfg.stream = stream;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CLUSTER;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    // persistent grid: one CTA (pair) per resident slot, at most one per unit
    static unsigned long long attr_set = 0;
    static int max_clusters[64] = {};
    const int dev = current_device(), dev_slot = dev >= 0 && dev < 64 ? dev : 0;
    if (first_use_on_device(&attr_set)) {
        VR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_PP_SMEM_BYTES));
        int n = num_sms() / CLUSTER;
        if (CLUSTER > 1) {
            cfg.gridDim = dim3(num_sms() / CLUSTER * CLUSTER);
            VR_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
        }
        max_clusters[dev_slot] = n;
    }
    const PPSched sch = pp_schedule(g.M, g.N, g.K, CLUSTER, l2_slices);
    VR_REQUIRE(max_clusters[dev_slot] > 0, "vr_gemm: no %d-CTA cluster of the ping-pong kernel fits on this device", CLUSTER);
    const int units = sch.num_units();
    const int clusters = units < max_clusters[dev_slot] ? units : max_clusters[dev_slot];
    cfg.gridDim = dim3(clusters * CLUSTER);
    VR_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, ta, tb, g, sch));
    return 0;
}

// Output types: F16 = false (bf16 operands) writes bf16 or fp32, F16 = true (fp16 operands) fp16 or fp32. Checked before
// any CUDA call; the bf16 messages are the ones the bf16-only library gave.
template <bool F16>
static int check_out_dtype(const vr_gemm_epilogue& e) {
    if (F16) {
        if (e.mode == VR_EPI_LINEAR && e.out_dtype == VR_F32) {
            VR_REQUIRE(!e.act_gelu, "vr_gemm: GELU epilogue writes fp16 only (fp16 operands)");
            return 0;
        }
        if (e.mode == VR_EPI_LINEAR)
            VR_REQUIRE(e.out_dtype == VR_F16, "vr_gemm: with fp16 operands out_dtype must be VR_F16 or VR_F32");
        else
            VR_REQUIRE(e.out_dtype == VR_F16, "vr_gemm: with fp16 operands ROPE / SWIGLU write fp16: out_dtype must be VR_F16");
        return 0;
    }
    if (e.mode != VR_EPI_LINEAR) return 0;  // ROPE / SWIGLU write bf16 whatever out_dtype says
    if (e.out_dtype == VR_F32) {
        VR_REQUIRE(!e.act_gelu, "vr_gemm: GELU epilogue writes bf16 only");
        return 0;
    }
    VR_REQUIRE(e.out_dtype == VR_BF16, "vr_gemm: out_dtype must be VR_BF16 or VR_F32");
    return 0;
}

// feature-major accumulator kernel (block_n == 3): LINEAR epilogues only
template <bool F16>
static int dispatch_swapped(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t s) {
    const vr_gemm_epilogue& e = g.epi;
    VR_REQUIRE(e.mode == VR_EPI_LINEAR, "vr_gemm: block_n=3 (feature-major accumulator) supports LINEAR epilogues only");
    if (int rc = check_out_dtype<F16>(e)) return rc;
    if (e.out_dtype == VR_F32) return launch_gemm<F16, 128, VR_EPI_LINEAR, true, false, true>(A, lda, B, ldb, g, s);
    if (e.act_gelu) return launch_gemm<F16, 128, VR_EPI_LINEAR, false, true, true>(A, lda, B, ldb, g, s);
    return launch_gemm<F16, 128, VR_EPI_LINEAR, false, false, true>(A, lda, B, ldb, g, s);
}

// BN > 0: tile width of the cooperative kernel. BN < 0: the ping-pong kernel (128 x 128 tiles), as the block_n selector
// -BN names it: PP (L2-sliced tile order), PP_NFAST (plain n-fastest order), PP_MC (CTA pairs with B multicast).
// LEAN selects the ping-pong kernel's lean epilogue (16-bit LINEAR, bias [+ GELU] only); the cooperative kernel ignores it.
constexpr int PP = 2, PP_MC = 4, PP_NFAST = 5;
template <bool F16, int BN, int MODE, bool OUT_F32, bool GELU, bool LEAN = false>
static int launch_any(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t s) {
    if constexpr (BN < 0)
        return launch_pingpong<F16, MODE, OUT_F32, GELU, -BN == PP_MC ? 2 : 1, LEAN>(A, lda, B, ldb, g, -BN != PP_NFAST, s);
    else return launch_gemm<F16, BN, MODE, OUT_F32, GELU>(A, lda, B, ldb, g, s);
}

template <bool F16, int BN>
static int dispatch_mode(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t s) {
    const vr_gemm_epilogue& e = g.epi;
    switch (e.mode) {
        case VR_EPI_LINEAR: {
            if (int rc = check_out_dtype<F16>(e)) return rc;
            if (e.out_dtype == VR_F32) return launch_any<F16, BN, VR_EPI_LINEAR, true, false>(A, lda, B, ldb, g, s);
            // a NULL bias keeps the generic epilogue: adding a zero bias would turn an accumulator of -0 into +0
            const bool lean = BN < 0 && e.bias && e.scale == 1.0f && !e.rowadd && !e.resid;
            if (e.act_gelu)
                return lean ? launch_any<F16, BN, VR_EPI_LINEAR, false, true, true>(A, lda, B, ldb, g, s)
                            : launch_any<F16, BN, VR_EPI_LINEAR, false, true>(A, lda, B, ldb, g, s);
            return lean ? launch_any<F16, BN, VR_EPI_LINEAR, false, false, true>(A, lda, B, ldb, g, s)
                        : launch_any<F16, BN, VR_EPI_LINEAR, false, false>(A, lda, B, ldb, g, s);
        }
        case VR_EPI_ROPE:
            VR_REQUIRE(e.positions && e.rope_cos && e.rope_sin, "vr_gemm: ROPE epilogue needs positions/cos/sin");
            VR_REQUIRE(g.N % 64 == 0 && e.rope_cols % 64 == 0, "vr_gemm: ROPE needs N and rope_cols multiples of 64");
            if (int rc = check_out_dtype<F16>(e)) return rc;
            return launch_any<F16, BN, VR_EPI_ROPE, false, false>(A, lda, B, ldb, g, s);
        case VR_EPI_SWIGLU:
            VR_REQUIRE(g.N % 64 == 0, "vr_gemm: SWIGLU needs N multiple of 64");
            if (int rc = check_out_dtype<F16>(e)) return rc;
            return launch_any<F16, BN, VR_EPI_SWIGLU, false, false>(A, lda, B, ldb, g, s);
        default:
            set_error("vr_gemm: unknown epilogue mode %d", e.mode);
            return 2;
    }
}

template <bool F16>
static int dispatch_block_n(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, int bn, cudaStream_t s) {
    if (bn == PP) return dispatch_mode<F16, -PP>(A, lda, B, ldb, g, s);
    if (bn == PP_MC) return dispatch_mode<F16, -PP_MC>(A, lda, B, ldb, g, s);
    if (bn == PP_NFAST) return dispatch_mode<F16, -PP_NFAST>(A, lda, B, ldb, g, s);
    if (bn == 3) return dispatch_swapped<F16>(A, lda, B, ldb, g, s);
    if (bn == 256) return dispatch_mode<F16, 256>(A, lda, B, ldb, g, s);
    if (bn == 192) return dispatch_mode<F16, 192>(A, lda, B, ldb, g, s);
    if (bn == 128) return dispatch_mode<F16, 128>(A, lda, B, ldb, g, s);
    if (bn == 64) return dispatch_mode<F16, 64>(A, lda, B, ldb, g, s);
    set_error("vr_gemm: block_n must be 0 (auto), 64, 128, 192, 256, 2 / 4 / 5 (ping-pong) or 3 (feature-major accumulator)");
    return 2;
}

}  // namespace vr

extern "C" int vr_gemm_tuned(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M,
                             int32_t N, int32_t K, const vr_gemm_epilogue* epi, int32_t block_n, void* stream) {
    using namespace vr;
    VR_REQUIRE(A && B && epi && epi->out, "vr_gemm: null pointer argument");
    VR_REQUIRE(M > 0 && N > 0 && K > 0, "vr_gemm: empty problem M=%d N=%d K=%d", M, N, K);
    VR_REQUIRE(ab_dtype == VR_BF16 || ab_dtype == VR_F16, "vr_gemm: operands must be bf16 or fp16 (got dtype %d)", ab_dtype);
    VR_REQUIRE(N % 8 == 0, "vr_gemm: N=%d must be a multiple of 8", N);
    VR_REQUIRE(K % 8 == 0, "vr_gemm: K=%d must be a multiple of 8 (16-byte TMA rows)", K);
    const int64_t out_cols = epi->mode == VR_EPI_SWIGLU ? N / 2 : N;
    VR_REQUIRE(epi->ldo >= out_cols && epi->ldo % 8 == 0, "vr_gemm: ldo=%lld too small or not a multiple of 8",
               (long long)epi->ldo);
    // the ping-pong kernel stores a 16-bit LINEAR output 16 bytes at a time (ldo % 8 == 0 keeps every row aligned)
    VR_REQUIRE(epi->mode != VR_EPI_LINEAR || (reinterpret_cast<uintptr_t>(epi->out) & 15) == 0,
               "vr_gemm: a LINEAR out must be 16-byte aligned (out=%p)", epi->out);
    // the other bases, at the width of their widest access: A / B are TMA sources; the epilogues read bias, rowadd, resid
    // and the RoPE tables as float2 and positions as int32, and ROPE / SWIGLU store 16-bit pairs
    VR_REQUIRE_ALIGNED("vr_gemm", "A", A, 16);
    VR_REQUIRE_ALIGNED("vr_gemm", "B", B, 16);
    VR_REQUIRE_ALIGNED("vr_gemm", "bias", epi->bias, 8);
    VR_REQUIRE_ALIGNED("vr_gemm", "rowadd", epi->rowadd, 8);
    VR_REQUIRE_ALIGNED("vr_gemm", "resid", epi->resid, 8);
    VR_REQUIRE_ALIGNED("vr_gemm", "rope_cos", epi->rope_cos, 8);
    VR_REQUIRE_ALIGNED("vr_gemm", "rope_sin", epi->rope_sin, 8);
    VR_REQUIRE_ALIGNED("vr_gemm", "positions", epi->positions, 4);
    VR_REQUIRE_ALIGNED("vr_gemm", "out", epi->out, 4);
    GemmArgs g;
    g.M = M; g.N = N; g.K = K; g.epi = *epi;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int bn = block_n;
    if (bn == 0) {
        // M <= 128 (a few queries): one row tile, the kernel only streams the weight - 64-wide feature tiles spread that
        // stream over 4x as many SMs as 256-wide ones (o_proj 2304x2304: 36 CTAs instead of 9). Otherwise the ping-pong
        // kernel in CTA pairs with the B tile multicast: one warpgroup's epilogue runs under the other's MMAs, and the
        // pair reads 24 KB instead of 32 KB from L2 per stage. On H100 it was the fastest or tied on every GEMM class of
        // the encode step (tools/bench_gemm.py); single-CTA ping-pong was slower than the cooperative kernel on
        // mainloop-bound ones (gate|up, RoPE qkv).
        bn = M <= 128 ? 64 : PP_MC;
    }
    return ab_dtype == VR_F16 ? dispatch_block_n<true>(A, lda, B, ldb, g, bn, s) : dispatch_block_n<false>(A, lda, B, ldb, g, bn, s);
}

extern "C" int vr_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M, int32_t N,
                       int32_t K, const vr_gemm_epilogue* epi, void* stream) {
    return vr_gemm_tuned(A, lda, B, ldb, ab_dtype, M, N, K, epi, 0, stream);
}
