#include "common.h"
#include "gemm.cuh"

namespace vr {

template <int BN, int MODE, bool OUT_F32, bool GELU, bool SWAP = false>
static int launch_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    CUtensorMap ta, tb;
    // the MMA's M operand is staged in 128-row boxes, its N operand in 64-row boxes: SWAP hands the weight to the M side
    // (128 features per tile) and the activations to the N side (BN tokens per tile)
    if (int rc = make_tmap_2d(SWAP ? &tb : &ta, A, g.M, g.K, lda, SWAP ? 64 : GEMM_BM, GEMM_BK, 128, true)) return rc;
    if (int rc = make_tmap_2d(SWAP ? &ta : &tb, B, g.N, g.K, ldb, SWAP ? GEMM_BM : 64, GEMM_BK, 128, true)) return rc;
    auto kern = gemm_wgmma_kernel<BN, MODE, OUT_F32, GELU, SWAP>;
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

// feature-major accumulator kernel (block_n == 3): LINEAR epilogues only
static int dispatch_swapped(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t s) {
    const vr_gemm_epilogue& e = g.epi;
    VR_REQUIRE(e.mode == VR_EPI_LINEAR, "vr_gemm: block_n=3 (feature-major accumulator) supports LINEAR epilogues only");
    if (e.out_dtype == VR_F32) {
        VR_REQUIRE(!e.act_gelu, "vr_gemm: GELU epilogue writes bf16 only");
        return launch_gemm<128, VR_EPI_LINEAR, true, false, true>(A, lda, B, ldb, g, s);
    }
    VR_REQUIRE(e.out_dtype == VR_BF16, "vr_gemm: out_dtype must be VR_BF16 or VR_F32");
    if (e.act_gelu) return launch_gemm<128, VR_EPI_LINEAR, false, true, true>(A, lda, B, ldb, g, s);
    return launch_gemm<128, VR_EPI_LINEAR, false, false, true>(A, lda, B, ldb, g, s);
}

template <int BN>
static int dispatch_mode(const void* A, int64_t lda, const void* B, int64_t ldb, const GemmArgs& g, cudaStream_t s) {
    const vr_gemm_epilogue& e = g.epi;
    switch (e.mode) {
        case VR_EPI_LINEAR:
            if (e.out_dtype == VR_F32) {
                VR_REQUIRE(!e.act_gelu, "vr_gemm: GELU epilogue writes bf16 only");
                return launch_gemm<BN, VR_EPI_LINEAR, true, false>(A, lda, B, ldb, g, s);
            }
            VR_REQUIRE(e.out_dtype == VR_BF16, "vr_gemm: out_dtype must be VR_BF16 or VR_F32");
            if (e.act_gelu) return launch_gemm<BN, VR_EPI_LINEAR, false, true>(A, lda, B, ldb, g, s);
            return launch_gemm<BN, VR_EPI_LINEAR, false, false>(A, lda, B, ldb, g, s);
        case VR_EPI_ROPE:
            VR_REQUIRE(e.positions && e.rope_cos && e.rope_sin, "vr_gemm: ROPE epilogue needs positions/cos/sin");
            VR_REQUIRE(g.N % 64 == 0 && e.rope_cols % 64 == 0, "vr_gemm: ROPE needs N and rope_cols multiples of 64");
            return launch_gemm<BN, VR_EPI_ROPE, false, false>(A, lda, B, ldb, g, s);
        case VR_EPI_SWIGLU:
            VR_REQUIRE(g.N % 64 == 0, "vr_gemm: SWIGLU needs N multiple of 64");
            return launch_gemm<BN, VR_EPI_SWIGLU, false, false>(A, lda, B, ldb, g, s);
        default:
            set_error("vr_gemm: unknown epilogue mode %d", e.mode);
            return 2;
    }
}

}  // namespace vr

extern "C" int vr_gemm_tuned(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M,
                             int32_t N, int32_t K, const vr_gemm_epilogue* epi, int32_t block_n, void* stream) {
    using namespace vr;
    VR_REQUIRE(A && B && epi && epi->out, "vr_gemm: null pointer argument");
    VR_REQUIRE(M > 0 && N > 0 && K > 0, "vr_gemm: empty problem M=%d N=%d K=%d", M, N, K);
    VR_REQUIRE(ab_dtype == VR_BF16, "vr_gemm: only bf16 operands are instantiated (got dtype %d)", ab_dtype);
    VR_REQUIRE(N % 8 == 0, "vr_gemm: N=%d must be a multiple of 8", N);
    VR_REQUIRE(K % 8 == 0, "vr_gemm: K=%d must be a multiple of 8 (16-byte TMA rows)", K);
    const int64_t out_cols = epi->mode == VR_EPI_SWIGLU ? N / 2 : N;
    VR_REQUIRE(epi->ldo >= out_cols && epi->ldo % 8 == 0, "vr_gemm: ldo=%lld too small or not a multiple of 8",
               (long long)epi->ldo);
    GemmArgs g;
    g.M = M; g.N = N; g.K = K; g.epi = *epi;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int bn = block_n;
    if (bn == 0) {
        // M <= 128 (a few queries): one row tile, the kernel only streams the weight - 64-wide feature tiles spread that
        // stream over 4x as many SMs as 256-wide ones (o_proj 2304x2304: 36 CTAs instead of 9). Otherwise the widest tile
        // (most reuse of the A rows per byte staged), except where 192 tiles N exactly and 256 does not (N = 1152:
        // 6 x 192 instead of 4.5 x 256).
        bn = M <= 128 ? 64 : (N < 256 ? 128 : ((N % 192 == 0 && N % 256 != 0) ? 192 : 256));
    }
    if (bn == 3) return dispatch_swapped(A, lda, B, ldb, g, s);
    if (bn == 256) return dispatch_mode<256>(A, lda, B, ldb, g, s);
    if (bn == 192) return dispatch_mode<192>(A, lda, B, ldb, g, s);
    if (bn == 128) return dispatch_mode<128>(A, lda, B, ldb, g, s);
    if (bn == 64) return dispatch_mode<64>(A, lda, B, ldb, g, s);
    set_error("vr_gemm: block_n must be 0 (auto), 64, 128, 192, 256 or 3 (feature-major accumulator)");
    return 2;
}

extern "C" int vr_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M, int32_t N,
                       int32_t K, const vr_gemm_epilogue* epi, void* stream) {
    return vr_gemm_tuned(A, lda, B, ldb, ab_dtype, M, N, K, epi, 0, stream);
}
