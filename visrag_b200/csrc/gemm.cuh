// Persistent warp-specialised wgmma GEMM:  C[M,N] = A[M,K] * B[N,K]^T  (both K-major).
//
//   warpgroup 0 (one lane)  TMA producer : A/B 128B-swizzled tiles -> multi-stage smem ring; the ring runs ahead
//                                          into the next tile while the consumers are in their epilogue
//   warpgroups 1, 2         consumers    : each owns 64 of the tile's 128 rows: wgmma m64 x BN x k16 from shared
//                                          memory, fp32 accumulators in registers (BN/2 per thread), then the fused
//                                          epilogue (bias / GELU / residual / RoPE / SwiGLU) straight from the
//                                          accumulator fragments: a thread holds pairs of adjacent columns, so
//                                          global accesses are 8-byte (fp32) or 4-byte (bf16 / fp16) and a quad of lanes
//                                          covers one 32-byte sector of a row.
//
// Two mbarrier arrays: smem full (TMA -> consumers, transaction bytes) and empty (8 consumer warps -> TMA).
// Tiles are scheduled round-robin over a grid of min(#tiles, #SMs) CTAs, n-block fastest so
// that CTAs running together share the same A rows in L2.
//
// gemm_pingpong_kernel (below) is the same pipeline with a different consumer schedule: each consumer warpgroup owns a
// whole 128 x 128 tile and the two take turns on the tensor cores, so one tile's epilogue overlaps the next tile's
// MMAs. vr_gemm uses it, in CTA pairs that share the B tile by multicast, for every problem with more than one row tile.
// Its LINEAR epilogue stores a 16-bit output 16 bytes per thread after a transpose across each quad of lanes.
#pragma once
#include "ptx.cuh"
#include "../../include/visrag_b200.h"

namespace vr {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;  // 64 bf16 / fp16 = 128 B = one swizzle-128B row
constexpr int GEMM_THREADS = 3 * 128;  // producer warpgroup + two consumer warpgroups

template <int BN>
struct GemmCfg {
    static_assert(BN % 64 == 0 && BN <= 256, "tile width: 64, 128, 192 or 256");
    static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
    static constexpr int B_BYTES = BN * GEMM_BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (192 * 1024) / STAGE_BYTES;  // 4 / 4 / 6 / 8 stages in 192 KB of the SM's 227 KB
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct GemmArgs {
    int M, N, K;
    vr_gemm_epilogue epi;
};

// Exact-erf GELU (timm Mlp uses nn.GELU, erf form). erf through Abramowitz-Stegun 7.1.26: |error| <= 1.5e-7 absolute, far
// below the bf16 rounding of the result, at ~1/3 of erff()'s instruction count (the fc1 epilogue is issue bound).
__device__ __forceinline__ float erf_as(float x) {
    const float ax = fabsf(x);
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
    float p = fmaf(1.061405429f, t, -1.453152027f);
    p = fmaf(p, t, 1.421413741f);
    p = fmaf(p, t, -0.284496736f);
    p = fmaf(p, t, 0.254829592f);
    p *= t;
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * ax * ax));
    return copysignf(fmaf(-p, e, 1.0f), x);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f)); }

#ifndef VR_GELU_POLY
#define VR_GELU_POLY 1
#endif
#if VR_GELU_POLY
// erf without the SFU: z = clamp(x/sqrt2, +-3.2), erf(z) = z * P(u), u = z^2 * (2/3.2^2) - 1 in [-1, 1], P = degree-10
// near-minimax polynomial (Chebyshev fit of erf(z)/z, evaluated by Horner in the mapped variable so the coefficients stay
// O(1) and nothing cancels). |erf error| <= 3.2e-6 in fp32 incl. the clamp (past it erf(z) is replaced by P's value at
// 3.2, 1 - 2.9e-6), so |GELU error| = 0.5 |x| |erf error| <= 1.6e-6 |x| plus fp32 rounding: it grows with |x| (1.6e-4 at
// |x| = 100) but stays about 2^-19 relative to the input, far below the bf16 rounding of the result
// (tests/kernel_bounds.py derives the GEMM's GELU bound from this). The Abramowitz-Stegun form below needs two MUFU ops per
// element (rcp + ex2): 65536 per 128x256 tile = 4096 SFU cycles on the critical path of the fc1 epilogue. This form is 14 FMA-pipe instructions per element and no MUFU.
// N GELUs as N interleaved chains: each step is done for all N values before the next, so consecutive FMAs are
// independent (a single chain stalls on every FMA's latency). Per value the operations are the same for every N.
template <int N>
__device__ __forceinline__ void gelu_erf_n(float (&x)[N]) {
    constexpr float R2 = 0.70710678118654752f, ZMAX = 3.2f, A = 2.0f / (ZMAX * ZMAX);
    // P's coefficients, highest degree first
    constexpr float C[11] = {2.982273671e-03f, -7.046153472e-03f, 7.957076705e-03f, -1.521942819e-02f, 3.318292224e-02f,
                             -5.471928813e-02f, 8.062700147e-02f, -1.136467381e-01f, 1.543549678e-01f, -2.173077339e-01f,
                             4.413341836e-01f};
    float z[N], u[N], p[N];
#pragma unroll
    for (int i = 0; i < N; ++i) z[i] = fminf(fmaxf(x[i] * R2, -ZMAX), ZMAX);
#pragma unroll
    for (int i = 0; i < N; ++i) u[i] = fmaf(fmaf(z[i], z[i], 0.0f), A, -1.0f);
#pragma unroll
    for (int i = 0; i < N; ++i) p[i] = fmaf(u[i], C[0], C[1]);
#pragma unroll
    for (int k = 2; k < 11; ++k) {
#pragma unroll
        for (int i = 0; i < N; ++i) p[i] = fmaf(p[i], u[i], C[k]);
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const float r = fmaf(p[i], z[i], 0.0f);  // erf(z)
        const float h = 0.5f * x[i];
        x[i] = fmaf(h, r, h);
    }
}
__device__ __forceinline__ void gelu_erf2(float& x0, float& x1) {
    float x[2] = {x0, x1};
    gelu_erf_n(x);
    x0 = x[0];
    x1 = x[1];
}
#else
// two independent GELUs side by side (instruction-level parallelism for the Horner chains)
__device__ __forceinline__ void pk_fma(float& d0, float& d1, float a0, float a1, float b0, float b1, float c0, float c1) {
    d0 = fmaf(a0, b0, c0);
    d1 = fmaf(a1, b1, c1);
}
__device__ __forceinline__ void gelu_erf2(float& x0, float& x1) {
    constexpr float R2 = 0.70710678118654752f;
    const float a0 = fabsf(x0) * R2, a1 = fabsf(x1) * R2;  // |z|, z = x / sqrt(2)
    float d0, d1, t0, t1, p0, p1, q0, q1, e0, e1, r0, r1;
    pk_fma(d0, d1, a0, a1, 0.3275911f, 0.3275911f, 1.0f, 1.0f);
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
    pk_fma(p0, p1, t0, t1, 1.061405429f, 1.061405429f, -1.453152027f, -1.453152027f);
    pk_fma(p0, p1, p0, p1, t0, t1, 1.421413741f, 1.421413741f);
    pk_fma(p0, p1, p0, p1, t0, t1, -0.284496736f, -0.284496736f);
    pk_fma(p0, p1, p0, p1, t0, t1, 0.254829592f, 0.254829592f);
    pk_fma(p0, p1, p0, p1, t0, t1, 0.0f, 0.0f);
    pk_fma(q0, q1, a0, a1, a0, a1, 0.0f, 0.0f);
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(q0 * -1.4426950408889634f));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(q1 * -1.4426950408889634f));
    pk_fma(r0, r1, p0, p1, -e0, -e1, 1.0f, 1.0f);  // erf(|z|)
    r0 = copysignf(r0, x0);
    r1 = copysignf(r1, x1);
    const float h0 = 0.5f * x0, h1 = 0.5f * x1;
    pk_fma(x0, x1, h0, h1, r0, r1, h0, h1);
}
template <int N>
__device__ __forceinline__ void gelu_erf_n(float (&x)[N]) {
#pragma unroll
    for (int i = 0; i < N; i += 2) gelu_erf2(x[i], x[i + 1]);
}
#endif
// x * sigmoid(x) with two SFU ops (ex2 + rcp, ~1e-6 relative) instead of an IEEE division
__device__ __forceinline__ float silu(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
}

// ---------------------------------------------------------------------------------------
// Epilogue, per accumulator fragment pair (two adjacent columns of one row).
// ---------------------------------------------------------------------------------------
// F16: the operands are fp16 and every 16-bit output is fp16 (else bf16); the fp32 arithmetic does not change.
// LINEAR: out = [resid +] scale * gelu?(acc + bias) [+ rowadd[row % period]]; columns col, col + 1 (col even, N % 8 == 0)
template <bool F16, bool OUT_F32, bool GELU>
__device__ __forceinline__ void epi_linear2(const GemmArgs& g, int row, int col, float x0, float x1) {
    const vr_gemm_epilogue& e = g.epi;
    if (row >= g.M || col >= g.N) return;
    if (e.bias) {
        const float2 b = *reinterpret_cast<const float2*>(e.bias + col);
        x0 += b.x; x1 += b.y;
    }
    if (GELU) gelu_erf2(x0, x1);
    if (e.scale != 1.0f) { x0 *= e.scale; x1 *= e.scale; }
    if (e.rowadd) {
        const float2 a2 = *reinterpret_cast<const float2*>(e.rowadd + static_cast<long long>(row % e.rowadd_period) * g.N + col);
        x0 += a2.x; x1 += a2.y;
    }
    const long long o = static_cast<long long>(row) * e.ldo + col;
    if (e.resid) {
        const float2 r2 = *reinterpret_cast<const float2*>(e.resid + o);
        x0 += r2.x; x1 += r2.y;
    }
    if (OUT_F32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(e.out) + o) = make_float2(x0, x1);
    else *reinterpret_cast<uint32_t*>(reinterpret_cast<half16_t<F16>*>(e.out) + o) = pack16x2<F16>(x0, x1);
}

// LINEAR, feature-major accumulator (SWAP kernels: the WEIGHT tile is the MMA's M operand, tokens are its N): one element
template <bool F16, bool OUT_F32, bool GELU>
__device__ __forceinline__ void epi_linear_t(const GemmArgs& g, int tok, int f, float x) {
    const vr_gemm_epilogue& e = g.epi;
    if (tok >= g.M || f >= g.N) return;
    if (e.bias) x += e.bias[f];
    if (GELU) {
        float y = x;
        gelu_erf2(x, y);
    }
    if (e.scale != 1.0f) x *= e.scale;
    if (e.rowadd) x += e.rowadd[static_cast<long long>(tok % e.rowadd_period) * g.N + f];
    const long long o = static_cast<long long>(tok) * e.ldo + f;
    if (e.resid) x += e.resid[o];
    if (OUT_F32) reinterpret_cast<float*>(e.out)[o] = x;
    else reinterpret_cast<half16_t<F16>*>(e.out)[o] = to_half16<F16>(x);
}

// RoPE (modeling_minicpm.py:259-290): a head is 64 columns [lo(32) | hi(32)];
//   lo' = lo*cos - hi*sin ; hi' = hi*cos + lo*sin   with cos/sin[pos, 0..31].
// (lo0, lo1) are columns head0 + c, head0 + c + 1 and (hi0, hi1) the columns 32 further, c even in [0, 32).
template <bool F16>
__device__ __forceinline__ void epi_rope2(const GemmArgs& g, int row, int head0, int c, float lo0, float lo1, float hi0,
                                          float hi1) {
    const vr_gemm_epilogue& e = g.epi;
    if (row >= g.M || head0 >= g.N) return;
    if (head0 < e.rope_cols) {
        const long long pos = e.positions[row];
        const float2 cs = *reinterpret_cast<const float2*>(e.rope_cos + pos * 32 + c);
        const float2 sn = *reinterpret_cast<const float2*>(e.rope_sin + pos * 32 + c);
        const float a0 = lo0, a1 = lo1, b0 = hi0, b1 = hi1;
        lo0 = a0 * cs.x - b0 * sn.x; hi0 = b0 * cs.x + a0 * sn.x;
        lo1 = a1 * cs.y - b1 * sn.y; hi1 = b1 * cs.y + a1 * sn.y;
    }
    half16_t<F16>* o = reinterpret_cast<half16_t<F16>*>(e.out) + static_cast<long long>(row) * e.ldo + head0 + c;
    *reinterpret_cast<uint32_t*>(o) = pack16x2<F16>(lo0, lo1);
    *reinterpret_cast<uint32_t*>(o + 32) = pack16x2<F16>(hi0, hi1);
}

// SwiGLU (modeling_minicpm.py:333): accumulator columns [gate(32) | up(32)] -> 32 16-bit outputs at column blk0/2.
template <bool F16>
__device__ __forceinline__ void epi_swiglu2(const GemmArgs& g, int row, int blk0, int c, float g0, float g1, float u0, float u1) {
    const vr_gemm_epilogue& e = g.epi;
    if (row >= g.M || blk0 >= g.N) return;
    half16_t<F16>* o = reinterpret_cast<half16_t<F16>*>(e.out) + static_cast<long long>(row) * e.ldo + (blk0 >> 1) + c;
    *reinterpret_cast<uint32_t*>(o) = pack16x2<F16>(silu(g0) * u0, silu(g1) * u1);
}

// ---------------------------------------------------------------------------------------
// SWAP = true (LINEAR only): the host passes the WEIGHT map as tmap_a and the activation map as tmap_b; accumulator
// rows are output features (128 per tile), accumulator columns are tokens (BN per tile). g keeps its meaning
// (M tokens, N features). wgmma's M is fixed at 64 while its N goes down to 8, so this is the form for few tokens.
// Feature blocks vary fastest so that co-running CTAs share one activation tile in L2.
template <bool F16, int BN, int MODE, bool OUT_F32, bool GELU, bool SWAP = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmArgs g) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int wg = threadIdx.x >> 7;
    const int warp = (threadIdx.x >> 5) & 3;  // inside the warpgroup
    const int lane = threadIdx.x & 31;

    static_assert(!SWAP || MODE == VR_EPI_LINEAR, "feature-major accumulators are implemented for LINEAR epilogues");
    const int tiles_m = ((SWAP ? g.N : g.M) + GEMM_BM - 1) / GEMM_BM;
    const int tiles_n = ((SWAP ? g.M : g.N) + BN - 1) / BN;
    const int num_tiles = tiles_m * tiles_n;
    const int num_kb = (g.K + GEMM_BK - 1) / GEMM_BK;
    // tile -> (first accumulator row, first accumulator column)
    auto tile_m0 = [&](int t) { return (SWAP ? t % tiles_m : t / tiles_n) * GEMM_BM; };
    auto tile_n0 = [&](int t) { return (SWAP ? t / tiles_m : t % tiles_n) * BN; };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int m0 = tile_m0(t);
                const int n0 = tile_n0(t);
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    tma_load_2d(&tmap_a, &full_bar[stage], smem_a + stage * Cfg::A_BYTES, kb * GEMM_BK, m0);
                    // B boxes are 64 rows (a box is at most 256 rows; 64 divides every tile width); rows past the
                    // matrix read as zeros and still count their bytes
#pragma unroll
                    for (int h = 0; h < BN / 64; ++h)
                        tma_load_2d(&tmap_b, &full_bar[stage], smem_b + stage * Cfg::B_BYTES + h * (64 * GEMM_BK * 2),
                                    kb * GEMM_BK, n0 + h * 64);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ------------------------------------------------------------ consumers: main loop + epilogue
        setmaxnreg_inc<232>();
        const int cw = wg - 1;  // rows [64 cw, 64 cw + 64) of the tile
        // descriptor = constant high word | (address >> 4); K-major SW128: LBO unused, SBO 1024 B (8 rows)
        const uint64_t desc_hi = make_smem_desc(0, 16, 1024, kLayoutSW128);
        const uint32_t a_lo0 = (smem_u32(smem_a) + cw * (64 * GEMM_BK * 2)) >> 4, b_lo0 = smem_u32(smem_b) >> 4;
        const int g8 = lane >> 2, q = lane & 3;
        int stage = 0;
        uint32_t phase = 0;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            float acc[BN / 2];
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t ad = desc_hi | static_cast<uint64_t>(a_lo0 + stage * (Cfg::A_BYTES >> 4));
                const uint64_t bd = desc_hi | static_cast<uint64_t>(b_lo0 + stage * (Cfg::B_BYTES >> 4));
                wgmma_fence();
                // +32 B (= +2 in the >>4 address field) per 16-element K step inside the 128 B swizzle row
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_ss<F16, false>(acc, ad + 2 * kk, bd + 2 * kk, (kb | kk) != 0, std::integral_constant<int, BN>());
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();  // the MMAs of the previous k-block retired: hand its slot back
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            wgmma_touch(acc);

            const int r0 = tile_m0(t) + cw * 64 + warp * 16 + g8;  // accumulator rows r0 and r0 + 8
            const int n0 = tile_n0(t);
            if (MODE == VR_EPI_LINEAR) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = n0 + j * 8 + q * 2;
                    if (SWAP) {
                        epi_linear_t<F16, OUT_F32, GELU>(g, c, r0, acc[4 * j]);
                        epi_linear_t<F16, OUT_F32, GELU>(g, c + 1, r0, acc[4 * j + 1]);
                        epi_linear_t<F16, OUT_F32, GELU>(g, c, r0 + 8, acc[4 * j + 2]);
                        epi_linear_t<F16, OUT_F32, GELU>(g, c + 1, r0 + 8, acc[4 * j + 3]);
                    } else {
                        epi_linear2<F16, OUT_F32, GELU>(g, r0, c, acc[4 * j], acc[4 * j + 1]);
                        epi_linear2<F16, OUT_F32, GELU>(g, r0 + 8, c, acc[4 * j + 2], acc[4 * j + 3]);
                    }
                }
            } else {
                // 64-column blocks (a RoPE head / a gate|up pair): columns c and c + 32 sit in the same thread
#pragma unroll
                for (int hb = 0; hb < BN / 64; ++hb) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int lo = 4 * (hb * 8 + j), hi = 4 * (hb * 8 + j + 4);
                        const int blk0 = n0 + hb * 64, c = j * 8 + q * 2;
                        if (MODE == VR_EPI_ROPE) {
                            epi_rope2<F16>(g, r0, blk0, c, acc[lo], acc[lo + 1], acc[hi], acc[hi + 1]);
                            epi_rope2<F16>(g, r0 + 8, blk0, c, acc[lo + 2], acc[lo + 3], acc[hi + 2], acc[hi + 3]);
                        } else {
                            epi_swiglu2<F16>(g, r0, blk0, c, acc[lo], acc[lo + 1], acc[hi], acc[hi + 1]);
                            epi_swiglu2<F16>(g, r0 + 8, blk0, c, acc[lo + 2], acc[lo + 3], acc[hi + 2], acc[hi + 3]);
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// Ping-pong schedule: each consumer warpgroup owns a whole 128 x 128 tile (two m64n128k16 row halves per k16 step,
// 128 accumulator registers per thread) and the CTA's tiles alternate between the two warpgroups (tile i of the CTA
// goes to warpgroup 1 + i % 2). The producer fills one ring in tile order, so warpgroup w finds tile i's k-blocks at
// ring position i * num_kb. The mainloops take turns through a named-barrier handoff: a warpgroup waits for its turn,
// issues its whole k-loop, passes the turn on, and only then waits for its MMAs and runs its epilogue - so the epilogue
// of one tile runs while the other warpgroup's MMAs of the next tile keep the tensor cores busy.
constexpr int GEMM_PP_BN = 128;
constexpr int GEMM_PP_A_BYTES = GEMM_BM * GEMM_BK * 2;
constexpr int GEMM_PP_B_BYTES = GEMM_PP_BN * GEMM_BK * 2;
constexpr int GEMM_PP_STAGE_BYTES = GEMM_PP_A_BYTES + GEMM_PP_B_BYTES;               // 32 KB
constexpr int GEMM_PP_STAGES = (192 * 1024) / GEMM_PP_STAGE_BYTES;                    // 6
// + align slack + barriers + the lean epilogue's bias slots (128 fp32 per consumer warpgroup). With the 1 KB the
// system reserves per block this is 195.25 KB, within the 196 KB shared-memory carveout that the kernel needs
// without the slots, so the SM's L1 keeps the same size.
constexpr int GEMM_PP_SMEM_BYTES = GEMM_PP_STAGES * GEMM_PP_STAGE_BYTES + 1024 + 256 + 2 * GEMM_PP_BN * 4;
constexpr int GEMM_PP_BAR_BIAS = 3;  // named barriers 3 and 4: the lean epilogue's bias slot of warpgroup 1 / 2 is full
constexpr int GEMM_PP_BAR_TURN = 1;  // named barriers 1 (warpgroup 1's turn) and 2 (warpgroup 2's turn); 0 is __syncthreads

// Tile order. A wave of CTAs reads its weight tiles from L2 only if the weight columns it works on stay resident while
// the wave sweeps down M. So the N tiles are cut into the fewest equal slices whose weight (128 rows x K bf16 per tile)
// fits in GEMM_PP_L2_SLICE bytes - under half of the 50 MB L2, leaving room for the A rows in flight and the output
// stream - and the tiles are ordered slice by slice, then by M row, N tile fastest. A wave then covers about
// grid / slice_width M rows of one slice. Where the whole weight fits (all ViT GEMMs, LM o_proj) there is one slice
// and this is plain n-fastest order; LM qkv (54 tiles) and down (18 tiles at K = 5760) take 2 slices, gate|up (90) 3,
// so each weight tile is read from HBM about once per slice instead of once per M row of the wave.
constexpr long long GEMM_PP_L2_SLICE = 20ll << 20;

// The schedule works on units: a unit is CLUSTER vertically adjacent tiles of one N column (one tile without clusters,
// the two tiles of a CTA pair with them). Computed on the host; slice_w = tiles_n gives plain n-fastest order.
struct PPSched {
    int units_m, tiles_n, slice_w;
    __host__ __device__ int num_units() const { return units_m * tiles_n; }
    // unit -> (M unit index, N tile index)
    __device__ void coords(int u, int& um, int& tn) const {
        const int slice_units = units_m * slice_w;
        const int s = u / slice_units, r = u - s * slice_units;
        const int w = min(slice_w, tiles_n - s * slice_w);  // the last slice may be narrower
        um = r / w;
        tn = s * slice_w + r % w;
    }
};

inline PPSched pp_schedule(int M, int N, int K, int cluster, bool l2_slices) {
    PPSched s;
    s.units_m = ((M + GEMM_BM - 1) / GEMM_BM + cluster - 1) / cluster;
    s.tiles_n = (N + GEMM_PP_BN - 1) / GEMM_PP_BN;
    s.slice_w = s.tiles_n;
    if (l2_slices) {
        long long fit = GEMM_PP_L2_SLICE / (static_cast<long long>(GEMM_PP_BN) * K * 2);
        if (fit < 1) fit = 1;
        if (fit < s.tiles_n) {
            const int slices = static_cast<int>((s.tiles_n + fit - 1) / fit);
            s.slice_w = (s.tiles_n + slices - 1) / slices;
        }
    }
    return s;
}

// 4 x 4 transpose of 32-bit words across the 4 lanes of a quad (lane q = lane % 4): on entry lane q holds w[j] = E(q, j),
// on exit w[j] = E(j, q). Two butterfly stages (lane ^ 2, then lane ^ 1), each exchanging the two words whose index bit
// differs from the lane's. Every lane of the warp must take part.
__device__ __forceinline__ void quad_transpose4(uint32_t (&w)[4], int q) {
    const bool b1 = q & 2, b0 = q & 1;
    uint32_t r0 = __shfl_xor_sync(0xffffffffu, b1 ? w[0] : w[2], 2);
    uint32_t r1 = __shfl_xor_sync(0xffffffffu, b1 ? w[1] : w[3], 2);
    if (b1) { w[0] = r0; w[1] = r1; } else { w[2] = r0; w[3] = r1; }
    r0 = __shfl_xor_sync(0xffffffffu, b0 ? w[0] : w[1], 1);
    r1 = __shfl_xor_sync(0xffffffffu, b0 ? w[2] : w[3], 1);
    if (b0) { w[0] = r0; w[2] = r1; } else { w[1] = r0; w[3] = r1; }
}

// LINEAR epilogue of one 64 x 128 row half, the same arithmetic as epi_linear2 in the same order. The output may be the
// residual itself (in place), so the compiler cannot move a load above an earlier store: written pair by pair, every
// fragment pair waits for a full memory round trip. Here the loads of PP_EPI_BATCH column groups (both rows) are
// issued together before any of their stores - one round trip per batch.
constexpr int PP_EPI_BATCH = 4;
template <bool F16, bool OUT_F32, bool GELU>
__device__ __forceinline__ void pp_epilogue_linear(const GemmArgs& g, const float (&acc)[64], int r0, int n0, int q2) {
    const vr_gemm_epilogue& e = g.epi;
    const bool row_ok[2] = {r0 < g.M, r0 + 8 < g.M};
    const long long o[2] = {static_cast<long long>(r0) * e.ldo, static_cast<long long>(r0 + 8) * e.ldo};
    long long ra[2] = {0, 0};
    if (e.rowadd) {
        ra[0] = static_cast<long long>(r0 % e.rowadd_period) * g.N;
        ra[1] = static_cast<long long>((r0 + 8) % e.rowadd_period) * g.N;
    }
#pragma unroll
    for (int jb = 0; jb < GEMM_PP_BN / 8; jb += PP_EPI_BATCH) {
        float2 bias[PP_EPI_BATCH], add[PP_EPI_BATCH][2], res[PP_EPI_BATCH][2];
#pragma unroll
        for (int j = 0; j < PP_EPI_BATCH; ++j) {
            const int c = n0 + (jb + j) * 8 + q2;
            const bool col_ok = c < g.N;
            bias[j] = make_float2(0.0f, 0.0f);
            if (e.bias && col_ok) bias[j] = __ldg(reinterpret_cast<const float2*>(e.bias + c));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                add[j][h] = res[j][h] = make_float2(0.0f, 0.0f);
                if (e.rowadd && col_ok && row_ok[h]) add[j][h] = __ldg(reinterpret_cast<const float2*>(e.rowadd + ra[h] + c));
                if (e.resid && col_ok && row_ok[h]) res[j][h] = *reinterpret_cast<const float2*>(e.resid + o[h] + c);
            }
        }
        uint32_t w16[2][PP_EPI_BATCH];  // 16-bit output: the packed pairs, stored below 16 bytes per thread
#pragma unroll
        for (int j = 0; j < PP_EPI_BATCH; ++j) {
            const int c = n0 + (jb + j) * 8 + q2;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (OUT_F32 && (!row_ok[h] || c >= g.N)) continue;
                float x0 = acc[4 * (jb + j) + 2 * h], x1 = acc[4 * (jb + j) + 2 * h + 1];
                if (e.bias) { x0 += bias[j].x; x1 += bias[j].y; }
                if (GELU) gelu_erf2(x0, x1);
                if (e.scale != 1.0f) { x0 *= e.scale; x1 *= e.scale; }
                if (e.rowadd) { x0 += add[j][h].x; x1 += add[j][h].y; }
                if (e.resid) { x0 += res[j][h].x; x1 += res[j][h].y; }
                if (OUT_F32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(e.out) + o[h] + c) = make_float2(x0, x1);
                else w16[h][j] = pack16x2<F16>(x0, x1);
            }
        }
        if (!OUT_F32) {
            // lane q of a quad holds columns 8 (jb + j) + 2q, +1 of the batch's column groups j; after the transpose it
            // holds all 8 columns of column group jb + q: one 16-byte store per row instead of four 4-byte ones (a
            // warp's store then fills whole 32-byte sectors of its 8 rows instead of half of each)
            static_assert(PP_EPI_BATCH == 4, "the quad transpose moves 4 column groups");
            const int q = q2 >> 1, c = n0 + (jb + q) * 8;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                quad_transpose4(w16[h], q);
                if (row_ok[h] && c < g.N)
                    *reinterpret_cast<uint4*>(reinterpret_cast<half16_t<F16>*>(e.out) + o[h] + c) =
                        make_uint4(w16[h][0], w16[h][1], w16[h][2], w16[h][3]);
            }
        }
    }
}

// The lean LINEAR epilogue: 16-bit output, a bias, GELU or not, scale 1, no row add, no residual - every 16-bit LINEAR
// class of the encode step (ViT qkv and fc1, resampler k / v). An epilogue warpgroup has one warp per SM sub-partition,
// so nothing hides its latencies and its time is its instruction path. This one has no code for the absent terms,
// reads the bias from a shared-memory slot that was filled while the MMAs ran (pp_stage_bias), runs a batch's 16 GELUs
// as interleaved chains, and an interior tile (GUARD = false) stores without row or column tests. Per element the
// arithmetic is pp_epilogue_linear's (acc + bias, then GELU), so the bits are the same.
// The bias stays out of registers: 128 accumulators plus 32 bias registers leave ptxas too few to interleave the GELUs.
// Thread t of a consumer warpgroup copies bias column n0 + t of its tile into the warpgroup's slot (none past N: those
// columns are not stored).
__device__ __forceinline__ void pp_stage_bias(float* slot, const GemmArgs& g, int n0, int t) {
    if (n0 + t < g.N) cp_async_4(slot + t, g.epi.bias + n0 + t);
}
template <bool F16, bool GELU, bool GUARD>
__device__ __forceinline__ void pp_epilogue_lean(const GemmArgs& g, const float (&acc)[64], const float* bias, int r0, int n0,
                                                 int q) {
    const vr_gemm_epilogue& e = g.epi;
    // after the quad transpose lane q stores the 8 columns of group jb + q: base column n0 + 8 q
    half16_t<F16>* out = reinterpret_cast<half16_t<F16>*>(e.out) + static_cast<long long>(r0) * e.ldo + n0 + 8 * q;
    const long long row8 = 8 * e.ldo;
    const bool row_ok[2] = {r0 < g.M, r0 + 8 < g.M};
#pragma unroll
    for (int jb = 0; jb < GEMM_PP_BN / 8; jb += 4) {
        float x[16];  // x[4 j + 2 h + k] = acc[4 (jb + j) + 2 h + k]: column group jb + j, row r0 + 8 h, column 2 (lane % 4) + k
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 b = ld_shared_f2(bias + 8 * (jb + j) + 2 * q);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                x[4 * j + 2 * h] = acc[4 * (jb + j) + 2 * h] + b.x;
                x[4 * j + 2 * h + 1] = acc[4 * (jb + j) + 2 * h + 1] + b.y;
            }
        }
        if (GELU) gelu_erf_n(x);
        uint32_t w16[2][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) w16[h][j] = pack16x2<F16>(x[4 * j + 2 * h], x[4 * j + 2 * h + 1]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            quad_transpose4(w16[h], q);
            if (!GUARD || (row_ok[h] && n0 + 8 * (jb + q) < g.N))
                *reinterpret_cast<uint4*>(out + h * row8 + 8 * jb) = make_uint4(w16[h][0], w16[h][1], w16[h][2], w16[h][3]);
        }
    }
}

// epilogue of one 64 x 128 row half: accumulator rows r0 and r0 + 8, columns n0 + 8 j + q2 (+1), q2 = 2 (lane % 4)
template <bool F16, int MODE, bool OUT_F32, bool GELU>
__device__ __forceinline__ void pp_epilogue(const GemmArgs& g, const float (&acc)[64], int r0, int n0, int q2) {
    if (MODE == VR_EPI_LINEAR) {
        pp_epilogue_linear<F16, OUT_F32, GELU>(g, acc, r0, n0, q2);
    } else {
        // 64-column blocks (a RoPE head / a gate|up pair): columns c and c + 32 sit in the same thread
#pragma unroll
        for (int hb = 0; hb < GEMM_PP_BN / 64; ++hb) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int lo = 4 * (hb * 8 + j), hi = 4 * (hb * 8 + j + 4);
                const int blk0 = n0 + hb * 64, c = j * 8 + q2;
                if (MODE == VR_EPI_ROPE) {
                    epi_rope2<F16>(g, r0, blk0, c, acc[lo], acc[lo + 1], acc[hi], acc[hi + 1]);
                    epi_rope2<F16>(g, r0 + 8, blk0, c, acc[lo + 2], acc[lo + 3], acc[hi + 2], acc[hi + 3]);
                } else {
                    epi_swiglu2<F16>(g, r0, blk0, c, acc[lo], acc[lo + 1], acc[hi], acc[hi + 1]);
                    epi_swiglu2<F16>(g, r0 + 8, blk0, c, acc[lo + 2], acc[lo + 3], acc[hi + 2], acc[hi + 3]);
                }
            }
        }
    }
}

// CLUSTER = 2: CTA pairs take M tiles 2u and 2u + 1 of the same N tile. Each CTA loads its own A box and one 64-row
// half of the shared B tile, multicast to both CTAs, so each CTA stages its full 32 KB stage while it reads only 24 KB
// from L2. A stage is refilled only when the consumers of BOTH CTAs are done with it (the partner's producer writes
// into it too): every consumer warp arrives on the empty barrier of both CTAs. Both CTAs walk the same unit sequence,
// so their rings stay in step. With an odd number of M tiles the last pair's second tile lies past M: TMA fills it
// with zeros (the bytes still count) and the epilogue's row guard drops it.
// LEAN: the lean 16-bit LINEAR epilogue (pp_epilogue_lean); the host selects it when the epilogue is exactly bias [+ GELU].
template <bool F16, int MODE, bool OUT_F32, bool GELU, int CLUSTER, bool LEAN = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmArgs g,
                     const PPSched sch) {
    static_assert(CLUSTER == 1 || CLUSTER == 2, "CTA pairs at most");
    static_assert(!LEAN || (MODE == VR_EPI_LINEAR && !OUT_F32), "the lean epilogue writes 16-bit LINEAR outputs");
    constexpr int STAGES = GEMM_PP_STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * GEMM_PP_A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * GEMM_PP_STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    float* bias_slots = reinterpret_cast<float*>(smem + STAGES * GEMM_PP_STAGE_BYTES + 256);

    const int wg = threadIdx.x >> 7;
    const int warp = (threadIdx.x >> 5) & 3;
    const int lane = threadIdx.x & 31;
    const int num_kb = (g.K + GEMM_BK - 1) / GEMM_BK;
    const int rank = CLUSTER == 1 ? 0 : static_cast<int>(cluster_ctarank());
    const int unit0 = blockIdx.x / CLUSTER, unit_step = gridDim.x / CLUSTER;  // the pair's units: unit0 + k unit_step
    const int num_units = sch.num_units();

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 4 * CLUSTER);  // each warp of the owning warpgroup, in every CTA of the cluster
        }
        fence_mbar_init();  // release at cluster scope: the partner arrives on these barriers and multicasts into them
    }
    if (CLUSTER == 1) __syncthreads();
    else cluster_sync_all();  // both CTAs' barriers are initialised before either issues a multicast or remote arrive

    if (wg == 0) {
        // ------------------------------------------------------------ TMA producer: the CTA's tiles in order
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int u = unit0; u < num_units; u += unit_step) {
                int um, tn;
                sch.coords(u, um, tn);
                const int m0 = (um * CLUSTER + rank) * GEMM_BM, n0 = tn * GEMM_PP_BN;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], GEMM_PP_STAGE_BYTES);
                    // rows past the matrix (A or B) read as zeros and count their bytes
                    tma_load_2d(&tmap_a, &full_bar[stage], smem_a + stage * GEMM_PP_A_BYTES, kb * GEMM_BK, m0);
                    uint8_t* b_dst = smem_b + stage * GEMM_PP_B_BYTES;
                    if (CLUSTER == 1) {
#pragma unroll
                        for (int h = 0; h < GEMM_PP_BN / 64; ++h)
                            tma_load_2d(&tmap_b, &full_bar[stage], b_dst + h * (64 * GEMM_BK * 2), kb * GEMM_BK, n0 + h * 64);
                    } else {
                        tma_load_2d_multicast(&tmap_b, &full_bar[stage], b_dst + rank * (64 * GEMM_BK * 2), kb * GEMM_BK,
                                              n0 + rank * 64, 0x3);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ------------------------------------------------------------ consumers: tiles i = wg - 1, wg + 1, ...
        setmaxnreg_inc<232>();
        const int me = wg - 1;
        const uint64_t desc_hi = make_smem_desc(0, 16, 1024, kLayoutSW128);
        const uint32_t a_lo0 = smem_u32(smem_a) >> 4, b_lo0 = smem_u32(smem_b) >> 4;
        constexpr uint32_t HALF = (64 * GEMM_BK * 2) >> 4;  // rows 64..127 of the A stage
        const int g8 = lane >> 2, q = lane & 3;
        float* bias_slot = bias_slots + me * GEMM_PP_BN;  // LEAN only
        // release a stage: one arrival per warp on the empty barrier of every CTA of the cluster
        auto release = [&](int s) {
            if (lane != 0) return;
            if (CLUSTER == 1) {
                mbar_arrive(&empty_bar[s]);
            } else {
#pragma unroll
                for (int r = 0; r < CLUSTER; ++r) mbar_arrive_cluster(&empty_bar[s], r);
            }
        };
        for (int i = me, u = unit0 + me * unit_step; u < num_units; i += 2, u += 2 * unit_step) {
            const int pos = i * num_kb;  // ring position of this tile's first k-block
            int stage = pos % STAGES;
            uint32_t phase = (pos / STAGES) & 1;
            if (i > 0) named_bar_sync(GEMM_PP_BAR_TURN + me, 256);  // the previous tile's MMAs are all issued
            if constexpr (LEAN) {
                // every warp of this warpgroup has passed the turn barrier, so its reads of the previous tile's bias
                // are done; the copy completes under the mainloop
                int um, tn;
                sch.coords(u, um, tn);
                pp_stage_bias(bias_slot, g, tn * GEMM_PP_BN, threadIdx.x & 127);
            }
            float acc0[64], acc1[64];  // rows 0..63 and 64..127 of the tile
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t ad = desc_hi | static_cast<uint64_t>(a_lo0 + stage * (GEMM_PP_A_BYTES >> 4));
                const uint64_t bd = desc_hi | static_cast<uint64_t>(b_lo0 + stage * (GEMM_PP_B_BYTES >> 4));
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    wgmma_ss<F16, false>(acc0, ad + 2 * kk, bd + 2 * kk, (kb | kk) != 0, std::integral_constant<int, 128>());
                    wgmma_ss<F16, false>(acc1, ad + HALF + 2 * kk, bd + 2 * kk, (kb | kk) != 0,
                                           std::integral_constant<int, 128>());
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();
                    release(prev);
                }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            // pass the turn on only if the CTA has a next tile: every arrive then meets exactly one bar.sync
            if (u + unit_step < num_units) named_bar_arrive(GEMM_PP_BAR_TURN + (me ^ 1), 256);
            wgmma_wait<0>();
            release(prev);
            wgmma_touch(acc0);
            wgmma_touch(acc1);

            int um, tn;
            sch.coords(u, um, tn);
            const int m0 = (um * CLUSTER + rank) * GEMM_BM, n0 = tn * GEMM_PP_BN;
            if constexpr (LEAN) {
                cp_async_wait_all();
                named_bar_sync(GEMM_PP_BAR_BIAS + me, 128);  // every thread's bias column has landed
                if (m0 + GEMM_BM <= g.M && n0 + GEMM_PP_BN <= g.N) {
                    pp_epilogue_lean<F16, GELU, false>(g, acc0, bias_slot, m0 + warp * 16 + g8, n0, q);
                    pp_epilogue_lean<F16, GELU, false>(g, acc1, bias_slot, m0 + 64 + warp * 16 + g8, n0, q);
                } else {
                    pp_epilogue_lean<F16, GELU, true>(g, acc0, bias_slot, m0 + warp * 16 + g8, n0, q);
                    pp_epilogue_lean<F16, GELU, true>(g, acc1, bias_slot, m0 + 64 + warp * 16 + g8, n0, q);
                }
            } else {
                pp_epilogue<F16, MODE, OUT_F32, GELU>(g, acc0, m0 + warp * 16 + g8, n0, q * 2);
                pp_epilogue<F16, MODE, OUT_F32, GELU>(g, acc1, m0 + 64 + warp * 16 + g8, n0, q * 2);
            }
        }
    }
    // The partner may still multicast into this CTA's ring or arrive on its barriers until it has drained its own
    // work: neither CTA exits before both are done.
    if (CLUSTER == 2) cluster_sync_all();
}

}  // namespace vr
