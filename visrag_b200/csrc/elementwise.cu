// HBM-bound kernels of the encode path: patch unfold + normalise, LayerNorm, RMSNorm, LM input
// assembly, final norm + pooling + L2 normalise. All of them stream the activation once with 16-byte
// accesses; row statistics are computed in fp32 with a warp per row (rows are <= 9 KB, so the second
// and third sweep of a row hit L1).
#include "common.h"
#include "ptx.cuh"
#include "../../include/visrag_b200.h"

namespace vr {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------
// im2col + normalise. One CTA per (slice, patch row): the strip of `patch` full-width pixel rows is ONE contiguous,
// 4-byte aligned span of patch*w*3 bytes; it is staged in shared memory with 16-byte (or 4-byte) coalesced loads,
// then every thread builds 8 consecutive output columns (col = c*p*p + ky*p + kx) of one patch from shared memory and
// writes them with one 16-byte store (a warp writes 512 contiguous bytes). ToTensor + Normalize(0.5, 0.5) is one
// FFMA: bf16(fma(u, 2/255, -1)) == bf16((u/255 - 0.5)/0.5) for all 256 byte values (tests/test_gpu_kernels.py checks
// every value), so the division of the fp32 reference is not needed for a bit-identical bf16 result. The same holds for
// fp16 (F16): fp16(fma(u, 2/255, -1)) == fp16((u/255 - 0.5)/0.5) for all 256 values (tests/test_fp16_host.py).
// CHUNKED: for strips wider than the shared-memory buffer (patch 14: 347 patches = 4858 pixels and wider). A CTA then takes
// one chunk of at most `cg` patch columns of a strip, staged row by row (the chunk's pixel rows are `patch` spans of
// cg*patch*3 bytes, w*3 bytes apart); every output value is computed by the same FFMA, so the result is the same bits.
// ---------------------------------------------------------------------------------------------
constexpr int IM2COL_THREADS = 256;

template <bool F16, bool CHUNKED>
__global__ void __launch_bounds__(IM2COL_THREADS)
im2col_norm_kernel(const uint8_t* __restrict__ px, int n_strips, int gw, int patch, half16_t<F16>* __restrict__ out,
                   long long ldo, int cg) {
    extern __shared__ __align__(16) uint8_t strip[];  // [patch][pitch] + offset table [groups*8] (uint16)
    const int w3 = CHUNKED ? 0 : gw * patch * 3;
    const int pitch = CHUNKED ? (cg * patch * 3 + 15) & ~15 : w3;  // bytes per staged pixel row (chunks: 16-byte multiple)
    const int strip_bytes = patch * pitch;
    const int groups = static_cast<int>(ldo / 8);
    const int pp = patch * patch, kvalid = 3 * pp;
    const int n_chunks = CHUNKED ? (gw + cg - 1) / cg : 1;
    unsigned short* off = reinterpret_cast<unsigned short*>(strip + ((strip_bytes + 15) & ~15));
    // column -> (ky << 8 | kx*3 + c): position inside the strip relative to the patch's first pixel (0xFFFF = pad column)
    for (int col = threadIdx.x; col < groups * 8; col += IM2COL_THREADS) {
        unsigned short o = 0xFFFFu;
        if (col < kvalid) {
            const int c = col / pp, rem = col - c * pp;
            const int ky = rem / patch, kx = rem - ky * patch;
            o = static_cast<unsigned short>((ky << 8) | (kx * 3 + c));
        }
        off[col] = o;
    }
    for (int unit = blockIdx.x; unit < n_strips * n_chunks; unit += gridDim.x) {
        const int sidx = CHUNKED ? unit / n_chunks : unit;
        const int p0 = CHUNKED ? (unit - sidx * n_chunks) * cg : 0;  // first patch column of the chunk
        const int pc = CHUNKED ? min(cg, gw - p0) : gw;              // patch columns in the chunk
        __syncthreads();  // previous strip fully consumed (and the offset table written, first iteration)
        if constexpr (CHUNKED) {
            const long long row_bytes = static_cast<long long>(gw) * patch * 3;
            const uint8_t* src = px + static_cast<long long>(sidx) * patch * row_bytes + static_cast<long long>(p0) * patch * 3;
            const int cb = pc * patch * 3;  // bytes of the chunk in each pixel row
            const uintptr_t al = reinterpret_cast<uintptr_t>(src) | static_cast<uintptr_t>(row_bytes) | static_cast<uintptr_t>(cb);
            if ((al & 3) == 0) {
                const int vpr = cb >> 2;
                for (int i = threadIdx.x; i < patch * vpr; i += IM2COL_THREADS) {
                    const int r = i / vpr, c = i - r * vpr;
                    *reinterpret_cast<uint32_t*>(strip + r * pitch + c * 4) = __ldg(reinterpret_cast<const uint32_t*>(src + r * row_bytes) + c);
                }
            } else {
                for (int i = threadIdx.x; i < patch * cb; i += IM2COL_THREADS) {
                    const int r = i / cb, c = i - r * cb;
                    strip[r * pitch + c] = __ldg(src + r * row_bytes + c);
                }
            }
        } else {
            const uint8_t* src = px + static_cast<long long>(sidx) * strip_bytes;
            if (((reinterpret_cast<uintptr_t>(src) | static_cast<uintptr_t>(strip_bytes)) & 15) == 0) {
                const uint4* s4 = reinterpret_cast<const uint4*>(src);
                uint4* d4 = reinterpret_cast<uint4*>(strip);
                for (int i = threadIdx.x; i < (strip_bytes >> 4); i += IM2COL_THREADS) d4[i] = __ldg(s4 + i);
            } else if (((reinterpret_cast<uintptr_t>(src) | static_cast<uintptr_t>(strip_bytes)) & 3) == 0) {
                const uint32_t* s1 = reinterpret_cast<const uint32_t*>(src);
                uint32_t* d1 = reinterpret_cast<uint32_t*>(strip);
                for (int i = threadIdx.x; i < (strip_bytes >> 2); i += IM2COL_THREADS) d1[i] = __ldg(s1 + i);
            } else {
                for (int i = threadIdx.x; i < strip_bytes; i += IM2COL_THREADS) strip[i] = __ldg(src + i);
            }
        }
        __syncthreads();
        half16_t<F16>* orow0 = out + (static_cast<long long>(sidx) * gw + p0) * ldo;
        const int items = pc * groups;
        for (int it = threadIdx.x; it < items; it += IM2COL_THREADS) {
            const int p = it / groups, g = it - p * groups;
            const uint4 o8 = *reinterpret_cast<const uint4*>(off + g * 8);
            const uint8_t* base = strip + p * patch * 3;
            const uint32_t ow[4] = {o8.x, o8.y, o8.z, o8.w};
            uint32_t pk[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t oa = ow[j] & 0xFFFFu, ob = ow[j] >> 16;
                const uint32_t aa = (oa >> 8) * pitch + (oa & 0xFFu), ab = (ob >> 8) * pitch + (ob & 0xFFu);
                const float va = oa == 0xFFFFu ? 0.f : fmaf(static_cast<float>(base[aa]), 2.0f / 255.0f, -1.0f);
                const float vb = ob == 0xFFFFu ? 0.f : fmaf(static_cast<float>(base[ab]), 2.0f / 255.0f, -1.0f);
                pk[j] = pack16x2<F16>(va, vb);
            }
            *reinterpret_cast<uint4*>(orow0 + static_cast<long long>(p) * ldo + g * 8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        }
    }
}

// Patch 14 (the only size the model uses): one thread per (patch, pixel row) = 42 contiguous source bytes -> three runs
// of 14 bf16 (one per channel) in the patch's output row. Bytes become floats with one PRMT each (0x4B0000xx = 2^23 + u,
// then - 2^23: exact, and no I2F on the quarter-rate conversion pipe), the output rows of the strip are assembled in
// shared memory and leave with ONE bulk (TMA) store per strip while the next strip is being loaded.
constexpr int IM2COL14_THREADS = 224;  // 7 warps: 14 pixel rows x 16 patches per round

// BULK: the pixel rows are 16-byte multiples at 16-byte aligned addresses -> the strip is staged by 14 bulk (TMA) row
// copies onto an mbarrier, double buffered: strip i+1 streams in while strip i is converted (a version with ordinary
// loads is latency bound: too few loads in flight per SM).
template <bool BULK, bool F16>
__global__ void __launch_bounds__(IM2COL14_THREADS)
im2col_norm14_kernel(const uint8_t* __restrict__ px, int n_strips, int gw, half16_t<F16>* __restrict__ out, int ldo) {
    constexpr int P = 14, RUN = P * 3;  // 42 bytes per (patch, pixel row)
    constexpr int NBUF = BULK ? 2 : 1;
    extern __shared__ __align__(16) uint8_t smem14[];
    __shared__ __align__(8) uint64_t bars[2];
    const int w3 = gw * RUN;            // bytes per pixel row of the strip (a multiple of 42, hence even)
    // shared-memory row pitch: 16-byte multiple with an odd number of 16-byte units, so that the 14 pixel rows of a patch
    // (consecutive lanes) start in different banks (w3 itself is 1344 B = 16 banks apart for 448-pixel slices)
    const int pitch = (((w3 + 15) >> 4) | 1) << 4;
    const int in_bytes = P * pitch + 16;  // + 16: the last item's 12-word window reads past its 42 bytes
    uint8_t* tile = smem14 + NBUF * in_bytes;  // [gw][ldo] 16-bit, exactly the layout of the strip's output rows
    const int tile_bytes = gw * ldo * 2;
    const int strip_bytes = P * w3;
    // zero the padding columns once: they are never written again
    for (int i = threadIdx.x; i < gw * (ldo - 3 * P * P); i += IM2COL14_THREADS) {
        const int p = i / (ldo - 3 * P * P), c = i - p * (ldo - 3 * P * P);
        reinterpret_cast<half16_t<F16>*>(tile)[p * ldo + 3 * P * P + c] = to_half16<F16>(0.f);
    }
    for (int i = threadIdx.x; i < NBUF * in_bytes / 4; i += IM2COL14_THREADS) reinterpret_cast<uint32_t*>(smem14)[i] = 0;
    if (BULK && threadIdx.x == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
    }
    fence_proxy_async_smem();  // the zero fill above must be ordered before the bulk copies into the same buffers
    __syncthreads();
    auto issue = [&](int sidx, int buf) {  // thread 0 only
        const uint8_t* src = px + static_cast<long long>(sidx) * strip_bytes;
        mbar_expect_tx(&bars[buf], static_cast<uint32_t>(strip_bytes));
        for (int r = 0; r < P; ++r) bulk_load_1d(smem14 + buf * in_bytes + r * pitch, src + r * w3, static_cast<uint32_t>(w3), &bars[buf]);
    };
    if (BULK && threadIdx.x == 0 && blockIdx.x < n_strips) issue(blockIdx.x, 0);
    int k = 0;
    for (int sidx = blockIdx.x; sidx < n_strips; sidx += gridDim.x, ++k) {
        uint8_t* strip = smem14 + (BULK ? (k & 1) * in_bytes : 0);
        if (BULK) {
            // buffer (k+1)&1 was read by iteration k-1, which every thread left through the barrier below
            if (threadIdx.x == 0 && sidx + static_cast<int>(gridDim.x) < n_strips) issue(sidx + gridDim.x, (k + 1) & 1);
            mbar_wait(&bars[k & 1], (k >> 1) & 1);
        } else {
            const uint8_t* src = px + static_cast<long long>(sidx) * strip_bytes;
            if ((w3 & 3) == 0) {  // 4-byte aligned rows (the strip start always is: 588*gw bytes per strip)
                const int vpr = w3 >> 2;
                for (int i = threadIdx.x; i < P * vpr; i += IM2COL14_THREADS) {
                    const int r = i / vpr, c = i - r * vpr;
                    *reinterpret_cast<uint32_t*>(strip + r * pitch + c * 4) = __ldcs(reinterpret_cast<const uint32_t*>(src) + i);
                }
            } else {  // odd grid width: rows are only 2-byte aligned
                const int vpr = w3 >> 1;
                for (int i = threadIdx.x; i < P * vpr; i += IM2COL14_THREADS) {
                    const int r = i / vpr, c = i - r * vpr;
                    *reinterpret_cast<unsigned short*>(strip + r * pitch + c * 2) = __ldcs(reinterpret_cast<const unsigned short*>(src) + i);
                }
            }
        }
        if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // previous strip's tile has left
        __syncthreads();
        for (int it = threadIdx.x; it < gw * P; it += IM2COL14_THREADS) {
            const int p = it / P, ky = it - p * P;
            const int off = ky * pitch + p * RUN;  // even
            const uint32_t* wsrc = reinterpret_cast<const uint32_t*>(strip + (off & ~3));
            uint32_t w[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) w[i] = wsrc[i];
            if (off & 2) {
#pragma unroll
                for (int i = 0; i < 11; ++i) w[i] = __funnelshift_r(w[i], w[i + 1], 16);
            }
            uint32_t* dst = reinterpret_cast<uint32_t*>(tile + (p * ldo + ky * P) * 2);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
#pragma unroll
                for (int i = 0; i < P / 2; ++i) {
                    const int k0 = (2 * i) * 3 + c, k1 = (2 * i + 1) * 3 + c;  // byte index of pixel 2i / 2i+1, channel c
                    const float f0 = __uint_as_float(__byte_perm(w[k0 >> 2], 0x4B000000u, 0x7540 | (k0 & 3))) - 8388608.0f;
                    const float f1 = __uint_as_float(__byte_perm(w[k1 >> 2], 0x4B000000u, 0x7540 | (k1 & 3))) - 8388608.0f;
                    dst[c * (P * P / 2) + i] = pack16x2<F16>(fmaf(f0, 2.0f / 255.0f, -1.0f), fmaf(f1, 2.0f / 255.0f, -1.0f));
                }
            }
        }
        fence_proxy_async_smem();  // generic-proxy writes -> visible to the bulk copy engine
        __syncthreads();
        if (threadIdx.x == 0) {
            half16_t<F16>* gdst = out + static_cast<long long>(sidx) * gw * ldo;
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(tile)),
                         "r"(tile_bytes)
                         : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// LayerNorm / RMSNorm: one warp per row, dim % 4 == 0. Statistics in fp32; the output is stored as bf16 or (F16) fp16.
// ---------------------------------------------------------------------------------------------
template <bool RMS, bool F16>
__global__ void norm_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma,
                            const float* __restrict__ beta, float eps, int rows, int dim,
                            half16_t<F16>* __restrict__ out, long long ldo, half16_t<F16>* __restrict__ out2,
                            const float* __restrict__ add, int add_period) {
    const int warps_per_block = blockDim.x >> 5;
    const int lane = threadIdx.x & 31;
    const int nvec = dim >> 2;
    for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps_per_block) {
        const float4* xr = reinterpret_cast<const float4*>(x + static_cast<long long>(row) * ldx);
        float mean = 0.f;
        if (!RMS) {
            float s = 0.f;
            for (int i = lane; i < nvec; i += 32) {
                const float4 v = xr[i];
                s += (v.x + v.y) + (v.z + v.w);
            }
            mean = warp_sum(s) / static_cast<float>(dim);
        }
        float ss = 0.f;
        for (int i = lane; i < nvec; i += 32) {
            const float4 v = xr[i];
            const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
            ss += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(ss) / static_cast<float>(dim) + eps);
        half16_t<F16>* orow = out + static_cast<long long>(row) * ldo;
        half16_t<F16>* orow2 = out2 ? out2 + static_cast<long long>(row) * ldo : nullptr;
        const float* arow = add ? add + static_cast<long long>(row % add_period) * dim : nullptr;
        for (int i = lane; i < nvec; i += 32) {
            const float4 v = xr[i];
            const float4 g = reinterpret_cast<const float4*>(gamma)[i];
            float y0 = (v.x - mean) * rstd * g.x, y1 = (v.y - mean) * rstd * g.y;
            float y2 = (v.z - mean) * rstd * g.z, y3 = (v.w - mean) * rstd * g.w;
            if (!RMS) {
                const float4 bb = reinterpret_cast<const float4*>(beta)[i];
                y0 += bb.x; y1 += bb.y; y2 += bb.z; y3 += bb.w;
            }
            uint2 pk;
            pk.x = pack16x2<F16>(y0, y1);
            pk.y = pack16x2<F16>(y2, y3);
            reinterpret_cast<uint2*>(orow)[i] = pk;
            if (orow2) {
                const float4 aa = reinterpret_cast<const float4*>(arow)[i];
                uint2 pk2;
                pk2.x = pack16x2<F16>(y0 + aa.x, y1 + aa.y);
                pk2.y = pack16x2<F16>(y2 + aa.z, y3 + aa.w);
                reinterpret_cast<uint2*>(orow2)[i] = pk2;
            }
        }
    }
}

// Register-resident variant for dim == VPL * 128 (1152 -> VPL 9, 2304 -> VPL 18): the row is read from HBM exactly once.
template <bool RMS, int VPL, bool F16>
__global__ void __launch_bounds__(256)
norm_kernel_reg(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
                float eps, int rows, half16_t<F16>* __restrict__ out, long long ldo, half16_t<F16>* __restrict__ out2,
                const float* __restrict__ add, int add_period) {
    constexpr int DIM = VPL * 128;
    const int warps_per_block = blockDim.x >> 5;
    const int lane = threadIdx.x & 31;
    for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps_per_block) {
        const float4* xr = reinterpret_cast<const float4*>(x + static_cast<long long>(row) * ldx);
        float4 v[VPL];
#pragma unroll
        for (int i = 0; i < VPL; ++i) v[i] = xr[lane + i * 32];
        float mean = 0.f;
        if (!RMS) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < VPL; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
            mean = warp_sum(s) * (1.0f / DIM);
        }
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            ss += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(ss) * (1.0f / DIM) + eps);
        uint2* orow = reinterpret_cast<uint2*>(out + static_cast<long long>(row) * ldo);
        uint2* orow2 = out2 ? reinterpret_cast<uint2*>(out2 + static_cast<long long>(row) * ldo) : nullptr;
        const float4* arow = add ? reinterpret_cast<const float4*>(add + static_cast<long long>(row % add_period) * DIM) : nullptr;
#pragma unroll
        for (int i = 0; i < VPL; ++i) {
            const int c = lane + i * 32;
            const float4 g = reinterpret_cast<const float4*>(gamma)[c];
            float y0 = (v[i].x - mean) * rstd * g.x, y1 = (v[i].y - mean) * rstd * g.y;
            float y2 = (v[i].z - mean) * rstd * g.z, y3 = (v[i].w - mean) * rstd * g.w;
            if (!RMS) {
                const float4 bb = reinterpret_cast<const float4*>(beta)[c];
                y0 += bb.x; y1 += bb.y; y2 += bb.z; y3 += bb.w;
            }
            uint2 pk;
            pk.x = pack16x2<F16>(y0, y1);
            pk.y = pack16x2<F16>(y2, y3);
            orow[c] = pk;
            if (orow2) {
                const float4 aa = arow[c];
                uint2 pk2;
                pk2.x = pack16x2<F16>(y0 + aa.x, y1 + aa.y);
                pk2.y = pack16x2<F16>(y2 + aa.z, y3 + aa.w);
                orow2[c] = pk2;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// LM input assembly: one warp per token row.
// ---------------------------------------------------------------------------------------------
template <bool F16>
__global__ void build_lm_input_kernel(const int* __restrict__ src, int tokens, int dim,
                                      const half16_t<F16>* __restrict__ embed, float scale_emb,
                                      const float* __restrict__ vision, long long ldv, float* __restrict__ h,
                                      long long ldh) {
    const int warps_per_block = blockDim.x >> 5;
    const int lane = threadIdx.x & 31;
    for (int t = blockIdx.x * warps_per_block + (threadIdx.x >> 5); t < tokens; t += gridDim.x * warps_per_block) {
        const int s = src[t];
        float4* dst = reinterpret_cast<float4*>(h + static_cast<long long>(t) * ldh);
        if (s >= 0) {
            const float4* v = reinterpret_cast<const float4*>(vision + static_cast<long long>(s) * ldv);
            for (int i = lane; i < (dim >> 2); i += 32) dst[i] = v[i];
        } else {
            const uint2* e = reinterpret_cast<const uint2*>(embed + static_cast<long long>(-(s + 1)) * dim);
            for (int i = lane; i < (dim >> 2); i += 32) {
                const uint2 raw = e[i];
                const float2 a = unpack16x2<F16>(raw.x), b = unpack16x2<F16>(raw.y);  // exact
                dst[i] = make_float4(a.x * scale_emb, a.y * scale_emb, b.x * scale_emb, b.y * scale_emb);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Final RMSNorm + pooling + L2 normalise: one thread-block CLUSTER of 8 (or 4) CTAs per sequence, every row read from HBM once.
// The sum order is fixed by 8 virtual ranks of 4 warps each, whatever the cluster size: warp w of virtual rank v takes
// the weighted rows t_lo + 4v + w + 32k in increasing k. An 8-CTA cluster runs virtual rank v in CTA v; a 4-CTA cluster
// runs virtual ranks r and r + 4 in CTA r, one after the other, into two partial vectors. So the embedding's bits do
// not depend on the cluster size, i.e. on the batch size, nor on which other sequences share the launch.
//   phase 1: a warp holds one row in registers (VPL float4 per lane), computes 1/rms and adds w_t/rms_t * x_t into its
//            accumulator (its shared-memory staging row), one row after the other;
//   phase 2: the virtual rank's partial = ((warp 0 + warp 1) + warp 2) + warp 3, per column through shared memory;
//   phase 3: after a cluster barrier CTA 0 sums the 8 partials in virtual-rank order over distributed shared memory,
//            applies gamma / sum(w), reduces the squared norm, normalises and writes the embedding.
// pooling: 0 = wmean (w_t = t+1), 1 = mean, 2 = lasttoken, 3 = cls (dense_retrieval_model.py:170-218).
// ---------------------------------------------------------------------------------------------
constexpr int POOL_THREADS = 128;  // 4 warps x ~164 registers: three CTAs per SM (256 threads left one)
constexpr int POOL_WARPS = POOL_THREADS / 32;
constexpr int POOL_VRANKS = 8;  // virtual ranks per sequence; the cluster has 8 CTAs, or 4 when that lets every cluster be resident at once

template <int VPL, bool EXACT>
__global__ void __launch_bounds__(POOL_THREADS, VPL <= 18 ? 5 : 2)
pool_norm_kernel(const float* __restrict__ h, long long ldh, const float* __restrict__ gamma, float eps,
                 const int* __restrict__ cu, int dim, int pooling, int normalize, float* __restrict__ reps) {
    // [POOL_WARPS][VPL*128] staging, reused as the partial of the CTA's last virtual rank; with 4 CTAs one more [VPL*128]
    // holds the partial of its first
    extern __shared__ __align__(16) float pool_smem[];
    __shared__ float red[POOL_WARPS];
    __shared__ float total;
    constexpr int COLS = VPL * 128;
    const unsigned csize = cluster_nctarank();  // set by the launcher (cudaLaunchAttributeClusterDimension)
    const int b = blockIdx.x / csize;
    const unsigned rank = cluster_ctarank();
    const int begin = cu[b], len = cu[b + 1] - begin;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nvec = dim >> 2;
    float* out = reps + static_cast<long long>(b) * dim;
    if (len <= 0) {  // uniform over the cluster: nobody reaches a cluster barrier
        if (rank == 0)
            for (int c = threadIdx.x; c < dim; c += POOL_THREADS) out[c] = 0.f;
        return;
    }
    int t_lo = 0, t_hi = len;  // rows that carry weight
    if (pooling == 2) t_lo = len - 1;
    if (pooling == 3) t_hi = 1;
    // the warp's accumulator lives in its shared-memory staging row (registers hold one input row: ~100 per thread,
    // five CTAs per SM; with a register accumulator it was 164 and three)
    float4* stage = reinterpret_cast<float4*>(pool_smem) + warp * (COLS / 4);
    float4* first = reinterpret_cast<float4*>(pool_smem) + POOL_WARPS * (COLS / 4);  // 4-CTA cluster: partial of virtual rank `rank`
    for (int v = static_cast<int>(rank); v < POOL_VRANKS; v += static_cast<int>(csize)) {
        const bool last = v + static_cast<int>(csize) >= POOL_VRANKS;
#pragma unroll
        for (int i = 0; i < VPL; ++i) stage[lane + i * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int t = t_lo + v * POOL_WARPS + warp; t < t_hi; t += POOL_VRANKS * POOL_WARPS) {
            const float4* xr = reinterpret_cast<const float4*>(h + static_cast<long long>(begin + t) * ldh);
            float4 x[VPL];
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                const int c = lane + i * 32;
                x[i] = (EXACT || c < nvec) ? __ldcs(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < VPL; ++i) ss += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
            ss = warp_sum(ss);
            const float w = (pooling == 0) ? static_cast<float>(t + 1) : 1.0f;
            const float sc = w * rsqrtf(ss / static_cast<float>(dim) + eps);
#pragma unroll
            for (int i = 0; i < VPL; ++i) {
                float4 a = stage[lane + i * 32];
                a.x += sc * x[i].x; a.y += sc * x[i].y; a.z += sc * x[i].z; a.w += sc * x[i].w;
                stage[lane + i * 32] = a;
            }
        }
        __syncthreads();
        // partial of virtual rank v: column-wise sum over the warps, written over warp 0's staging area (last) or `first`
        float4* dst = last ? reinterpret_cast<float4*>(pool_smem) : first;
        for (int c = threadIdx.x; c < COLS / 4; c += POOL_THREADS) {
            float4 s4 = reinterpret_cast<const float4*>(pool_smem)[c];
#pragma unroll
            for (int wv = 1; wv < POOL_WARPS; ++wv) {
                const float4 o = reinterpret_cast<const float4*>(pool_smem)[wv * (COLS / 4) + c];
                s4.x += o.x; s4.y += o.y; s4.z += o.z; s4.w += o.w;
            }
            dst[c] = s4;  // column c of warp 0's area is read only by this thread
        }
        if (!last) __syncthreads();  // the staging rows are zeroed again for the next virtual rank
    }
    cluster_sync_all();
    if (rank == 0) {
        // sum(w) over the weighted rows in closed form (exact in fp32 for len < 4096; float otherwise)
        const float n = static_cast<float>(t_hi - t_lo);
        const float wsum = (pooling == 0) ? 0.5f * n * (n + 1.0f) : n;
        const uint32_t my = smem_u32(pool_smem);
        float sq = 0.f;
        float4 mine[(COLS / 4 + POOL_THREADS - 1) / POOL_THREADS];
#pragma unroll
        for (int k = 0; k < (COLS / 4 + POOL_THREADS - 1) / POOL_THREADS; ++k) {
            const int c = threadIdx.x + k * POOL_THREADS;
            float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < nvec) {
                for (unsigned v = 0; v < POOL_VRANKS; ++v) {  // virtual rank v's partial: CTA v % csize, `first` unless it is that CTA's last
                    const uint32_t off = v + csize >= POOL_VRANKS ? 0u : POOL_WARPS * COLS * 4u;
                    const float4 o = ld_shared_cluster_f4(mapa_u32(my + off + c * 16, v % csize));
                    s4.x += o.x; s4.y += o.y; s4.z += o.z; s4.w += o.w;
                }
                const float4 g = reinterpret_cast<const float4*>(gamma)[c];
                s4.x = s4.x * g.x / wsum; s4.y = s4.y * g.y / wsum; s4.z = s4.z * g.z / wsum; s4.w = s4.w * g.w / wsum;
                sq += (s4.x * s4.x + s4.y * s4.y) + (s4.z * s4.z + s4.w * s4.w);
            }
            mine[k] = s4;
        }
        sq = warp_sum(sq);
        if (lane == 0) red[warp] = sq;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s1 = 0.f;
            for (int i = 0; i < POOL_WARPS; ++i) s1 += red[i];
            total = s1;
        }
        __syncthreads();
        const float inv = normalize ? 1.0f / fmaxf(sqrtf(total), 1e-12f) : 1.0f;
#pragma unroll
        for (int k = 0; k < (COLS / 4 + POOL_THREADS - 1) / POOL_THREADS; ++k) {
            const int c = threadIdx.x + k * POOL_THREADS;
            if (c < nvec)
                reinterpret_cast<float4*>(out)[c] = make_float4(mine[k].x * inv, mine[k].y * inv, mine[k].z * inv, mine[k].w * inv);
        }
    }
    cluster_sync_all();  // the peers' shared memory must stay alive until CTA 0 has read it
}

static int grid_for(long long work_items, int per_block) {
    long long blocks = (work_items + per_block - 1) / per_block;
    const long long cap = static_cast<long long>(num_sms()) * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return static_cast<int>(blocks);
}

template <bool F16>
static int im2col_norm_impl(const uint8_t* pixels, int32_t n_slices, int32_t h, int32_t w, int32_t patch, void* out, int64_t ldo,
                            cudaStream_t st) {
    const int gw = w / patch;
    const long long n_strips = static_cast<long long>(n_slices) * (h / patch);
    VR_REQUIRE(n_strips < (1ll << 31), "vr_im2col_norm: too many patch rows");
    half16_t<F16>* o = reinterpret_cast<half16_t<F16>*>(out);
    long long blocks = n_strips;
    if (patch == 14 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(pixels) & 3) == 0 && (ldo & 7) == 0) {
        const size_t pitch14 = static_cast<size_t>((((w * 3 + 15) >> 4) | 1) << 4);
        const bool bulk = ((w * 3) & 15) == 0 && (reinterpret_cast<uintptr_t>(pixels) & 15) == 0;
        const size_t smem14 = (bulk ? 2 : 1) * (14 * pitch14 + 16) + static_cast<size_t>(gw) * ldo * 2;
        if (smem14 <= 200 * 1024) {
            static unsigned long long configured14 = 0;
            if (first_use_on_device(&configured14)) {
                VR_CHECK_CUDA(cudaFuncSetAttribute(im2col_norm14_kernel<true, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
                VR_CHECK_CUDA(cudaFuncSetAttribute(im2col_norm14_kernel<false, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            }
            const long long per_sm = (200 * 1024) / static_cast<long long>(smem14) < 4 ? (200 * 1024) / static_cast<long long>(smem14) : 4;
            const long long cap14 = static_cast<long long>(num_sms()) * (per_sm < 1 ? 1 : per_sm);
            if (blocks > cap14) blocks = cap14;
            if (bulk)
                im2col_norm14_kernel<true, F16><<<static_cast<int>(blocks), IM2COL14_THREADS, smem14, st>>>(
                    pixels, static_cast<int>(n_strips), gw, o, static_cast<int>(ldo));
            else
                im2col_norm14_kernel<false, F16><<<static_cast<int>(blocks), IM2COL14_THREADS, smem14, st>>>(
                    pixels, static_cast<int>(n_strips), gw, o, static_cast<int>(ldo));
            VR_CHECK_CUDA(cudaGetLastError());
            return 0;
        }
    }
    const size_t smem = ((static_cast<size_t>(patch) * w * 3 + 15) & ~static_cast<size_t>(15)) + static_cast<size_t>(ldo) * 2;
    const long long cap = static_cast<long long>(num_sms()) * 8;
    static unsigned long long configured = 0;
    if (first_use_on_device(&configured)) {
        VR_CHECK_CUDA(cudaFuncSetAttribute(im2col_norm_kernel<F16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VR_CHECK_CUDA(cudaFuncSetAttribute(im2col_norm_kernel<F16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    if (smem <= 200 * 1024) {  // the whole strip fits
        if (blocks > cap) blocks = cap;
        im2col_norm_kernel<F16, false><<<static_cast<int>(blocks), IM2COL_THREADS, smem, st>>>(pixels, static_cast<int>(n_strips), gw,
                                                                                               patch, o, ldo, gw);
        VR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    // chunks of at most cg patch columns: the largest count whose pixel rows (each padded to 16 bytes, so that the 4-byte
    // stores of every row stay aligned) fit next to the offset table, then evened out over the chunks of a strip
    const long long avail = 200 * 1024 - static_cast<long long>(ldo) * 2;
    auto rows_bytes = [&](long long c) { return patch * ((c * patch * 3 + 15) & ~15ll); };
    VR_REQUIRE(rows_bytes(1) <= avail, "vr_im2col_norm: ldo=%lld leaves no shared memory for one %d-pixel patch", (long long)ldo, patch);
    long long max_cg = avail / (3ll * patch * patch);
    while (rows_bytes(max_cg) > avail) --max_cg;
    const long long n_chunks = (gw + max_cg - 1) / max_cg;
    const int cg = static_cast<int>((gw + n_chunks - 1) / n_chunks);
    VR_REQUIRE(n_strips * n_chunks < (1ll << 31), "vr_im2col_norm: too many patch rows");
    const size_t smem_c = static_cast<size_t>(rows_bytes(cg)) + static_cast<size_t>(ldo) * 2;
    blocks = n_strips * n_chunks;
    if (blocks > cap) blocks = cap;
    im2col_norm_kernel<F16, true><<<static_cast<int>(blocks), IM2COL_THREADS, smem_c, st>>>(pixels, static_cast<int>(n_strips), gw,
                                                                                            patch, o, ldo, cg);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <bool RMS, bool F16>
static int norm_impl(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t rows, int32_t dim,
                     void* out, int64_t ldo, void* out2, const float* add, int32_t add_period, cudaStream_t s) {
    half16_t<F16>* o = reinterpret_cast<half16_t<F16>*>(out);
    half16_t<F16>* o2 = reinterpret_cast<half16_t<F16>*>(out2);
    if (dim == 2304)
        norm_kernel_reg<RMS, 18, F16><<<grid_for(rows, 8), 256, 0, s>>>(x, ldx, gamma, beta, eps, rows, o, ldo, o2, add, add_period);
    else if (!RMS && dim == 1152)
        norm_kernel_reg<RMS, 9, F16><<<grid_for(rows, 8), 256, 0, s>>>(x, ldx, gamma, beta, eps, rows, o, ldo, o2, add, add_period);
    else
        norm_kernel<RMS, F16><<<grid_for(rows, 8), 256, 0, s>>>(x, ldx, gamma, beta, eps, rows, dim, o, ldo, o2, add, add_period);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vr

using namespace vr;

extern "C" int vr_im2col_norm_ex(const uint8_t* pixels, int32_t n_slices, int32_t h, int32_t w, int32_t patch, void* out,
                                 int64_t ldo, int32_t out_dtype, void* stream) {
    VR_REQUIRE(pixels && out, "vr_im2col_norm: null pointer");
    VR_REQUIRE(n_slices > 0 && h > 0 && w > 0 && patch > 0 && h % patch == 0 && w % patch == 0,
               "vr_im2col_norm: bad geometry n=%d h=%d w=%d patch=%d", n_slices, h, w, patch);
    VR_REQUIRE(ldo % 8 == 0 && ldo >= 3 * patch * patch, "vr_im2col_norm: ldo=%lld must be a multiple of 8 and >= %d",
               (long long)ldo, 3 * patch * patch);
    VR_REQUIRE(patch <= 85, "vr_im2col_norm: patch=%d exceeds 85", patch);
    VR_REQUIRE(out_dtype == VR_BF16 || out_dtype == VR_F16, "vr_im2col_norm: out_dtype must be VR_BF16 or VR_F16 (got %d)", out_dtype);
    // every path stores 8 output columns (16 bytes) at a time; the pixel loads pick their width from the alignment
    VR_REQUIRE_ALIGNED("vr_im2col_norm", "out", out, 16);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return out_dtype == VR_F16 ? im2col_norm_impl<true>(pixels, n_slices, h, w, patch, out, ldo, st)
                               : im2col_norm_impl<false>(pixels, n_slices, h, w, patch, out, ldo, st);
}

extern "C" int vr_im2col_norm(const uint8_t* pixels, int32_t n_slices, int32_t h, int32_t w, int32_t patch, void* out,
                              int64_t ldo, void* stream) {
    return vr_im2col_norm_ex(pixels, n_slices, h, w, patch, out, ldo, VR_BF16, stream);
}

extern "C" int vr_layernorm_ex(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t rows,
                               int32_t dim, void* out, int64_t ldo, void* out2, const float* add, int32_t add_period,
                               int32_t out_dtype, void* stream) {
    VR_REQUIRE(x && gamma && beta && out, "vr_layernorm: null pointer");
    VR_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0, "vr_layernorm: bad shape rows=%d dim=%d",
               rows, dim);
    VR_REQUIRE(!out2 || (add && add_period > 0), "vr_layernorm: out2 needs add/add_period");
    VR_REQUIRE(out_dtype == VR_BF16 || out_dtype == VR_F16, "vr_layernorm: out_dtype must be VR_BF16 or VR_F16 (got %d)", out_dtype);
    // float4 loads of x, gamma, beta and add; 8-byte stores of out and out2
    VR_REQUIRE_ALIGNED("vr_layernorm", "x", x, 16);
    VR_REQUIRE_ALIGNED("vr_layernorm", "gamma", gamma, 16);
    VR_REQUIRE_ALIGNED("vr_layernorm", "beta", beta, 16);
    VR_REQUIRE_ALIGNED("vr_layernorm", "add", add, 16);
    VR_REQUIRE_ALIGNED("vr_layernorm", "out", out, 8);
    VR_REQUIRE_ALIGNED("vr_layernorm", "out2", out2, 8);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    return out_dtype == VR_F16 ? norm_impl<false, true>(x, ldx, gamma, beta, eps, rows, dim, out, ldo, out2, add, add_period, s)
                               : norm_impl<false, false>(x, ldx, gamma, beta, eps, rows, dim, out, ldo, out2, add, add_period, s);
}

extern "C" int vr_layernorm(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t rows,
                            int32_t dim, void* out, int64_t ldo, void* out2, const float* add, int32_t add_period,
                            void* stream) {
    return vr_layernorm_ex(x, ldx, gamma, beta, eps, rows, dim, out, ldo, out2, add, add_period, VR_BF16, stream);
}

extern "C" int vr_rmsnorm_ex(const float* x, int64_t ldx, const float* gamma, float eps, int32_t rows, int32_t dim, void* out,
                             int64_t ldo, int32_t out_dtype, void* stream) {
    VR_REQUIRE(x && gamma && out, "vr_rmsnorm: null pointer");
    VR_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0, "vr_rmsnorm: bad shape rows=%d dim=%d",
               rows, dim);
    VR_REQUIRE(out_dtype == VR_BF16 || out_dtype == VR_F16, "vr_rmsnorm: out_dtype must be VR_BF16 or VR_F16 (got %d)", out_dtype);
    VR_REQUIRE_ALIGNED("vr_rmsnorm", "x", x, 16);
    VR_REQUIRE_ALIGNED("vr_rmsnorm", "gamma", gamma, 16);
    VR_REQUIRE_ALIGNED("vr_rmsnorm", "out", out, 8);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    return out_dtype == VR_F16 ? norm_impl<true, true>(x, ldx, gamma, nullptr, eps, rows, dim, out, ldo, nullptr, nullptr, 1, s)
                               : norm_impl<true, false>(x, ldx, gamma, nullptr, eps, rows, dim, out, ldo, nullptr, nullptr, 1, s);
}

extern "C" int vr_rmsnorm(const float* x, int64_t ldx, const float* gamma, float eps, int32_t rows, int32_t dim, void* out,
                          int64_t ldo, void* stream) {
    return vr_rmsnorm_ex(x, ldx, gamma, eps, rows, dim, out, ldo, VR_BF16, stream);
}

extern "C" int vr_build_lm_input_ex(const int32_t* src, int32_t tokens, int32_t dim, const void* embed, int32_t embed_dtype,
                                    float scale_emb, const float* vision, int64_t ldv, float* h, int64_t ldh, void* stream) {
    VR_REQUIRE(src && embed && h, "vr_build_lm_input: null pointer");
    VR_REQUIRE(tokens > 0 && dim % 4 == 0 && ldh % 4 == 0 && (vision == nullptr || ldv % 4 == 0),
               "vr_build_lm_input: bad shape tokens=%d dim=%d", tokens, dim);
    VR_REQUIRE(embed_dtype == VR_BF16 || embed_dtype == VR_F16, "vr_build_lm_input: embed_dtype must be VR_BF16 or VR_F16 (got %d)",
               embed_dtype);
    // int32 loads of src, 8-byte loads of embed rows (dim % 4 == 0 keeps every row aligned), float4 copies of vision and h
    VR_REQUIRE_ALIGNED("vr_build_lm_input", "src", src, 4);
    VR_REQUIRE_ALIGNED("vr_build_lm_input", "embed", embed, 8);
    VR_REQUIRE_ALIGNED("vr_build_lm_input", "vision", vision, 16);
    VR_REQUIRE_ALIGNED("vr_build_lm_input", "h", h, 16);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (embed_dtype == VR_F16)
        build_lm_input_kernel<true><<<grid_for(tokens, 8), 256, 0, s>>>(src, tokens, dim, reinterpret_cast<const __half*>(embed),
                                                                        scale_emb, vision, ldv, h, ldh);
    else
        build_lm_input_kernel<false><<<grid_for(tokens, 8), 256, 0, s>>>(
            src, tokens, dim, reinterpret_cast<const __nv_bfloat16*>(embed), scale_emb, vision, ldv, h, ldh);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_build_lm_input(const int32_t* src, int32_t tokens, int32_t dim, const void* embed_bf16, float scale_emb,
                                 const float* vision, int64_t ldv, float* h, int64_t ldh, void* stream) {
    return vr_build_lm_input_ex(src, tokens, dim, embed_bf16, VR_BF16, scale_emb, vision, ldv, h, ldh, stream);
}

extern "C" int vr_pool_norm(const float* h, int64_t ldh, const float* gamma, float eps, const int32_t* cu, int32_t batch,
                            int32_t dim, int32_t pooling, int32_t normalize, float* reps, void* stream) {
    VR_REQUIRE(h && gamma && cu && reps, "vr_pool_norm: null pointer");
    VR_REQUIRE(batch > 0 && dim > 0 && dim % 4 == 0 && dim <= 4096 && ldh % 4 == 0,
               "vr_pool_norm: bad shape batch=%d dim=%d", batch, dim);
    VR_REQUIRE(pooling >= 0 && pooling <= 3, "vr_pool_norm: pooling must be 0..3");
    VR_REQUIRE((reinterpret_cast<uintptr_t>(h) & 15) == 0 && (reinterpret_cast<uintptr_t>(reps) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(gamma) & 15) == 0,
               "vr_pool_norm: h, gamma and reps must be 16-byte aligned");
    VR_REQUIRE_ALIGNED("vr_pool_norm", "cu", cu, 4);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    // 8 CTAs per sequence while all clusters fit on the GPU at once (5 CTAs per SM), else 4: one wave of longer CTAs beats
    // a second wave of whole clusters (the kernel is a latency chain: load rows -> CTA sum -> cluster sum -> normalise).
    // Both sum in the same order (virtual ranks), so the choice does not change the result.
    const unsigned csize = static_cast<long long>(batch) * POOL_VRANKS <= static_cast<long long>(num_sms()) * 5 ? POOL_VRANKS : POOL_VRANKS / 2;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(batch) * csize);
    cfg.blockDim = dim3(POOL_THREADS);
    cfg.stream = s;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = csize; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
#define VR_POOL_LAUNCH(VPL, EXACT)                                                                                        \
    do {                                                                                                                  \
        const int row_bytes = (VPL) * 128 * static_cast<int>(sizeof(float));                                              \
        static unsigned long long configured = 0;                                                                         \
        if (first_use_on_device(&configured))                                                                             \
            VR_CHECK_CUDA(cudaFuncSetAttribute(pool_norm_kernel<VPL, EXACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                               (POOL_WARPS + 1) * row_bytes));                                            \
        cfg.dynamicSmemBytes = (POOL_WARPS + (csize < POOL_VRANKS ? 1 : 0)) * row_bytes;                                  \
        VR_CHECK_CUDA(cudaLaunchKernelEx(&cfg, pool_norm_kernel<VPL, EXACT>, h, static_cast<long long>(ldh), gamma, eps, cu, dim, \
                                         pooling, normalize, reps));                                                      \
    } while (0)
    if (dim == 2304) VR_POOL_LAUNCH(18, true);
    else if (dim <= 512) VR_POOL_LAUNCH(4, false);
    else if (dim <= 2048) VR_POOL_LAUNCH(16, false);
    else VR_POOL_LAUNCH(32, false);
#undef VR_POOL_LAUNCH
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}
