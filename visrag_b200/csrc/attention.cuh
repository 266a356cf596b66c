// Flash-style attention on wgmma for the three attention shapes of VisRAG-Ret
// (ViT 16x72 non-causal, MiniCPM 36x64 causal var-len, Resampler 18x128 cross-attention).
//
// One CTA = one (64*NWG-query tile, head, sequence):
//   warpgroup 0 (one lane) : TMA producer. Q once, then K and V tiles of 128 keys through two-stage rings.
//   warpgroups 1..NWG      : each owns 64 query rows and walks the same K/V stream:
//               S = Q K^T  (m64 x n128 x k=head_stride, operands from shared memory) -> fp32 registers
//               softmax on the accumulator fragments (a row lives in the 4 lanes of a quad: two shuffles per
//               reduction), running max / sum in registers
//               O += P V   (P stays in registers: the accumulator fragment layout of S is the A-operand layout of
//               the next MMA; V is read MN-major from the same swizzled tile TMA wrote)
// NWG = 2 (sequences longer than 64 queries) stages every K/V tile once for 128 queries and hides the softmax under the
// other warpgroup's MMAs (ping-pong): named barriers 1 and 2 pass the turn to issue MMAs back and forth, so while one
// warpgroup runs its softmax, the tensor cores work on the other's S = Q K^T and O += P V. Each turn issues
// S_{j+1} = Q K_{j+1}^T and O += P_j V_j back to back as one batch. The source waits for S_{j+1}, runs its softmax and
// then waits for P_j V_j, but ptxas (CUDA 12.9) moves that second wait up to the first shuffle of the row max. So the
// exponentials do not run under the warpgroup's own PV MMA; the overlap comes from the ping-pong alone.
// Its softmax is branch-free: full key tiles take no mask, partial and diagonal tiles set masked scores to -inf with
// selects, and each p is one FFMA plus one ex2.approx.ftz.
// At head stride 128 (no caller in the model has more than 64 queries there), O, S and P of this form would not fit the
// register budget together, so that stride keeps the sequential per-tile loop for both warpgroups.
// NWG = 1 is the kernel for sequences of up to 64 queries (the resampler's 64 learned queries).
// Both loops run the same arithmetic per query row: the same S MMAs, the same masked att_softmax_tile, O rescaled by alpha
// before P V is added, and the same store. Key tiles past a row's causal limit change nothing (alpha = 1, p = 0). So a
// sequence's output does not depend on which form ran it, and hence not on max_q or on the other sequences of the batch.
//
// Head dims that are not multiples of 64 (ViT: 72, stored padded to 80 with zero columns) are
// split into a 64-wide 128B-swizzled chunk plus a 16-wide 32B-swizzled chunk, each with its own
// TMA box and MMA descriptor.
#pragma once
#include "ptx.cuh"
#include "../../include/visrag_b200.h"

namespace vr {

constexpr int ATT_BN = 128;  // keys per iteration
constexpr int ATT_STAGES = 2;

template <int HS, int NWG>
struct AttCfg {
    static constexpr int BM = 64 * NWG;                 // queries per CTA
    static constexpr int THREADS = 384;                 // producer + two more warpgroups (with NWG = 1 the third only donates registers)
    static constexpr int NCH = HS / 64;                 // 64-wide swizzle-128B chunks
    static constexpr bool HAS16 = (HS % 64) == 16;      // extra 16-wide swizzle-32B chunk
    static_assert(HS == 64 || HS == 80 || HS == 128, "head stride must be 64, 80 or 128");
    static constexpr int Q_CHUNK = BM * 128;            // one 64-column chunk of the Q tile
    static constexpr int Q_BYTES = NCH * Q_CHUNK + (HAS16 ? BM * 32 : 0);
    static constexpr int TILE_BYTES = NCH * 16384 + (HAS16 ? 4096 : 0);  // 128 keys x HS x 2B
    static constexpr int OFF_Q = 0;
    static constexpr int OFF_K = (Q_BYTES + 1023) & ~1023;
    static constexpr int OFF_V = OFF_K + ATT_STAGES * TILE_BYTES;
    static constexpr int OFF_BAR = OFF_V + ATT_STAGES * TILE_BYTES;
    static constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;  // 10 mbarriers of 8 B in the 128 at OFF_BAR
};

struct AttArgs {
    int q_col0, k_col0, v_col0;
    int head_dim;  // output columns per head
    int heads, batch;
    const int* cu_q;
    const int* cu_k;
    int max_q;
    float scale_log2;  // scale * log2(e)
    void* out;         // bf16, or fp16 when the kernel's F16 is set
    long long ldo;
};

struct AttMaps {
    CUtensorMap q64, q16, k64, k16, v64, v16;
};

// Write O / l for the two accumulator rows of this thread (head_dim columns; the zero pad columns of a 72->80 head are
// dropped). l_a / l_b are this thread's partial row sums; the quad reduces them here.
template <bool F16, int NCH, bool HAS16>
__device__ __forceinline__ void att_store(const AttArgs& a, const float (&o)[NCH][32], const float (&o16)[8], float l_a, float l_b,
                                          int row_a, int len_q, int q_begin, int b, int head, int q4) {
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int q_idx = row_a + 8 * half;
        if (q_idx >= len_q) continue;
        const float inv = 1.0f / (half ? l_b : l_a);
        const long long row = a.cu_q ? (long long)(q_begin + q_idx) : (long long)b * a.max_q + q_idx;
        half16_t<F16>* dst = reinterpret_cast<half16_t<F16>*>(a.out) + row * a.ldo + head * a.head_dim;
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = c * 64 + j * 8 + q4 * 2;
                if (col < a.head_dim)
                    *reinterpret_cast<uint32_t*>(dst + col) = pack16x2<F16>(o[c][4 * j + 2 * half] * inv, o[c][4 * j + 2 * half + 1] * inv);
            }
        if (HAS16) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int col = NCH * 64 + j * 8 + q4 * 2;
                if (col < a.head_dim)
                    *reinterpret_cast<uint32_t*>(dst + col) = pack16x2<F16>(o16[4 * j + 2 * half] * inv, o16[4 * j + 2 * half + 1] * inv);
            }
        }
    }
}

// Online softmax of one key tile on the S fragments (registers 4j+0/1 = row a, 4j+2/3 = row b, keys 8j + 2 q4 + 0/1);
// masked scores are already -inf. s becomes p; m / l are updated and alpha (the factor for O) is returned.
// c = scale * log2(e). p = ex2(s c - m c) is one FFMA on the rounded product m c, and alpha = ex2(m_old c - m c) uses the
// same rounded products, so a row's rounding of the shift is a common factor of O and l and cancels in O / l.
__device__ __forceinline__ void att_softmax_tile(float (&s)[64], float c, float& m_a, float& m_b, float& l_a, float& l_b,
                                                 float& alpha_a, float& alpha_b) {
    float mt_a = m_a, mt_b = m_b;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        mt_a = fmaxf(mt_a, fmaxf(s[4 * j], s[4 * j + 1]));
        mt_b = fmaxf(mt_b, fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
    mt_a = fmaxf(mt_a, __shfl_xor_sync(0xffffffffu, mt_a, 1));
    mt_a = fmaxf(mt_a, __shfl_xor_sync(0xffffffffu, mt_a, 2));
    mt_b = fmaxf(mt_b, __shfl_xor_sync(0xffffffffu, mt_b, 1));
    mt_b = fmaxf(mt_b, __shfl_xor_sync(0xffffffffu, mt_b, 2));
    // a row that has seen no key yet keeps m = -inf: shift by 0 (its p are all 0), and alpha = ex2(-inf) = 0
    // __fmul_rn: m c must be the rounded product here too, so no FFMA contraction into the alpha argument
    const float mc_a = mt_a == -INFINITY ? 0.f : __fmul_rn(mt_a, c), mc_b = mt_b == -INFINITY ? 0.f : __fmul_rn(mt_b, c);
    alpha_a = ex2_ftz(__fmul_rn(m_a, c) - mc_a);
    alpha_b = ex2_ftz(__fmul_rn(m_b, c) - mc_b);
    m_a = mt_a;
    m_b = mt_b;
    float lt_a = 0.f, lt_b = 0.f;  // this thread's 32 p of each row, summed in order
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            s[4 * j + e] = ex2_ftz(__fmaf_rn(s[4 * j + e], c, -mc_a));
            s[4 * j + 2 + e] = ex2_ftz(__fmaf_rn(s[4 * j + 2 + e], c, -mc_b));
            lt_a += s[4 * j + e];
            lt_b += s[4 * j + 2 + e];
        }
    }
    l_a = l_a * alpha_a + lt_a;
    l_b = l_b * alpha_b + lt_b;
}

// F16: Q, K, V, P and the output are fp16 (else bf16). P is rounded to nearest with no flush, so p below 2^-14 enter the
// P V MMA as fp16 subnormals instead of zeros. The softmax and everything kept in fp32 are the same in both types.
template <int HS, bool CAUSAL, int NWG, bool F16>
// Register file: 384 threads x 168 as compiled; the producer warpgroup (and, with NWG = 1, the idle third one) hands its
// share to the consumers: 40 / 232 / 232 resp. 40 / 232 / 40. The same block shape for both forms keeps every role
// branch warpgroup-uniform with a known register budget.
__global__ void __launch_bounds__(384, 1)
attention_wgmma_kernel(const __grid_constant__ AttMaps maps, const AttArgs a) {
    using Cfg = AttCfg<HS, NWG>;
    constexpr int NCH = Cfg::NCH;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem + Cfg::OFF_Q;
    uint8_t* sK = smem + Cfg::OFF_K;
    uint8_t* sV = smem + Cfg::OFF_V;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
    uint64_t* q_bar = bars + 0;
    uint64_t* k_full = bars + 1;                   // [ATT_STAGES]
    uint64_t* k_empty = k_full + ATT_STAGES;
    uint64_t* v_full = k_empty + ATT_STAGES;
    uint64_t* v_empty = v_full + ATT_STAGES;
    uint64_t* v_tail = v_empty + ATT_STAGES;       // TMA of a partial last V tile, before its rows past len_k are zeroed

    const int wg = threadIdx.x >> 7;
    const int warp = (threadIdx.x >> 5) & 3;
    const int lane = threadIdx.x & 31;
    const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;

    const int k_begin = a.cu_k[b];
    const int len_k = a.cu_k[b + 1] - k_begin;
    const int q_begin = a.cu_q ? a.cu_q[b] : 0;
    const int len_q = a.cu_q ? a.cu_q[b + 1] - q_begin : a.max_q;
    const int q0 = qt * Cfg::BM;
    if (q0 >= len_q || len_k <= 0) return;  // uniform per CTA: nothing set up yet

    int nkt = (len_k + ATT_BN - 1) / ATT_BN;
    if (CAUSAL) {
        // keys visible to the last query row of this tile: index <= q + (len_k - len_q)
        const int last_q = min(q0 + Cfg::BM, len_q) - 1;
        const int max_key = last_q + (len_k - len_q);
        nkt = min(nkt, max_key / ATT_BN + 1);
    }

    if (threadIdx.x == 0) {
        mbar_init(q_bar, 1);
        for (int i = 0; i < ATT_STAGES; ++i) {
            mbar_init(&k_full[i], 1);
            mbar_init(&v_full[i], 1);
            mbar_init(&k_empty[i], NWG * 4);  // one arrival per consumer warp
            mbar_init(&v_empty[i], NWG * 4);
        }
        mbar_init(v_tail, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0 || wg > NWG) {
        // ---------------------------------------------------------------- TMA producer (warpgroup 0)
        setmaxnreg_dec<40>();
        if (wg == 0 && warp == 0) {
            // Sequences are packed, so a last tile that ends past len_k holds the next sequence's K and V rows. Its K rows
            // only give scores that the consumers replace by -inf, but P V would still multiply their p = 0 by those V
            // rows, and 0 * inf or 0 * NaN is NaN. So the V rows [tail, 128) of that tile are zeroed before the
            // consumers may read it: its TMA lands on v_tail, this warp clears the rows, and only then arrives on v_full.
            const int tail = len_k - (nkt - 1) * ATT_BN;  // keys of the last loaded tile inside the sequence
            const int st_last = (nkt - 1) % ATT_STAGES;
            if (lane == 0) {
                const int qcol = a.q_col0 + head * HS, kcol = a.k_col0 + head * HS, vcol = a.v_col0 + head * HS;
                mbar_expect_tx(q_bar, Cfg::Q_BYTES);
#pragma unroll
                for (int c = 0; c < NCH; ++c) tma_load_2d(&maps.q64, q_bar, sQ + c * Cfg::Q_CHUNK, qcol + c * 64, q_begin + q0);
                if (Cfg::HAS16) tma_load_2d(&maps.q16, q_bar, sQ + NCH * Cfg::Q_CHUNK, qcol + NCH * 64, q_begin + q0);
                auto load_tile = [&](const CUtensorMap* m64, const CUtensorMap* m16, uint64_t* bar, uint8_t* dst, int col, int row) {
                    mbar_expect_tx(bar, Cfg::TILE_BYTES);
#pragma unroll
                    for (int c = 0; c < NCH; ++c) tma_load_2d(m64, bar, dst + c * 16384, col + c * 64, row);
                    if (Cfg::HAS16) tma_load_2d(m16, bar, dst + NCH * 16384, col + NCH * 64, row);
                };
                for (int kt = 0; kt < nkt; ++kt) {
                    const int st = kt % ATT_STAGES;
                    const uint32_t ph = (kt / ATT_STAGES) & 1;
                    mbar_wait(&k_empty[st], ph ^ 1);
                    load_tile(&maps.k64, &maps.k16, &k_full[st], sK + st * Cfg::TILE_BYTES, kcol, k_begin + kt * ATT_BN);
                    mbar_wait(&v_empty[st], ph ^ 1);
                    load_tile(&maps.v64, &maps.v16, kt == nkt - 1 && tail < ATT_BN ? v_tail : &v_full[st],
                              sV + st * Cfg::TILE_BYTES, vcol, k_begin + kt * ATT_BN);
                }
            }
            __syncwarp();
            if (tail < ATT_BN) {
                // A key row is contiguous in both layouts (128 B in a 64-wide 128B-swizzled chunk, 32 B in the 16-wide
                // 32B-swizzled one: the swizzles permute 16-byte units within a row), so rows [tail, 128) are one range.
                uint8_t* dst = sV + st_last * Cfg::TILE_BYTES;
                const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
                mbar_wait(v_tail, 0);
#pragma unroll
                for (int c = 0; c < NCH; ++c)
                    for (int i = tail * 8 + lane; i < ATT_BN * 8; i += 32) reinterpret_cast<uint4*>(dst + c * 16384)[i] = zero;
                if (Cfg::HAS16)
                    for (int i = tail * 2 + lane; i < ATT_BN * 2; i += 32) reinterpret_cast<uint4*>(dst + NCH * 16384)[i] = zero;
                fence_proxy_async_smem();  // the generic-proxy stores, before the consumers' wgmma reads them
                __syncwarp();
                if (lane == 0) mbar_arrive(&v_full[st_last]);
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumers
    setmaxnreg_inc<232>();
    const int cw = wg - 1;
    const int g8 = lane >> 2, q4 = lane & 3;
    const int row_a = q0 + cw * 64 + warp * 16 + g8;  // query index (inside the sequence) of accumulator rows g8 / g8 + 8
    const int row_b = row_a + 8;
    const int causal_shift = len_k - len_q;
    const uint32_t q_addr = smem_u32(sQ) + cw * (64 * 128);
    const uint32_t q16_addr = smem_u32(sQ) + NCH * Cfg::Q_CHUNK + cw * (64 * 32);

    if constexpr (NWG == 2 && HS != 128) {
        const float c = a.scale_log2;
        float o[NCH][32];
        float o16[8];
#pragma unroll
        for (int cc = 0; cc < NCH; ++cc)
#pragma unroll
            for (int j = 0; j < 32; ++j) o[cc][j] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) o16[j] = 0.f;
        float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f, alpha_a, alpha_b;
        float s[64];
        uint32_t pa[ATT_BN / 16][4];  // P in bf16 / fp16 as the A operand: k step kk = accumulator column blocks 2kk, 2kk+1

        auto issue_s = [&](int kt) {  // S = Q K_kt^T
            const uint32_t k_addr = smem_u32(sK) + (kt % ATT_STAGES) * Cfg::TILE_BYTES;
#pragma unroll
            for (int cc = 0; cc < NCH; ++cc) {
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_ss<F16, false>(s, make_smem_desc(q_addr + cc * Cfg::Q_CHUNK + kk * 32, 16, 1024, kLayoutSW128),
                                           make_smem_desc(k_addr + cc * 16384 + kk * 32, 16, 1024, kLayoutSW128), (cc | kk) != 0,
                                           std::integral_constant<int, 128>());
            }
            if (Cfg::HAS16)
                wgmma_ss<F16, false>(s, make_smem_desc(q16_addr, 16, 256, kLayoutSW32),
                                       make_smem_desc(k_addr + NCH * 16384, 16, 256, kLayoutSW32), 1, std::integral_constant<int, 128>());
            wgmma_commit();
        };
        auto issue_pv = [&](int kt) {  // O += P V_kt
            const uint32_t v_addr = smem_u32(sV) + (kt % ATT_STAGES) * Cfg::TILE_BYTES;
#pragma unroll
            for (int kk = 0; kk < ATT_BN / 16; ++kk) {
#pragma unroll
                for (int cc = 0; cc < NCH; ++cc)  // V chunk: [128 keys][64 dims], 128 B per key row -> MN-major
                    wgmma_rs_tb<F16>(o[cc], pa[kk], make_smem_desc(v_addr + cc * 16384 + kk * 2048, 16, 1024, kLayoutSW128), 1,
                                std::integral_constant<int, 64>());
                if (Cfg::HAS16)  // [128 keys][16 dims], 32 B per key row
                    wgmma_rs_tb<F16>(o16, pa[kk], make_smem_desc(v_addr + NCH * 16384 + kk * 512, 16, 256, kLayoutSW32), 1,
                                std::integral_constant<int, 16>());
            }
            wgmma_commit();
        };
        // S of key tile kt has landed in s: mask it where needed, then s -> p
        const int row0 = q0 + cw * 64;  // first query row of this warpgroup
        auto softmax = [&](int kt) {
            const int key0 = kt * ATT_BN;
            // full tile: every key exists, and (causal) every row of the warpgroup sees every key. Warpgroup-uniform.
            const bool full = key0 + ATT_BN <= len_k && (!CAUSAL || key0 + ATT_BN - 1 <= row0 + causal_shift);
            if (!full) {
                int lim_a = len_k - key0, lim_b = lim_a;  // keys [0, lim) of this tile exist for the row
                if (CAUSAL) {
                    lim_a = min(lim_a, row_a + causal_shift - key0 + 1);
                    lim_b = min(lim_b, row_b + causal_shift - key0 + 1);
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int key = j * 8 + q4 * 2 + e;
                        s[4 * j + e] = key < lim_a ? s[4 * j + e] : -INFINITY;
                        s[4 * j + 2 + e] = key < lim_b ? s[4 * j + 2 + e] : -INFINITY;
                    }
                }
            }
            att_softmax_tile(s, c, m_a, m_b, l_a, l_b, alpha_a, alpha_b);
        };
        auto pack_p = [&] {
#pragma unroll
            for (int kk = 0; kk < ATT_BN / 16; ++kk) {
                pa[kk][0] = pack16x2<F16>(s[8 * kk + 0], s[8 * kk + 1]);
                pa[kk][1] = pack16x2<F16>(s[8 * kk + 2], s[8 * kk + 3]);
                pa[kk][2] = pack16x2<F16>(s[8 * kk + 4], s[8 * kk + 5]);
                pa[kk][3] = pack16x2<F16>(s[8 * kk + 6], s[8 * kk + 7]);
            }
        };
        auto rescale_o = [&] {
#pragma unroll
            for (int cc = 0; cc < NCH; ++cc)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[cc][4 * j] *= alpha_a; o[cc][4 * j + 1] *= alpha_a;
                    o[cc][4 * j + 2] *= alpha_b; o[cc][4 * j + 3] *= alpha_b;
                }
            if (Cfg::HAS16) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    o16[4 * j] *= alpha_a; o16[4 * j + 1] *= alpha_a;
                    o16[4 * j + 2] *= alpha_b; o16[4 * j + 3] *= alpha_b;
                }
            }
        };
        // Ping-pong turn to issue MMAs: warpgroup cw waits on named barrier 1 + cw and passes the turn on 2 - cw (256
        // threads each: 128 waiting, 128 arriving). Both warpgroups take nkt + 1 turns, so the counts match; warpgroup 1's
        // first arrival lets warpgroup 0 start, and warpgroup 0 takes warpgroup 1's last arrival before it leaves.
        auto turn_wait = [&] { named_bar_sync(1 + cw, 256); };
        auto turn_pass = [&] { named_bar_arrive(2 - cw, 256); };
        if (cw == 1) named_bar_arrive(1, 256);

        // prologue: S_0 and its softmax
        mbar_wait(q_bar, 0);
        mbar_wait(&k_full[0], 0);
        turn_wait();
        wgmma_fence();
        issue_s(0);
        turn_pass();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&k_empty[0]);
        wgmma_touch(s);
        softmax(0);
        pack_p();
        // steady state: one turn issues S_{kt+1} and P_kt V_kt; then the softmax of S_{kt+1} and the rescale of O
        for (int kt = 0; kt + 1 < nkt; ++kt) {
            const int st = kt % ATT_STAGES, st1 = (kt + 1) % ATT_STAGES;
            mbar_wait(&k_full[st1], ((kt + 1) / ATT_STAGES) & 1);
            mbar_wait(&v_full[st], (kt / ATT_STAGES) & 1);
            turn_wait();
            wgmma_fence();
            issue_s(kt + 1);
            issue_pv(kt);
            turn_pass();
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(&k_empty[st1]);
            wgmma_touch(s);
            softmax(kt + 1);
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&v_empty[st]);
#pragma unroll
            for (int cc = 0; cc < NCH; ++cc) wgmma_touch(o[cc]);
            wgmma_touch(o16);
            rescale_o();
            pack_p();
        }
        // last key tile: P V only
        {
            const int kt = nkt - 1, st = kt % ATT_STAGES;
            mbar_wait(&v_full[st], (kt / ATT_STAGES) & 1);
            turn_wait();
            wgmma_fence();
            issue_pv(kt);
            turn_pass();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&v_empty[st]);
#pragma unroll
            for (int cc = 0; cc < NCH; ++cc) wgmma_touch(o[cc]);
            wgmma_touch(o16);
        }
        if (cw == 0) turn_wait();
        att_store<F16, NCH, Cfg::HAS16>(a, o, o16, l_a, l_b, row_a, len_q, q_begin, b, head, q4);
    } else {  // NWG = 1, and NWG = 2 at head stride 128: each warpgroup takes each key tile in turn
        float o[NCH][32];
        float o16[8];
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int j = 0; j < 32; ++j) o[c][j] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) o16[j] = 0.f;
        float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;

        mbar_wait(q_bar, 0);
        for (int kt = 0; kt < nkt; ++kt) {
            const int st = kt % ATT_STAGES;
            const uint32_t ph = (kt / ATT_STAGES) & 1;
            const uint32_t k_addr = smem_u32(sK) + st * Cfg::TILE_BYTES, v_addr = smem_u32(sV) + st * Cfg::TILE_BYTES;
            // ---- S = Q K^T
            float s[64];
            mbar_wait(&k_full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_ss<F16, false>(s, make_smem_desc(q_addr + c * Cfg::Q_CHUNK + kk * 32, 16, 1024, kLayoutSW128),
                                           make_smem_desc(k_addr + c * 16384 + kk * 32, 16, 1024, kLayoutSW128), (c | kk) != 0,
                                           std::integral_constant<int, 128>());
            }
            if (Cfg::HAS16)
                wgmma_ss<F16, false>(s, make_smem_desc(q16_addr, 16, 256, kLayoutSW32),
                                       make_smem_desc(k_addr + NCH * 16384, 16, 256, kLayoutSW32), 1, std::integral_constant<int, 128>());
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&k_empty[st]);
            wgmma_touch(s);

            // ---- softmax on the fragments: masked scores -> -inf, then the same arithmetic as the pipelined form, so a
            // sequence gets the same bits from either form (and from either side of the max_q <= 64 dispatch)
            const int key0 = kt * ATT_BN;
            int lim_a = len_k - key0, lim_b = lim_a;  // keys [0, lim) of this tile exist for the row
            if (CAUSAL) {
                lim_a = min(lim_a, row_a + causal_shift - key0 + 1);
                lim_b = min(lim_b, row_b + causal_shift - key0 + 1);
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int key = j * 8 + q4 * 2 + e;
                    s[4 * j + e] = key < lim_a ? s[4 * j + e] : -INFINITY;
                    s[4 * j + 2 + e] = key < lim_b ? s[4 * j + 2 + e] : -INFINITY;
                }
            }
            float alpha_a, alpha_b;
            att_softmax_tile(s, a.scale_log2, m_a, m_b, l_a, l_b, alpha_a, alpha_b);
            // ---- O = O * alpha + P V
#pragma unroll
            for (int c = 0; c < NCH; ++c)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[c][4 * j] *= alpha_a; o[c][4 * j + 1] *= alpha_a;
                    o[c][4 * j + 2] *= alpha_b; o[c][4 * j + 3] *= alpha_b;
                }
            if (Cfg::HAS16) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    o16[4 * j] *= alpha_a; o16[4 * j + 1] *= alpha_a;
                    o16[4 * j + 2] *= alpha_b; o16[4 * j + 3] *= alpha_b;
                }
            }
            // P as the A operand: 16 keys = accumulator column blocks 2kk, 2kk+1 -> the four A registers of k step kk. All of
            // them are written before the fence: register operands of an MMA must not change between fence and wait.
            uint32_t pa[ATT_BN / 16][4];
#pragma unroll
            for (int kk = 0; kk < ATT_BN / 16; ++kk) {
                pa[kk][0] = pack16x2<F16>(s[8 * kk + 0], s[8 * kk + 1]);
                pa[kk][1] = pack16x2<F16>(s[8 * kk + 2], s[8 * kk + 3]);
                pa[kk][2] = pack16x2<F16>(s[8 * kk + 4], s[8 * kk + 5]);
                pa[kk][3] = pack16x2<F16>(s[8 * kk + 6], s[8 * kk + 7]);
            }
            mbar_wait(&v_full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < ATT_BN / 16; ++kk) {
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    // V chunk: [128 keys][64 dims], 128 B per key row -> MN-major, 8-key groups 1024 B apart
                    wgmma_rs_tb<F16>(o[c], pa[kk], make_smem_desc(v_addr + c * 16384 + kk * 2048, 16, 1024, kLayoutSW128), 1,
                                std::integral_constant<int, 64>());
                }
                if (Cfg::HAS16) {
                    // [128 keys][16 dims], 32 B per key row
                    wgmma_rs_tb<F16>(o16, pa[kk], make_smem_desc(v_addr + NCH * 16384 + kk * 512, 16, 256, kLayoutSW32), 1,
                                std::integral_constant<int, 16>());
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&v_empty[st]);
#pragma unroll
            for (int c = 0; c < NCH; ++c) wgmma_touch(o[c]);
            wgmma_touch(o16);
        }

        att_store<F16, NCH, Cfg::HAS16>(a, o, o16, l_a, l_b, row_a, len_q, q_begin, b, head, q4);
    }
}

}  // namespace vr
