// Dense query x corpus similarity + top-k (reference: torch.matmul + torch.topk, fp32, in
// retriever/dense_retriever.py:25-30), built so that the [nq, nd] score matrix never touches HBM and the
// result is the EXACT fp32 top-k:
//
//  1. score_filter_kernel : wgmma GEMM on fp16 copies of Q and D (fp32 accumulate in registers). Each CTA owns a
//     (128-query block, contiguous range of 256-doc tiles); its MMA threads keep the 16 best approximate scores of
//     their rows in registers across all tiles of the range. Output: per query
//     `lists = ranges*2` sorted candidate lists of 16 (score, doc) pairs.
//  2. rescore_topk_kernel : one CTA per query recomputes every candidate's score in fp32 on CUDA cores
//     (q . d, 2304 FMAs each), selects the top-k by (score desc, doc id asc), and PROVES the selection: every
//     doc that was dropped by a list has approximate score <= that list's 16th entry, hence exact score
//     <= tail + eps with eps = fp16 rounding bound * |q| * max|d|. If max(tail) + eps < k-th exact score the
//     result equals the full fp32 scan; otherwise the query is flagged and the caller reruns it through
//  3. exact_scores_kernel + topk_rows_kernel : plain fp32 scan (also the path for tiny problems).
//
// Tie rule everywhere: higher score first, then lower doc id.
#include "common.h"
#include "gemm.cuh"
#include <math.h>
#include <type_traits>

namespace vr {

constexpr int SC_KT = 16;    // candidates kept per list
constexpr int SC_BN = 256;   // docs per tile
constexpr int SC_MAX_RANGES = 64;  // doc ranges (= candidate lists per query) the filter may use

// Work decomposition of the filter: the unit of work is one 256-query x 256-doc tile (one CTA pair). The doc axis
// is cut into R equal ranges; item i = r*QB + b (QB = 256-query blocks) is the sweep of query block b over doc range r,
// and pair p runs items p, p+P, p+2P, ... Items have the same length and start together, so all pairs of a wave walk
// their doc range in lockstep: at any moment the whole GPU reads at most ceil(P/QB)+1 distinct doc tiles and every doc
// tile is fetched from HBM once and then served to the other query blocks from L2. (A contiguous "stream-K" split of
// the b-major tile list balances perfectly but de-phases the pairs, and every pair then streams its own doc tiles from
// DRAM.) R is chosen by the host to fill whole waves
// (score_plan); every item emits ONE 16-entry candidate list per query, so a query has R lists. Items of later waves
// start from the threshold the finished items of the same query published (tau, see the epilogue).
struct ScoreArgs {
    int nq;
    long long nd;
    int dim;
    int lists;         // candidate lists per query (>= R; the ones beyond R are written empty)
    int T;             // doc tiles
    int R;             // doc ranges
    int QB;            // 256-query blocks
    int items;         // R * QB
    float* cand_scores;  // [nq, lists*SC_KT]
    int* cand_ids;
};

// A mask set (vr_doc_masks on the device): query row r searches mask of_query[r] (of_query NULL: mask 0 for every row),
// and doc i is eligible for mask m when bit i & 31 of words[m * pitch + (i >> 5)] is set. A single doc mask is the set of
// one with pitch ceil(nd / 32).
struct DocMasks {
    const uint32_t* words;
    long long pitch;
    const int* of_query;
};

// The mask words of query row `row`.
__device__ __forceinline__ const uint32_t* mask_of_row(const DocMasks& m, long long row) {
    return m.of_query ? m.words + static_cast<long long>(__ldg(m.of_query + row)) * m.pitch : m.words;
}

struct MaskedScoreArgs : ScoreArgs {
    DocMasks masks;
};

struct GroupedScoreArgs : ScoreArgs {
    const int* doc_groups;     // [nd]: the group (document) of each doc (page)
};

struct MaskedGroupedScoreArgs : MaskedScoreArgs {
    const int* doc_groups;
};

// Range search ((Masked)RangeScoreArgs): instead of lists, every doc whose approximate score is >= the row's drop
// threshold t - eps is appended to the row's candidate region (see the epilogue).
struct RangeFields {
    const float* thresholds;    // [nq] t of each query row
    const float* qnorms;        // [nq] fp32 L2 norm of each query row
    const float* max_doc_norm;  // [1] max L2 norm of the doc rows
    int cap;                    // candidate slots per query row
    int* counts;                // [nq] candidates found (zeroed by the host); > cap: the row overflowed
    int* cand;                  // [nq, cap] their doc ids, in no particular order
};

struct RangeScoreArgs : ScoreArgs {
    RangeFields range;
};

struct MaskedRangeScoreArgs : MaskedScoreArgs {
    RangeFields range;
};

template <typename Args>
constexpr bool kMasked = std::is_base_of<MaskedScoreArgs, Args>::value;
template <typename Args>
constexpr bool kGrouped = std::is_same<Args, GroupedScoreArgs>::value || std::is_same<Args, MaskedGroupedScoreArgs>::value;
template <typename Args>
constexpr bool kRange = std::is_same<Args, RangeScoreArgs>::value || std::is_same<Args, MaskedRangeScoreArgs>::value;

// The bound of the filter: |approximate score - exact fp32 score| <= score_eps(|q|, max|d|, dim) for finite fp16 copies of
// both operands. fp16 operand rounding (2^-11 each) + fp32 accumulation slack, times |q| * max|d|, plus an absolute term
// for fp16 subnormals (elements below 6.1e-5 carry an absolute error up to 2^-25). The one statement of eps: the top-k
// proof (proof_flag) and the range filter's drop threshold both call it.
__device__ __forceinline__ float score_eps(float qnorm, float dn, int dim) {
    return (9.765625e-4f + static_cast<float>(dim) * 1.1920929e-7f) * qnorm * dn +
           sqrtf(static_cast<float>(dim)) * 5.9604645e-8f * (qnorm + dn) + 1e-6f;
}

// The range filter's drop threshold of query row `row`: t - eps rounded toward -inf, so that every doc with exact
// score >= t has approximate score >= it. NaN (no comparison passes, nothing is appended) for rows past nq and for rows
// without a bound: a query or max doc norm that is not < 65504 (inf / NaN included) means some fp16 operand may have
// overflowed, and lane `mark` records such a row as overflowed so that the host reruns it through the fp32 scan.
__device__ __forceinline__ float range_drop_threshold(const RangeFields& f, int row, int nq, int dim, bool mark) {
    if (row >= nq) return __int_as_float(0x7fffffff);
    const float qn = __ldg(f.qnorms + row), dn = __ldg(f.max_doc_norm);
    if (!(qn < 65504.f) || !(dn < 65504.f)) {
        if (mark) atomicMax(f.counts + row, f.cap + 1);
        return __int_as_float(0x7fffffff);
    }
    return __fsub_rd(__ldg(f.thresholds + row), score_eps(qn, dn, dim));
}

struct Score2Cfg {
    static constexpr int STAGES = 6;
    static constexpr int SUB_BN = 128;                      // docs per MMA sub-tile (a 256-doc tile is two of them)
    static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;   // this CTA's 128 query rows
    static constexpr int B_BYTES = SUB_BN * GEMM_BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // 32 KB
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

__device__ __forceinline__ void topk_insert(float (&sc)[SC_KT], int (&id)[SC_KT], float v, int i) {
    // precondition: v > sc[SC_KT-1]; lists are sorted descending, ties keep the earlier entry first
    sc[SC_KT - 1] = v;
    id[SC_KT - 1] = i;
#pragma unroll
    for (int j = SC_KT - 1; j > 0; --j) {
        const bool sw = sc[j] > sc[j - 1];
        const float a = sc[j], b = sc[j - 1];
        const int ia = id[j], ib = id[j - 1];
        sc[j - 1] = sw ? a : b;
        sc[j] = sw ? b : a;
        id[j - 1] = sw ? ia : ib;
        id[j] = sw ? ib : ia;
    }
}

// Group-distinct lists: a list holds at most one doc per group. A doc whose group already has an entry replaces it only
// when its score is higher, and is dropped otherwise; a doc of a new group goes in as topk_insert puts it (precondition
// then: v > sc[SC_KT-1]). Every dropped doc is therefore <= the list's final tail or <= its own group's entry. The groups
// of the entries are looked up, not kept in registers: this runs on the rare insertion path only.
__device__ __forceinline__ void group_insert(float (&sc)[SC_KT], int (&id)[SC_KT], float v, int i,
                                             const int* __restrict__ groups) {
    const int gi = __ldg(groups + i);
    bool same = false, up = false;
#pragma unroll
    for (int j = 0; j < SC_KT; ++j) {
        if (id[j] >= 0 && __ldg(groups + id[j]) == gi) {
            same = true;
            if (v > sc[j]) { sc[j] = v; id[j] = i; up = true; }
        }
    }
    if (!same) {
        topk_insert(sc, id, v, i);
    } else if (up) {  // the raised entry moves up to its place (one pass from the bottom carries it)
#pragma unroll
        for (int j = SC_KT - 1; j > 0; --j) {
            const bool sw = sc[j] > sc[j - 1];
            const float a = sc[j], b = sc[j - 1];
            const int ia = id[j], ib = id[j - 1];
            sc[j - 1] = sw ? a : b;
            sc[j] = sw ? b : a;
            id[j - 1] = sw ? ia : ib;
            id[j] = sw ? ib : ia;
        }
    }
}

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// A pair of CTAs (blocks 2p, 2p+1) shares one work item: 256 queries x a range of 256-doc tiles, 128 queries per CTA,
// fp16 operands, fp32 wgmma accumulators in registers. Roles as in gemm.cuh: a TMA producer warpgroup and two consumer
// warpgroups of 64 query rows each; a doc tile is computed as two 128-doc sub-tiles. A query row of the accumulator
// lives in the 4 lanes of a quad (each lane holds a quarter of the columns), so every lane keeps a sorted top-16 of ITS
// columns for each of its two rows over all tiles of the item; the four lists of a row are merged by shuffles at the end
// of the item (top-16 of the union: its tail bounds everything any lane dropped) into one list per (query, doc range).
// MASKED: every query row has its own mask of the set (mask_of_row), one eligibility bit per doc. An ineligible doc's score
// becomes -inf before anything looks at it, so it never enters that row's lists, never raises the row's thr and never
// reaches the row's published tau: every tail of a query, and so the rescoring kernel's bound, is a tail over that query's
// eligible docs only. A thread's two accumulator rows (g8, g8 + 8) are two queries, each with its own mask words.
// The mask travels in its own argument type, so the unmasked form keeps the parameter list it has without the mask (an
// unused parameter or ScoreArgs field changes its register allocation and code).
// GROUPED ((Masked)GroupedScoreArgs): doc_groups gives each doc its group, and every list is group-distinct (group_insert,
// in the slow path and in the quad merge); the fast path is that of the page-level form with the same masking. The quad merge keeps the merged tail >= each lane's tail
// (each lane's 16 groups have an entry at least that high in the union), so thr stays a valid drop threshold, and a
// published tau is the tail of a group-distinct list.
// RANGE ((Masked)RangeScoreArgs): no lists, no quad merge, no tau. Each accumulator row has one fixed drop threshold
// thr = t - eps (range_drop_threshold); the fast path is max >= thr over the lane's 32 scores, and the slow path appends
// every column with score >= thr to the row's candidate region: the quad's four lanes take their slots with ONE atomicAdd
// on the row's counter, and write only while slot < cap (the counter keeps counting, so counts > cap marks an overflow).
// Masked-out columns become NaN, which no comparison passes (-inf would pass a threshold of -inf).
template <typename Args>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
score_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                    const Args g) {
    constexpr bool GROUPED = kGrouped<Args>;
    constexpr bool MASKED = kMasked<Args>;
    constexpr bool RANGE = kRange<Args>;
    using Cfg = Score2Cfg;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int rank = blockIdx.x & 1;
    const int pair = blockIdx.x >> 1;
    const int num_pairs = gridDim.x >> 1;
    const int num_kb = (g.dim + GEMM_BK - 1) / GEMM_BK;
    // item -> (query block b, doc tiles [t0, t1))
    auto item_b = [&](int item) { return item % g.QB; };
    auto item_t0 = [&](int item) { return static_cast<int>(static_cast<long long>(g.T) * (item / g.QB) / g.R); };
    auto item_t1 = [&](int item) { return static_cast<int>(static_cast<long long>(g.T) * (item / g.QB + 1) / g.R); };

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_d);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int item = pair; item < g.items; item += num_pairs) {
                const int m0 = item_b(item) * 2 * GEMM_BM + rank * GEMM_BM;
                const int t1 = item_t1(item);
                for (int u = 2 * item_t0(item); u < 2 * t1; ++u) {  // 128-doc sub-tiles
                    const int n0 = u * Cfg::SUB_BN;
                    for (int kb = 0; kb < num_kb; ++kb) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                        tma_load_2d(&tmap_q, &full_bar[stage], smem_a + stage * Cfg::A_BYTES, kb * GEMM_BK, m0);
                        tma_load_2d(&tmap_d, &full_bar[stage], smem_b + stage * Cfg::B_BYTES, kb * GEMM_BK, n0);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int cw = wg - 1;
    const uint64_t desc_hi = make_smem_desc(0, 16, 1024, kLayoutSW128);
    const uint32_t a_lo0 = (smem_u32(smem_a) + cw * (64 * GEMM_BK * 2)) >> 4, b_lo0 = smem_u32(smem_b) >> 4;
    const int g8 = lane >> 2, q4 = lane & 3;
    float sc[2][SC_KT];  // [accumulator row g8 / g8 + 8]
    int id[2][SC_KT];
    int stage = 0;
    uint32_t phase = 0;
    for (int item = pair; item < g.items; item += num_pairs) {
        const int b = item_b(item), r = item / g.QB;
        const int row0 = b * 2 * GEMM_BM + rank * GEMM_BM + cw * 64 + warp * 16 + g8;
        // tau: a lower bound on what this query can still use, published by the items of this query that already
        // finished (the 16th best score of their doc range). Dropping everything <= tau is covered by the proof: the
        // rescoring kernel's bound is the maximum over all list tails, and tau is one of them.
        float* tau_ptr[2];
        float tau[2], thr[2];  // thr = max(tau, best tail of the quad's four lists: the merged list's tail is no lower)
        const uint32_t* mrow[2];  // MASKED: the mask words of each row's query
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if constexpr (RANGE) {
                thr[h] = range_drop_threshold(g.range, row0 + 8 * h, g.nq, g.dim, q4 == 0);
            } else {
                tau_ptr[h] = g.cand_scores + (static_cast<long long>(min(row0 + 8 * h, g.nq - 1)) * g.lists + g.lists - 1) * SC_KT;
                thr[h] = tau[h] = __ldcg(tau_ptr[h]);
            }
            if constexpr (MASKED) mrow[h] = mask_of_row(g.masks, min(row0 + 8 * h, g.nq - 1));
            if constexpr (!RANGE) {
#pragma unroll
                for (int j = 0; j < SC_KT; ++j) { sc[h][j] = -INFINITY; id[h][j] = -1; }
            }
        }
        const int t1 = item_t1(item);
        for (int u = 2 * item_t0(item); u < 2 * t1; ++u) {
            // each row's 4 mask words of the sub-tile, loaded before the k-loop so the latency hides under the MMAs (words
            // at or past the end of a mask read as 0: those columns are >= nd and skipped below anyway)
            uint32_t mw[2][4];
            if constexpr (MASKED) {
                const long long w0 = static_cast<long long>(u) * (Cfg::SUB_BN / 32), nw = (g.nd + 31) / 32;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 4; ++i) mw[h][i] = w0 + i < nw ? __ldg(mrow[h] + w0 + i) : 0u;
            }
            float acc[Cfg::SUB_BN / 2];
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t ad = desc_hi | static_cast<uint64_t>(a_lo0 + stage * (Cfg::A_BYTES >> 4));
                const uint64_t bd = desc_hi | static_cast<uint64_t>(b_lo0 + stage * (Cfg::B_BYTES >> 4));
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wgmma_ss<true, false>(acc, ad + 2 * kk, bd + 2 * kk, (kb | kk) != 0, std::integral_constant<int, Cfg::SUB_BN>());
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            wgmma_touch(acc);

            const long long col_base = static_cast<long long>(u) * Cfg::SUB_BN + q4 * 2;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                // this lane's 32 scores of the row: v[2j + e] = column 8j + 2 q4 + e of the sub-tile
                uint32_t v[32];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    v[2 * j] = __float_as_uint(acc[4 * j + 2 * h]);
                    v[2 * j + 1] = __float_as_uint(acc[4 * j + 2 * h + 1]);
                }
                if constexpr (MASKED) {
                    // bit 2j + e of elig = eligibility of this lane's column 8j + 2 q4 + e for row h's query: word j >> 2,
                    // bit 8 (j & 3) + 2 q4 + e
                    uint32_t elig = 0;
#pragma unroll
                    for (int w = 0; w < 4; ++w) {
                        const uint32_t x = mw[h][w] >> (2 * q4);
                        elig |= ((x & 0x3u) | ((x >> 6) & 0xCu) | ((x >> 12) & 0x30u) | ((x >> 18) & 0xC0u)) << (8 * w);
                    }
                    if constexpr (RANGE) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = (elig >> j) & 1u ? v[j] : 0x7fffffffu;
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = (elig >> j) & 1u ? v[j] : __float_as_uint(-INFINITY);
                    }
                }
                // fast path: nothing of the 32 scores beats the threshold (the common case after the first tiles)
                float mx = fmaxf(__uint_as_float(v[0]), __uint_as_float(v[1]));
#pragma unroll
                for (int j = 2; j < 32; j += 2) mx = fmaxf(mx, fmaxf(__uint_as_float(v[j]), __uint_as_float(v[j + 1])));
                if constexpr (RANGE) {
                    const bool hit = mx >= thr[h];
                    if (__any_sync(0xffffffffu, hit)) {  // warp-uniform: the quad exchange below needs every lane
                        uint32_t m = 0;
                        if (hit) {
#pragma unroll
                            for (int j = 0; j < 32; ++j)
                                m |= (__uint_as_float(v[j]) >= thr[h] && col_base + (j >> 1) * 8 + (j & 1) < g.nd ? 1u : 0u) << j;
                        }
                        // slots of the quad's lanes: an exclusive prefix of their counts, one atomicAdd for the row
                        const int n = __popc(m);
                        int pre = n;
                        int o = __shfl_up_sync(0xffffffffu, pre, 1, 4);
                        if (q4 >= 1) pre += o;
                        o = __shfl_up_sync(0xffffffffu, pre, 2, 4);
                        if (q4 >= 2) pre += o;
                        const int total = __shfl_sync(0xffffffffu, pre, 3, 4);
                        const int row = row0 + 8 * h;
                        int base = 0;
                        if (q4 == 0 && total > 0) base = atomicAdd(g.range.counts + row, total);
                        int slot = __shfl_sync(0xffffffffu, base, 0, 4) + pre - n;
                        int* dst = g.range.cand + static_cast<long long>(row) * g.range.cap;
#pragma unroll 1
                        while (m) {
                            const int j = __ffs(m) - 1;
                            m &= m - 1;
                            if (slot < g.range.cap) dst[slot] = static_cast<int>(col_base + (j >> 1) * 8 + (j & 1));
                            ++slot;
                        }
                    }
                    continue;
                }
                if (mx > thr[h]) {
                    // slow path, ONE compact instance of the insertion code per row (a fully unrolled form - 32 inlined
                    // insertions - would thrash the instruction cache)
                    uint32_t mask = 0;
#pragma unroll
                    for (int j = 0; j < 32; ++j) mask |= (__uint_as_float(v[j]) > thr[h] ? 1u : 0u) << j;
#pragma unroll 1
                    while (mask) {
                        const int j = __ffs(mask) - 1;
                        mask &= mask - 1;
                        // v[j] with a run-time j: binary select tree over the register array
                        uint32_t s16[16], s8[8], s4[4], s2[2];
#pragma unroll
                        for (int i = 0; i < 16; ++i) s16[i] = (j & 1) ? v[2 * i + 1] : v[2 * i];
#pragma unroll
                        for (int i = 0; i < 8; ++i) s8[i] = (j & 2) ? s16[2 * i + 1] : s16[2 * i];
#pragma unroll
                        for (int i = 0; i < 4; ++i) s4[i] = (j & 4) ? s8[2 * i + 1] : s8[2 * i];
#pragma unroll
                        for (int i = 0; i < 2; ++i) s2[i] = (j & 8) ? s4[2 * i + 1] : s4[2 * i];
                        const float sv = __uint_as_float((j & 16) ? s2[1] : s2[0]);
                        const long long col = col_base + (j >> 1) * 8 + (j & 1);
                        if (sv > thr[h] && col < g.nd) {
                            if constexpr (GROUPED) group_insert(sc[h], id[h], sv, static_cast<int>(col), g.doc_groups);
                            else topk_insert(sc[h], id[h], sv, static_cast<int>(col));
                            thr[h] = fmaxf(thr[h], sc[h][SC_KT - 1]);
                        }
                    }
                }
                thr[h] = fmaxf(thr[h], quad_max(sc[h][SC_KT - 1]));
            }
        }
        if constexpr (RANGE) continue;  // the candidates are already in their regions
        // one candidate list per (query row, doc range): merge the quad's four column subsets (after the two exchange
        // steps every lane of the quad holds the top-16 of the union), write it, publish its tail as the query's new tau
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int step = 1; step <= 2; ++step) {
                float os[SC_KT];
                int oi[SC_KT];
#pragma unroll
                for (int j = 0; j < SC_KT; ++j) {
                    os[j] = __shfl_xor_sync(0xffffffffu, sc[h][j], step);
                    oi[j] = __shfl_xor_sync(0xffffffffu, id[h][j], step);
                }
#pragma unroll 1
                for (int j = 0; j < SC_KT; ++j) {
                    // os[j] with a run-time j (one compact instance of the insertion code)
                    float v2 = os[0];
                    int i2 = oi[0];
#pragma unroll
                    for (int i = 1; i < SC_KT; ++i)
                        if (i == j) { v2 = os[i]; i2 = oi[i]; }
                    if (v2 > sc[h][SC_KT - 1]) {
                        if constexpr (GROUPED) group_insert(sc[h], id[h], v2, i2, g.doc_groups);
                        else topk_insert(sc[h], id[h], v2, i2);
                    }
                }
            }
            const int row = row0 + 8 * h;
            if (q4 == 0 && row < g.nq) {
                const long long base = (static_cast<long long>(row) * g.lists + r) * SC_KT;
#pragma unroll
                for (int j4 = 0; j4 < SC_KT / 4; ++j4) {
                    *reinterpret_cast<float4*>(g.cand_scores + base + j4 * 4) =
                        make_float4(sc[h][j4 * 4], sc[h][j4 * 4 + 1], sc[h][j4 * 4 + 2], sc[h][j4 * 4 + 3]);
                    *reinterpret_cast<int4*>(g.cand_ids + base + j4 * 4) =
                        make_int4(id[h][j4 * 4], id[h][j4 * 4 + 1], id[h][j4 * 4 + 2], id[h][j4 * 4 + 3]);
                }
                const float tail = sc[h][SC_KT - 1];
                if (tail > tau[h]) {  // float max through the integer atomics (tail may be negative)
                    // branch on the sign BIT: -0.0 goes to the unsigned min, where its pattern is the least of all
                    // negative floats (as a signed int it is INT_MIN, which a signed max never stores over -inf or
                    // a negative tau)
                    if (__float_as_int(tail) >= 0) atomicMax(reinterpret_cast<int*>(tau_ptr[h]), __float_as_int(tail));
                    else atomicMin(reinterpret_cast<unsigned int*>(tau_ptr[h]), __float_as_uint(tail));
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// (score, id) ordering: a before b  <=>  a.s > b.s || (a.s == b.s && a.id < b.id)
__device__ __forceinline__ bool before(float sa, long long ia, float sb, long long ib) {
    return sa > sb || (sa == sb && ia < ib);
}

// Warp arg-max in (score, id) order: every lane ends with the warp's best pair.
__device__ __forceinline__ void warp_argmax(float& bs, long long& bi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, bs, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (before(os, oi, bs, bi)) { bs = os; bi = oi; }
    }
}

// Block arg-max over WARPS warps through the per-warp slots red_s / red_i: every thread ends with the block's best pair.
// The second barrier lets the next call reuse the slots.
template <int WARPS>
__device__ __forceinline__ void block_argmax(float& bs, long long& bi, float* red_s, long long* red_i) {
    warp_argmax(bs, bi);
    if ((threadIdx.x & 31) == 0) { red_s[threadIdx.x >> 5] = bs; red_i[threadIdx.x >> 5] = bi; }
    __syncthreads();
    bs = red_s[0]; bi = red_i[0];
    for (int i = 1; i < WARPS; ++i)
        if (before(red_s[i], red_i[i], bs, bi)) { bs = red_s[i]; bi = red_i[i]; }
    __syncthreads();
}

constexpr int RS_THREADS = 128;
constexpr int RS_MAX_KEEP = 256;

// Exact fp32 q . d of one doc row, by one warp (every lane returns it): lane-strided float4 FMAs, then warp_sum_f. This
// is the order of exact_scores_kernel, so the rescored scores have the bits of vr_score_exact.
__device__ __forceinline__ float warp_dot_row(const float* qs, const float* __restrict__ d, int dim, int lane) {
    const float4* drow = reinterpret_cast<const float4*>(d);
    const float4* q4 = reinterpret_cast<const float4*>(qs);
    float a = 0.f;
    for (int i = lane; i < (dim >> 2); i += 32) {
        const float4 x = drow[i], y = q4[i];
        a = fmaf(x.x, y.x, a);
        a = fmaf(x.y, y.y, a);
        a = fmaf(x.z, y.z, a);
        a = fmaf(x.w, y.w, a);
    }
    return warp_sum_f(a);
}

// The proof of the rescoring kernels: 1 (rerun the query through the fp32 scan) unless bound + eps < kth, where bound
// covers every candidate that was not rescored exactly (-inf: none) and kth is the k-th exact score.
__device__ __forceinline__ int proof_flag(float bound, float kth, float qnorm, float dn, int dim) {
    const float eps = score_eps(qnorm, dn, dim);
    int flag = 0;
    if (bound > -INFINITY && !(bound + eps < kth)) flag = 1;  // something was dropped that might belong
    // the bound assumes finite fp16 copies of both operands: a row norm >= 65504 (or inf / NaN, for which the
    // comparison is false as well) means some |x| may have overflowed fp16 -> rerun this query through the fp32 scan
    if (!(qnorm < 65504.f) || !(dn < 65504.f)) flag = 1;
    return flag;
}

// Step 1 of the rescoring kernels (warp 0, every lane returns the bound): a multi-way merge of the list heads sends the
// `keep` best candidates by approximate score to sel[] (-1 pads when the lists run out) and, with SCORES, their scores to
// sel_s[]; the return value bounds everything else: the list tails and the best pruned head.
template <bool SCORES>
__device__ __forceinline__ float merge_list_heads(const float* __restrict__ cs, const int* __restrict__ ci, int lists,
                                                  int keep, int lane, int* sel, float* sel_s) {
    // lane l owns lists l, l+32, ...: head position per owned list (<= 2 lists per lane for lists <= 64; general loop)
    float tail = -INFINITY;
    for (int l = lane; l < lists; l += 32) tail = fmaxf(tail, cs[l * SC_KT + SC_KT - 1]);
    int head[(SC_MAX_RANGES + 31) / 32 + 1];
#pragma unroll
    for (int j = 0; j < (SC_MAX_RANGES + 31) / 32 + 1; ++j) head[j] = 0;
    for (int m = 0; m < keep; ++m) {
        // best head of this lane
        float bs = -INFINITY;
        int bj = -1;
#pragma unroll
        for (int j = 0; j < (SC_MAX_RANGES + 31) / 32 + 1; ++j) {
            const int l = lane + j * 32;
            if (l < lists && head[j] < SC_KT) {
                const float v = cs[l * SC_KT + head[j]];
                if (ci[l * SC_KT + head[j]] >= 0 && (bj < 0 || v > bs)) { bs = v; bj = j; }
            }
        }
        // warp arg-max (ties: lower lane)
        float ws = bs;
        int wl = bj >= 0 ? lane : 64;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float os = __shfl_xor_sync(0xffffffffu, ws, o);
            const int ol = __shfl_xor_sync(0xffffffffu, wl, o);
            if (ol < 64 && (wl >= 64 || os > ws || (os == ws && ol < wl))) { ws = os; wl = ol; }
        }
        if (wl >= 64) {  // every list exhausted
            for (int r = m + lane; r < keep; r += 32) sel[r] = -1;
            break;
        }
        if (lane == wl) {
#pragma unroll
            for (int j = 0; j < (SC_MAX_RANGES + 31) / 32 + 1; ++j)
                if (j == bj) {
                    sel[m] = ci[(lane + j * 32) * SC_KT + head[j]];
                    if constexpr (SCORES) sel_s[m] = ws;
                    ++head[j];
                }
        }
    }
    // what is left in the lists was pruned: bounded by the best remaining head
    float rem = -INFINITY;
#pragma unroll
    for (int j = 0; j < (SC_MAX_RANGES + 31) / 32 + 1; ++j) {
        const int l = lane + j * 32;
        if (l < lists && head[j] < SC_KT && ci[l * SC_KT + head[j]] >= 0) rem = fmaxf(rem, cs[l * SC_KT + head[j]]);
    }
    float bnd = fmaxf(tail, rem);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) bnd = fmaxf(bnd, __shfl_xor_sync(0xffffffffu, bnd, o));
    return bnd;
}

// One CTA per query. The filter hands over `lists` sorted 16-entry candidate lists (approximate scores). Step 1 (warp 0):
// multi-way merge of the list heads keeps the `keep` best candidates by approximate score; everything else - docs a list
// dropped (<= that list's 16th entry) and candidates pruned here (<= the best remaining head) - is bounded by `bound`.
// Step 2: exact fp32 rescoring of the kept candidates, one warp per candidate. Step 3: top-k by (score desc, id asc)
// and the proof  bound + eps < k-th exact score  (else the query is flagged for the fp32 scan).
// It takes no mask, with a mask set or without: a masked filter's lists of query q hold q's eligible docs only, and every
// tail of them is a tail over q's eligible docs, so the candidates, the bound and the proof are already q's own.
__global__ void __launch_bounds__(RS_THREADS)
rescore_topk_kernel(const float* __restrict__ Q, const float* __restrict__ D, long long nd, int dim, int lists, int keep,
                    const float* __restrict__ cand_scores, const int* __restrict__ cand_ids,
                    const float* __restrict__ max_doc_norm, int k, long long id_offset, float* __restrict__ out_scores,
                    long long* __restrict__ out_ids, int* __restrict__ flags) {
    extern __shared__ float sm[];
    float* qs = sm;                                   // [dim]
    float* ex = sm + dim;                             // [keep] exact scores
    int* sel = reinterpret_cast<int*>(ex + keep);     // [keep] doc ids of the kept candidates (-1 = none)
    __shared__ float red_s[RS_THREADS / 32];
    __shared__ long long red_i[RS_THREADS / 32];
    __shared__ float sh_bound, sh_qnorm;
    const int q = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* qrow = Q + static_cast<long long>(q) * dim;
    const float* cs = cand_scores + static_cast<long long>(q) * lists * SC_KT;
    const int* ci = cand_ids + static_cast<long long>(q) * lists * SC_KT;
    if (warp == 0) {
        const float bnd = merge_list_heads<false>(cs, ci, lists, keep, lane, sel, nullptr);
        if (lane == 0) sh_bound = bnd;
    }
    float qq = 0.f;
    for (int i = threadIdx.x; i < dim; i += RS_THREADS) {
        const float v = qrow[i];
        qs[i] = v;
        qq += v * v;
    }
    qq = warp_sum_f(qq);
    if (lane == 0) red_s[warp] = qq;
    __syncthreads();  // qs, sel, sh_bound, red_s visible
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < RS_THREADS / 32; ++i) s += red_s[i];
        sh_qnorm = sqrtf(s);
    }
    // exact fp32 rescoring: one warp per kept candidate
    for (int c = warp; c < keep; c += RS_THREADS / 32) {
        const int id = sel[c];
        const float s = id >= 0 ? warp_dot_row(qs, D + static_cast<long long>(id) * dim, dim, lane) : -INFINITY;
        if (lane == 0) ex[c] = s;
    }
    __syncthreads();  // ex[] complete, red_s reusable
    // k rounds of block arg-max in (score desc, id asc) order, strictly after the previous winner
    float last_s = INFINITY;
    long long last_i = -1;
    float kth = -INFINITY;
    for (int round = 0; round < k; ++round) {
        float bs = -INFINITY;
        long long bi = 0x7fffffffffffffffll;
        for (int c = threadIdx.x; c < keep; c += RS_THREADS) {
            const int id = sel[c];
            if (id < 0) continue;
            const float s = ex[c];
            if (!before(last_s, last_i, s, id)) continue;  // already emitted (or equal to the previous winner)
            if (before(s, id, bs, bi)) { bs = s; bi = id; }
        }
        block_argmax<RS_THREADS / 32>(bs, bi, red_s, red_i);
        const bool valid = bi != 0x7fffffffffffffffll;
        if (threadIdx.x == 0) {
            out_scores[static_cast<long long>(q) * k + round] = valid ? bs : -INFINITY;
            out_ids[static_cast<long long>(q) * k + round] = valid ? bi + id_offset : -1;
        }
        if (!valid) {
            for (int r2 = round + 1 + threadIdx.x; r2 < k; r2 += RS_THREADS) {
                out_scores[static_cast<long long>(q) * k + r2] = -INFINITY;
                out_ids[static_cast<long long>(q) * k + r2] = -1;
            }
            kth = -INFINITY;
            break;
        }
        last_s = bs; last_i = bi; kth = bs;
    }
    if (threadIdx.x == 0) flags[q] = proof_flag(sh_bound, kth, sh_qnorm, *max_doc_norm, dim);
}

// ---------------------------------------------------------------------------------------------
// Document-level (grouped) rescoring. doc_groups [nd] gives every doc (page) its group (document); the CSR group_offsets
// [G+1] / group_pages lists each group's pages, ascending. The score of a group is the maximum exact score over its
// eligible pages, its best page the lowest of those with that maximum; groups rank by (score desc, best page asc).
// Candidate lists may come from either filter: group-distinct lists (every dropped page <= the list's tail or <= its own
// group's entry in that list) or page lists (every dropped page <= the tail, which satisfies the same invariant).
constexpr int RG_PAGE_BUDGET = 4096;  // pages one query may fully rescore (36 KB of fp32 rows each at dim 2304)

// One CTA per query. Step 1: the list-head merge and bound of rescore_topk_kernel. Step 2: the distinct groups of the kept
// candidates, in approximate order; as long as their pages fit RG_PAGE_BUDGET, each is FULLY rescored (every eligible
// page, exact fp32, the FMA order and warp reduction of the page kernels, so the same bits); the first group that does
// not fit ends the walk, and it and every later kept group enter the bound with their best approximate entry. Step 3:
// top-k of the rescored groups and the proof  B + eps < k-th group score, B = max(list tails, pruned heads, approximate
// entries of kept groups not rescored). A group that was not rescored has every page p either dropped by a list
// (approx(p) <= that list's tail, or <= its group's entry there, which was kept - so in B - or pruned - so <= a pruned
// head) or pruned or kept (in B): exact(p) <= B + eps < k-th. Otherwise the query is flagged.
__global__ void __launch_bounds__(RS_THREADS, 1)  // without the 1, ptxas caps it at 32 registers and spills
rescore_groups_kernel(const float* __restrict__ Q, const float* __restrict__ D, int dim, int lists, int keep,
                      const float* __restrict__ cand_scores, const int* __restrict__ cand_ids,
                      const int* __restrict__ doc_groups, const int* __restrict__ group_offsets,
                      const int* __restrict__ group_pages, const DocMasks masks,
                      const float* __restrict__ max_doc_norm, int k, long long id_offset, float* __restrict__ out_scores,
                      long long* __restrict__ out_pages, long long* __restrict__ out_groups, int* __restrict__ flags) {
    extern __shared__ float sm[];
    float* qs = sm;                                      // [dim]
    float* ex = qs + dim;                                // [RG_PAGE_BUDGET] exact scores of the rescored pages
    int* pg = reinterpret_cast<int*>(ex + RG_PAGE_BUDGET);  // [RG_PAGE_BUDGET] their pages (-1: ineligible)
    float* sel_s = reinterpret_cast<float*>(pg + RG_PAGE_BUDGET);  // [keep] approximate scores of the kept candidates
    int* sel = reinterpret_cast<int*>(sel_s + keep);     // [keep] their pages
    int* first = sel + keep;                             // [keep] group of the candidate if it is its group's first, else -1
    int* gstart = first + keep;                          // [keep + 1] rescored group s owns pg[gstart[s], gstart[s+1])
    int* gid = gstart + keep + 1;                        // [keep] its group
    float* gs = reinterpret_cast<float*>(gid + keep);    // [keep] its score
    int* gp = reinterpret_cast<int*>(gs + keep);         // [keep] its best page (-1: no eligible page)
    __shared__ float red_s[RS_THREADS / 32];
    __shared__ long long red_i[RS_THREADS / 32];
    __shared__ float sh_bound, sh_qnorm;
    __shared__ int sh_ng;
    const int q = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* qrow = Q + static_cast<long long>(q) * dim;
    const uint32_t* doc_mask = masks.words ? mask_of_row(masks, q) : nullptr;  // this query's mask (NULL: every page)
    if (warp == 0) {
        const float bnd = merge_list_heads<true>(cand_scores + static_cast<long long>(q) * lists * SC_KT,
                                           cand_ids + static_cast<long long>(q) * lists * SC_KT, lists, keep, lane, sel, sel_s);
        if (lane == 0) sh_bound = bnd;
    }
    float qq = 0.f;
    for (int i = threadIdx.x; i < dim; i += RS_THREADS) {
        const float v = qrow[i];
        qs[i] = v;
        qq += v * v;
    }
    qq = warp_sum_f(qq);
    if (lane == 0) red_s[warp] = qq;
    __syncthreads();  // qs, sel, sel_s, sh_bound, red_s visible
    for (int c = threadIdx.x; c < keep; c += RS_THREADS) {
        const int p = sel[c];
        int g = p >= 0 ? __ldg(doc_groups + p) : -1;
        for (int j = 0; j < c && g >= 0; ++j)
            if (sel[j] >= 0 && __ldg(doc_groups + sel[j]) == g) g = -1;
        first[c] = g;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < RS_THREADS / 32; ++i) s += red_s[i];
        sh_qnorm = sqrtf(s);
        float bnd = sh_bound;
        int ng = 0, total = 0;
        bool full = false;
        for (int c = 0; c < keep; ++c) {
            const int g = first[c];
            if (g < 0) continue;
            const int n = __ldg(group_offsets + g + 1) - __ldg(group_offsets + g);
            if (!full && n <= RG_PAGE_BUDGET - total) {
                gid[ng] = g;
                gstart[ng++] = total;
                total += n;
            } else {
                full = true;
                bnd = fmaxf(bnd, sel_s[c]);  // the group's best kept entry (candidates are in approximate order)
            }
        }
        gstart[ng] = total;
        sh_ng = ng;
        sh_bound = bnd;
    }
    __syncthreads();
    const int ng = sh_ng, total = gstart[ng];
    for (int s = 0; s < ng; ++s) {
        const int* src = group_pages + __ldg(group_offsets + gid[s]);
        const int n = gstart[s + 1] - gstart[s];
        for (int i = threadIdx.x; i < n; i += RS_THREADS) {
            const int p = __ldg(src + i);
            pg[gstart[s] + i] = doc_mask && !((__ldg(doc_mask + (p >> 5)) >> (p & 31)) & 1u) ? -1 : p;
        }
    }
    __syncthreads();
    // exact fp32 rescoring of every eligible page of the rescored groups: one warp per page
    for (int t = warp; t < total; t += RS_THREADS / 32) {
        const int id = pg[t];
        const float s = id >= 0 ? warp_dot_row(qs, D + static_cast<long long>(id) * dim, dim, lane) : -INFINITY;
        if (lane == 0) ex[t] = s;
    }
    __syncthreads();
    // each group: max over its eligible pages (NaN never selected), lowest page on ties (pages ascend)
    for (int s = threadIdx.x; s < ng; s += RS_THREADS) {
        float best = -INFINITY;
        int bp = -1;
        for (int t = gstart[s]; t < gstart[s + 1]; ++t) {
            const float v = ex[t];
            if (pg[t] >= 0 && !isnan(v) && (bp < 0 || v > best)) { best = v; bp = pg[t]; }
        }
        gs[s] = best;
        gp[s] = bp;
    }
    __syncthreads();
    // k rounds of block arg-max over the rescored groups in (score desc, best page asc) order
    float last_s = INFINITY;
    long long last_i = -1;
    float kth = -INFINITY;
    for (int round = 0; round < k; ++round) {
        float bs = -INFINITY;
        long long bi = 0x7fffffffffffffffll;
        for (int c = threadIdx.x; c < ng; c += RS_THREADS) {
            const int id = gp[c];
            if (id < 0) continue;
            const float s = gs[c];
            if (!before(last_s, last_i, s, id)) continue;
            if (before(s, id, bs, bi)) { bs = s; bi = id; }
        }
        block_argmax<RS_THREADS / 32>(bs, bi, red_s, red_i);
        const bool valid = bi != 0x7fffffffffffffffll;
        const long long o = static_cast<long long>(q) * k;
        if (threadIdx.x == 0) {
            out_scores[o + round] = valid ? bs : -INFINITY;
            out_pages[o + round] = valid ? bi + id_offset : -1;
            out_groups[o + round] = valid ? __ldg(doc_groups + bi) : -1;
        }
        if (!valid) {
            for (int r2 = round + 1 + threadIdx.x; r2 < k; r2 += RS_THREADS) {
                out_scores[o + r2] = -INFINITY;
                out_pages[o + r2] = -1;
                out_groups[o + r2] = -1;
            }
            kth = -INFINITY;
            break;
        }
        last_s = bs; last_i = bi; kth = bs;
    }
    if (threadIdx.x == 0) flags[q] = proof_flag(sh_bound, kth, sh_qnorm, *max_doc_norm, dim);
}

// ---------------------------------------------------------------------------------------------
// Plain fp32 scan: scores[q, doc] = Q[q] . D[doc].  Block = 8 warps; each warp owns docs, up to 8 queries per pass.
// ---------------------------------------------------------------------------------------------
constexpr int EX_QB = 8;   // queries per pass (their rows sit in shared memory)
constexpr int EX_DW = 4;   // docs per warp per pass: each query float4 read from shared memory feeds 4 doc rows

template <int NQ>  // queries per pass this instantiation is compiled for (1, 2, 4 or EX_QB): fewer accumulators, deeper unroll
__global__ void __launch_bounds__(256)
exact_scores_kernel(const float* __restrict__ Q, int nq, const float* __restrict__ D, long long nd, int dim,
                    float* __restrict__ scores) {
    extern __shared__ float qsm[];  // [NQ, dim]
    const int q0 = blockIdx.y * NQ;
    const int nqb = min(NQ, nq - q0);
    for (int i = threadIdx.x; i < nqb * dim; i += blockDim.x) qsm[i] = Q[static_cast<long long>(q0) * dim + i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nv = dim >> 2;
    const long long groups = (nd + EX_DW - 1) / EX_DW;
    for (long long gi = static_cast<long long>(blockIdx.x) * 8 + warp; gi < groups; gi += static_cast<long long>(gridDim.x) * 8) {
        const long long doc0 = gi * EX_DW;
        const float4* drow[EX_DW];
#pragma unroll
        for (int d = 0; d < EX_DW; ++d) drow[d] = reinterpret_cast<const float4*>(D + min(doc0 + d, nd - 1) * dim);
        float acc[EX_DW][NQ];
#pragma unroll
        for (int d = 0; d < EX_DW; ++d)
#pragma unroll
            for (int j = 0; j < NQ; ++j) acc[d][j] = 0.f;
#pragma unroll(NQ <= 2 ? 3 : 1)
        for (int i = lane; i < nv; i += 32) {
            float4 x[EX_DW];
#pragma unroll
            for (int d = 0; d < EX_DW; ++d) x[d] = __ldcs(drow[d] + i);  // streamed once: do not keep in L1
#pragma unroll
            for (int j = 0; j < NQ; ++j) {
                if (j < nqb) {
                    const float4 y = reinterpret_cast<const float4*>(qsm + j * dim)[i];
#pragma unroll
                    for (int d = 0; d < EX_DW; ++d) {
                        acc[d][j] = fmaf(x[d].x, y.x, acc[d][j]);
                        acc[d][j] = fmaf(x[d].y, y.y, acc[d][j]);
                        acc[d][j] = fmaf(x[d].z, y.z, acc[d][j]);
                        acc[d][j] = fmaf(x[d].w, y.w, acc[d][j]);
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < NQ; ++j) {
            if (j < nqb) {
#pragma unroll
                for (int d = 0; d < EX_DW; ++d) {
                    const float s = warp_sum_f(acc[d][j]);
                    if (lane == d && doc0 + d < nd) scores[static_cast<long long>(q0 + j) * nd + doc0 + d] = s;
                }
            }
        }
    }
}

// Column c is eligible when bit c & 31 of mask word c >> 5 is set (the layout of one mask of a DocMasks set).
__device__ __forceinline__ bool col_eligible(const uint32_t* __restrict__ mask, long long c) {
    return (__ldg(mask + (c >> 5)) >> (c & 31)) & 1u;
}

// top-k of each row of a dense [rows, cols] fp32 matrix (optionally with explicit ids per entry).
// MASKED (ids == NULL only): row r's ineligible columns (by the mask of row r's query) are skipped like negative ids -
// never represented by a -inf score, which would count as a valid entry.
// The body of topk_rows_kernel, also the rerun of select_rows_kernel for rows that repeat a (score, id) pair.
template <bool MASKED>
__device__ __forceinline__ void topk_rows_block(const float* __restrict__ scores, const long long* __restrict__ ids,
                                                long long cols, int k, long long id_offset, long long chunk_cols,
                                                float* __restrict__ out_scores, long long* __restrict__ out_ids,
                                                const DocMasks& masks) {
    // block (row, chunk): top-k of columns [chunk*chunk_cols, ...) of one row, written as list `row*gridDim.y + chunk`
    __shared__ float red_s[8];
    __shared__ long long red_i[8];
    const long long c_lo = static_cast<long long>(blockIdx.y) * chunk_cols;
    const long long c_hi = min(cols, c_lo + chunk_cols);
    const float* srow = scores + static_cast<long long>(blockIdx.x) * cols;
    const long long* irow = ids ? ids + static_cast<long long>(blockIdx.x) * cols : nullptr;
    const long long row = static_cast<long long>(blockIdx.x) * gridDim.y + blockIdx.y;  // output list
    const uint32_t* mask = MASKED ? mask_of_row(masks, blockIdx.x) : nullptr;
    float last_s = INFINITY;
    long long last_i = -1;
    for (int round = 0; round < k; ++round) {
        float bs = -INFINITY;
        long long bi = 0x7fffffffffffffffll;
        for (long long c = c_lo + threadIdx.x; c < c_hi; c += 256) {
            const long long id = irow ? irow[c] : c;
            if (id < 0) continue;
            if (MASKED && !col_eligible(mask, c)) continue;
            const float s = srow[c];
            if (!before(last_s, last_i, s, id)) continue;
            if (before(s, id, bs, bi)) { bs = s; bi = id; }
        }
        block_argmax<8>(bs, bi, red_s, red_i);
        const bool valid = bi != 0x7fffffffffffffffll;
        if (threadIdx.x == 0) {
            out_scores[row * k + round] = valid ? bs : -INFINITY;
            out_ids[row * k + round] = valid ? bi + id_offset : -1;
        }
        if (!valid) {
            for (int r2 = round + 1 + threadIdx.x; r2 < k; r2 += 256) {
                out_scores[row * k + r2] = -INFINITY;
                out_ids[row * k + r2] = -1;
            }
            break;
        }
        last_s = bs; last_i = bi;
    }
}

template <bool MASKED>
__global__ void __launch_bounds__(256)
topk_rows_kernel(const float* __restrict__ scores, const long long* __restrict__ ids, long long cols, int k,
                 long long id_offset, long long chunk_cols, float* __restrict__ out_scores,
                 long long* __restrict__ out_ids, const DocMasks masks) {
    topk_rows_block<MASKED>(scores, ids, cols, k, id_offset, chunk_cols, out_scores, out_ids, masks);
}

// Short rows (cols <= 32*NPL): one WARP per row, the row lives in registers, k rounds of shuffle arg-max - no block barriers.
// This is the merge of per-rank / per-shard partial top-k lists ([nq, world*k]) and the second pass of the chunked top-k.
template <int NPL, bool MASKED>
__global__ void __launch_bounds__(256)
topk_rows_warp_kernel(const float* __restrict__ scores, const long long* __restrict__ ids, int rows, int cols, int k,
                      long long id_offset, float* __restrict__ out_scores, long long* __restrict__ out_ids,
                      const DocMasks masks) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const uint32_t* mask = MASKED ? mask_of_row(masks, row) : nullptr;
    const float* srow = scores + static_cast<long long>(row) * cols;
    const long long* irow = ids ? ids + static_cast<long long>(row) * cols : nullptr;
    float s[NPL];
    long long id[NPL];
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
        const int c = lane + j * 32;
        const bool in = c < cols && (!MASKED || col_eligible(mask, c));
        id[j] = in ? (irow ? irow[c] : static_cast<long long>(c)) : -1;
        s[j] = (in && id[j] >= 0) ? srow[c] : -INFINITY;
    }
    float last_s = INFINITY;
    long long last_i = -1;
    for (int round = 0; round < k; ++round) {
        float bs = -INFINITY;
        long long bi = 0x7fffffffffffffffll;
#pragma unroll
        for (int j = 0; j < NPL; ++j) {
            if (id[j] < 0) continue;
            if (!before(last_s, last_i, s[j], id[j])) continue;
            if (before(s[j], id[j], bs, bi)) { bs = s[j]; bi = id[j]; }
        }
        warp_argmax(bs, bi);
        const bool valid = bi != 0x7fffffffffffffffll;
        if (lane == 0) {
            out_scores[static_cast<long long>(row) * k + round] = valid ? bs : -INFINITY;
            out_ids[static_cast<long long>(row) * k + round] = valid ? bi + id_offset : -1;
        }
        if (!valid) {
            for (int r2 = round + 1 + lane; r2 < k; r2 += 32) {
                out_scores[static_cast<long long>(row) * k + r2] = -INFINITY;
                out_ids[static_cast<long long>(row) * k + r2] = -1;
            }
            break;
        }
        last_s = bs; last_i = bi;
    }
}

template <bool MASKED>
static int launch_topk_rows(const float* scores, const long long* ids, int rows, long long cols, int k, long long id_offset,
                            float* out_scores, long long* out_ids, const DocMasks& mask, cudaStream_t s) {
    if (cols <= 128)
        topk_rows_warp_kernel<4, MASKED><<<(rows + 7) / 8, 256, 0, s>>>(scores, ids, rows, static_cast<int>(cols), k, id_offset,
                                                                        out_scores, out_ids, mask);
    else if (cols <= 512)
        topk_rows_warp_kernel<16, MASKED><<<(rows + 7) / 8, 256, 0, s>>>(scores, ids, rows, static_cast<int>(cols), k, id_offset,
                                                                         out_scores, out_ids, mask);
    else
        topk_rows_kernel<MASKED><<<rows, 256, 0, s>>>(scores, ids, cols, k, id_offset, cols, out_scores, out_ids, mask);
    return 0;
}

// Exact grouped path, after vr_score_exact: every (row, group) of scores [rows, nd] reduces to its maximum over the
// group's eligible pages (NaN never selected) and the lowest page with it, as one 64-bit key per (row, group):
// the score's order-preserving bits above ~page, so the largest key is (highest score, lowest page) and atomicMax gives
// the same answer in any order. -0 counts as +0 (they are equal scores: the lower page wins). Each thread takes a run of
// GK_RUN consecutive pages of one row and issues one atomic per group run, so any group size - one group of every page
// included - spreads over the whole grid.
constexpr int GK_RUN = 8;

__device__ __forceinline__ unsigned long long page_key(float v, int p) {
    uint32_t b = __float_as_uint(v);
    if (b == 0x80000000u) b = 0u;
    const uint32_t o = (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // > 0 for every non-NaN score: key 0 = no page
    return (static_cast<unsigned long long>(o) << 32) | static_cast<uint32_t>(~p);
}

__global__ void __launch_bounds__(256)
group_key_kernel(const float* __restrict__ scores, int rows, long long nd, int G, const int* __restrict__ doc_groups,
                 const DocMasks masks, unsigned long long* __restrict__ keys) {
    const long long runs = (nd + GK_RUN - 1) / GK_RUN, n = static_cast<long long>(rows) * runs;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long row = i / runs, p0 = (i - row * runs) * GK_RUN;
        const float* srow = scores + row * nd;
        unsigned long long* krow = keys + row * G;
        const uint32_t* mask = masks.words ? mask_of_row(masks, row) : nullptr;  // the row's mask (NULL: every page)
        int cur = -1;
        unsigned long long best = 0;
#pragma unroll
        for (int j = 0; j < GK_RUN; ++j) {
            const long long p = p0 + j;
            if (p >= nd || (mask && !col_eligible(mask, p))) continue;
            const float v = srow[p];
            if (isnan(v)) continue;
            const int g = __ldg(doc_groups + p);
            if (g != cur) {
                if (best) atomicMax(krow + cur, best);
                cur = g;
                best = 0;
            }
            const unsigned long long key = page_key(v, static_cast<int>(p));
            best = key > best ? key : best;
        }
        if (best) atomicMax(krow + cur, best);
    }
}

// keys [rows, G] -> best pages (in place; -1: no eligible page) and their scores, read back from the score rows so they
// keep their bits (a -0 stays -0)
__global__ void __launch_bounds__(256)
group_decode_kernel(const float* __restrict__ scores, int rows, long long nd, int G, long long* __restrict__ pages,
                    float* __restrict__ gscores) {
    const long long n = static_cast<long long>(rows) * G;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const unsigned long long key = static_cast<unsigned long long>(pages[i]);
        const int p = key ? static_cast<int>(~static_cast<uint32_t>(key)) : -1;
        gscores[i] = p >= 0 ? scores[(i / G) * nd + p] : -INFINITY;
        pages[i] = p;
    }
}

// The group of each emitted page (page ids carry id_offset; -1 stays -1).
__global__ void page_groups_kernel(const long long* __restrict__ pages, long long n, long long id_offset,
                                   const int* __restrict__ doc_groups, long long* __restrict__ groups) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x)
        groups[i] = pages[i] >= 0 ? __ldg(doc_groups + (pages[i] - id_offset)) : -1;
}

// ---------------------------------------------------------------------------------------------
// Candidate lists (vr_doc_lists on the device): query row r scores the docs ids[offsets[m], offsets[m+1]) of list
// m = of_query[r] (of_query NULL: list 0 for every row).
struct DocLists {
    const long long* offsets;
    const int* ids;
    int count;
    const int* of_query;
};

// Status bits of list_scores_kernel (OR-ed into the caller's word)
constexpr int LS_TRUNCATED = 1;   // a list is longer than `width`: only its first `width` entries were scored
constexpr int LS_BAD_LIST = 2;    // an of_query value outside [0, count): the row was given an empty list

// Exact fp32 scores of the listed docs only, into a padded block [nq, width]: position j of row r holds
// (q_r . D[L(r)[j]], L(r)[j]) for j < |L(r)| and (-inf, -1) after it, and with doc_groups the group of the entry (-1 for
// padding) in out_groups. Ids outside [0, nd) are skipped: they give (-inf, -1) and are never read. Block (x, y) takes
// the NQ query rows [x NQ, x NQ + NQ) and list positions [y chunk, (y + 1) chunk). Consecutive rows with the same list
// (a run: the caller sorts rows by list) are scored together: a warp reads EX_DW listed rows once and applies them to
// every query of the run from shared memory, as exact_scores_kernel does for the whole index; a row that is alone in
// its list streams its own rows. A lane's FMA chain and the warp reduction are those of exact_scores_kernel and
// warp_dot_row (float4s lane, lane + 32, ..., x y z w in turn, then warp_sum_f), so every score has the bits
// vr_score_exact gives the same (query, doc) pair.
template <int NQ>
__global__ void __launch_bounds__(256)
list_scores_kernel(const float* __restrict__ Q, int nq, const float* __restrict__ D, long long nd, int dim,
                   const DocLists lists, int width, int chunk, const int* __restrict__ doc_groups,
                   float* __restrict__ out_scores, long long* __restrict__ out_ids, long long* __restrict__ out_groups,
                   int* __restrict__ status) {
    extern __shared__ float qsm[];  // [NQ, dim]: the query rows of the current run
    __shared__ int row_list[NQ];
    const int q0 = blockIdx.x * NQ;
    const int nqb = min(NQ, nq - q0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nv = dim >> 2;
    const int p_lo = blockIdx.y * chunk, p_hi = min(width, p_lo + chunk);
    if (threadIdx.x < nqb) {
        int m = lists.of_query ? __ldg(lists.of_query + q0 + threadIdx.x) : 0;
        if (m < 0 || m >= lists.count) {
            atomicOr(status, LS_BAD_LIST);
            m = -1;
        }
        row_list[threadIdx.x] = m;
    }
    __syncthreads();
    for (int a = 0; a < nqb;) {  // runs [a, b) of rows with one list (block-uniform)
        const int m = row_list[a];
        int b = a + 1;
        while (b < nqb && row_list[b] == m) ++b;
        const int nr = b - a;
        long long off = 0, len = 0;
        if (m >= 0) {
            off = __ldg(lists.offsets + m);
            len = __ldg(lists.offsets + m + 1) - off;
        }
        if (len > width && blockIdx.y == 0 && threadIdx.x == 0) atomicOr(status, LS_TRUNCATED);
        const int n = static_cast<int>(max(0ll, min(len, static_cast<long long>(width))));
        if (p_lo < n)
            for (int i = threadIdx.x; i < nr * dim; i += blockDim.x) qsm[i] = Q[static_cast<long long>(q0 + a) * dim + i];
        __syncthreads();
        for (int pos0 = p_lo + warp * EX_DW; pos0 < p_hi; pos0 += 8 * EX_DW) {
            if (pos0 >= n) {  // past the list: padding only
                for (int t = lane; t < nr * EX_DW; t += 32) {
                    const int pos = pos0 + t % EX_DW;
                    if (pos < p_hi) {
                        const long long o = static_cast<long long>(q0 + a + t / EX_DW) * width + pos;
                        out_scores[o] = -INFINITY;
                        out_ids[o] = -1;
                        if (out_groups) out_groups[o] = -1;
                    }
                }
                continue;
            }
            int id[EX_DW];
            const float4* drow[EX_DW];
#pragma unroll
            for (int d = 0; d < EX_DW; ++d) {
                const int v = pos0 + d < n ? __ldg(lists.ids + off + pos0 + d) : -1;
                id[d] = v >= 0 && v < nd ? v : -1;
                drow[d] = reinterpret_cast<const float4*>(D + static_cast<long long>(id[d] >= 0 ? id[d] : 0) * dim);
            }
            float acc[EX_DW][NQ];
#pragma unroll
            for (int d = 0; d < EX_DW; ++d)
#pragma unroll
                for (int j = 0; j < NQ; ++j) acc[d][j] = 0.f;
#pragma unroll(NQ <= 2 ? 3 : 1)
            for (int i = lane; i < nv; i += 32) {
                float4 x[EX_DW];
#pragma unroll
                for (int d = 0; d < EX_DW; ++d) x[d] = __ldg(drow[d] + i);  // other query tiles may read the row next
#pragma unroll
                for (int j = 0; j < NQ; ++j) {
                    if (j < nr) {
                        const float4 y = reinterpret_cast<const float4*>(qsm + j * dim)[i];
#pragma unroll
                        for (int d = 0; d < EX_DW; ++d) {
                            acc[d][j] = fmaf(x[d].x, y.x, acc[d][j]);
                            acc[d][j] = fmaf(x[d].y, y.y, acc[d][j]);
                            acc[d][j] = fmaf(x[d].z, y.z, acc[d][j]);
                            acc[d][j] = fmaf(x[d].w, y.w, acc[d][j]);
                        }
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < NQ; ++j) {
                if (j < nr) {
#pragma unroll
                    for (int d = 0; d < EX_DW; ++d) {
                        const float s = warp_sum_f(acc[d][j]);
                        if (lane == d && pos0 + d < p_hi) {
                            const long long o = static_cast<long long>(q0 + a + j) * width + pos0 + d;
                            out_scores[o] = id[d] >= 0 ? s : -INFINITY;
                            out_ids[o] = id[d];
                            if (out_groups) out_groups[o] = id[d] >= 0 ? __ldg(doc_groups + id[d]) : -1;
                        }
                    }
                }
            }
        }
        __syncthreads();  // qsm is reloaded by the next run
        a = b;
    }
}

// Merge of per-rank partial group lists [rows, cols] (score, page, group; page < 0 = empty): the first k distinct groups
// in (score desc, page asc) order, one warp per row, the row in registers. Each round takes the best live entry and then
// retires every entry of its group: the first entry of a group in that order is its best.
template <int NPL>
__global__ void __launch_bounds__(256)
merge_groups_warp_kernel(const float* __restrict__ scores, const long long* __restrict__ pages,
                         const long long* __restrict__ groups, int rows, int cols, int k, float* __restrict__ out_scores,
                         long long* __restrict__ out_pages, long long* __restrict__ out_groups) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const long long base = static_cast<long long>(row) * cols;
    float s[NPL];
    long long id[NPL], gr[NPL];
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
        const int c = lane + j * 32;
        id[j] = c < cols ? pages[base + c] : -1;
        gr[j] = id[j] >= 0 ? groups[base + c] : -1;
        s[j] = id[j] >= 0 ? scores[base + c] : -INFINITY;
    }
    for (int round = 0; round < k; ++round) {
        float bs = -INFINITY;
        long long bi = 0x7fffffffffffffffll, bg = -1;
#pragma unroll
        for (int j = 0; j < NPL; ++j)
            if (id[j] >= 0 && before(s[j], id[j], bs, bi)) { bs = s[j]; bi = id[j]; bg = gr[j]; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float os = __shfl_xor_sync(0xffffffffu, bs, o);
            const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
            const long long og = __shfl_xor_sync(0xffffffffu, bg, o);
            if (before(os, oi, bs, bi)) { bs = os; bi = oi; bg = og; }
        }
        const bool valid = bi != 0x7fffffffffffffffll;
        const long long o = static_cast<long long>(row) * k;
        if (lane == 0) {
            out_scores[o + round] = valid ? bs : -INFINITY;
            out_pages[o + round] = valid ? bi : -1;
            out_groups[o + round] = valid ? bg : -1;
        }
        if (!valid) {
            for (int r2 = round + 1 + lane; r2 < k; r2 += 32) {
                out_scores[o + r2] = -INFINITY;
                out_pages[o + r2] = -1;
                out_groups[o + r2] = -1;
            }
            break;
        }
#pragma unroll
        for (int j = 0; j < NPL; ++j)
            if (gr[j] == bg) id[j] = -1;
    }
}

// fp32 -> fp16 rows, with the row L2 norms and their maximum (norms are >= 0, so the int view orders them).
__global__ void f32_to_f16_rows_kernel(const float* __restrict__ src, long long rows, int dim, __half* __restrict__ dst,
                                       float* __restrict__ norms, float* __restrict__ max_norm) {
    constexpr int CH = 6;  // float4 per lane in flight (dim 2304 = 3 chunks of 6 x 32 float4)
    const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
    const int nv = dim >> 2;
    for (long long r = static_cast<long long>(blockIdx.x) * warps + (threadIdx.x >> 5); r < rows;
         r += static_cast<long long>(gridDim.x) * warps) {
        const float4* s4 = reinterpret_cast<const float4*>(src + r * dim);
        uint2* d2 = reinterpret_cast<uint2*>(dst + r * dim);
        float ss = 0.f;
        for (int i0 = 0; i0 < nv; i0 += CH * 32) {
            float4 v[CH];
#pragma unroll
            for (int j = 0; j < CH; ++j) {
                const int i = i0 + j * 32 + lane;
                v[j] = i < nv ? __ldcs(s4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int j = 0; j < CH; ++j) {
                const int i = i0 + j * 32 + lane;
                ss += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
                if (i < nv) {
                    uint2 pk;
                    pk.x = pack_f16x2(v[j].x, v[j].y);
                    pk.y = pack_f16x2(v[j].z, v[j].w);
                    d2[i] = pk;
                }
            }
        }
        ss = warp_sum_f(ss);
        if (lane == 0) {
            const float n = sqrtf(ss);
            if (norms) norms[r] = n;
            if (max_norm) atomicMax(reinterpret_cast<int*>(max_norm), __float_as_int(n));
        }
    }
}

// Before the filter: every list slot beyond the R real ones becomes an empty list (-inf, -1). The LAST slot doubles as
// the query's running threshold tau (its first score; id -1 keeps the rescoring kernel from reading it as a candidate).
__global__ void score_init_lists_kernel(float* __restrict__ cand_scores, int* __restrict__ cand_ids, int nq, int lists, int R) {
    const int per_row = (lists - R) * SC_KT;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < static_cast<long long>(nq) * per_row;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long row = i / per_row;
        const long long o = (row * lists + R) * SC_KT + (i - row * per_row);
        cand_scores[o] = -INFINITY;
        cand_ids[o] = -1;
    }
}

// CTA pairs of the (persistent) filter kernel: one CTA per SM
static int score_pairs() { return num_sms() / 2; }

struct ScorePlan {
    int T, R, QB, items, lists, pairs;
};

static ScorePlan score_plan(int nq, long long nd) {
    ScorePlan p;
    p.QB = (nq + 2 * GEMM_BM - 1) / (2 * GEMM_BM);
    p.T = static_cast<int>((nd + SC_BN - 1) / SC_BN);
    const int P = score_pairs();
    // time ~ waves * tiles per item, plus half a tile per item for the pipeline fill, the merge of the quad's lists and
    // the list write-out
    double best = 1e30;
    p.R = 1;
    for (int R = 1; R <= SC_MAX_RANGES && R <= p.T; ++R) {
        const long long waves = (static_cast<long long>(p.QB) * R + P - 1) / P;
        const double cost = static_cast<double>(waves) * ((p.T + R - 1) / R + 0.5);
        if (cost < best * 0.98) { best = cost; p.R = R; }  // a larger R must win by 2 %: fewer lists to rescore
    }
    p.items = p.QB * p.R;
    p.pairs = p.items < P ? p.items : P;
    p.lists = 2 * ((p.R + 2) / 2);  // >= R + 1: the last slot carries the per-query threshold (score_init_lists_kernel)
    return p;
}

static int score_ranges_for(int nq, long long nd) { return score_plan(nq, nd).lists / 2; }

// A doc mask as the _masked entry points take it: present and 4-byte aligned (one uint32 word per 32 docs).
static bool mask_ok(const uint32_t* mask) { return mask && (reinterpret_cast<uintptr_t>(mask) & 3) == 0; }

static const DocMasks kNoMasks = {nullptr, 0, nullptr};

// A single doc mask (the _masked entry points, the doc_mask arguments) is the mask set of one.
static DocMasks one_mask(const uint32_t* words, long long nd) { return DocMasks{words, (nd + 31) / 32, nullptr}; }

// A mask set as the _masks entry points take it, refused before any CUDA call unless every row it names can be read for
// nd docs. The values of of_query lie in device memory: the caller keeps them in [0, count).
static int masks_check(const char* fn, const vr_doc_masks* m, long long nd) {
    VR_REQUIRE(m, "%s: masks must not be NULL", fn);
    VR_REQUIRE(m->words, "%s: masks->words must not be NULL", fn);
    VR_REQUIRE_ALIGNED(fn, "masks->words", m->words, 4);
    VR_REQUIRE(m->count >= 1, "%s: masks->count=%d, needs at least one mask", fn, m->count);
    VR_REQUIRE(m->pitch >= (nd + 31) / 32, "%s: masks->pitch=%lld words is below ceil(nd / 32) = %lld", fn,
               (long long)m->pitch, (long long)((nd + 31) / 32));
    VR_REQUIRE(m->count == 1 || m->of_query, "%s: masks->of_query is NULL with masks->count=%d masks", fn, m->count);
    VR_REQUIRE_ALIGNED(fn, "masks->of_query", m->of_query, 4);
    return 0;
}
#define VR_REQUIRE_MASKS(fn, m, nd)                                   \
    do {                                                              \
        if (int rc_ = masks_check((fn), (m), (nd))) return rc_;       \
    } while (0)

static DocMasks device_masks(const vr_doc_masks* m) { return DocMasks{m->words, m->pitch, m->of_query}; }

// The list initialisation (range forms: the zeroing of the candidate counters), then score_filter_kernel<Args> over
// `plan`, after the caller's argument checks. masks, doc_groups and range go to the forms whose Args carry them.
template <typename Args>
static int launch_score_filter(const ScorePlan& plan, const void* q_f16, int nq, const void* d_f16, long long nd, int dim,
                               float* cand_scores, int* cand_ids, const DocMasks& masks, const int* doc_groups,
                               cudaStream_t st, const RangeFields* range = nullptr) {
    using Cfg = Score2Cfg;
    CUtensorMap tq, td;
    if (int rc = make_tmap_2d(&tq, q_f16, nq, dim, dim, GEMM_BM, GEMM_BK, 128, false)) return rc;
    if (int rc = make_tmap_2d(&td, d_f16, nd, dim, dim, 128, GEMM_BK, 128, false)) return rc;
    static unsigned long long attr_set = 0;
    if (first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(score_filter_kernel<Args>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    Args g;
    g.nq = nq; g.nd = nd; g.dim = dim; g.lists = plan.lists; g.T = plan.T; g.R = plan.R; g.QB = plan.QB; g.items = plan.items;
    g.cand_scores = cand_scores; g.cand_ids = cand_ids;
    if constexpr (kMasked<Args>) g.masks = masks;
    if constexpr (kGrouped<Args>) g.doc_groups = doc_groups;
    if constexpr (kRange<Args>) {
        g.range = *range;
        VR_CHECK_CUDA(cudaMemsetAsync(range->counts, 0, static_cast<size_t>(nq) * sizeof(int), st));
    } else {
        const long long n = static_cast<long long>(nq) * (plan.lists - plan.R) * SC_KT;
        long long blocks = (n + 255) / 256;
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        score_init_lists_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(cand_scores, cand_ids, nq, plan.lists, plan.R);
        VR_CHECK_CUDA(cudaGetLastError());
    }
    score_filter_kernel<Args><<<2 * plan.pairs, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tq, td, g);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// vr_score_filter(_masked, _masks): the page lists, masked when masks is not NULL (after the caller's mask checks)
static int score_filter(const char* fn, const void* q_f16, int nq, const void* d_f16, long long nd, int dim, int ranges,
                        const DocMasks* masks, float* cand_scores, int* cand_ids, void* stream) {
    VR_REQUIRE(q_f16 && d_f16 && cand_scores && cand_ids, "%s: null pointer", fn);
    VR_REQUIRE(nq > 0 && nd > 0 && nd < 2147483647ll && dim % 8 == 0, "%s: bad shape nq=%d nd=%lld dim=%d", fn, nq,
               (long long)nd, dim);
    VR_REQUIRE(nq < (1 << 30), "%s: too many queries", fn);
    const ScorePlan plan = score_plan(nq, nd);
    VR_REQUIRE(ranges * 2 == plan.lists, "%s: ranges must come from vr_score_ranges()", fn);
    // q / d are TMA sources; the candidate lists are written 16 bytes at a time
    VR_REQUIRE_ALIGNED(fn, "q_f16", q_f16, 16);
    VR_REQUIRE_ALIGNED(fn, "d_f16", d_f16, 16);
    VR_REQUIRE_ALIGNED(fn, "cand_scores", cand_scores, 16);
    VR_REQUIRE_ALIGNED(fn, "cand_ids", cand_ids, 16);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (masks)
        return launch_score_filter<MaskedScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, cand_scores, cand_ids, *masks, nullptr, st);
    return launch_score_filter<ScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, cand_scores, cand_ids, kNoMasks, nullptr, st);
}

// vr_topk_rows(_masked, _masks), after the mask checks: the masked form when masks is not NULL (ids is NULL then)
static int topk_rows(const char* fn, const float* scores, const int64_t* ids, int rows, long long cols, int k,
                     long long id_offset, float* out_scores, int64_t* out_ids, const DocMasks* masks, void* stream) {
    VR_REQUIRE(scores && out_scores && out_ids, "%s: null pointer", fn);
    VR_REQUIRE(rows > 0 && cols > 0 && k > 0, "%s: bad shape", fn);
    const long long* i = reinterpret_cast<const long long*>(ids);
    long long* oi = reinterpret_cast<long long*>(out_ids);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (masks) launch_topk_rows<true>(scores, i, rows, cols, k, id_offset, out_scores, oi, *masks, s);
    else launch_topk_rows<false>(scores, i, rows, cols, k, id_offset, out_scores, oi, kNoMasks, s);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// vr_topk_rows_chunked(_masked, _masks), after the mask checks: the masked form when masks is not NULL
static int topk_rows_chunked(const char* fn, const float* scores, int rows, long long cols, int k, long long id_offset,
                             int chunks, float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids,
                             const DocMasks* masks, void* stream) {
    VR_REQUIRE(scores && ws_scores && ws_ids && out_scores && out_ids, "%s: null pointer", fn);
    VR_REQUIRE(rows > 0 && cols > 0 && k > 0 && chunks > 0 && chunks <= 65535, "%s: bad shape", fn);
    long long* wi = reinterpret_cast<long long*>(ws_ids);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const long long chunk_cols = (cols + chunks - 1) / chunks;
    // pass 1: every (row, chunk) block reduces its column range to a sorted top-k list (ids = column + id_offset)
    if (masks)
        topk_rows_kernel<true><<<dim3(rows, chunks), 256, 0, s>>>(scores, nullptr, cols, k, id_offset, chunk_cols, ws_scores,
                                                                  wi, *masks);
    else
        topk_rows_kernel<false><<<dim3(rows, chunks), 256, 0, s>>>(scores, nullptr, cols, k, id_offset, chunk_cols, ws_scores,
                                                                   wi, kNoMasks);
    VR_CHECK_CUDA(cudaGetLastError());
    // pass 2: merge the `chunks` lists of each row (explicit ids; exhausted lists carry id -1 and are skipped)
    launch_topk_rows<false>(ws_scores, wi, rows, static_cast<long long>(chunks) * k, k, 0, out_scores,
                            reinterpret_cast<long long*>(out_ids), kNoMasks, s);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Candidates rescored per query (the best by approximate score), for vr_score_rescore(_groups)
static int rescore_keep(int k, int lists) {
    int keep = 2 * k > 32 ? 2 * k : 32;
    if (keep > lists * SC_KT) keep = lists * SC_KT;
    if (keep > RS_MAX_KEEP) keep = RS_MAX_KEEP;
    return keep;
}

// ---------------------------------------------------------------------------------------------------- range search
// Every eligible doc with exact score s >= t of its query row, ordered by (score desc, id asc). Two producers fill a
// per-row REGION (scores, ids, a row pitch, a count per row) in no particular order: the candidate rescoring after the
// range filter, and the selection over rows of the fp32 scan. One ordering step (vr_range_sort) turns any region into
// CSR rows.

// Exact fp32 rescoring of the filter's candidates: block (x, y) takes candidates y, y + gridDim.y * 8, ... of query row
// x, one warp per candidate through warp_dot_row (the bits of vr_score_exact), and appends those with s >= t to the
// row's region [cap] (kept[row] counts them; zeroed by the host). A row whose counter says it overflowed (count > cap)
// is skipped: the host reruns it through the fp32 scan.
constexpr int RR_THREADS = 256;

__global__ void __launch_bounds__(RR_THREADS)
range_rescore_kernel(const float* __restrict__ Q, const float* __restrict__ D, int dim, const float* __restrict__ thresholds,
                     int cap, const int* __restrict__ counts, const int* __restrict__ cand, float* __restrict__ out_scores,
                     int* __restrict__ out_ids, int* __restrict__ kept) {
    extern __shared__ float qs[];  // [dim]
    const int q = blockIdx.x;
    const int n = __ldg(counts + q);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c0 = blockIdx.y * (RR_THREADS / 32) + warp, stride = gridDim.y * (RR_THREADS / 32);
    if (n > cap || blockIdx.y * (RR_THREADS / 32) >= n) return;  // block-uniform
    const float* qrow = Q + static_cast<long long>(q) * dim;
    for (int i = threadIdx.x; i < dim; i += RR_THREADS) qs[i] = qrow[i];
    __syncthreads();
    const float t = __ldg(thresholds + q);
    const long long base = static_cast<long long>(q) * cap;
    for (int c = c0; c < n; c += stride) {
        const int id = __ldg(cand + base + c);
        const float s = warp_dot_row(qs, D + static_cast<long long>(id) * dim, dim, lane);
        if (lane == 0 && s >= t) {
            const int o = atomicAdd(kept + q, 1);
            out_scores[base + o] = s;
            out_ids[base + o] = id;
        }
    }
}

// Selection over rows of vr_score_exact output [rows, nd]: the eligible columns (by the mask of each row, masks.words
// NULL: every column) with s >= t_row, appended to the row's region [pitch] with one atomicAdd per warp (counts zeroed by
// the host). NaN scores never pass. Block (x, y): row y, column strides of 256 from 256 x.
__global__ void __launch_bounds__(256)
range_select_kernel(const float* __restrict__ scores, long long nd, const float* __restrict__ thresholds, const DocMasks masks,
                    long long pitch, float* __restrict__ out_scores, int* __restrict__ out_ids, int* __restrict__ counts) {
    const int row = blockIdx.y, lane = threadIdx.x & 31;
    const float t = __ldg(thresholds + row);
    const uint32_t* mask = masks.words ? mask_of_row(masks, row) : nullptr;
    const float* srow = scores + static_cast<long long>(row) * nd;
    const long long o_row = static_cast<long long>(row) * pitch;
    for (long long c0 = static_cast<long long>(blockIdx.x) * 256; c0 < nd; c0 += static_cast<long long>(gridDim.x) * 256) {
        const long long c = c0 + threadIdx.x;
        float s = 0.f;
        bool keep = false;
        if (c < nd) {
            s = srow[c];
            keep = s >= t && (!mask || col_eligible(mask, c));
        }
        const uint32_t b = __ballot_sync(0xffffffffu, keep);
        if (b) {
            int base = 0;
            if (lane == 0) base = atomicAdd(counts + row, __popc(b));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (keep) {
                const int o = base + __popc(b & ((1u << lane) - 1u));
                out_scores[o_row + o] = s;
                out_ids[o_row + o] = static_cast<int>(c);
            }
        }
    }
}

// Sort key of an entry: ascending keys = (score desc, id asc), the before() order. High word: the order-preserving bits
// of the score, inverted; -0 is canonicalised to +0 (they tie under before(), so the id decides). Low word: id << 1, and
// bit 0 remembers a -0 so that the output keeps the score's own bits (it never decides an order: ids are distinct).
// The all-ones key is the padding: it would need a NaN score, which no producer emits.
// Order-preserving bits of a score (raw bits b): increasing in the score, -0 as +0 (NaNs land beyond +-inf).
__device__ __forceinline__ uint32_t score_order(uint32_t b) {
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long range_key(float s, int id) {
    const uint32_t b = __float_as_uint(s);
    const uint32_t negzero = b == 0x80000000u ? 1u : 0u;
    const uint32_t o = score_order(b);
    return (static_cast<unsigned long long>(~o) << 32) | (static_cast<uint32_t>(id) << 1) | negzero;
}

__device__ __forceinline__ void range_unkey(unsigned long long key, float& s, long long& id) {
    const uint32_t o = ~static_cast<uint32_t>(key >> 32), lo = static_cast<uint32_t>(key);
    const uint32_t b = (lo & 1u) ? 0x80000000u : (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    s = __uint_as_float(b);
    id = static_cast<long long>(lo >> 1);
}

constexpr int RSORT_TILE = 4096;   // entries a block orders in shared memory (32 KB of keys)
constexpr int RSORT_THREADS = 512;

// One bitonic compare-exchange stage (k, j) over keys[0, n) of shared memory; idx0 is the global index of keys[0], which
// sets the direction of each pair (ascending when (index & k) == 0).
__device__ __forceinline__ void bitonic_stage(unsigned long long* keys, int n, long long idx0, long long k, int j) {
    for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const unsigned long long a = keys[i], b = keys[i + j];
        const bool up = ((idx0 + i) & k) == 0;
        if ((a > b) == up) { keys[i] = b; keys[i + j] = a; }
    }
    __syncthreads();
}

__device__ __forceinline__ long long region_row(const int* row_of, int i) {
    return row_of ? static_cast<long long>(__ldg(row_of + i)) : i;
}

// Rows of at most RSORT_TILE entries: block i loads region row r = row_of[i] as keys (padded to a power of two), sorts
// them in shared memory and writes the CSR row at out_offsets[r].
__global__ void __launch_bounds__(RSORT_THREADS)
range_sort_smem_kernel(const float* __restrict__ scores, const int* __restrict__ ids, long long pitch,
                       const int* __restrict__ counts, const int* __restrict__ row_of, const long long* __restrict__ out_offsets,
                       long long id_offset, float* __restrict__ out_scores, long long* __restrict__ out_ids) {
    __shared__ unsigned long long keys[RSORT_TILE];
    const long long r = region_row(row_of, blockIdx.x);
    const int n = __ldg(counts + r);
    if (n <= 0) return;
    int P = 1;
    while (P < n) P <<= 1;
    for (int j = threadIdx.x; j < P; j += RSORT_THREADS)
        keys[j] = j < n ? range_key(scores[r * pitch + j], ids[r * pitch + j]) : ~0ull;
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) bitonic_stage(keys, P, 0, k, j);
    const long long o = __ldg(out_offsets + r);
    for (int j = threadIdx.x; j < n; j += RSORT_THREADS) {
        float s;
        long long id;
        range_unkey(keys[j], s, id);
        out_scores[o + j] = s;
        out_ids[o + j] = id + id_offset;
    }
}

// Longer rows: a bitonic sort of P = 2^m >= RSORT_TILE keys per row in the workspace [rows, P]. Stages with j >= TILE
// run over global memory (range_bitonic_global_kernel, one launch per stage); all stages with j < TILE of one k run in
// shared memory, tile by tile (range_bitonic_tile_kernel).
__global__ void __launch_bounds__(256)
range_keys_kernel(const float* __restrict__ scores, const int* __restrict__ ids, long long pitch, const int* __restrict__ counts,
                  const int* __restrict__ row_of, long long P, unsigned long long* __restrict__ ws) {
    const long long r = region_row(row_of, blockIdx.y);
    const int n = __ldg(counts + r);
    unsigned long long* w = ws + static_cast<long long>(blockIdx.y) * P;
    for (long long j = blockIdx.x * 256ll + threadIdx.x; j < P; j += static_cast<long long>(gridDim.x) * 256)
        w[j] = j < n ? range_key(scores[r * pitch + j], ids[r * pitch + j]) : ~0ull;
}

// k_lo == 2: every stage of k = 2 .. TILE (each tile sorted in the direction its global index gives); else the stages
// j = TILE/2 .. 1 of k = k_lo.
__global__ void __launch_bounds__(RSORT_THREADS)
range_bitonic_tile_kernel(unsigned long long* __restrict__ ws, long long P, long long k_lo) {
    __shared__ unsigned long long keys[RSORT_TILE];
    const long long idx0 = static_cast<long long>(blockIdx.x) * RSORT_TILE;
    unsigned long long* w = ws + static_cast<long long>(blockIdx.y) * P + idx0;
    for (int j = threadIdx.x; j < RSORT_TILE; j += RSORT_THREADS) keys[j] = w[j];
    __syncthreads();
    if (k_lo == 2) {
        for (int k = 2; k <= RSORT_TILE; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) bitonic_stage(keys, RSORT_TILE, idx0, k, j);
    } else {
        for (int j = RSORT_TILE / 2; j > 0; j >>= 1) bitonic_stage(keys, RSORT_TILE, idx0, k_lo, j);
    }
    for (int j = threadIdx.x; j < RSORT_TILE; j += RSORT_THREADS) w[j] = keys[j];
}

__global__ void __launch_bounds__(256)
range_bitonic_global_kernel(unsigned long long* __restrict__ ws, long long P, long long k, long long j) {
    unsigned long long* w = ws + static_cast<long long>(blockIdx.y) * P;
    for (long long t = blockIdx.x * 256ll + threadIdx.x; t < P / 2; t += static_cast<long long>(gridDim.x) * 256) {
        const long long i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const unsigned long long a = w[i], b = w[i + j];
        const bool up = (i & k) == 0;
        if ((a > b) == up) { w[i] = b; w[i + j] = a; }
    }
}

__global__ void __launch_bounds__(256)
range_emit_kernel(const unsigned long long* __restrict__ ws, long long P, const int* __restrict__ counts,
                  const int* __restrict__ row_of, const long long* __restrict__ out_offsets, long long id_offset,
                  float* __restrict__ out_scores, long long* __restrict__ out_ids) {
    const long long r = region_row(row_of, blockIdx.y);
    const int n = __ldg(counts + r);
    const long long o = __ldg(out_offsets + r);
    const unsigned long long* w = ws + static_cast<long long>(blockIdx.y) * P;
    for (long long j = blockIdx.x * 256ll + threadIdx.x; j < n; j += static_cast<long long>(gridDim.x) * 256) {
        float s;
        long long id;
        range_unkey(w[j], s, id);
        out_scores[o + j] = s;
        out_ids[o + j] = id + id_offset;
    }
}

// The workspace of vr_range_sort: none up to RSORT_TILE entries a row, else rows x P keys.
static long long range_sort_P(int max_count) {
    long long P = RSORT_TILE;
    while (P < max_count) P <<= 1;
    return P;
}

static long long range_sort_ws(int rows, int max_count) {
    return max_count <= RSORT_TILE ? 0 : static_cast<long long>(rows) * range_sort_P(max_count) * 8;
}

// vr_range_groups: a region reduced to one entry per group (document) of each row, the group's first entry in the
// before() order with that entry's own score bits, appended to the output region in no particular order. Pass 1 takes
// the atomicMax of page_key per (row, group): the order bits of the score above ~page, so the largest key is the highest
// score and then the lowest page (-0 as +0), whatever order the atomics run in. Pass 2: the entry whose key equals its
// group's slot claims the slot (an atomicCAS back to 0, so a repeated entry is emitted once) and appends itself. The
// per-row table is an open-addressing hash of P >= 2 * max_count slots (key u64, group int32; load <= 1/2): in shared
// memory up to RGROUP_SMEM_MAX entries a row, one block per row, else in the caller's workspace [rows, P] with blocks
// spread over each row. An entry counts when its score is not NaN, its id lies in [0, nd) and its group in [0, G).
constexpr int RGROUP_SMEM_MAX = 4096;  // 8192 slots, 96 KB
constexpr int RGROUP_THREADS = 512;

__device__ __forceinline__ uint32_t rgroup_hash(uint32_t g) {  // the finaliser of MurmurHash3: spreads strided group ids
    g ^= g >> 16; g *= 0x85ebca6bu; g ^= g >> 13; g *= 0xc2b2ae35u; g ^= g >> 16;
    return g;
}

// One pass over entries [j0, n) (step `step`) of a region row (at `base`) against its table (keys tk, groups tg, P = mask + 1
// slots). INSERT: atomicMax of each entry's key into its group's slot (taking an empty slot when the group has none).
// Else: the entry holding its slot's key claims it and goes to the output row at `obase` (count in *emitted).
template <bool INSERT>
__device__ __forceinline__ void rgroup_pass(const float* __restrict__ scores, const int* __restrict__ ids, long long base,
                                            int j0, int n, int step, long long nd, const int* __restrict__ doc_groups, int G,
                                            unsigned long long* tk, int* tg, uint32_t mask, float* __restrict__ out_scores,
                                            int* __restrict__ out_ids, long long obase, int* emitted) {
    for (int j = j0; j < n; j += step) {
        const float s = scores[base + j];
        const int id = ids[base + j];
        if (isnan(s) || id < 0 || id >= nd) continue;
        const int g = __ldg(doc_groups + id);
        if (g < 0 || g >= G) continue;
        const unsigned long long key = page_key(s, id);
        uint32_t h = rgroup_hash(static_cast<uint32_t>(g)) & mask;
        for (;;) {  // the group's slot: pass 2 finds it before any empty slot
            const int cur = INSERT ? atomicCAS(tg + h, -1, g) : tg[h];
            if (cur == -1 || cur == g) break;
            h = (h + 1) & mask;
        }
        if (INSERT) {
            atomicMax(tk + h, key);
        } else if (atomicCAS(tk + h, key, 0ull) == key) {
            const int o = atomicAdd(emitted, 1);
            out_scores[obase + o] = s;
            out_ids[obase + o] = id;
        }
    }
}

__device__ __forceinline__ int rgroup_count(const int* counts, long long r, int max_count) {
    return max(0, min(__ldg(counts + r), max_count));  // the caller keeps counts <= max_count; the table holds no more
}

__global__ void __launch_bounds__(RGROUP_THREADS)
range_groups_smem_kernel(const float* __restrict__ scores, const int* __restrict__ ids, long long pitch,
                         const int* __restrict__ counts, int max_count, long long nd, const int* __restrict__ doc_groups,
                         int G, int P, float* __restrict__ out_scores, int* __restrict__ out_ids, int* __restrict__ out_counts) {
    extern __shared__ unsigned long long rg_keys[];  // [P] keys, then [P] groups
    int* rg_groups = reinterpret_cast<int*>(rg_keys + P);
    __shared__ int emitted;
    const long long r = blockIdx.x, base = r * pitch;
    const int n = rgroup_count(counts, r, max_count);
    for (int j = threadIdx.x; j < P; j += RGROUP_THREADS) { rg_keys[j] = 0; rg_groups[j] = -1; }
    if (threadIdx.x == 0) emitted = 0;
    __syncthreads();
    rgroup_pass<true>(scores, ids, base, threadIdx.x, n, RGROUP_THREADS, nd, doc_groups, G, rg_keys, rg_groups, P - 1,
                      nullptr, nullptr, 0, nullptr);
    __syncthreads();
    rgroup_pass<false>(scores, ids, base, threadIdx.x, n, RGROUP_THREADS, nd, doc_groups, G, rg_keys, rg_groups, P - 1,
                       out_scores, out_ids, base, &emitted);
    __syncthreads();
    if (threadIdx.x == 0) out_counts[r] = emitted;
}

// The workspace form: block (x, y) takes entries 256 x, 256 (x + gridDim.x), ... of row y; one launch per pass (the
// output counts are zeroed by the host).
template <bool INSERT>
__global__ void __launch_bounds__(256)
range_groups_ws_kernel(const float* __restrict__ scores, const int* __restrict__ ids, long long pitch,
                       const int* __restrict__ counts, int max_count, long long nd, const int* __restrict__ doc_groups, int G,
                       long long P, unsigned long long* __restrict__ ws, float* __restrict__ out_scores,
                       int* __restrict__ out_ids, int* __restrict__ out_counts) {
    const long long r = blockIdx.y, base = r * pitch;
    const int n = rgroup_count(counts, r, max_count);
    unsigned long long* tk = ws + r * P;
    int* tg = reinterpret_cast<int*>(ws + gridDim.y * P) + r * P;
    rgroup_pass<INSERT>(scores, ids, base, blockIdx.x * 256 + threadIdx.x, n, gridDim.x * 256, nd, doc_groups, G, tk, tg,
                        static_cast<uint32_t>(P - 1), out_scores, out_ids, base, out_counts + r);
}

static long long range_groups_P(int max_count) {
    long long P = 2;
    while (P < 2ll * max_count) P <<= 1;
    return P;
}

// The workspace of vr_range_groups: none up to RGROUP_SMEM_MAX entries a row, else rows x P slots of 12 bytes.
static long long range_groups_ws(int rows, int max_count) {
    return max_count <= RGROUP_SMEM_MAX ? 0 : static_cast<long long>(rows) * range_groups_P(max_count) * 12;
}

// ---------------------------------------------------------------------------------------------------- radix select
// vr_select_rows: the top-k of each row with the bits and order of vr_topk_rows, in passes over the row whose number does
// not grow with k (DESIGN §4, "Deep top-k"). An entry counts when its id is >= 0, its column is eligible under the row's
// mask and its score is not NaN; its key is score_order(score) (-0 as +0, the tie rule of before()). Digit passes of 8
// bits, each a shared-memory histogram of the entries that match the digits chosen so far, find the key B of the k-th
// entry and how many entries of key B it takes; a pass whose chosen bin holds exactly that many ends the search early.
// When the boundary splits the entries of key B, digit passes over their ids (from the top byte of the largest) find the
// highest id taken. The winners - key > B, or key == B and id <= that id - are gathered in shared memory and sorted
// bitonically by (key desc, id asc). vr_topk_rows emits a repeated (score, id) pair once: a block whose winners repeat a
// pair (only an input that repeats one can) reruns its row through topk_rows_block, so the result is that kernel's in
// every case.
constexpr int SEL_THREADS = 256;
constexpr int SEL_MAX_K = 4096;
constexpr int SEL_K_MIN = 32;  // k above this: vr_group_topk_rows selects with the radix select (retriever.SELECT_K_MIN)

struct SelState {
    int need;           // entries still to take from the matching bins
    int total;          // entries counted by the last histogram
    int bin_count;      // entries in the chosen bin
    unsigned int bin;   // the chosen bin
};

// Warp 0 after a histogram: the bin holding the need-th entry, bins walked from 255 down (DESC) or from 0 up. Sets
// st.bin and st.bin_count, lowers st.need by the entries of the bins walked past, and sets st.total.
template <bool DESC>
__device__ __forceinline__ void select_bin(const unsigned int* hist, SelState& st) {
    const int lane = threadIdx.x;
    int h[8], sum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int b = lane * 8 + j;
        h[j] = static_cast<int>(hist[DESC ? 255 - b : b]);
        sum += h[j];
    }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    const int need = st.need;
    __syncwarp();
    int past = incl - sum;
    bool found = !(past < need && need <= incl);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (!found && past + h[j] >= need) {
            found = true;
            st.bin = DESC ? 255 - (lane * 8 + j) : lane * 8 + j;
            st.bin_count = h[j];
            st.need = need - past;
        }
        past += h[j];
    }
    if (lane == 31) st.total = incl;
    __syncwarp();
}

template <bool MASKED>
__global__ void __launch_bounds__(SEL_THREADS, 4)  // without the 4, ptxas caps the unmasked form at 48 registers and spills
select_rows_kernel(const float* __restrict__ scores, const long long* __restrict__ ids, long long cols, int k,
                   long long id_offset, long long chunk_cols, float* __restrict__ out_scores,
                   long long* __restrict__ out_ids, const DocMasks masks) {
    // block (row, chunk) as in topk_rows_kernel. Dynamic shared memory: [P] sort words (~key << 32 | score bits), then
    // [P] ids, P = the power of two >= k.
    extern __shared__ unsigned long long sel_words[];
    __shared__ unsigned int hist[256];
    __shared__ SelState st;
    __shared__ unsigned long long id_max;
    __shared__ int taken, repeat;
    const long long c_lo = static_cast<long long>(blockIdx.y) * chunk_cols;
    const long long c_hi = min(cols, c_lo + chunk_cols);
    const float* srow = scores + static_cast<long long>(blockIdx.x) * cols;
    const long long* irow = ids ? ids + static_cast<long long>(blockIdx.x) * cols : nullptr;
    const long long row = static_cast<long long>(blockIdx.x) * gridDim.y + blockIdx.y;  // output list
    const uint32_t* mask = MASKED ? mask_of_row(masks, blockIdx.x) : nullptr;
    const int lane = threadIdx.x & 31;

    // column c: false when it does not count, else its key, raw score bits and id
    auto entry = [&](long long c, uint32_t& key, uint32_t& bits, long long& id) -> bool {
        if (c >= c_hi) return false;
        id = irow ? irow[c] : c;
        if (id < 0 || (MASKED && !col_eligible(mask, c))) return false;
        const float s = srow[c];
        bits = __float_as_uint(s);
        key = score_order(bits);
        return !isnan(s);
    };
    // hist[d] = the entries whose digit_of is d (256: not counted), one shared atomic per distinct digit of a warp
    auto histogram = [&](auto digit_of) {
        for (int i = threadIdx.x; i < 256; i += SEL_THREADS) hist[i] = 0;
        __syncthreads();
        for (long long c0 = c_lo; c0 < c_hi; c0 += SEL_THREADS) {
            const unsigned int d = digit_of(c0 + threadIdx.x);
            const unsigned int peers = __match_any_sync(0xffffffffu, d);
            if (d < 256 && lane == __ffs(peers) - 1) atomicAdd(hist + d, static_cast<unsigned int>(__popc(peers)));
        }
        __syncthreads();
    };

    // winners: key > thr, or key == thr and id <= id_hi
    uint32_t thr = 0, pmask = 0;
    long long id_hi = 0x7fffffffffffffffll;
    bool split = true;  // the boundary splits the entries of key thr
    if (threadIdx.x == 0) st.need = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        histogram([&](long long c) -> unsigned int {
            uint32_t key, bits;
            long long id;
            if (!entry(c, key, bits, id) || (key & pmask) != thr) return 256u;
            return (key >> shift) & 255u;
        });
        if (threadIdx.x < 32) select_bin<true>(hist, st);
        __syncthreads();
        if (shift == 24 && st.total <= k) {  // k or fewer entries: every one is a winner
            split = false;
            break;
        }
        thr |= st.bin << shift;
        pmask |= 255u << shift;
        if (st.bin_count == st.need) {  // the whole bin is taken: key >= thr
            split = false;
            break;
        }
    }
    if (split) {  // the lowest st.need ids of key thr
        if (threadIdx.x == 0) id_max = 0;
        __syncthreads();
        for (long long c = c_lo + threadIdx.x; c < c_hi; c += SEL_THREADS) {
            uint32_t key, bits;
            long long id;
            if (entry(c, key, bits, id) && key == thr) atomicMax(&id_max, static_cast<unsigned long long>(id));
        }
        __syncthreads();
        const unsigned long long top = id_max;
        unsigned long long ip = 0, imask = 0;
        int shift = top ? (63 - __clzll(static_cast<long long>(top))) & ~7 : 0;
        for (;; shift -= 8) {
            histogram([&](long long c) -> unsigned int {
                uint32_t key, bits;
                long long id;
                if (!entry(c, key, bits, id) || key != thr || (static_cast<unsigned long long>(id) & imask) != ip) return 256u;
                return static_cast<unsigned int>(id >> shift) & 255u;
            });
            if (threadIdx.x < 32) select_bin<false>(hist, st);
            __syncthreads();
            ip |= static_cast<unsigned long long>(st.bin) << shift;
            imask |= 255ull << shift;
            if (shift == 0 || st.bin_count == st.need) break;
        }
        id_hi = static_cast<long long>(ip | ((1ull << shift) - 1));  // ids of key thr sit below 2^(shift + 8)
    }

    int P = 1;
    while (P < k) P <<= 1;
    unsigned long long* wk = sel_words;
    long long* wi = reinterpret_cast<long long*>(sel_words + P);
    if (threadIdx.x == 0) { taken = 0; repeat = 0; }
    __syncthreads();
    for (long long c = c_lo + threadIdx.x; c < c_hi; c += SEL_THREADS) {
        uint32_t key, bits;
        long long id;
        if (entry(c, key, bits, id) && (key > thr || (key == thr && id <= id_hi))) {
            const int slot = atomicAdd(&taken, 1);
            if (slot < k) {
                wk[slot] = (static_cast<unsigned long long>(~key) << 32) | bits;
                wi[slot] = id;
            }
        }
    }
    __syncthreads();
    const int n = taken;
    if (n <= k) {
        int P2 = 1;
        while (P2 < n) P2 <<= 1;
        for (int j = n + threadIdx.x; j < P2; j += SEL_THREADS) { wk[j] = ~0ull; wi[j] = 0x7fffffffffffffffll; }
        __syncthreads();
        for (int kk = 2; kk <= P2; kk <<= 1) {
            for (int j = kk >> 1; j > 0; j >>= 1) {
                for (int t = threadIdx.x; t < P2 / 2; t += SEL_THREADS) {
                    const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                    const unsigned long long a = wk[i], b = wk[i + j];
                    const long long ia = wi[i], ib = wi[i + j];
                    const bool later = (a >> 32) > (b >> 32) || ((a >> 32) == (b >> 32) && ia > ib);
                    if (later == ((i & kk) == 0)) { wk[i] = b; wk[i + j] = a; wi[i] = ib; wi[i + j] = ia; }
                }
                __syncthreads();
            }
        }
        for (int j = threadIdx.x; j + 1 < n; j += SEL_THREADS)
            if ((wk[j] >> 32) == (wk[j + 1] >> 32) && wi[j] == wi[j + 1]) repeat = 1;
        __syncthreads();
    }
    if (n > k || repeat) {  // block-uniform
        topk_rows_block<MASKED>(scores, ids, cols, k, id_offset, chunk_cols, out_scores, out_ids, masks);
        return;
    }
    for (int j = threadIdx.x; j < k; j += SEL_THREADS) {
        out_scores[row * k + j] = j < n ? __uint_as_float(static_cast<uint32_t>(wk[j])) : -INFINITY;
        out_ids[row * k + j] = j < n ? wi[j] + id_offset : -1;
    }
}

// ---------------------------------------------------------------------------------------------------- MMR selection
// Maximal marginal relevance over each query row's candidates (DESIGN §4). One thread-block cluster of C CTAs per query
// row: CTA c holds candidate rows [c * R, c * R + R) (R = ceil(fetch / C)) in shared memory, read from HBM once by 1-D
// bulk copies. Pick 1 is candidate 0. Each later pick is one round: every CTA reads the previous pick's row from its
// owner over DSMEM and folds sim(c_j, pick) into r_j of its own unpicked rows (one warp per row, warp_dot_row: the bits
// of vr_score_exact), takes its best key of v_j = fl(fl(lambda * s_j) - fl(mu * r_j)), and stores it into slot
// [round & 1][rank] of every CTA. After one cluster barrier every CTA reduces the same C slots and so agrees on the pick.
// The other parity lets a CTA write round t + 1's key while a slower one still reads round t's; round t + 2 needs the
// barrier of round t + 1, which the slower CTA passes only after reading.
constexpr int MMR_THREADS = 256;
constexpr int MMR_WARPS = MMR_THREADS / 32;
constexpr int MMR_MAX_FETCH = 128;
constexpr long long MMR_MAX_ELEMS = 128ll * 2304;   // fetch * dim
constexpr int MMR_CTA_BYTES = 144 * 1024;           // candidate rows held by one CTA
constexpr int MMR_MAX_CLUSTER = 8;

// (v, position j) as one key, larger = picked first: v's order bits (any NaN = 1, below -inf; -0 = +0) above ~j, so
// equal values go to the lower position. 0 is no candidate.
__device__ __forceinline__ unsigned long long mmr_key(float v, int j) {
    unsigned o = 1u;
    if (!isnan(v)) {
        const unsigned b = v == 0.f ? 0u : __float_as_uint(v);
        o = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    }
    return (static_cast<unsigned long long>(o) << 32) | (0xffffffffu - static_cast<unsigned>(j));
}

__global__ void __launch_bounds__(MMR_THREADS, 1)
mmr_select_kernel(const float* __restrict__ emb, long long nd, int dim, const float* __restrict__ cand_scores,
                  const long long* __restrict__ cand_ids, int fetch, const float* __restrict__ lambda, int k, int R,
                  long long id_offset, float* __restrict__ out_scores, long long* __restrict__ out_ids) {
    extern __shared__ __align__(16) float mmr_rows[];   // [R][dim]: this CTA's candidate rows, then [dim]: the pick's row
    __shared__ long long cid[MMR_MAX_FETCH];            // the row's candidate ids
    __shared__ float rel[MMR_MAX_FETCH], red[MMR_MAX_FETCH];  // s_j and r_j of this CTA's rows
    __shared__ int taken[MMR_MAX_FETCH], picks[MMR_MAX_FETCH];
    __shared__ unsigned long long slots[2][MMR_MAX_CLUSTER];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int sh_n;
    const unsigned C = cluster_nctarank(), rank = cluster_ctarank();
    const int q = blockIdx.x / C;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* cs = cand_scores + static_cast<long long>(q) * fetch;
    if (threadIdx.x == 0) {
        sh_n = fetch;
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    // the first id outside [0, nd) ends the row's candidates
    for (int j = threadIdx.x; j < fetch; j += MMR_THREADS) {
        const long long id = cand_ids[static_cast<long long>(q) * fetch + j];
        cid[j] = id;
        if (id < 0 || id >= nd) atomicMin(&sh_n, j);
    }
    __syncthreads();
    const int n = sh_n;
    const int base = static_cast<int>(rank) * R;
    const int own = max(0, min(R, n - base));
    const uint32_t row_bytes = static_cast<uint32_t>(dim) * 4;
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, row_bytes * own);
        for (int j = 0; j < own; ++j)
            bulk_load_1d(mmr_rows + static_cast<long long>(j) * dim, emb + cid[base + j] * dim, row_bytes, &bar);
    }
    for (int j = threadIdx.x; j < own; j += MMR_THREADS) {
        rel[j] = cs[base + j];
        red[j] = -INFINITY;
        taken[j] = 0;
    }
    const float lam = lambda[q];
    const float mu = __fsub_rn(1.f, lam);
    const int npick = min(k, n);
    mbar_wait(&bar, 0);
    cluster_sync_all();  // every CTA of the cluster runs and holds its rows
    int p = 0;           // the latest pick
    float* prow = mmr_rows + static_cast<long long>(R) * dim;
    for (int t = 1; t < npick; ++t) {
        // one copy of the pick's row per CTA: every warp reading it over DSMEM for each of its rows would make the
        // owner's SM serve C * R rows a round
        const int owner = p / R;
        const float4* src = reinterpret_cast<const float4*>(
            map_cluster_ptr(mmr_rows + static_cast<long long>(p - owner * R) * dim, owner));
        for (int i = threadIdx.x; i < (dim >> 2); i += MMR_THREADS) reinterpret_cast<float4*>(prow)[i] = src[i];
        __syncthreads();
        for (int j = warp; j < own; j += MMR_WARPS) {
            if (taken[j] || base + j == p) continue;
            const float s = warp_dot_row(prow, mmr_rows + static_cast<long long>(j) * dim, dim, lane);
            if (lane == 0) red[j] = fmaxf(red[j], s);  // maxNum: a NaN similarity leaves r_j as it is
        }
        __syncthreads();
        if (warp == 0) {
            if (lane == 0 && p >= base && p < base + own) taken[p - base] = 1;
            __syncwarp();
            unsigned long long best = 0;
            for (int j = lane; j < own; j += 32) {
                if (taken[j]) continue;
                const float v = __fsub_rn(__fmul_rn(lam, rel[j]), __fmul_rn(mu, red[j]));
                const unsigned long long key = mmr_key(v, base + j);
                best = key > best ? key : best;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
                best = other > best ? other : best;
            }
            if (lane < static_cast<int>(C)) st_shared_cluster_u64(mapa_u32(smem_u32(&slots[t & 1][rank]), lane), best);
        }
        cluster_sync_all();  // also the last DSMEM access of the round: no CTA exits while another reads its rows
        unsigned long long best = slots[t & 1][0];
        for (unsigned c = 1; c < C; ++c) best = slots[t & 1][c] > best ? slots[t & 1][c] : best;
        p = static_cast<int>(0xffffffffu - static_cast<unsigned>(best & 0xffffffffu));
        if (threadIdx.x == 0) picks[t] = p;
    }
    if (rank != 0) return;
    if (threadIdx.x == 0) picks[0] = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < k; t += MMR_THREADS) {
        const long long o = static_cast<long long>(q) * k + t;
        out_scores[o] = t < npick ? cs[picks[t]] : -INFINITY;
        out_ids[o] = t < npick ? cid[picks[t]] + id_offset : -1;
    }
}

// Cluster size of a call: the smallest of 1, 2, 4, 8 CTAs whose share of the fetch rows fits MMR_CTA_BYTES, provided
// that share and the pick's row fit MMR_SMEM_BYTES (0: none).
constexpr int MMR_SMEM_BYTES = 200 * 1024;
static int mmr_cluster(int fetch, int dim) {
    for (int c = 1; c <= MMR_MAX_CLUSTER; c *= 2) {
        const long long rows = (fetch + c - 1) / c;
        if (rows * dim * 4 <= MMR_CTA_BYTES) return (rows + 1) * dim * 4 <= MMR_SMEM_BYTES ? c : 0;
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Per-document top-m: the m best eligible pages of given groups (DESIGN §4, capped top-k and inner hits).
// ---------------------------------------------------------------------------------------------
constexpr int GROUP_PAGES_MAX = 256;   // m: pages kept per (row, slot, piece)
constexpr int GROUP_PIECE_MAX = 4096;  // pages of one group a block scores

// Block (row * kg + slot, piece) scores pages [piece * y, piece * (y + 1)) of group g = groups[row, slot] through the
// CSR, one warp per page (warp_dot_row: the lane loop of exact_scores_kernel, so every score has the bits
// vr_score_exact gives that pair), with the query row in shared memory. An ineligible page is never read and counts as
// NaN, which is never selected. fuse(row, page, s) turns each eligible page's score into the score it is ranked by
// (NoFuse: s itself). Page keys are distinct, so each entry's rank in (score desc, page asc) order is the number of
// entries before it: the entries of rank < m go straight to their slot, and the rest of the m slots get (-inf, -1). A
// group outside [0, G) is empty: padding, and nothing is read. The body of group_pages_topm_kernel and
// group_pages_fused_kernel.
template <class Fuse>
__device__ __forceinline__ void group_pages_block(const float* __restrict__ Q, const float* __restrict__ D, int dim,
                                                  const long long* __restrict__ groups, int kg, const int* __restrict__ offsets,
                                                  const int* __restrict__ pages, int G, const DocMasks& masks, int m,
                                                  int piece, long long id_offset, const Fuse& fuse,
                                                  float* __restrict__ out_scores, long long* __restrict__ out_pages) {
    extern __shared__ float gsm[];  // [dim] query row, then [piece] scores and [piece] pages
    float* qs = gsm;
    float* ps = gsm + dim;
    int* pp = reinterpret_cast<int*>(ps + piece);
    const long long rs = blockIdx.x;
    const long long row = rs / kg;
    const long long o = (rs * gridDim.y + blockIdx.y) * m;
    const long long g = groups[rs];
    int n = 0, lo = 0;
    if (g >= 0 && g < G) {
        lo = __ldg(offsets + g) + static_cast<int>(blockIdx.y) * piece;
        n = min(__ldg(offsets + g + 1) - lo, piece);
    }
    if (n <= 0) {  // block-uniform
        for (int t = threadIdx.x; t < m; t += blockDim.x) {
            out_scores[o + t] = -INFINITY;
            out_pages[o + t] = -1;
        }
        return;
    }
    for (int i = threadIdx.x; i < dim; i += blockDim.x) qs[i] = Q[row * dim + i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    const uint32_t* mask = masks.words ? mask_of_row(masks, row) : nullptr;
    for (int j = warp; j < n; j += warps) {
        const int p = __ldg(pages + lo + j);
        const bool eligible = !mask || col_eligible(mask, p);
        const float s = eligible ? warp_dot_row(qs, D + static_cast<long long>(p) * dim, dim, lane) : NAN;
        if (lane == 0) { ps[j] = eligible ? fuse(row, p, s) : s; pp[j] = p; }
    }
    __syncthreads();
    int valid = 0;
    for (int t0 = 0; t0 < n; t0 += blockDim.x) {  // uniform trip count: __syncthreads_count in every iteration
        const int t = t0 + threadIdx.x;
        const bool live = t < n && !isnan(ps[t]);
        if (live) {
            const float s = ps[t];
            const int p = pp[t];
            int rank = 0;
            for (int j = 0; j < n && rank < m; ++j) rank += !isnan(ps[j]) && before(ps[j], pp[j], s, p);
            if (rank < m) {
                out_scores[o + rank] = s;
                out_pages[o + rank] = p + id_offset;
            }
        }
        valid += __syncthreads_count(live);
    }
    for (int t = min(valid, m) + threadIdx.x; t < m; t += blockDim.x) {
        out_scores[o + t] = -INFINITY;
        out_pages[o + t] = -1;
    }
}

struct NoFuse {
    __device__ __forceinline__ float operator()(long long, int, float s) const { return s; }
};

__global__ void __launch_bounds__(256)
group_pages_topm_kernel(const float* __restrict__ Q, const float* __restrict__ D, int dim, const long long* __restrict__ groups,
                        int kg, const int* __restrict__ offsets, const int* __restrict__ pages, int G, const DocMasks masks,
                        int m, int piece, long long id_offset, float* __restrict__ out_scores,
                        long long* __restrict__ out_pages) {
    group_pages_block(Q, D, dim, groups, kg, offsets, pages, G, masks, m, piece, id_offset, NoFuse{}, out_scores, out_pages);
}

// ---------------------------------------------------------------------------------------------
// Hybrid retrieval: the dense score fused with an external score per (query, page) (DESIGN §4, "Hybrid retrieval").
// A hit list is CSR over query rows: row r's hits are ids / values [offsets[r], offsets[r + 1]).
// ---------------------------------------------------------------------------------------------
constexpr int FUSE_DENSE_MAX = 4096;  // dense entries per row vr_fuse_rows hashes (k of score_topk, or the RRF window)
constexpr int FUSE_THREADS = 256;

// The weighted sum with the two roundings of fp32 torch, fl(s + fl(w * v)): no contraction into an FMA.
__device__ __forceinline__ float fuse_sum(float s, float w, float v) { return __fadd_rn(s, __fmul_rn(w, v)); }

// The RRF term of a rank (from 1): fl(1 / fl(c + rank)), rounded to nearest.
__device__ __forceinline__ float rrf_term(int c, long long rank) {
    return __frcp_rn(static_cast<float>(static_cast<long long>(c) + rank));
}

// The weighted-sum fusion of vr_group_pages_fused: row r's hits sorted by id, looked up by a binary search.
struct HitsFuse {
    const long long* offsets;
    const int* ids;
    const float* values;
    float w;
    __device__ __forceinline__ float operator()(long long row, int p, float s) const {
        long long a = __ldg(offsets + row), b = __ldg(offsets + row + 1);
        while (a < b) {
            const long long mid = (a + b) >> 1;
            if (__ldg(ids + mid) < p) a = mid + 1;
            else b = mid;
        }
        return a < __ldg(offsets + row + 1) && __ldg(ids + a) == p ? fuse_sum(s, w, __ldg(values + a)) : s;
    }
};

__global__ void __launch_bounds__(256)
group_pages_fused_kernel(const float* __restrict__ Q, const float* __restrict__ D, int dim, const long long* __restrict__ groups,
                         int kg, const int* __restrict__ offsets, const int* __restrict__ pages, int G, const DocMasks masks,
                         const HitsFuse fuse, int piece, long long id_offset, float* __restrict__ out_scores,
                         long long* __restrict__ out_pages) {
    group_pages_block(Q, D, dim, groups, kg, offsets, pages, G, masks, 1, piece, id_offset, fuse, out_scores, out_pages);
}

// One block per query row. The row's dense entries (ids distinct, a negative id is empty) go into an open-addressing
// hash of P = 2^m >= 2 kd slots in shared memory (id -> slot; load <= 1/2), so the table fits whatever the length of the
// hit list. Each hit probes it: a hit whose page is a dense entry retires that entry and carries both scores. Output
// row r of [rows, width]: slots [0, kd) the dense entries that are not hits, then slot kd + i for hit i, then (-inf, -1).
// SUM: a hit scores fuse_sum(dense, w, v), a dense entry its own score. RRF: the dense rank of slot j is j + 1 and the
// external rank of hit i is i + 1 (the caller orders each row by (value desc, id asc)); a score is
// fl(rrf_term(dense rank) + rrf_term(external rank)), a missing rank contributing 0.
__global__ void __launch_bounds__(FUSE_THREADS)
fuse_rows_kernel(const float* __restrict__ dense_scores, const long long* __restrict__ dense_ids, int kd,
                 const long long* __restrict__ hit_offsets, const int* __restrict__ hit_ids,
                 const float* __restrict__ hit_values, const float* __restrict__ hit_dense, long long hit_pitch, bool rrf,
                 float w, int c, long long width, int P, float* __restrict__ out_scores, long long* __restrict__ out_ids,
                 int* __restrict__ status) {
    extern __shared__ int fsm[];  // [P] keys (page id, -1 empty), [P] dense slot, [kd] retired flags
    int* tk = fsm;
    int* tj = fsm + P;
    int* gone = fsm + 2 * P;
    const long long r = blockIdx.x;
    const uint32_t mask = static_cast<uint32_t>(P - 1);
    for (int i = threadIdx.x; i < P; i += blockDim.x) tk[i] = -1;
    for (int j = threadIdx.x; j < kd; j += blockDim.x) gone[j] = 0;
    __syncthreads();
    const long long* di = dense_ids + r * kd;
    for (int j = threadIdx.x; j < kd; j += blockDim.x) {
        const long long id = di[j];
        if (id < 0 || id > 0x7fffffffll) continue;
        const int key = static_cast<int>(id);
        for (uint32_t h = rgroup_hash(static_cast<uint32_t>(key)) & mask;; h = (h + 1) & mask) {
            const int prev = atomicCAS(tk + h, -1, key);
            if (prev == -1) { tj[h] = j; break; }
            if (prev == key) break;  // a repeated dense id keeps its first slot
        }
    }
    __syncthreads();
    const long long off = __ldg(hit_offsets + r);
    const long long len = __ldg(hit_offsets + r + 1) - off;
    const long long n = min(len, width - kd);
    if (len > n && threadIdx.x == 0) atomicOr(status, 1);
    float* os = out_scores + r * width;
    long long* oi = out_ids + r * width;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int p = __ldg(hit_ids + off + i);
        int j = -1;
        for (uint32_t h = rgroup_hash(static_cast<uint32_t>(p)) & mask;; h = (h + 1) & mask) {
            const int key = tk[h];
            if (key == -1) break;
            if (key == p) { j = tj[h]; break; }
        }
        if (j >= 0) gone[j] = 1;
        float s;
        if (rrf) s = __fadd_rn(j >= 0 ? rrf_term(c, j + 1) : 0.f, rrf_term(c, i + 1));
        else s = fuse_sum(__ldg(hit_dense + r * hit_pitch + i), w, __ldg(hit_values + off + i));
        os[kd + i] = s;
        oi[kd + i] = p;
    }
    __syncthreads();
    const float* ds = dense_scores + r * kd;
    for (int j = threadIdx.x; j < kd; j += blockDim.x) {
        const long long id = di[j];
        const bool live = id >= 0 && !gone[j];
        os[j] = live ? (rrf ? rrf_term(c, j + 1) : ds[j]) : -INFINITY;
        oi[j] = live ? id : -1;
    }
    for (long long t = kd + n + threadIdx.x; t < width; t += blockDim.x) {
        os[t] = -INFINITY;
        oi[t] = -1;
    }
}

}  // namespace vr

using namespace vr;

extern "C" int vr_score_ranges(int32_t nq, int64_t nd) { return score_ranges_for(nq, nd); }
extern "C" int vr_score_plan(int32_t nq, int64_t nd, int32_t* out6) {
    VR_REQUIRE(out6 && nq > 0 && nd > 0, "vr_score_plan: bad arguments");
    const ScorePlan p = score_plan(nq, nd);
    out6[0] = p.T; out6[1] = p.R; out6[2] = p.QB; out6[3] = p.items; out6[4] = p.pairs; out6[5] = p.lists;
    return 0;
}
extern "C" int vr_score_list_len(void) { return SC_KT; }

extern "C" int vr_f32_to_f16_rows(const float* src, int64_t rows, int32_t dim, void* dst_f16, float* norms, float* max_norm,
                                  void* stream) {
    VR_REQUIRE(src && dst_f16, "vr_f32_to_f16_rows: null pointer");
    VR_REQUIRE(rows > 0 && dim > 0 && dim % 4 == 0, "vr_f32_to_f16_rows: bad shape rows=%lld dim=%d", (long long)rows, dim);
    VR_REQUIRE_ALIGNED("vr_f32_to_f16_rows", "src", src, 16);  // float4 loads, 8-byte stores
    VR_REQUIRE_ALIGNED("vr_f32_to_f16_rows", "dst_f16", dst_f16, 8);
    long long blocks = (rows + 7) / 8;
    const long long cap = static_cast<long long>(num_sms()) * 16;
    if (blocks > cap) blocks = cap;
    f32_to_f16_rows_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        src, rows, dim, reinterpret_cast<__half*>(dst_f16), norms, max_norm);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_score_filter(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                               float* cand_scores, int32_t* cand_ids, void* stream) {
    return score_filter("vr_score_filter", q_f16, nq, d_f16, nd, dim, ranges, nullptr, cand_scores, cand_ids, stream);
}

extern "C" int vr_score_filter_masked(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim,
                                      int32_t ranges, float* cand_scores, int32_t* cand_ids, const uint32_t* doc_mask,
                                      void* stream) {
    VR_REQUIRE(mask_ok(doc_mask), "vr_score_filter_masked: doc_mask must be a non-null, 4-byte aligned pointer");
    const DocMasks m = one_mask(doc_mask, nd);
    return score_filter("vr_score_filter", q_f16, nq, d_f16, nd, dim, ranges, &m, cand_scores, cand_ids, stream);
}

extern "C" int vr_score_filter_masks(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim,
                                     int32_t ranges, float* cand_scores, int32_t* cand_ids, const vr_doc_masks* masks,
                                     void* stream) {
    VR_REQUIRE_MASKS("vr_score_filter_masks", masks, nd);
    const DocMasks m = device_masks(masks);
    return score_filter("vr_score_filter_masks", q_f16, nq, d_f16, nd, dim, ranges, &m, cand_scores, cand_ids, stream);
}

extern "C" int vr_score_rescore(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, int32_t ranges,
                                const float* cand_scores, const int32_t* cand_ids, const float* max_doc_norm, int32_t k,
                                int64_t id_offset, float* out_scores, int64_t* out_ids, int32_t* flags, void* stream) {
    VR_REQUIRE(q_f32 && d_f32 && cand_scores && cand_ids && max_doc_norm && out_scores && out_ids && flags,
               "vr_score_rescore: null pointer");
    VR_REQUIRE(nq > 0 && k > 0 && dim % 4 == 0, "vr_score_rescore: bad shape");
    VR_REQUIRE_ALIGNED("vr_score_rescore", "d_f32", d_f32, 16);  // float4 rows (dim % 4 == 0 keeps every row aligned)
    const int lists = ranges * 2;
    VR_REQUIRE(ranges > 0 && lists <= SC_MAX_RANGES + 2, "vr_score_rescore: ranges must come from vr_score_ranges()");
    const int keep = rescore_keep(k, lists);
    const size_t smem = (static_cast<size_t>(dim) + 2 * static_cast<size_t>(keep)) * sizeof(float);
    VR_REQUIRE(smem <= 200 * 1024, "vr_score_rescore: dim too large for shared memory (%zu bytes)", smem);
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(rescore_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    rescore_topk_kernel<<<nq, RS_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
        q_f32, d_f32, nd, dim, lists, keep, cand_scores, cand_ids, max_doc_norm, k, id_offset, out_scores,
        reinterpret_cast<long long*>(out_ids), flags);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_score_exact(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, float* scores,
                              void* stream) {
    VR_REQUIRE(q_f32 && d_f32 && scores, "vr_score_exact: null pointer");
    VR_REQUIRE(nq > 0 && nd > 0 && dim % 4 == 0, "vr_score_exact: bad shape");
    VR_REQUIRE_ALIGNED("vr_score_exact", "d_f32", d_f32, 16);
    const int NQ = nq >= EX_QB ? EX_QB : (nq >= 4 ? 4 : (nq >= 2 ? 2 : 1));
    const size_t smem = static_cast<size_t>(NQ) * dim * sizeof(float);
    VR_REQUIRE(smem <= 200 * 1024, "vr_score_exact: dim too large");
    long long bx = (nd + 8 * EX_DW - 1) / (8 * EX_DW);
    const long long cap = static_cast<long long>(num_sms()) * 3;
    if (bx > cap) bx = cap;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // grid.y is one query block of NQ; past 65535 blocks the queries go in several launches (a query's scores do not
    // depend on which launch, or which block, computes them)
    const int chunk = 65535 * NQ;
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        const int n = nq - q0 < chunk ? nq - q0 : chunk;
        const float* q = q_f32 + static_cast<long long>(q0) * dim;
        float* out = scores + static_cast<long long>(q0) * nd;
        dim3 grid(static_cast<unsigned>(bx), (n + NQ - 1) / NQ);
#define VR_EXACT_LAUNCH(N)                                                                                               \
    do {                                                                                                                 \
        static unsigned long long attr_set = 0;                                                                          \
        if (smem > 48 * 1024 && first_use_on_device(&attr_set))                                                          \
            VR_CHECK_CUDA(cudaFuncSetAttribute(exact_scores_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
        exact_scores_kernel<N><<<grid, 256, smem, st>>>(q, n, d_f32, nd, dim, out);                                      \
    } while (0)
        if (NQ == EX_QB) VR_EXACT_LAUNCH(EX_QB);
        else if (NQ == 4) VR_EXACT_LAUNCH(4);
        else if (NQ == 2) VR_EXACT_LAUNCH(2);
        else VR_EXACT_LAUNCH(1);
#undef VR_EXACT_LAUNCH
        VR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

extern "C" int vr_topk_rows(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                            float* out_scores, int64_t* out_ids, void* stream) {
    return topk_rows("vr_topk_rows", scores, ids, rows, cols, k, id_offset, out_scores, out_ids, nullptr, stream);
}

extern "C" int vr_topk_rows_masked(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k,
                                   int64_t id_offset, float* out_scores, int64_t* out_ids, const uint32_t* doc_mask,
                                   void* stream) {
    VR_REQUIRE(mask_ok(doc_mask), "vr_topk_rows_masked: doc_mask must be a non-null, 4-byte aligned pointer");
    VR_REQUIRE(!ids, "vr_topk_rows_masked: the mask indexes columns, so ids must be NULL");
    const DocMasks m = one_mask(doc_mask, cols);
    return topk_rows("vr_topk_rows_masked", scores, ids, rows, cols, k, id_offset, out_scores, out_ids, &m, stream);
}

extern "C" int vr_topk_rows_masks(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k,
                                  int64_t id_offset, float* out_scores, int64_t* out_ids, const vr_doc_masks* masks,
                                  void* stream) {
    VR_REQUIRE_MASKS("vr_topk_rows_masks", masks, cols);
    VR_REQUIRE(!ids, "vr_topk_rows_masks: the masks index columns, so ids must be NULL");
    const DocMasks m = device_masks(masks);
    return topk_rows("vr_topk_rows_masks", scores, ids, rows, cols, k, id_offset, out_scores, out_ids, &m, stream);
}

extern "C" int vr_topk_rows_chunked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                    int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                                    int64_t* out_ids, void* stream) {
    return topk_rows_chunked("vr_topk_rows_chunked", scores, rows, cols, k, id_offset, chunks, ws_scores, ws_ids, out_scores,
                             out_ids, nullptr, stream);
}

extern "C" int vr_topk_rows_chunked_masked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                           int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                                           int64_t* out_ids, const uint32_t* doc_mask, void* stream) {
    VR_REQUIRE(mask_ok(doc_mask), "vr_topk_rows_chunked_masked: doc_mask must be a non-null, 4-byte aligned pointer");
    const DocMasks m = one_mask(doc_mask, cols);
    return topk_rows_chunked("vr_topk_rows_chunked_masked", scores, rows, cols, k, id_offset, chunks, ws_scores, ws_ids,
                             out_scores, out_ids, &m, stream);
}

extern "C" int vr_topk_rows_chunked_masks(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                          int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                                          int64_t* out_ids, const vr_doc_masks* masks, void* stream) {
    VR_REQUIRE_MASKS("vr_topk_rows_chunked_masks", masks, cols);
    const DocMasks m = device_masks(masks);
    return topk_rows_chunked("vr_topk_rows_chunked_masks", scores, rows, cols, k, id_offset, chunks, ws_scores, ws_ids,
                             out_scores, out_ids, &m, stream);
}

// ---------------------------------------------------------------------------------------------- document-level top-k
// A group table as the _groups entry points take it: 4-byte aligned int32 arrays, G >= 1, nd within the int32 ids.
static bool i32_ok(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

// The mask of a _groups call: the set of a _masks entry point (checked here, so that the refusals keep the order of the
// other arguments' checks), else the optional single doc_mask of the plain entry point.
static int group_masks(const char* fn, const uint32_t* doc_mask, const vr_doc_masks* set, long long nd, DocMasks* out,
                       bool* masked) {
    if (set) {
        VR_REQUIRE_MASKS(fn, set, nd);
        *out = device_masks(set);
    } else {
        VR_REQUIRE(!doc_mask || mask_ok(doc_mask), "%s: doc_mask must be NULL or 4-byte aligned", fn);
        *out = doc_mask ? one_mask(doc_mask, nd) : kNoMasks;
    }
    *masked = set || doc_mask;
    return 0;
}

// vr_score_filter_groups(_masks)
static int score_filter_groups(const char* fn, const void* q_f16, int nq, const void* d_f16, long long nd, int dim,
                               int ranges, float* cand_scores, int* cand_ids, const int* doc_groups, const uint32_t* doc_mask,
                               const vr_doc_masks* set, void* stream) {
    VR_REQUIRE(i32_ok(doc_groups), "%s: doc_groups must be a non-null, 4-byte aligned pointer", fn);
    DocMasks masks;
    bool masked;
    if (int rc = group_masks(fn, doc_mask, set, nd, &masks, &masked)) return rc;
    VR_REQUIRE(q_f16 && d_f16 && cand_scores && cand_ids, "%s: null pointer", fn);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(nq > 0 && nq < (1 << 30) && dim % 8 == 0, "%s: bad shape", fn);
    const ScorePlan plan = score_plan(nq, nd);
    VR_REQUIRE(ranges * 2 == plan.lists, "%s: ranges must come from vr_score_ranges()", fn);
    VR_REQUIRE_ALIGNED(fn, "q_f16", q_f16, 16);
    VR_REQUIRE_ALIGNED(fn, "d_f16", d_f16, 16);
    VR_REQUIRE_ALIGNED(fn, "cand_scores", cand_scores, 16);
    VR_REQUIRE_ALIGNED(fn, "cand_ids", cand_ids, 16);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (masked)
        return launch_score_filter<MaskedGroupedScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, cand_scores, cand_ids, masks,
                                                           doc_groups, st);
    return launch_score_filter<GroupedScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, cand_scores, cand_ids, kNoMasks, doc_groups, st);
}

extern "C" int vr_score_filter_groups(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim,
                                      int32_t ranges, float* cand_scores, int32_t* cand_ids, const int32_t* doc_groups,
                                      const uint32_t* doc_mask, void* stream) {
    return score_filter_groups("vr_score_filter_groups", q_f16, nq, d_f16, nd, dim, ranges, cand_scores, cand_ids, doc_groups,
                               doc_mask, nullptr, stream);
}

extern "C" int vr_score_filter_groups_masks(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim,
                                            int32_t ranges, float* cand_scores, int32_t* cand_ids, const int32_t* doc_groups,
                                            const vr_doc_masks* masks, void* stream) {
    VR_REQUIRE(masks, "vr_score_filter_groups_masks: masks must not be NULL");
    return score_filter_groups("vr_score_filter_groups_masks", q_f16, nq, d_f16, nd, dim, ranges, cand_scores, cand_ids,
                               doc_groups, nullptr, masks, stream);
}

// vr_score_rescore_groups(_masks)
static int score_rescore_groups(const char* fn, const float* q_f32, int nq, const float* d_f32, long long nd, int dim,
                                int ranges, const float* cand_scores, const int* cand_ids, const int* doc_groups,
                                const int* group_offsets, const int* group_pages, int G, const uint32_t* doc_mask,
                                const vr_doc_masks* set, const float* max_doc_norm, int k, long long id_offset,
                                float* out_scores, int64_t* out_pages, int64_t* out_groups, int* flags, void* stream) {
    VR_REQUIRE(i32_ok(doc_groups) && i32_ok(group_offsets) && i32_ok(group_pages),
               "%s: doc_groups, group_offsets and group_pages must be non-null, 4-byte aligned pointers", fn);
    DocMasks masks;
    bool masked;
    if (int rc = group_masks(fn, doc_mask, set, nd, &masks, &masked)) return rc;
    VR_REQUIRE(G > 0, "%s: G=%d, needs at least one group", fn, G);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(q_f32 && d_f32 && cand_scores && cand_ids && max_doc_norm && out_scores && out_pages && out_groups && flags,
               "%s: null pointer", fn);
    VR_REQUIRE(nq > 0 && k > 0 && dim % 4 == 0, "%s: bad shape", fn);
    VR_REQUIRE_ALIGNED(fn, "d_f32", d_f32, 16);
    const int lists = ranges * 2;
    VR_REQUIRE(ranges > 0 && lists <= SC_MAX_RANGES + 2, "%s: ranges must come from vr_score_ranges()", fn);
    const int keep = rescore_keep(k, lists);
    const size_t smem = (static_cast<size_t>(dim) + 2 * RG_PAGE_BUDGET + 7 * static_cast<size_t>(keep) + 1) * sizeof(float);
    VR_REQUIRE(smem <= 200 * 1024, "%s: dim too large for shared memory (%zu bytes)", fn, smem);
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(rescore_groups_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    rescore_groups_kernel<<<nq, RS_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
        q_f32, d_f32, dim, lists, keep, cand_scores, cand_ids, doc_groups, group_offsets, group_pages, masks, max_doc_norm,
        k, id_offset, out_scores, reinterpret_cast<long long*>(out_pages), reinterpret_cast<long long*>(out_groups), flags);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_score_rescore_groups(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                                       int32_t ranges, const float* cand_scores, const int32_t* cand_ids,
                                       const int32_t* doc_groups, const int32_t* group_offsets, const int32_t* group_pages,
                                       int32_t G, const uint32_t* doc_mask, const float* max_doc_norm, int32_t k,
                                       int64_t id_offset, float* out_scores, int64_t* out_pages, int64_t* out_groups,
                                       int32_t* flags, void* stream) {
    return score_rescore_groups("vr_score_rescore_groups", q_f32, nq, d_f32, nd, dim, ranges, cand_scores, cand_ids,
                                doc_groups, group_offsets, group_pages, G, doc_mask, nullptr, max_doc_norm, k, id_offset,
                                out_scores, out_pages, out_groups, flags, stream);
}

extern "C" int vr_score_rescore_groups_masks(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                                             int32_t ranges, const float* cand_scores, const int32_t* cand_ids,
                                             const int32_t* doc_groups, const int32_t* group_offsets,
                                             const int32_t* group_pages, int32_t G, const vr_doc_masks* masks,
                                             const float* max_doc_norm, int32_t k, int64_t id_offset, float* out_scores,
                                             int64_t* out_pages, int64_t* out_groups, int32_t* flags, void* stream) {
    VR_REQUIRE(masks, "vr_score_rescore_groups_masks: masks must not be NULL");
    return score_rescore_groups("vr_score_rescore_groups_masks", q_f32, nq, d_f32, nd, dim, ranges, cand_scores, cand_ids,
                                doc_groups, group_offsets, group_pages, G, nullptr, masks, max_doc_norm, k, id_offset,
                                out_scores, out_pages, out_groups, flags, stream);
}

// workspace of vr_group_topk_rows: best pages [rows, G] i64, group scores [rows, G] f32, and with chunks >= 2 the first
// pass's lists [rows, chunks, k] (i64 ids, f32 scores)
static long long group_topk_ws(int rows, int G, int k, int chunks) {
    const long long n = static_cast<long long>(rows) * G, w = chunks >= 2 ? static_cast<long long>(rows) * chunks * k : 0;
    return ((n * 12 + 15) / 16) * 16 + w * 12;
}

extern "C" int64_t vr_group_topk_ws_bytes(int32_t rows, int32_t G, int32_t k, int32_t chunks) {
    return rows > 0 && G > 0 && k > 0 ? group_topk_ws(rows, G, k, chunks) : -1;
}

static int select_rows(const char* fn, const float* scores, const int64_t* ids, int rows, long long cols, int k,
                       long long id_offset, int chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                       int64_t* out_ids, const DocMasks* masks, void* stream);

// vr_group_topk_rows(_masks)
static int group_topk_rows(const char* fn, const float* scores, int rows, long long nd, const int* doc_groups, int G,
                           const uint32_t* doc_mask, const vr_doc_masks* set, int k, long long id_offset, int chunks, void* ws,
                           long long ws_bytes, float* out_scores, int64_t* out_pages, int64_t* out_groups, void* stream) {
    VR_REQUIRE(i32_ok(doc_groups), "%s: doc_groups must be a non-null, 4-byte aligned pointer", fn);
    DocMasks masks;
    bool masked;
    if (int rc = group_masks(fn, doc_mask, set, nd, &masks, &masked)) return rc;
    VR_REQUIRE(G > 0, "%s: G=%d, needs at least one group", fn, G);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(scores && out_scores && out_pages && out_groups, "%s: null pointer", fn);
    VR_REQUIRE(rows > 0 && k > 0 && chunks >= 0 && chunks <= 65535, "%s: bad shape", fn);
    VR_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0 && ws_bytes >= group_topk_ws(rows, G, k, chunks),
               "%s: workspace too small or misaligned (%lld bytes, need %lld, 16-byte aligned)", fn,
               (long long)ws_bytes, group_topk_ws(rows, G, k, chunks));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long n = static_cast<long long>(rows) * G;
    long long* gpages = reinterpret_cast<long long*>(ws);
    float* gscores = reinterpret_cast<float*>(gpages + n);
    VR_CHECK_CUDA(cudaMemsetAsync(gpages, 0, n * sizeof(long long), st));  // keys: 0 = no page yet
    const long long runs = static_cast<long long>(rows) * ((nd + GK_RUN - 1) / GK_RUN);
    long long blocks = (runs + 255) / 256;
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    group_key_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(scores, rows, nd, G, doc_groups, masks,
                                                               reinterpret_cast<unsigned long long*>(gpages));
    VR_CHECK_CUDA(cudaGetLastError());
    blocks = (n + 255) / 256;
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    group_decode_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(scores, rows, nd, G, gpages, gscores);
    VR_CHECK_CUDA(cudaGetLastError());
    long long* op = reinterpret_cast<long long*>(out_pages);
    long long* ws_i = reinterpret_cast<long long*>(reinterpret_cast<char*>(ws) + ((n * 12 + 15) / 16) * 16);
    float* ws_s = reinterpret_cast<float*>(ws_i + static_cast<long long>(rows) * chunks * k);
    if (k > SEL_K_MIN && k <= SEL_MAX_K) {  // the radix select over the group rows, with the best pages as ids (same bits)
        if (int rc = select_rows(fn, gscores, reinterpret_cast<const int64_t*>(gpages), rows, G, k, id_offset,
                                 chunks >= 2 ? chunks : 1, ws_s, reinterpret_cast<int64_t*>(ws_i), out_scores, out_pages,
                                 nullptr, stream))
            return rc;
    } else if (chunks >= 2) {  // few rows x many groups: spread each row over `chunks` blocks, then merge their lists
        topk_rows_kernel<false><<<dim3(rows, chunks), 256, 0, st>>>(gscores, gpages, G, k, id_offset, (G + chunks - 1) / chunks,
                                                                    ws_s, ws_i, kNoMasks);
        VR_CHECK_CUDA(cudaGetLastError());
        launch_topk_rows<false>(ws_s, ws_i, rows, static_cast<long long>(chunks) * k, k, 0, out_scores, op, kNoMasks, st);
    } else {
        launch_topk_rows<false>(gscores, gpages, rows, G, k, id_offset, out_scores, op, kNoMasks, st);
    }
    VR_CHECK_CUDA(cudaGetLastError());
    const long long m = static_cast<long long>(rows) * k;
    page_groups_kernel<<<static_cast<int>((m + 255) / 256 < 4096 ? (m + 255) / 256 : 4096), 256, 0, st>>>(
        op, m, id_offset, doc_groups, reinterpret_cast<long long*>(out_groups));
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}


extern "C" int vr_group_topk_rows(const float* scores, int32_t rows, int64_t nd, const int32_t* doc_groups, int32_t G,
                                  const uint32_t* doc_mask, int32_t k, int64_t id_offset, int32_t chunks, void* ws,
                                  int64_t ws_bytes, float* out_scores, int64_t* out_pages, int64_t* out_groups,
                                  void* stream) {
    return group_topk_rows("vr_group_topk_rows", scores, rows, nd, doc_groups, G, doc_mask, nullptr, k, id_offset, chunks, ws,
                           ws_bytes, out_scores, out_pages, out_groups, stream);
}

extern "C" int vr_group_topk_rows_masks(const float* scores, int32_t rows, int64_t nd, const int32_t* doc_groups, int32_t G,
                                        const vr_doc_masks* masks, int32_t k, int64_t id_offset, int32_t chunks, void* ws,
                                        int64_t ws_bytes, float* out_scores, int64_t* out_pages, int64_t* out_groups,
                                        void* stream) {
    VR_REQUIRE(masks, "vr_group_topk_rows_masks: masks must not be NULL");
    return group_topk_rows("vr_group_topk_rows_masks", scores, rows, nd, doc_groups, G, nullptr, masks, k, id_offset, chunks,
                           ws, ws_bytes, out_scores, out_pages, out_groups, stream);
}

extern "C" int vr_merge_group_topk(const float* scores, const int64_t* pages, const int64_t* groups, int32_t rows,
                                   int32_t cols, int32_t k, float* out_scores, int64_t* out_pages, int64_t* out_groups,
                                   void* stream) {
    VR_REQUIRE(scores && pages && groups && out_scores && out_pages && out_groups, "vr_merge_group_topk: null pointer");
    VR_REQUIRE(rows > 0 && cols > 0 && cols <= 512 && k > 0, "vr_merge_group_topk: bad shape (rows=%d, cols=%d <= 512, k=%d)",
               rows, cols, k);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long* p = reinterpret_cast<const long long*>(pages);
    const long long* g = reinterpret_cast<const long long*>(groups);
    long long* op = reinterpret_cast<long long*>(out_pages);
    long long* og = reinterpret_cast<long long*>(out_groups);
    if (cols <= 128)
        merge_groups_warp_kernel<4><<<(rows + 7) / 8, 256, 0, st>>>(scores, p, g, rows, cols, k, out_scores, op, og);
    else
        merge_groups_warp_kernel<16><<<(rows + 7) / 8, 256, 0, st>>>(scores, p, g, rows, cols, k, out_scores, op, og);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------- candidate lists
// A list set as vr_score_lists takes it, refused before any CUDA call unless its arrays can be read. The offsets, the ids
// and the values of of_query lie in device memory: the caller keeps them consistent (ids outside [0, nd) are skipped,
// an of_query value outside [0, count) and a list longer than width are reported in *status).
static int lists_check(const char* fn, const vr_doc_lists* l) {
    VR_REQUIRE(l, "%s: lists must not be NULL", fn);
    VR_REQUIRE(l->offsets, "%s: lists->offsets must not be NULL", fn);
    VR_REQUIRE(l->ids, "%s: lists->ids must not be NULL", fn);
    VR_REQUIRE_ALIGNED(fn, "lists->offsets", l->offsets, 8);
    VR_REQUIRE_ALIGNED(fn, "lists->ids", l->ids, 4);
    VR_REQUIRE(l->count >= 1, "%s: lists->count=%d, needs at least one list", fn, l->count);
    VR_REQUIRE(l->count == 1 || l->of_query, "%s: lists->of_query is NULL with lists->count=%d lists", fn, l->count);
    VR_REQUIRE_ALIGNED(fn, "lists->of_query", l->of_query, 4);
    return 0;
}

extern "C" int vr_score_lists(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                              const vr_doc_lists* lists, int32_t width, const int32_t* doc_groups, float* out_scores,
                              int64_t* out_ids, int64_t* out_groups, int32_t* status, void* stream) {
    const char* fn = "vr_score_lists";
    if (int rc = lists_check(fn, lists)) return rc;
    VR_REQUIRE(q_f32 && d_f32 && out_scores && out_ids && status, "%s: null pointer", fn);
    VR_REQUIRE(!doc_groups == !out_groups, "%s: doc_groups and out_groups go together (both or neither)", fn);
    VR_REQUIRE(width >= 1, "%s: width=%d, needs at least 1", fn, width);
    VR_REQUIRE(nq > 0 && dim > 0 && dim % 4 == 0, "%s: bad shape nq=%d dim=%d (dim %% 4 == 0)", fn, nq, dim);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE_ALIGNED(fn, "q_f32", q_f32, 4);
    VR_REQUIRE_ALIGNED(fn, "d_f32", d_f32, 16);  // float4 rows (dim % 4 == 0 keeps every row aligned)
    VR_REQUIRE_ALIGNED(fn, "doc_groups", doc_groups, 4);
    VR_REQUIRE_ALIGNED(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_ALIGNED(fn, "out_ids", out_ids, 8);
    VR_REQUIRE_ALIGNED(fn, "out_groups", out_groups, 8);
    VR_REQUIRE_ALIGNED(fn, "status", status, 4);
    // rows per tile: runs of rows sharing a list can only form when some list serves several rows
    const bool shared = !lists->of_query || lists->count < nq;
    const int NQ = !shared ? 1 : nq >= EX_QB ? EX_QB : (nq >= 4 ? 4 : (nq >= 2 ? 2 : 1));
    const size_t smem = static_cast<size_t>(NQ) * dim * sizeof(float);
    VR_REQUIRE(smem <= 200 * 1024, "%s: dim too large", fn);
    // list positions per block: about four blocks per SM over the whole block, whole warps of EX_DW, <= 65535 chunks
    const long long tiles = (nq + NQ - 1) / NQ;
    long long chunk = static_cast<long long>(width) * tiles / (4ll * num_sms());
    if (chunk > 2048) chunk = 2048;
    if (chunk < (width + 65534ll) / 65535) chunk = (width + 65534ll) / 65535;
    chunk = (chunk + 8 * EX_DW - 1) / (8 * EX_DW) * (8 * EX_DW);
    if (chunk < 8 * EX_DW) chunk = 8 * EX_DW;
    const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>((width + chunk - 1) / chunk));
    const DocLists dl = {reinterpret_cast<const long long*>(lists->offsets), lists->ids, lists->count, lists->of_query};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    long long* oi = reinterpret_cast<long long*>(out_ids);
    long long* og = reinterpret_cast<long long*>(out_groups);
#define VR_LISTS_LAUNCH(N)                                                                                              \
    do {                                                                                                                \
        static unsigned long long attr_set = 0;                                                                         \
        if (smem > 48 * 1024 && first_use_on_device(&attr_set))                                                         \
            VR_CHECK_CUDA(cudaFuncSetAttribute(list_scores_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
        list_scores_kernel<N><<<grid, 256, smem, st>>>(q_f32, nq, d_f32, nd, dim, dl, width, static_cast<int>(chunk),      \
                                                       doc_groups, out_scores, oi, og, status);                         \
    } while (0)
    if (NQ == EX_QB) VR_LISTS_LAUNCH(EX_QB);
    else if (NQ == 4) VR_LISTS_LAUNCH(4);
    else if (NQ == 2) VR_LISTS_LAUNCH(2);
    else VR_LISTS_LAUNCH(1);
#undef VR_LISTS_LAUNCH
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------- range search
#define VR_REQUIRE_PTR(fn, name, ptr, bytes)                             \
    do {                                                                 \
        VR_REQUIRE((ptr), "%s: %s must not be NULL", fn, name);          \
        VR_REQUIRE_ALIGNED(fn, name, ptr, bytes);                        \
    } while (0)

extern "C" int vr_score_filter_range(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim,
                                     const float* thresholds, const float* q_norms, const float* max_doc_norm,
                                     const vr_doc_masks* masks, int32_t cap, int32_t* counts, int32_t* cand_ids,
                                     void* stream) {
    const char* fn = "vr_score_filter_range";
    if (masks) VR_REQUIRE_MASKS(fn, masks, nd);
    VR_REQUIRE_PTR(fn, "q_f16", q_f16, 16);  // TMA sources
    VR_REQUIRE_PTR(fn, "d_f16", d_f16, 16);
    VR_REQUIRE_PTR(fn, "thresholds", thresholds, 4);
    VR_REQUIRE_PTR(fn, "q_norms", q_norms, 4);
    VR_REQUIRE_PTR(fn, "max_doc_norm", max_doc_norm, 4);
    VR_REQUIRE_PTR(fn, "counts", counts, 4);
    VR_REQUIRE_PTR(fn, "cand_ids", cand_ids, 4);
    VR_REQUIRE(nq > 0 && nq < (1 << 30), "%s: nq=%d, needs 0 < nq < 2^30", fn, nq);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(dim > 0 && dim % 8 == 0, "%s: dim=%d, needs a positive multiple of 8", fn, dim);
    VR_REQUIRE(cap >= 1, "%s: cap=%d, needs at least 1", fn, cap);
    const ScorePlan plan = score_plan(nq, nd);
    const RangeFields rf = {thresholds, q_norms, max_doc_norm, cap, counts, cand_ids};
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (masks)
        return launch_score_filter<MaskedRangeScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, nullptr, nullptr,
                                                         device_masks(masks), nullptr, st, &rf);
    return launch_score_filter<RangeScoreArgs>(plan, q_f16, nq, d_f16, nd, dim, nullptr, nullptr, kNoMasks, nullptr, st, &rf);
}

extern "C" int vr_score_rescore_range(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                                      const float* thresholds, int32_t cap, const int32_t* counts, const int32_t* cand_ids,
                                      float* out_scores, int32_t* out_ids, int32_t* kept, void* stream) {
    const char* fn = "vr_score_rescore_range";
    VR_REQUIRE_PTR(fn, "q_f32", q_f32, 4);
    VR_REQUIRE_PTR(fn, "d_f32", d_f32, 16);  // float4 rows (dim % 4 == 0 keeps every row aligned)
    VR_REQUIRE_PTR(fn, "thresholds", thresholds, 4);
    VR_REQUIRE_PTR(fn, "counts", counts, 4);
    VR_REQUIRE_PTR(fn, "cand_ids", cand_ids, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 4);
    VR_REQUIRE_PTR(fn, "kept", kept, 4);
    VR_REQUIRE(nq > 0, "%s: nq=%d, needs at least 1", fn, nq);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(dim > 0 && dim % 4 == 0, "%s: dim=%d, needs a positive multiple of 4", fn, dim);
    VR_REQUIRE(cap >= 1, "%s: cap=%d, needs at least 1", fn, cap);
    const size_t smem = static_cast<size_t>(dim) * sizeof(float);
    VR_REQUIRE(smem <= 200 * 1024, "%s: dim=%d too large for shared memory", fn, dim);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    VR_CHECK_CUDA(cudaMemsetAsync(kept, 0, static_cast<size_t>(nq) * sizeof(int), st));
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(range_rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    // candidate blocks per row: about four blocks per SM over the whole call, no more than a row's slots need
    long long gy = (4ll * num_sms() + nq - 1) / nq;
    const long long most = (cap + RR_THREADS / 32 - 1) / (RR_THREADS / 32);
    if (gy > most) gy = most;
    if (gy > 65535) gy = 65535;
    range_rescore_kernel<<<dim3(nq, static_cast<unsigned>(gy)), RR_THREADS, smem, st>>>(q_f32, d_f32, dim, thresholds, cap,
                                                                                      counts, cand_ids, out_scores, out_ids, kept);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_range_rows(const float* scores, int32_t rows, int64_t nd, const float* thresholds, const vr_doc_masks* masks,
                             int64_t pitch, float* out_scores, int32_t* out_ids, int32_t* counts, void* stream) {
    const char* fn = "vr_range_rows";
    if (masks) VR_REQUIRE_MASKS(fn, masks, nd);
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "thresholds", thresholds, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 4);
    VR_REQUIRE_PTR(fn, "counts", counts, 4);
    VR_REQUIRE(rows > 0 && rows <= 65535, "%s: rows=%d, needs 0 < rows <= 65535", fn, rows);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(pitch >= nd, "%s: pitch=%lld is below nd=%lld", fn, (long long)pitch, (long long)nd);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    VR_CHECK_CUDA(cudaMemsetAsync(counts, 0, static_cast<size_t>(rows) * sizeof(int), st));
    long long gx = (nd + 255) / 256;
    const long long want = (8ll * num_sms() + rows - 1) / rows;
    if (gx > want) gx = want;
    const DocMasks m = masks ? device_masks(masks) : kNoMasks;
    range_select_kernel<<<dim3(static_cast<unsigned>(gx), rows), 256, 0, st>>>(scores, nd, thresholds, m, pitch, out_scores,
                                                                             out_ids, counts);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int64_t vr_range_sort_ws_bytes(int32_t rows, int32_t max_count) {
    return rows > 0 && max_count >= 0 ? range_sort_ws(rows, max_count) : -1;
}

extern "C" int vr_range_sort(const float* scores, const int32_t* ids, int64_t pitch, const int32_t* counts, int32_t rows,
                             const int32_t* row_of, const int64_t* out_offsets, int32_t max_count, int64_t id_offset, void* ws,
                             int64_t ws_bytes, float* out_scores, int64_t* out_ids, void* stream) {
    const char* fn = "vr_range_sort";
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "ids", ids, 4);
    VR_REQUIRE_PTR(fn, "counts", counts, 4);
    VR_REQUIRE_ALIGNED(fn, "row_of", row_of, 4);  // optional
    VR_REQUIRE_PTR(fn, "out_offsets", out_offsets, 8);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    VR_REQUIRE(rows > 0 && rows <= 65535, "%s: rows=%d, needs 0 < rows <= 65535", fn, rows);
    VR_REQUIRE(max_count >= 0 && max_count <= pitch, "%s: max_count=%d, needs 0 <= max_count <= pitch=%lld", fn, max_count,
               (long long)pitch);
    const long long need = range_sort_ws(rows, max_count);
    VR_REQUIRE(need == 0 || (ws && ws_bytes >= need), "%s: ws of %lld bytes, needs %lld (vr_range_sort_ws_bytes)", fn,
               (long long)ws_bytes, need);
    VR_REQUIRE_ALIGNED(fn, "ws", ws, 8);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    long long* oi = reinterpret_cast<long long*>(out_ids);
    const long long* oo = reinterpret_cast<const long long*>(out_offsets);
    if (max_count == 0) return 0;
    if (need == 0) {
        range_sort_smem_kernel<<<rows, RSORT_THREADS, 0, st>>>(scores, ids, pitch, counts, row_of, oo, id_offset, out_scores, oi);
        VR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    const long long P = range_sort_P(max_count);
    unsigned long long* w = reinterpret_cast<unsigned long long*>(ws);
    long long gx = P / 256;
    const long long cap = (8ll * num_sms() + rows - 1) / rows;
    if (gx > cap) gx = cap;
    const dim3 grid(static_cast<unsigned>(gx), rows), tiles(static_cast<unsigned>(P / RSORT_TILE), rows);
    range_keys_kernel<<<grid, 256, 0, st>>>(scores, ids, pitch, counts, row_of, P, w);
    range_bitonic_tile_kernel<<<tiles, RSORT_THREADS, 0, st>>>(w, P, 2);
    for (long long k = 2 * RSORT_TILE; k <= P; k <<= 1) {
        for (long long j = k >> 1; j >= RSORT_TILE; j >>= 1) range_bitonic_global_kernel<<<grid, 256, 0, st>>>(w, P, k, j);
        range_bitonic_tile_kernel<<<tiles, RSORT_THREADS, 0, st>>>(w, P, k);
    }
    range_emit_kernel<<<grid, 256, 0, st>>>(w, P, counts, row_of, oo, id_offset, out_scores, oi);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int64_t vr_range_groups_ws_bytes(int32_t rows, int32_t max_count) {
    return rows > 0 && max_count >= 0 ? range_groups_ws(rows, max_count) : -1;
}

extern "C" int vr_range_groups(const float* scores, const int32_t* ids, int64_t pitch, const int32_t* counts, int32_t rows,
                               int32_t max_count, const int32_t* doc_groups, int64_t nd, int32_t G, void* ws, int64_t ws_bytes,
                               float* out_scores, int32_t* out_ids, int32_t* out_counts, void* stream) {
    const char* fn = "vr_range_groups";
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "ids", ids, 4);
    VR_REQUIRE_PTR(fn, "counts", counts, 4);
    VR_REQUIRE_PTR(fn, "doc_groups", doc_groups, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 4);
    VR_REQUIRE_PTR(fn, "out_counts", out_counts, 4);
    VR_REQUIRE(rows > 0 && rows <= 65535, "%s: rows=%d, needs 0 < rows <= 65535", fn, rows);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(G > 0, "%s: G=%d, needs at least one group", fn, G);
    VR_REQUIRE(max_count >= 0 && max_count <= pitch, "%s: max_count=%d, needs 0 <= max_count <= pitch=%lld", fn, max_count,
               (long long)pitch);
    const long long need = range_groups_ws(rows, max_count);
    VR_REQUIRE(need == 0 || (ws && ws_bytes >= need), "%s: ws of %lld bytes, needs %lld (vr_range_groups_ws_bytes)", fn,
               (long long)ws_bytes, need);
    VR_REQUIRE_ALIGNED(fn, "ws", ws, 8);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (need == 0) {
        const int P = static_cast<int>(range_groups_P(max_count));
        const size_t smem = static_cast<size_t>(P) * 12;
        static unsigned long long attr_set = 0;
        if (first_use_on_device(&attr_set))  // the static `emitted` counts too: set it whatever this call's size
            VR_CHECK_CUDA(cudaFuncSetAttribute(range_groups_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(range_groups_P(RGROUP_SMEM_MAX)) * 12));
        range_groups_smem_kernel<<<rows, RGROUP_THREADS, smem, st>>>(scores, ids, pitch, counts, max_count, nd, doc_groups, G,
                                                                     P, out_scores, out_ids, out_counts);
        VR_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    const long long P = range_groups_P(max_count), slots = static_cast<long long>(rows) * P;
    unsigned long long* w = reinterpret_cast<unsigned long long*>(ws);
    VR_CHECK_CUDA(cudaMemsetAsync(w, 0, slots * 8, st));            // keys: 0 = no entry
    VR_CHECK_CUDA(cudaMemsetAsync(w + slots, 0xff, slots * 4, st));  // groups: -1 = empty slot
    VR_CHECK_CUDA(cudaMemsetAsync(out_counts, 0, static_cast<size_t>(rows) * sizeof(int), st));
    long long gx = (max_count + 255) / 256;
    const long long want = (8ll * num_sms() + rows - 1) / rows;
    if (gx > want) gx = want;
    const dim3 grid(static_cast<unsigned>(gx), rows);
    range_groups_ws_kernel<true><<<grid, 256, 0, st>>>(scores, ids, pitch, counts, max_count, nd, doc_groups, G, P, w,
                                                       out_scores, out_ids, out_counts);
    range_groups_ws_kernel<false><<<grid, 256, 0, st>>>(scores, ids, pitch, counts, max_count, nd, doc_groups, G, P, w,
                                                        out_scores, out_ids, out_counts);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// vr_select_rows(_masks) and the chunked forms, after the mask checks: select_rows_kernel over (rows, chunks) blocks; with
// chunks >= 2 each block writes its chunk's list (ids = column + id_offset) and a second launch selects from the
// [rows, chunks * k] lists, as topk_rows_chunked does.
static int select_rows(const char* fn, const float* scores, const int64_t* ids, int rows, long long cols, int k,
                       long long id_offset, int chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                       int64_t* out_ids, const DocMasks* masks, void* stream) {
    VR_REQUIRE(scores && out_scores && out_ids, "%s: null pointer", fn);
    VR_REQUIRE(chunks < 2 || (ws_scores && ws_ids), "%s: null pointer", fn);
    VR_REQUIRE(rows > 0 && cols > 0 && cols < 2147483647ll && k > 0 && chunks > 0 && chunks <= 65535, "%s: bad shape", fn);
    VR_REQUIRE(k <= SEL_MAX_K, "%s: k=%d, needs k <= %d", fn, k, SEL_MAX_K);
    static unsigned long long attr_set = 0;
    if (first_use_on_device(&attr_set)) {
        VR_CHECK_CUDA(cudaFuncSetAttribute(select_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SEL_MAX_K * 16));
        VR_CHECK_CUDA(cudaFuncSetAttribute(select_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SEL_MAX_K * 16));
    }
    int P = 1;
    while (P < k) P <<= 1;
    const size_t smem = static_cast<size_t>(P) * 16;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const long long* i = reinterpret_cast<const long long*>(ids);
    const long long chunk_cols = (cols + chunks - 1) / chunks;
    float* os = chunks >= 2 ? ws_scores : out_scores;
    long long* oi = reinterpret_cast<long long*>(chunks >= 2 ? ws_ids : out_ids);
    if (masks)
        select_rows_kernel<true><<<dim3(rows, chunks), SEL_THREADS, smem, s>>>(scores, i, cols, k, id_offset, chunk_cols, os,
                                                                               oi, *masks);
    else
        select_rows_kernel<false><<<dim3(rows, chunks), SEL_THREADS, smem, s>>>(scores, i, cols, k, id_offset, chunk_cols, os,
                                                                                oi, kNoMasks);
    VR_CHECK_CUDA(cudaGetLastError());
    if (chunks >= 2) {
        select_rows_kernel<false><<<rows, SEL_THREADS, smem, s>>>(ws_scores, oi, static_cast<long long>(chunks) * k, k, 0,
                                                                  static_cast<long long>(chunks) * k, out_scores,
                                                                  reinterpret_cast<long long*>(out_ids), kNoMasks);
        VR_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

extern "C" int vr_select_rows(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k,
                              int64_t id_offset, float* out_scores, int64_t* out_ids, void* stream) {
    const char* fn = "vr_select_rows";
    VR_REQUIRE_ALIGNED(fn, "ids", ids, 8);  // optional
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    return select_rows(fn, scores, ids, rows, cols, k, id_offset, 1, nullptr, nullptr, out_scores, out_ids, nullptr, stream);
}

extern "C" int vr_select_rows_masks(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k,
                                    int64_t id_offset, float* out_scores, int64_t* out_ids, const vr_doc_masks* masks,
                                    void* stream) {
    const char* fn = "vr_select_rows_masks";
    VR_REQUIRE_MASKS(fn, masks, cols);
    VR_REQUIRE(!ids, "%s: the masks index columns, so ids must be NULL", fn);
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    const DocMasks m = device_masks(masks);
    return select_rows(fn, scores, nullptr, rows, cols, k, id_offset, 1, nullptr, nullptr, out_scores, out_ids, &m, stream);
}

extern "C" int vr_select_rows_chunked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                      int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids,
                                      void* stream) {
    const char* fn = "vr_select_rows_chunked";
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "ws_scores", ws_scores, 4);
    VR_REQUIRE_PTR(fn, "ws_ids", ws_ids, 8);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    return select_rows(fn, scores, nullptr, rows, cols, k, id_offset, chunks, ws_scores, ws_ids, out_scores, out_ids, nullptr,
                       stream);
}

extern "C" int vr_select_rows_chunked_masks(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                            int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores,
                                            int64_t* out_ids, const vr_doc_masks* masks, void* stream) {
    const char* fn = "vr_select_rows_chunked_masks";
    VR_REQUIRE_MASKS(fn, masks, cols);
    VR_REQUIRE_PTR(fn, "scores", scores, 4);
    VR_REQUIRE_PTR(fn, "ws_scores", ws_scores, 4);
    VR_REQUIRE_PTR(fn, "ws_ids", ws_ids, 8);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    const DocMasks m = device_masks(masks);
    return select_rows(fn, scores, nullptr, rows, cols, k, id_offset, chunks, ws_scores, ws_ids, out_scores, out_ids, &m,
                       stream);
}

// ---------------------------------------------------------------------------------------------------- MMR selection
extern "C" int vr_mmr_select(const float* emb, int64_t nd, int32_t dim, const float* cand_scores, const int64_t* cand_ids,
                             int32_t nq, int32_t fetch, const float* lambda, int32_t k, int64_t id_offset, float* out_scores,
                             int64_t* out_ids, void* stream) {
    const char* fn = "vr_mmr_select";
    VR_REQUIRE_PTR(fn, "emb", emb, 16);  // bulk-copy sources
    VR_REQUIRE_PTR(fn, "cand_scores", cand_scores, 4);
    VR_REQUIRE_PTR(fn, "cand_ids", cand_ids, 8);
    VR_REQUIRE_PTR(fn, "lambda", lambda, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    VR_REQUIRE(nq > 0 && nq < (1 << 28), "%s: nq=%d, needs 0 < nq < 2^28", fn, nq);
    VR_REQUIRE(nd > 0, "%s: nd=%lld, needs at least 1", fn, (long long)nd);
    VR_REQUIRE(dim > 0 && dim % 4 == 0, "%s: dim=%d, needs a positive multiple of 4", fn, dim);
    VR_REQUIRE(fetch >= 1 && fetch <= MMR_MAX_FETCH, "%s: fetch=%d, needs 1 <= fetch <= %d", fn, fetch, MMR_MAX_FETCH);
    VR_REQUIRE(static_cast<long long>(fetch) * dim <= MMR_MAX_ELEMS, "%s: fetch=%d x dim=%d exceeds %lld floats of rows", fn,
               fetch, dim, MMR_MAX_ELEMS);
    const int C = mmr_cluster(fetch, dim);
    VR_REQUIRE(C > 0, "%s: fetch=%d rows of dim=%d do not fit %d CTAs of %d bytes (%d with the pick's row)", fn, fetch,
               dim, MMR_MAX_CLUSTER, MMR_CTA_BYTES, MMR_SMEM_BYTES);
    VR_REQUIRE(k >= 1 && k <= fetch, "%s: k=%d, needs 1 <= k <= fetch=%d", fn, k, fetch);
    const int R = (fetch + C - 1) / C;
    static unsigned long long attr_set = 0;
    if (first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(mmr_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MMR_SMEM_BYTES));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(nq) * C);
    cfg.blockDim = dim3(MMR_THREADS);
    cfg.dynamicSmemBytes = static_cast<size_t>(R + 1) * dim * sizeof(float);
    cfg.stream = reinterpret_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = C; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    VR_CHECK_CUDA(cudaLaunchKernelEx(&cfg, mmr_select_kernel, emb, static_cast<long long>(nd), static_cast<int>(dim),
                                     cand_scores, reinterpret_cast<const long long*>(cand_ids), static_cast<int>(fetch),
                                     lambda, static_cast<int>(k), R, static_cast<long long>(id_offset), out_scores,
                                     reinterpret_cast<long long*>(out_ids)));
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------- per-document top-m
extern "C" int vr_group_pages_topm(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                                   const int64_t* groups, int32_t kg, const int32_t* group_offsets, const int32_t* group_pages,
                                   int32_t G, const vr_doc_masks* masks, int32_t m, int32_t piece, int32_t pieces,
                                   int64_t id_offset, float* out_scores, int64_t* out_pages, void* stream) {
    const char* fn = "vr_group_pages_topm";
    if (masks) VR_REQUIRE_MASKS(fn, masks, nd);
    VR_REQUIRE_PTR(fn, "q_f32", q_f32, 4);
    VR_REQUIRE_PTR(fn, "d_f32", d_f32, 16);  // float4 rows (dim % 4 == 0 keeps every row aligned)
    VR_REQUIRE_PTR(fn, "groups", groups, 8);
    VR_REQUIRE_PTR(fn, "group_offsets", group_offsets, 4);
    VR_REQUIRE_PTR(fn, "group_pages", group_pages, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_pages", out_pages, 8);
    VR_REQUIRE(nq > 0, "%s: nq=%d, needs at least 1", fn, nq);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(dim > 0 && dim % 4 == 0, "%s: dim=%d, needs a positive multiple of 4", fn, dim);
    VR_REQUIRE(kg >= 1, "%s: kg=%d, needs at least 1", fn, kg);
    VR_REQUIRE(static_cast<long long>(nq) * kg < 2147483647ll, "%s: nq=%d x kg=%d rows, needs fewer than 2^31", fn, nq, kg);
    VR_REQUIRE(G >= 1, "%s: G=%d, needs at least 1", fn, G);
    VR_REQUIRE(m >= 1 && m <= GROUP_PAGES_MAX, "%s: m=%d, needs 1 <= m <= %d", fn, m, GROUP_PAGES_MAX);
    VR_REQUIRE(piece >= 1 && piece <= GROUP_PIECE_MAX, "%s: piece=%d, needs 1 <= piece <= %d", fn, piece, GROUP_PIECE_MAX);
    VR_REQUIRE(pieces >= 1 && pieces <= 65535, "%s: pieces=%d, needs 1 <= pieces <= 65535", fn, pieces);
    const size_t smem = static_cast<size_t>(dim) * sizeof(float) + static_cast<size_t>(piece) * 8;
    VR_REQUIRE(smem <= 200 * 1024, "%s: dim=%d with piece=%d too large for shared memory", fn, dim, piece);
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(group_pages_topm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    const int threads = 32 * (piece < 8 ? piece : 8);  // a warp per page: no idle warps for short documents
    const DocMasks dm = masks ? device_masks(masks) : kNoMasks;
    group_pages_topm_kernel<<<dim3(static_cast<unsigned>(nq * kg), static_cast<unsigned>(pieces)), threads, smem,
                              reinterpret_cast<cudaStream_t>(stream)>>>(
        q_f32, d_f32, dim, reinterpret_cast<const long long*>(groups), kg, group_offsets, group_pages, G, dm, m, piece,
        static_cast<long long>(id_offset), out_scores, reinterpret_cast<long long*>(out_pages));
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------- hybrid retrieval
extern "C" int vr_fuse_rows(const float* dense_scores, const int64_t* dense_ids, int32_t rows, int32_t kd,
                            const int64_t* hit_offsets, const int32_t* hit_ids, const float* hit_values,
                            const float* hit_dense, int64_t hit_pitch, int32_t mode, float weight, int32_t rrf_c,
                            int64_t width, float* out_scores, int64_t* out_ids, int32_t* status, void* stream) {
    const char* fn = "vr_fuse_rows";
    VR_REQUIRE(mode == VR_FUSE_SUM || mode == VR_FUSE_RRF, "%s: mode=%d, needs VR_FUSE_SUM (0) or VR_FUSE_RRF (1)", fn, mode);
    const bool rrf = mode == VR_FUSE_RRF;
    VR_REQUIRE_PTR(fn, "dense_scores", dense_scores, 4);
    VR_REQUIRE_PTR(fn, "dense_ids", dense_ids, 8);
    VR_REQUIRE_PTR(fn, "hit_offsets", hit_offsets, 8);
    VR_REQUIRE_PTR(fn, "hit_ids", hit_ids, 4);
    if (!rrf) {  // RRF reads neither the values nor the dense scores of the hits, only their order
        VR_REQUIRE_PTR(fn, "hit_values", hit_values, 4);
        VR_REQUIRE_PTR(fn, "hit_dense", hit_dense, 4);
    }
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_ids", out_ids, 8);
    VR_REQUIRE_PTR(fn, "status", status, 4);
    VR_REQUIRE(rows >= 1, "%s: rows=%d, needs at least 1", fn, rows);
    VR_REQUIRE(kd >= 1 && kd <= FUSE_DENSE_MAX, "%s: kd=%d, needs 1 <= kd <= %d", fn, kd, FUSE_DENSE_MAX);
    VR_REQUIRE(width >= kd && width < 2147483647ll, "%s: width=%lld, needs kd=%d <= width < 2^31", fn, (long long)width, kd);
    VR_REQUIRE(rrf || hit_pitch >= 1, "%s: hit_pitch=%lld, needs at least 1", fn, (long long)hit_pitch);
    VR_REQUIRE(rrf || (weight >= 0.f && weight <= 3.4028234663852886e38f),
               "%s: weight=%g, needs a finite weight >= 0", fn, static_cast<double>(weight));
    VR_REQUIRE(!rrf || rrf_c >= 0, "%s: rrf_c=%d, needs rrf_c >= 0", fn, rrf_c);
    int P = 2;
    while (P < 2 * kd) P <<= 1;
    const size_t smem = (2 * static_cast<size_t>(P) + kd) * sizeof(int);
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(fuse_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
    fuse_rows_kernel<<<rows, FUSE_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
        dense_scores, reinterpret_cast<const long long*>(dense_ids), kd, reinterpret_cast<const long long*>(hit_offsets),
        hit_ids, hit_values, hit_dense, static_cast<long long>(hit_pitch), rrf, weight, rrf_c, static_cast<long long>(width), P,
        out_scores, reinterpret_cast<long long*>(out_ids), status);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int vr_group_pages_fused(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                                    const int64_t* groups, int32_t kg, const int32_t* group_offsets,
                                    const int32_t* group_pages, int32_t G, const vr_doc_masks* masks,
                                    const int64_t* hit_offsets, const int32_t* hit_ids, const float* hit_values, float weight,
                                    int32_t piece, int32_t pieces, int64_t id_offset, float* out_scores, int64_t* out_pages,
                                    void* stream) {
    const char* fn = "vr_group_pages_fused";
    if (masks) VR_REQUIRE_MASKS(fn, masks, nd);
    VR_REQUIRE_PTR(fn, "q_f32", q_f32, 4);
    VR_REQUIRE_PTR(fn, "d_f32", d_f32, 16);  // float4 rows (dim % 4 == 0 keeps every row aligned)
    VR_REQUIRE_PTR(fn, "groups", groups, 8);
    VR_REQUIRE_PTR(fn, "group_offsets", group_offsets, 4);
    VR_REQUIRE_PTR(fn, "group_pages", group_pages, 4);
    VR_REQUIRE_PTR(fn, "hit_offsets", hit_offsets, 8);
    VR_REQUIRE_PTR(fn, "hit_ids", hit_ids, 4);
    VR_REQUIRE_PTR(fn, "hit_values", hit_values, 4);
    VR_REQUIRE_PTR(fn, "out_scores", out_scores, 4);
    VR_REQUIRE_PTR(fn, "out_pages", out_pages, 8);
    VR_REQUIRE(nq > 0, "%s: nq=%d, needs at least 1", fn, nq);
    VR_REQUIRE(nd > 0 && nd < 2147483647ll, "%s: nd=%lld beyond the int32 doc ids", fn, (long long)nd);
    VR_REQUIRE(dim > 0 && dim % 4 == 0, "%s: dim=%d, needs a positive multiple of 4", fn, dim);
    VR_REQUIRE(kg >= 1, "%s: kg=%d, needs at least 1", fn, kg);
    VR_REQUIRE(static_cast<long long>(nq) * kg < 2147483647ll, "%s: nq=%d x kg=%d rows, needs fewer than 2^31", fn, nq, kg);
    VR_REQUIRE(G >= 1, "%s: G=%d, needs at least 1", fn, G);
    VR_REQUIRE(weight >= 0.f && weight <= 3.4028234663852886e38f, "%s: weight=%g, needs a finite weight >= 0", fn,
               static_cast<double>(weight));
    VR_REQUIRE(piece >= 1 && piece <= GROUP_PIECE_MAX, "%s: piece=%d, needs 1 <= piece <= %d", fn, piece, GROUP_PIECE_MAX);
    VR_REQUIRE(pieces >= 1 && pieces <= 65535, "%s: pieces=%d, needs 1 <= pieces <= 65535", fn, pieces);
    const size_t smem = static_cast<size_t>(dim) * sizeof(float) + static_cast<size_t>(piece) * 8;
    VR_REQUIRE(smem <= 200 * 1024, "%s: dim=%d with piece=%d too large for shared memory", fn, dim, piece);
    static unsigned long long attr_set = 0;
    if (smem > 48 * 1024 && first_use_on_device(&attr_set))
        VR_CHECK_CUDA(cudaFuncSetAttribute(group_pages_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    const int threads = 32 * (piece < 8 ? piece : 8);  // a warp per page, as vr_group_pages_topm
    const DocMasks dm = masks ? device_masks(masks) : kNoMasks;
    const HitsFuse fuse = {reinterpret_cast<const long long*>(hit_offsets), hit_ids, hit_values, weight};
    group_pages_fused_kernel<<<dim3(static_cast<unsigned>(nq * kg), static_cast<unsigned>(pieces)), threads, smem,
                               reinterpret_cast<cudaStream_t>(stream)>>>(
        q_f32, d_f32, dim, reinterpret_cast<const long long*>(groups), kg, group_offsets, group_pages, G, dm, fuse, piece,
        static_cast<long long>(id_offset), out_scores, reinterpret_cast<long long*>(out_pages));
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}
