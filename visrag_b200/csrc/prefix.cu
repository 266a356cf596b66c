// Prefix-cache row assembly: the rows of every sequence become [cached prefix rows ; the sequence's own rows]. The
// cached path of the encoder runs it once per layer for the K|V columns (16-bit) and once for the fp32 residual stream
// before pooling. A pure copy, one pass with 16-byte accesses. A warp moves one chunk of a row, 128 vectors (2 KB): each
// lane issues its up to four loads before its stores, and a 9 KB row spreads over five warps, so that the hundred rows
// of a single query still spread over many SMs.
#include "common.h"
#include "../../include/visrag_b200.h"

namespace vr {

constexpr int PREFIX_THREADS = 256;
constexpr int PREFIX_UNROLL = 4;                  // vectors per lane and chunk
constexpr int PREFIX_CHUNK = 32 * PREFIX_UNROLL;  // vectors per warp item

__global__ void __launch_bounds__(PREFIX_THREADS)
prefix_rows_kernel(const uint4* __restrict__ prefix, long long ldp, const uint4* __restrict__ rows, long long ldr,
                   uint4* __restrict__ out, long long ldo, const int* __restrict__ cu_rows, const int* __restrict__ cu_out,
                   int batch, int prefix_len, long long items, int chunks, int vecs) {
    const int warps = PREFIX_THREADS / 32;
    const int lane = threadIdx.x & 31;
    for (long long it = static_cast<long long>(blockIdx.x) * warps + (threadIdx.x >> 5); it < items;
         it += static_cast<long long>(gridDim.x) * warps) {
        const int t = static_cast<int>(it / chunks);
        const int c0 = static_cast<int>(it - static_cast<long long>(t) * chunks) * PREFIX_CHUNK + lane;
        int lo = 0, hi = batch;  // the sequence b with cu_out[b] <= t < cu_out[b + 1] (the last such b: empty ones are skipped)
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(cu_out + mid) <= t) lo = mid;
            else hi = mid;
        }
        const int r = t - __ldg(cu_out + lo);
        const uint4* src = r < prefix_len ? prefix + static_cast<long long>(r) * ldp
                                          : rows + static_cast<long long>(__ldg(cu_rows + lo) + r - prefix_len) * ldr;
        uint4* dst = out + static_cast<long long>(t) * ldo;
        uint4 v[PREFIX_UNROLL];
#pragma unroll
        for (int j = 0; j < PREFIX_UNROLL; ++j)
            if (c0 + 32 * j < vecs) v[j] = src[c0 + 32 * j];
#pragma unroll
        for (int j = 0; j < PREFIX_UNROLL; ++j)
            if (c0 + 32 * j < vecs) dst[c0 + 32 * j] = v[j];
    }
}

}  // namespace vr

using namespace vr;

extern "C" int vr_prefix_rows(const void* prefix, int64_t ldp, const void* rows, int64_t ldr, void* out, int64_t ldo,
                              const int32_t* cu_rows, const int32_t* cu_out, int32_t batch, int32_t prefix_len,
                              int32_t out_rows, int32_t cols, int32_t elem_size, void* stream) {
    VR_REQUIRE(rows && out && cu_rows && cu_out && (prefix || prefix_len == 0), "vr_prefix_rows: null pointer");
    VR_REQUIRE(batch > 0 && prefix_len >= 0 && out_rows > 0 && cols > 0,
               "vr_prefix_rows: bad shape batch=%d prefix_len=%d out_rows=%d cols=%d", batch, prefix_len, out_rows, cols);
    VR_REQUIRE(elem_size == 2 || elem_size == 4, "vr_prefix_rows: elem_size must be 2 or 4 (got %d)", elem_size);
    VR_REQUIRE(ldp >= cols && ldr >= cols && ldo >= cols, "vr_prefix_rows: a leading dimension is below cols=%d", cols);
    const long long row_bytes = static_cast<long long>(cols) * elem_size;
    VR_REQUIRE(row_bytes % 16 == 0 && (ldp * elem_size) % 16 == 0 && (ldr * elem_size) % 16 == 0 && (ldo * elem_size) % 16 == 0,
               "vr_prefix_rows: cols and leading dimensions must be multiples of 16 bytes (cols=%d ldp=%lld ldr=%lld ldo=%lld, "
               "%d-byte elements)", cols, (long long)ldp, (long long)ldr, (long long)ldo, elem_size);
    VR_REQUIRE(((reinterpret_cast<uintptr_t>(prefix) | reinterpret_cast<uintptr_t>(rows) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
               "vr_prefix_rows: prefix, rows and out must be 16-byte aligned");
    VR_REQUIRE_ALIGNED("vr_prefix_rows", "cu_rows", cu_rows, 4);
    VR_REQUIRE_ALIGNED("vr_prefix_rows", "cu_out", cu_out, 4);
    const int per = elem_size == 2 ? 8 : 4;  // elements per 16-byte vector
    const int vecs = static_cast<int>(row_bytes / 16);
    const int chunks = (vecs + PREFIX_CHUNK - 1) / PREFIX_CHUNK;
    const long long items = static_cast<long long>(out_rows) * chunks;
    long long blocks = (items + PREFIX_THREADS / 32 - 1) / (PREFIX_THREADS / 32);
    const long long cap = static_cast<long long>(num_sms()) * 8;
    if (blocks > cap) blocks = cap;
    prefix_rows_kernel<<<static_cast<int>(blocks), PREFIX_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const uint4*>(prefix), ldp / per, reinterpret_cast<const uint4*>(rows), ldr / per,
        reinterpret_cast<uint4*>(out), ldo / per, cu_rows, cu_out, batch, prefix_len, items, chunks, vecs);
    VR_CHECK_CUDA(cudaGetLastError());
    return 0;
}
