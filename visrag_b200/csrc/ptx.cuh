// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA, fp32 accumulators in registers), fences, setmaxnreg.
// No CUTLASS / CuTe: every instruction is spelled out here once.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <type_traits>

namespace vr {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    return ok != 0;
}
// Spin on a phase parity. A pipeline bug must never hang the GPU: after ~2 s of
// spinning the kernel traps (the host then sees a launch failure instead of a hang).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t addr = smem_u32(bar);
    if (mbar_try_wait(addr, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(addr, parity)) {
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}

// 1-D bulk copy global -> shared (TMA without a tensor map): 16-byte aligned source, destination and size
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}


// ---------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same smem location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ float4 ld_shared_cluster_f4(uint32_t cluster_addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(cluster_addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared_cluster_u64(uint32_t cluster_addr, unsigned long long v) {
    asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(cluster_addr), "l"(v) : "memory");
}
// generic address of the same smem location in CTA `rank` of the cluster: ordinary loads through it read that CTA's
// shared memory (DSMEM)
template <typename T>
__device__ __forceinline__ T* map_cluster_ptr(T* p, uint32_t rank) {
    uint64_t r;
    asm volatile("mapa.u64 %0, %1, %2;" : "=l"(r) : "l"(p), "r"(rank));
    return reinterpret_cast<T*>(r);
}

// ---------------------------------------------------------------- fences
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 4-byte asynchronous copy global -> shared (no registers involved); cp_async_wait_all waits for the thread's own copies
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// 8-byte shared-memory load (the memory clobber keeps it after the waits and barriers that make the data visible)
__device__ __forceinline__ float2 ld_shared_f2(const void* p) {
    float2 v;
    asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(p)) : "memory");
    return v;
}

// 2-D tiled load: coordinates are (c0 = innermost/contiguous dim, c1 = row).
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem_dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// Same load written to the same smem offset of every CTA in cta_mask (bit r = cluster rank r); each destination CTA's
// mbarrier at `bar`'s offset receives the box's bytes.
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* m, uint64_t* bar, void* smem_dst, int c0, int c1,
                                                      uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
// arrive on the mbarrier at `bar`'s offset in CTA `rank` of the cluster. Default (CTA-scope release) semantics: the
// arrivals that use it hand back a shared-memory stage whose only readers were retired wgmma instructions, so there
// is no generic-proxy write to publish, and a cluster-scope release would cost a GPU-wide fence per arrival.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(mapa_u32(smem_u32(bar), rank)) : "memory");
}

// ---------------------------------------------------------------- warpgroup MMA (wgmma)
// Shared-memory matrix descriptor:
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4
//   [32,46) stride byte offset >> 4 [49,52) base offset = 0
//   [62,64) swizzle (0 none, 1 128B, 2 64B, 3 32B)
enum : uint64_t { kLayoutNone = 0, kLayoutSW128 = 1, kLayoutSW64 = 2, kLayoutSW32 = 3 };

__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint64_t layout) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= layout << 62;
    return d;
}

// Accumulator registers of other warpgroup-MMA groups may be touched only between fence and commit/wait.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving reads of the accumulators above the wait
template <int NR>
__device__ __forceinline__ void wgmma_touch(float (&d)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One m64nNk16 instruction, D (fp32, N/2 registers per thread) (+)= A * B. Register layout of D for thread t of the
// warpgroup (warp w = t / 32, g = (t % 32) / 4, q = t % 4): d[4j + 0/1] = row 16w + g, columns 8j + 2q + 0/1;
// d[4j + 2/3] = row 16w + g + 8, same columns.
//   F16    : operands are fp16 (else bf16)
//   TRANS_B: B tile is MN-major in shared memory (rows of the tile are K, N contiguous)
// Inline asm cannot build "{%0, ..., %(N/2-1)}" from a template parameter: the operand lists below are spelled out
// for every N the kernels use, and the overload is chosen by an integral_constant tag.
#define VR_R4(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define VR_R8(d, i) VR_R4(d, i), VR_R4(d, i + 4)
#define VR_R16(d, i) VR_R8(d, i), VR_R8(d, i + 8)
#define VR_R32(d, i) VR_R16(d, i), VR_R16(d, i + 16)
#define VR_R64(d, i) VR_R32(d, i), VR_R32(d, i + 32)

// register-name lists "%0, %1, ..." of 8 / 32 / 64 / 96 / 128 entries
#define VR_N8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define VR_N32 VR_N8 ", %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define VR_N64 VR_N32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define VR_N96 VR_N64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define VR_N128 VR_N96 ", %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"

// A and B from shared memory
#define VR_WGMMA_SS(NN, NREG, NAMES, REGS, A0, A1, A2)                                                                  \
    template <bool F16, bool TRANS_B>                                                                                   \
    __device__ __forceinline__ void wgmma_ss(float (&d)[NREG], uint64_t adesc, uint64_t bdesc, int accumulate,          \
                                             std::integral_constant<int, NN>) {                                         \
        if (F16)                                                                                                        \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #A2 ", 0;\n\t"                                         \
                         "wgmma.mma_async.sync.aligned.m64n" #NN "k16.f32.f16.f16 {" NAMES "}, %" #A0 ", %" #A1          \
                         ", p, 1, 1, 0, 0;\n\t}\n"                                                                      \
                         : REGS(d, 0)                                                                                   \
                         : "l"(adesc), "l"(bdesc), "r"(accumulate));                                                    \
        else if (TRANS_B)                                                                                               \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #A2 ", 0;\n\t"                                         \
                         "wgmma.mma_async.sync.aligned.m64n" #NN "k16.f32.bf16.bf16 {" NAMES "}, %" #A0 ", %" #A1        \
                         ", p, 1, 1, 0, 1;\n\t}\n"                                                                      \
                         : REGS(d, 0)                                                                                   \
                         : "l"(adesc), "l"(bdesc), "r"(accumulate));                                                    \
        else                                                                                                            \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #A2 ", 0;\n\t"                                         \
                         "wgmma.mma_async.sync.aligned.m64n" #NN "k16.f32.bf16.bf16 {" NAMES "}, %" #A0 ", %" #A1        \
                         ", p, 1, 1, 0, 0;\n\t}\n"                                                                      \
                         : REGS(d, 0)                                                                                   \
                         : "l"(adesc), "l"(bdesc), "r"(accumulate));                                                    \
    }
VR_WGMMA_SS(16, 8, VR_N8, VR_R8, 8, 9, 10)
VR_WGMMA_SS(64, 32, VR_N32, VR_R32, 32, 33, 34)
VR_WGMMA_SS(128, 64, VR_N64, VR_R64, 64, 65, 66)
#define VR_R96(d, i) VR_R64(d, i), VR_R32(d, i + 64)
VR_WGMMA_SS(192, 96, VR_N96, VR_R96, 96, 97, 98)
#define VR_R128(d, i) VR_R64(d, i), VR_R64(d, i + 64)
VR_WGMMA_SS(256, 128, VR_N128, VR_R128, 128, 129, 130)

// A (16-bit pairs, the m16n8k16 A-fragment layout of each warp) from registers, B MN-major from shared memory;
// F16: both operands fp16 (else bf16)
#define VR_WGMMA_RS(NN, NREG, NAMES, REGS, A0, A1, A2, A3, B0, P0)                                                      \
    template <bool F16>                                                                                                 \
    __device__ __forceinline__ void wgmma_rs_tb(float (&d)[NREG], const uint32_t (&a)[4], uint64_t bdesc, int accumulate, \
                                                std::integral_constant<int, NN>) {                                      \
        if (F16)                                                                                                        \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #P0 ", 0;\n\t"                                         \
                         "wgmma.mma_async.sync.aligned.m64n" #NN "k16.f32.f16.f16 {" NAMES "}, {%" #A0 ", %" #A1 ", %" #A2 \
                         ", %" #A3 "}, %" #B0 ", p, 1, 1, 1;\n\t}\n"                                                    \
                         : REGS(d, 0)                                                                                   \
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));                    \
        else                                                                                                            \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #P0 ", 0;\n\t"                                         \
                         "wgmma.mma_async.sync.aligned.m64n" #NN "k16.f32.bf16.bf16 {" NAMES "}, {%" #A0 ", %" #A1 ", %" #A2 \
                         ", %" #A3 "}, %" #B0 ", p, 1, 1, 1;\n\t}\n"                                                    \
                         : REGS(d, 0)                                                                                   \
                         : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));                    \
    }
VR_WGMMA_RS(16, 8, VR_N8, VR_R8, 8, 9, 10, 11, 12, 13)
VR_WGMMA_RS(64, 32, VR_N32, VR_R32, 32, 33, 34, 35, 36, 37)

// register budget per warpgroup role (all warps of the warpgroup execute it)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// signal a named barrier without waiting on it (the other side of a one-way handoff does bar.sync)
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------- misc
// 2^x on the MUFU, one instruction (exp2f is the non-ftz form: a range test and two scalings around the same MUFU.EX2).
// Results below 2^-126 flush to zero; relative error 2^-22 as for exp2f.
__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
// round to nearest even, no flush: results below 2^-14 become fp16 subnormals; beyond 65504 they become inf
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

// The kernels of the encode path store their 16-bit activations as bf16 or, with F16, as fp16 (one engine, one type).
template <bool F16>
using half16_t = typename std::conditional<F16, __half, __nv_bfloat16>::type;
template <bool F16>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
    return F16 ? pack_f16x2(lo, hi) : pack_bf16x2(lo, hi);
}
template <bool F16>
__device__ __forceinline__ half16_t<F16> to_half16(float x) {
    if constexpr (F16) return __float2half_rn(x);
    else return __float2bfloat16_rn(x);
}
// two 16-bit values of one 32-bit word -> fp32 (exact)
template <bool F16>
__device__ __forceinline__ float2 unpack16x2(uint32_t w) {
    if constexpr (F16) return __half22float2(*reinterpret_cast<const __half2*>(&w));
    else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}

}  // namespace vr
