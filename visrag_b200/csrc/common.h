// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor
// construction (driver entry point resolved at run time, so the library links against
// libcudart only and loads on a CPU-only box), device properties.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace vr {

void set_error(const char* fmt, ...);
int current_device();  // cudaGetDevice, -1 on failure
int num_sms();         // SM count of the CURRENT device (cached per device)
// Per-device one-time setup (cudaFuncSetAttribute and the occupancy queries are per device, the library is per process):
// returns true the first time it is called with `mask` while a given device is current. One mask per kernel instantiation.
bool first_use_on_device(unsigned long long* mask);

// 2-D row-major tensor [rows, cols] of 2-byte elements, box = [box_rows, box_cols].
// swizzle_bytes in {0 (none / 16B interleave), 32, 64, 128}; box_cols*2 must be <= swizzle span.
// Returns 0 on success.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols, int swizzle_bytes, bool is_bf16);

#define VR_CHECK_CUDA(expr)                                                                    \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            vr::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 1;                                                                          \
        }                                                                                      \
    } while (0)

#define VR_REQUIRE(cond, ...)          \
    do {                               \
        if (!(cond)) {                 \
            vr::set_error(__VA_ARGS__); \
            return 2;                  \
        }                              \
    } while (0)

// Base alignment of a pointer the kernels read or write with `bytes`-wide vector accesses (NULL passes: optional pointers
// are checked for presence elsewhere). A misaligned base is refused before any CUDA call, naming the argument; launched,
// it would be a misaligned-address fault that ends the CUDA context.
inline bool is_aligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
#define VR_REQUIRE_ALIGNED(fn, name, ptr, bytes)                                                                         \
    VR_REQUIRE(vr::is_aligned((ptr), (bytes)), "%s: %s must be %d-byte aligned (got %p)", fn, name, (int)(bytes), \
               (const void*)(ptr))

}  // namespace vr
