#include "common.h"
#include "../../include/visrag_b200.h"
#include <stdarg.h>
#include <string.h>
#include <mutex>

namespace vr {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int current_device() {
    int dev = -1;
    return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int num_sms() {
    static int cached[64] = {};
    const int dev = current_device();
    const int slot = (dev >= 0 && dev < 64) ? dev : 0;
    if (cached[slot] == 0) {
        int n = 0;
        cached[slot] = (dev >= 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;  // no device (host-only planning): an H100 SXM
    }
    return cached[slot];
}

bool first_use_on_device(unsigned long long* mask) {
    const int dev = current_device();
    if (dev < 0 || dev >= 64) return true;  // unknown device: redo the setup every time (correct, only slower)
    const unsigned long long bit = 1ull << dev;
    if (*mask & bit) return false;
    *mask |= bit;
    return true;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols, int swizzle_bytes, bool is_bf16) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
        return 1;
    }
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((ld_elems * 2) & 15) != 0) {
        set_error("TMA operand must be 16-byte aligned with a 16-byte-multiple row pitch (base=%p ld=%llu)", base,
                  (unsigned long long)ld_elems);
        return 2;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
    if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
    else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
    else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = fn(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                    const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u sw=%d)", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows, box_cols,
                  swizzle_bytes);
        return 1;
    }
    return 0;
}

}  // namespace vr

extern "C" const char* vr_last_error(void) { return vr::g_err; }
extern "C" int vr_abi_version(void) { return VR_ABI_VERSION; }
