// b2d_runtime.cu — error state, device queries, TMA tensor-map construction (driver entry point resolved at run time so
// that the library links without libcuda and loads on a GPU-less build box).
#include <stdarg.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <unordered_map>
#include <stdlib.h>
#include "b2d_internal.h"

namespace b2d {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

// The library links its own (static) CUDA runtime, whose per-thread "current device" is independent of the caller's
// (PyTorch's) runtime.  Autograd runs backward on a fresh host thread, and one process may drive several GPUs, so every
// entry point looks up the device that owns the buffer it was handed and makes it current for the calling thread
// whenever it differs from the one this thread was last bound to.
int bind_thread(const void* device_ptr) {
    static thread_local int bound = -1;
    cudaPointerAttributes at;
    cudaError_t e = cudaPointerGetAttributes(&at, device_ptr);
    if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "cudaPointerGetAttributes: %s", cudaGetErrorString(e));
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged)
        return set_error(B2D_ERR_ARG, "libb2d needs device pointers (got host/unregistered memory): no CPU fallback");
    if (at.device == bound) return B2D_OK;
    e = cudaSetDevice(at.device);
    if (e != cudaSuccess) return set_error(B2D_ERR_CUDA, "cudaSetDevice(%d): %s", at.device, cudaGetErrorString(e));
    cudaFree(0);  // make the primary context current for driver-API calls (cuTensorMapEncodeTiled)
    bound = at.device;
    return B2D_OK;
}

int device_sm_count() {
    static int cache[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return set_error(B2D_ERR_CUDA, "cudaGetDevice failed"), -1;
    if (dev < 64 && cache[dev] > 0) return cache[dev];
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return set_error(B2D_ERR_CUDA, "cudaDeviceGetAttribute(SM count) failed"), -1;
    if (dev < 64) cache[dev] = n;
    return n;
}

static std::atomic<int64_t> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

typedef CUresult (*encode_fn_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_fn_t get_encode() {
    static encode_fn_t fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<encode_fn_t>(p);
    });
    return fn;
}

int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int elem_bytes, int swizzle128) {
    encode_fn_t enc = get_encode();
    if (!enc) return set_error(B2D_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
    if (((uintptr_t)base & 15) != 0) return set_error(B2D_ERR_ALIGN, "tensor map base not 16-byte aligned");
    cuuint64_t gdim[5];
    cuuint64_t gstr[5];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = 1;
        if (i > 0) {
            gstr[i - 1] = strides_bytes[i - 1];
            if (gstr[i - 1] % 16) return set_error(B2D_ERR_ALIGN, "tensor map stride %d not a multiple of 16 bytes", i);
        }
    }
    CUresult r = enc(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                     (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(B2D_ERR_CUDA, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    return B2D_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* base, long long rows, long long cols, long long ld, int box_rows,
                 int box_cols) {
    if (box_cols != 64) return set_error(B2D_ERR_ARG, "make_tmap_2d: inner box must be 64 bf16 (128 B swizzle)");
    uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows};
    uint64_t strides[1] = {(uint64_t)ld * 2};
    uint32_t box[2] = {(uint32_t)box_cols, (uint32_t)box_rows};
    return make_tmap_nd(out, base, 2, dims, strides, box, 2, 1);
}

}  // namespace b2d

extern "C" int b2d_version(void) { return 2; }
extern "C" const char* b2d_last_error(void) { return b2d::g_err; }
extern "C" int64_t b2d_launch_count(void) { return b2d::g_launches.load(std::memory_order_relaxed); }
extern "C" int b2d_device_check(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return b2d::set_error(B2D_ERR_CUDA, "no CUDA device");
    int major = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess)
        return b2d::set_error(B2D_ERR_CUDA, "cannot query compute capability");
    if (major != 9) return b2d::set_error(B2D_ERR_ARCH, "device compute capability %d.x, need 9.0 (sm_90a)", major);
    return B2D_OK;
}
