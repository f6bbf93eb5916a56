// b2d_internal.h — host-side helpers shared by the .cu translation units of libb2d.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>
#include "../../include/b2d.h"

namespace b2d {

// printf-style; stores a thread-local message and returns `code`.
int set_error(int code, const char* fmt, ...);

// bind the calling host thread to the device owning `device_ptr` (first call per thread); see b2d_runtime.cu
int bind_thread(const void* device_ptr);
#define B2D_BIND(ptr)                                  \
    do {                                               \
        if (int rc__ = b2d::bind_thread(ptr)) return rc__; \
    } while (0)

// number of SMs of the current device (cached per device); <=0 on error
int device_sm_count();

// adds one to b2d_launch_count(); called once per kernel, after its launch error check passed
void count_launch();

// bf16 2-D tiled tensor map with 128-byte swizzle.  Tensor is row-major [rows, cols] with leading dimension `ld`
// (elements).  Box = box_cols (inner, must be 64 => 128 B) x box_rows.
int make_tmap_2d(CUtensorMap* out, const void* base, long long rows, long long cols, long long ld, int box_rows,
                 int box_cols);

// generic rank-N (N<=4) map: dims/strides innermost-first; strides in BYTES for dims 1..N-1; dtype bf16 or fp32.
int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int elem_bytes, int swizzle128);

// cluster_x > 1 launches thread-block clusters of cluster_x consecutive CTAs along x
template <typename... P, typename... A>
inline cudaError_t launch_kc(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x,
                             A&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    int n = 0;
    // programmatic dependent launch (b2d_ptx.cuh: griddep_*): every kernel launched here calls griddep_wait()
#ifndef B2D_NO_PDL
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
#endif
    if (cluster_x > 1) {
        at[n].id = cudaLaunchAttributeClusterDimension;
        at[n].val.clusterDim.x = (unsigned)cluster_x;
        at[n].val.clusterDim.y = 1;
        at[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = at;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...);
}

template <typename... P, typename... A>
inline cudaError_t launch_k(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
    return launch_kc(kern, grid, block, smem, st, 1, static_cast<A&&>(args)...);
}

#define B2D_CHECK_LAUNCH(name)                                                                     \
    do {                                                                                           \
        cudaError_t e__ = cudaGetLastError();                                                      \
        if (e__ != cudaSuccess) return b2d::set_error(B2D_ERR_CUDA, "%s launch: %s", name, cudaGetErrorString(e__)); \
        b2d::count_launch();                                                                       \
    } while (0)

}  // namespace b2d
