// b2d_ptx.cuh — thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), programmatic dependent launch
// and the wgmma shared-memory matrix descriptor.  Hand-written; bit layouts cross-checked against the PTX ISA
// (warpgroup-level matrix shared memory layout, matrix descriptor format).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "b2d_wgmma.cuh"

namespace b2d {

// ------------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    // with a suspend-time hint the waiting thread is parked by the hardware until the phase completes (or the hint
    // expires) instead of re-issuing the probe every few cycles and stealing issue slots from the compute warps
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ------------------------------------------------------------------------------------------------
// named barriers (ids 1-15; id 0 is __syncthreads).  `threads` counts every thread of the sync and arrive sides.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t threads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------------------------------------
// thread-block clusters (CTA pairs of the GEMM)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// every thread of every CTA in the cluster (not necessarily warp-converged)
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster.  Default (.release.cta)
// semantics: the GEMM signals with it that its wgmma reads of a stage are complete (wgmma.wait_group), which orders
// nothing in the generic proxy.  A .release.cluster arrive fences at cluster scope on every call, and at one arrival per
// k-block that halved the CTA-pair GEMM's main-loop rate on an H100.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
        "}\n" ::"r"(smem_u32(bar)), "r"(cta)
        : "memory");
}

// generic-proxy smem writes -> visible to the async proxy (UMMA / TMA reads of smem)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// the same box written to the same shared-memory offset of every CTA in `cta_mask`, completing bytes on each CTA's
// mbarrier at the offset of `bar`
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                               uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}
// 1-D bulk copy global -> shared (bytes % 16 == 0, 16-byte aligned), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// smem tile --> global, through the TMA unit (out-of-bounds elements of the box are not written)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Programmatic dependent launch.  Every kernel launched through launch_k / launch_kc carries the programmatic-stream-
// serialization attribute, so the NEXT kernel in the stream (or graph) may be scheduled onto SMs as soon as every CTA of
// this grid has executed griddep_launch_dependents() (first statement of each kernel) and resources free up: its launch
// latency and prologue (barrier init, tensor-memory allocation, descriptor prefetch) overlap this grid's tail.
// griddep_wait() blocks until every prerequisite grid has COMPLETED and its memory is visible; each kernel executes it
// before its first global-memory access (reads of earlier results, and writes that earlier kernels might still read).
#ifndef B2D_NO_PDL
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#else
__device__ __forceinline__ void griddep_launch_dependents() {}
__device__ __forceinline__ void griddep_wait() {}
#endif

// explicit shared-space accesses by 32-bit address.  Pointers derived from the re-aligned dynamic smem base lose their
// address space, and the compiler then emits GENERIC LD.E/ST.E with 64-bit address arithmetic for them (seen in the
// attention consumers' SASS); these keep the hot loops on LDS/STS.  volatile: ordered after the mbarrier waits.
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
// Four 8 x 8 bf16 matrices per warp instruction: lane l gives the 16-byte row (l % 8) of matrix l / 8, and register k
// holds matrix k's elements (row lane / 4, columns 2 (lane % 4) + {0, 1}), the accumulator fragment of mma / wgmma.
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&v)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3])
                 : "r"(addr)
                 : "memory");
}
__device__ __forceinline__ void stsm_x4(uint32_t addr, const uint32_t (&v)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]),
                 "r"(v[2]), "r"(v[3])
                 : "memory");
}

// ------------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, 128-byte swizzle (layout type 1 at bits [62,64)).
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4      [32,46) stride byte offset >> 4
// K-major SW128  : rows are 128 B (64 bf16 of K); 8-row groups are SBO = 1024 B apart; LBO unused.
// MN-major SW128 : each K-row holds 64 contiguous MN elements (128 B); 8 K-rows = 1024 B atom;
//                  SBO = distance between 8-K-row groups (1024 B), LBO = distance between 64-element MN atoms (8 KB).
// The high word is a constant; the low word advances by one integer add per 16-element k-step.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t SDESC_HI_SW128 = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sdesc_lo_kmajor(uint32_t smem_addr) { return ((smem_addr & 0x3FFFF) >> 4) | (1u << 16); }
__device__ __forceinline__ uint32_t sdesc_lo_mnmajor(uint32_t smem_addr) { return ((smem_addr & 0x3FFFF) >> 4) | (512u << 16); }
// MN-major with an explicit distance between the 64-element MN atoms (N > 64 stored as 64-column panels)
__device__ __forceinline__ uint32_t sdesc_lo_mnmajor(uint32_t smem_addr, uint32_t lbo_bytes) {
    return ((smem_addr & 0x3FFFF) >> 4) | ((lbo_bytes >> 4) << 16);
}
constexpr uint32_t SDESC_KSTEP_KMAJOR = 32 >> 4;     // +16 K elements inside a 128 B row
constexpr uint32_t SDESC_KSTEP_MNMAJOR = 2048 >> 4;  // +16 K rows of 128 B
__device__ __forceinline__ uint64_t sdesc(uint32_t lo) { return ((uint64_t)SDESC_HI_SW128 << 32) | lo; }

// register budget per warpgroup (producer warpgroups give registers to the math warpgroups)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ------------------------------------------------------------------------------------------------
// small math / packing helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// GELU(tanh) and derivative, fp32, on the MUFU tanh unit (tanh.approx.f32: rel. error 2^-11, below bf16 resolution)
__device__ __forceinline__ float tanh_approx(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float gelu_tanh(float x) {
    const float k0 = 0.7978845608028654f, k0k1 = 0.7978845608028654f * 0.044715f;
    float x2 = x * x;
    float t = tanh_approx(x * fmaf(k0k1, x2, k0));
    float hx = 0.5f * x;
    return fmaf(hx, t, hx);
}
__device__ __forceinline__ float dgelu_tanh(float x) {
    const float k0 = 0.7978845608028654f, k0k1 = 0.7978845608028654f * 0.044715f;
    float x2 = x * x;
    float t = tanh_approx(x * fmaf(k0k1, x2, k0));
    float du = fmaf(3.f * k0k1, x2, k0);
    float s = fmaf(-t, t, 1.f);
    return fmaf(0.5f * x * s, du, fmaf(0.5f, t, 0.5f));
}
__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.f + __expf(-x)); }

}  // namespace b2d
