// gsb_common.cuh -- shared device/host helpers for libgsplat_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/gsplat_b200.h"

#define GSB_VERSION 200

// ---- error plumbing (thread-local message, C ABI returns the code) -------------------------
void gsb_set_error(int code, const char *what, const char *file, int line);

#define GSB_CHECK_ARG(cond)                                                          \
    do {                                                                             \
        if (!(cond)) {                                                               \
            gsb_set_error(GSB_ERR_INVALID_ARG, "invalid argument: " #cond, __FILE__, __LINE__); \
            return GSB_ERR_INVALID_ARG;                                              \
        }                                                                            \
    } while (0)

#define GSB_CUDA(call)                                                               \
    do {                                                                             \
        cudaError_t e__ = (call);                                                    \
        if (e__ != cudaSuccess) {                                                    \
            gsb_set_error((int)e__, cudaGetErrorString(e__), __FILE__, __LINE__);    \
            return (int)e__;                                                         \
        }                                                                            \
    } while (0)

#define GSB_LAUNCH_CHECK() GSB_CUDA(cudaGetLastError())

static inline int gsb_div_up(int a, int b) { return (a + b - 1) / b; }
static inline size_t gsb_align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

#ifdef __CUDACC__
// ---- streaming loads/stores ------------------------------------------------------------------
__device__ __forceinline__ float4 ldg_stream4(const float4 *p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream4(float4 *p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- mbarrier + 1-D TMA bulk copy (cp.async.bulk -> SASS UBLKCP) ------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned; completes on `bar`.
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                            uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif  // __CUDACC__
