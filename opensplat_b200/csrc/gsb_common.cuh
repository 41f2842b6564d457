// gsb_common.cuh -- shared device/host helpers for libgsplat_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/gsplat_b200.h"

#define GSB_VERSION 800

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

// ---- warp / block scans of one int per thread --------------------------------------------------
__device__ __forceinline__ int warp_incl_scan(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// block-wide exclusive scan; returns the exclusive prefix and the block sum in *total.
// smem: THREADS/32 + 1 ints.
template <int THREADS>
__device__ __forceinline__ int block_excl_scan(int v, int *total, int *smem) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int inc = warp_incl_scan(v);
    if (lane == 31) smem[w] = inc;
    __syncthreads();
    if (w == 0) {
        const int x = (lane < THREADS / 32) ? smem[lane] : 0;
        const int xi = warp_incl_scan(x);
        if (lane < THREADS / 32) smem[lane] = xi - x;
        if (lane == 31) smem[THREADS / 32] = xi;
    }
    __syncthreads();
    const int res = smem[w] + inc - v;
    *total = smem[THREADS / 32];
    __syncthreads();
    return res;
}

// ---- tile bounding box of a projected Gaussian -------------------------------------------------
// get_tile_bbox (helpers.cuh:17-49): tiles [x0, x1) x [y0, y1) touched by the square of half-width
// `radius` around (cx, cy); (int) == cvt.rzi (saturating).  The projection (num_tiles_hit), both
// binning paths (keys, bins) and the blend records must agree on it bit for bit, so every one of
// them calls this; it contains no multiply-add, so --fmad does not change it.
__device__ __forceinline__ void gsb_tile_bbox(float cx, float cy, float radius, int tiles_x, int tiles_y,
                                              int &x0, int &x1, int &y0, int &y1) {
    const float tcx = cx / 16.f, tcy = cy / 16.f, tr = radius / 16.f;
    x0 = min(max(0, (int)(tcx - tr)), tiles_x);
    x1 = min(max(0, (int)(tcx + tr + 1.f)), tiles_x);
    y0 = min(max(0, (int)(tcy - tr)), tiles_y);
    y1 = min(max(0, (int)(tcy + tr + 1.f)), tiles_y);
}
#endif  // __CUDACC__
