// sh.cu -- spherical-harmonics colour evaluation, forward + VJP (S1/S2 of SURVEY.md section 8a).
//
// Replaces compute_sh_forward_kernel / compute_sh_backward_kernel (reference
// rasterizer/gsplat/sh.cuh:218-260, math :52-216).  Pure streaming work: 12+12K+12 bytes per
// Gaussian each way (K = number of SH bases), HBM-bound.  The reference reads the [N,K,3] AoS
// coefficient block with one thread per Gaussian (192-B stride between lanes at K=16).  Here a CTA
// moves its 128 Gaussians' coefficients as one contiguous span with 128-bit streaming accesses
// (fully coalesced, L1 bypassed) through a padded shared-memory transpose; rows are padded to
// 4*odd floats so the per-thread 128-bit row reads are bank-conflict free.  The multi-view forward stages the span
// once and evaluates it for several camera centres (a trainer's views of one step).
#include <type_traits>

#include "gsb_common.cuh"

int gsb_sm_count();

namespace {

constexpr int SH_THREADS = 128;

__host__ __device__ constexpr int sh_row_stride(int K) {
    int q = (3 * K + 3) / 4;
    return 4 * ((q & 1) ? q : q + 1);
}

// SH constants, sh.cuh:12-37.  ROUNDED_PRODUCTS: form the six second-order products with __fmul_rn, which the compiler
// never contracts into an FMA.  The single-view kernels compute them as separate multiplies; in the loop over views of
// sh_forward_multiview_kernel at K >= 16 the compiler would otherwise fold x * x into the subtractions of the degree-2
// and degree-3 bases, and its colours would no longer be bit-identical to gsb_sh_forward_rgb_cam's.  (At K = 9 the
// plain products contract as in the single-view kernel, and the rounded ones would not.)
template <bool ROUNDED_PRODUCTS = false>
__device__ __forceinline__ void sh_basis(int nb, float vx, float vy, float vz, float *Y) {
    Y[0] = 0.28209479177387814f;
    if (nb <= 1) return;
    // sh.cuh:67-72 normalises the direction inside the kernel
    float norm = sqrtf(vx * vx + vy * vy + vz * vz);
    float x = vx / norm, y = vy / norm, z = vz / norm;
    float xx, xy, xz, yy, yz, zz;
    if constexpr (ROUNDED_PRODUCTS) {
        xx = __fmul_rn(x, x); xy = __fmul_rn(x, y); xz = __fmul_rn(x, z);
        yy = __fmul_rn(y, y); yz = __fmul_rn(y, z); zz = __fmul_rn(z, z);
    } else {
        xx = x * x; xy = x * y; xz = x * z; yy = y * y; yz = y * z; zz = z * z;
    }
    Y[1] = -0.4886025119029199f * y;
    Y[2] = 0.4886025119029199f * z;
    Y[3] = -0.4886025119029199f * x;
    if (nb <= 4) return;
    Y[4] = 1.0925484305920792f * xy;
    Y[5] = -1.0925484305920792f * yz;
    Y[6] = 0.31539156525252005f * (2.f * zz - xx - yy);
    Y[7] = -1.0925484305920792f * xz;
    Y[8] = 0.5462742152960396f * (xx - yy);
    if (nb <= 9) return;
    Y[9] = -0.5900435899266435f * y * (3.f * xx - yy);
    Y[10] = 2.890611442640554f * xy * z;
    Y[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
    Y[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
    Y[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
    Y[14] = 1.445305721320277f * z * (xx - yy);
    Y[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
    if (nb <= 16) return;
    Y[16] = 2.5033429417967046f * xy * (xx - yy);
    Y[17] = -1.7701307697799304f * yz * (3.f * xx - yy);
    Y[18] = 0.9461746957575601f * xy * (7.f * zz - 1.f);
    Y[19] = -0.6690465435572892f * yz * (7.f * zz - 3.f);
    Y[20] = 0.10578554691520431f * (zz * (35.f * zz - 30.f) + 3.f);
    Y[21] = -0.6690465435572892f * xz * (7.f * zz - 3.f);
    Y[22] = 0.47308734787878004f * (xx - yy) * (7.f * zz - 1.f);
    Y[23] = -1.7701307697799304f * xz * (xx - 3.f * yy);
    Y[24] = 0.6258357354491761f * (xx * (xx - 3.f * yy) - yy * (3.f * xx - yy));
}

__device__ __forceinline__ int nb_of(int degrees_to_use) {
    return (degrees_to_use + 1) * (degrees_to_use + 1);
}

// rgbs = clamp_min(s, 0) with s = colour + bias (model.cpp:192), and the mask of its gradient (D17 of DESIGN.md).
// torch's clamp_min passes the gradient where s == min exactly, so the forward writes -0 at an exact tie and +0 below
// it; the mask passes where rgbs > 0 or rgbs is -0.  -0 == +0 wherever a colour is used (the blend kernels multiply
// and add it); only the mask reads the sign.  A +0 (e.g. torch.clamp_min's output) keeps the mask rgbs > 0.
__device__ __forceinline__ float clamp_rgb(float s) { return s > 0.f ? s : (s == 0.f ? -0.f : 0.f); }
__device__ __forceinline__ bool rgb_grad_passes(float rgb) { return rgb > 0.f || (rgb == 0.f && signbit(rgb)); }

template <int K>
__global__ void __launch_bounds__(SH_THREADS)
sh_forward_kernel(int n, int degrees_to_use, const float *__restrict__ viewdirs,
                  const float *__restrict__ coeffs, float *__restrict__ colors, int vec_ok, int fuse_rgb,
                  float bias,
                  // split inputs (gsb_sh_forward_split): coeffs = features_dc [n,3], rest = features_rest [n,K-1,3]
                  // (the two tensors Model::forward concatenates, model.cpp:186-188); cam_pos != NULL: `viewdirs`
                  // holds the MEANS and the direction means - cam_pos is formed here (model.cpp:176-177)
                  int split, const float *__restrict__ rest, const float *__restrict__ cam_pos) {
    constexpr int C = 3 * K;
    constexpr int S = sh_row_stride(K);
    __shared__ __align__(16) float tile[SH_THREADS * S];
    const int g0 = blockIdx.x * SH_THREADS;
    const int ng = min(SH_THREADS, n - g0);
    const int nb = min(nb_of(degrees_to_use), K);
    const float *src = coeffs + (size_t)g0 * C;
    const int total = ng * C;
    // ---- coalesced span load -> padded rows ----
    if (split) {
        const float *dc = coeffs + (size_t)g0 * 3, *rs = rest + (size_t)g0 * (C - 3);
        for (int e = threadIdx.x; e < ng * 3; e += SH_THREADS) tile[(e / 3) * S + (e % 3)] = __ldg(dc + e);
        if (C > 3)
            for (int e = threadIdx.x; e < ng * (C - 3); e += SH_THREADS) {
                const int g = e / (C - 3), j = e - g * (C - 3);
                tile[g * S + 3 + j] = __ldg(rs + e);
            }
    } else if (vec_ok && (C % 4 == 0)) {
        const float4 *src4 = reinterpret_cast<const float4 *>(src);
        for (int f = threadIdx.x; f < total / 4; f += SH_THREADS) {
            float4 v = ldg_stream4(src4 + f);
            int e = 4 * f, g = e / C, j = e - g * C;
            *reinterpret_cast<float4 *>(&tile[g * S + j]) = v;
        }
    } else {
        for (int e = threadIdx.x; e < total; e += SH_THREADS) {
            int g = e / C, j = e - g * C;
            tile[g * S + j] = __ldg(src + e);
        }
    }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= ng) return;
    const int g = g0 + t;
    float Y[K];
    {
        float vx = viewdirs[3 * g], vy = viewdirs[3 * g + 1], vz = viewdirs[3 * g + 2];
        if (cam_pos) { vx -= __ldg(cam_pos); vy -= __ldg(cam_pos + 1); vz -= __ldg(cam_pos + 2); }
        sh_basis(nb, vx, vy, vz, Y);
    }
    float row[S];
#pragma unroll
    for (int j = 0; j < S; j += 4) {
        float4 v = *reinterpret_cast<const float4 *>(&tile[t * S + j]);
        row[j] = v.x; row[j + 1] = v.y; row[j + 2] = v.z; row[j + 3] = v.w;
    }
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int b = 0; b < K; ++b) {
        if (b < nb) {
            c0 += Y[b] * row[3 * b];
            c1 += Y[b] * row[3 * b + 1];
            c2 += Y[b] * row[3 * b + 2];
        }
    }
    if (fuse_rgb) {  // fused glue of model.cpp:192: rgbs = clamp_min(colors + 0.5, 0), -0 at a tie
        c0 = clamp_rgb(c0 + bias);
        c1 = clamp_rgb(c1 + bias);
        c2 = clamp_rgb(c2 + bias);
    }
    colors[3 * g] = c0;
    colors[3 * g + 1] = c1;
    colors[3 * g + 2] = c2;
}

// Multi-view forward (a trainer's B camera views of one step): rgbs[v] = clamp_min(SH(means - cam_pos[v]) + bias, 0)
// for v < num_views.  The coefficient span of the CTA's 128 Gaussians is staged once through the same padded
// transpose as sh_forward_kernel and held in registers across the views, so the [n,K,3] block is read once per step
// instead of once per view.  Per view the arithmetic is sh_forward_kernel's with cam_pos (the same view direction,
// basis and accumulation order), so every view's rgbs are bit-identical to a gsb_sh_forward_rgb_cam call.
template <int K>
__global__ void __launch_bounds__(SH_THREADS)
sh_forward_multiview_kernel(int n, int degrees_to_use, const float *__restrict__ means, int num_views,
                            const float *__restrict__ cam_pos, const float *__restrict__ coeffs, float bias,
                            float *__restrict__ rgbs, int vec_ok) {
    constexpr int C = 3 * K;
    constexpr int S = sh_row_stride(K);
    __shared__ __align__(16) float tile[SH_THREADS * S];
    const int g0 = blockIdx.x * SH_THREADS;
    const int ng = min(SH_THREADS, n - g0);
    const int nb = min(nb_of(degrees_to_use), K);
    const float *src = coeffs + (size_t)g0 * C;
    const int total = ng * C;
    if (vec_ok && (C % 4 == 0)) {
        const float4 *src4 = reinterpret_cast<const float4 *>(src);
        for (int f = threadIdx.x; f < total / 4; f += SH_THREADS) {
            float4 v = ldg_stream4(src4 + f);
            int e = 4 * f, g = e / C, j = e - g * C;
            *reinterpret_cast<float4 *>(&tile[g * S + j]) = v;
        }
    } else {
        for (int e = threadIdx.x; e < total; e += SH_THREADS) {
            int g = e / C, j = e - g * C;
            tile[g * S + j] = __ldg(src + e);
        }
    }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= ng) return;
    const int g = g0 + t;
    const float mx = means[3 * g], my = means[3 * g + 1], mz = means[3 * g + 2];
    float row[S];
#pragma unroll
    for (int j = 0; j < S; j += 4) {
        float4 v = *reinterpret_cast<const float4 *>(&tile[t * S + j]);
        row[j] = v.x; row[j + 1] = v.y; row[j + 2] = v.z; row[j + 3] = v.w;
    }
    for (int view = 0; view < num_views; ++view) {
        float Y[K];
        {
            float vx = mx, vy = my, vz = mz;
            vx -= __ldg(cam_pos + 3 * view); vy -= __ldg(cam_pos + 3 * view + 1); vz -= __ldg(cam_pos + 3 * view + 2);
            sh_basis<(K >= 16)>(nb, vx, vy, vz, Y);
        }
        float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int b = 0; b < K; ++b) {
            if (b < nb) {
                c0 += Y[b] * row[3 * b];
                c1 += Y[b] * row[3 * b + 1];
                c2 += Y[b] * row[3 * b + 2];
            }
        }
        c0 = clamp_rgb(c0 + bias);
        c1 = clamp_rgb(c1 + bias);
        c2 = clamp_rgb(c2 + bias);
        float *out = rgbs + (size_t)view * 3 * n;
        out[3 * g] = c0;
        out[3 * g + 1] = c1;
        out[3 * g + 2] = c2;
    }
}

template <int K>
__global__ void __launch_bounds__(SH_THREADS)
sh_backward_kernel(int n, int degrees_to_use, const float *__restrict__ viewdirs,
                   const float *__restrict__ v_colors, float *__restrict__ v_coeffs, int vec_ok,
                   const float *__restrict__ rgb_mask,
                   // split outputs (gsb_sh_backward_split): v_coeffs = v_features_dc [n,3], v_rest [n,K-1,3];
                   // cam_pos != NULL: `viewdirs` holds the means
                   int split, float *__restrict__ v_rest, const float *__restrict__ cam_pos) {
    constexpr int C = 3 * K;
    constexpr int S = sh_row_stride(K);
    __shared__ __align__(16) float tile[SH_THREADS * S];
    const int g0 = blockIdx.x * SH_THREADS;
    const int ng = min(SH_THREADS, n - g0);
    const int nb = min(nb_of(degrees_to_use), K);
    const int t = threadIdx.x;
    if (t < ng) {
        const int g = g0 + t;
        float Y[K];
        {
            float vx = viewdirs[3 * g], vy = viewdirs[3 * g + 1], vz = viewdirs[3 * g + 2];
            if (cam_pos) { vx -= __ldg(cam_pos); vy -= __ldg(cam_pos + 1); vz -= __ldg(cam_pos + 2); }
            sh_basis(nb, vx, vy, vz, Y);
        }
        float v0 = v_colors[3 * g], v1 = v_colors[3 * g + 1], v2 = v_colors[3 * g + 2];
        if (rgb_mask) {  // gradient of clamp_min(colors + bias, 0): pass where the forward output was > 0 or -0
            v0 = rgb_grad_passes(rgb_mask[3 * g]) ? v0 : 0.f;
            v1 = rgb_grad_passes(rgb_mask[3 * g + 1]) ? v1 : 0.f;
            v2 = rgb_grad_passes(rgb_mask[3 * g + 2]) ? v2 : 0.f;
        }
        float row[S];
#pragma unroll
        for (int b = 0; b < K; ++b) {
            float yb = (b < nb) ? Y[b] : 0.f;  // bases above degrees_to_use stay 0 (bindings.cu:110)
            row[3 * b] = yb * v0;
            row[3 * b + 1] = yb * v1;
            row[3 * b + 2] = yb * v2;
        }
#pragma unroll
        for (int j = C; j < S; ++j) row[j] = 0.f;
#pragma unroll
        for (int j = 0; j < S; j += 4)
            *reinterpret_cast<float4 *>(&tile[t * S + j]) = make_float4(row[j], row[j + 1], row[j + 2], row[j + 3]);
    }
    __syncthreads();
    float *dst = v_coeffs + (size_t)g0 * C;
    const int total = ng * C;
    if (split) {
        float *dc = v_coeffs + (size_t)g0 * 3, *rs = v_rest + (size_t)g0 * (C - 3);
        for (int e = threadIdx.x; e < ng * 3; e += SH_THREADS) dc[e] = tile[(e / 3) * S + (e % 3)];
        if (C > 3)
            for (int e = threadIdx.x; e < ng * (C - 3); e += SH_THREADS) {
                const int g = e / (C - 3), j = e - g * (C - 3);
                rs[e] = tile[g * S + 3 + j];
            }
    } else if (vec_ok && (C % 4 == 0)) {
        float4 *dst4 = reinterpret_cast<float4 *>(dst);
        for (int f = threadIdx.x; f < total / 4; f += SH_THREADS) {
            int e = 4 * f, g = e / C, j = e - g * C;
            stg_stream4(dst4 + f, *reinterpret_cast<const float4 *>(&tile[g * S + j]));
        }
    } else {
        for (int e = threadIdx.x; e < total; e += SH_THREADS) {
            int g = e / C, j = e - g * C;
            dst[e] = tile[g * S + j];
        }
    }
}

// Multi-view SH VJP fused with the cross-GPU exchange (data-parallel training, SURVEY.md 8e): instead of
// all-reducing the [N,K,3] coefficient gradients (192 B/Gaussian at degree 3), every rank exposes only its
// view's colour gradient v_rgb_r [N,3] (12 B/Gaussian) in peer-mapped memory and THIS kernel forms
//   v_coeffs[g] = scale * sum_r Y(normalize(mean_g - cam_r)) (x) v_rgb_r[g]
// reading the peers' v_rgb_r directly over NVLink (P2P loads on mapped pointers) while it computes; the
// rank-1 structure of the SH VJP makes the local expansion exact.  NVLink traffic per rank drops from
// 2(G-1)/G x 192 B to (G-1) x 12 B per Gaussian and the separate sh_backward pass disappears.
// A CTA pulls each view's 1536-B span of its 128 Gaussians with fully coalesced loads (a warp request is one
// contiguous 128-B line of the peer's memory) into shared memory, all views of a batch in flight at once, then
// every thread expands its own Gaussian.
//
// The same launch also carries the all-reduce of the remaining per-Gaussian gradients (means, scales, quats,
// opacity: the `geom` prefix of the flat gradient buffer, 44 B/Gaussian): the first `geom_blocks` (4 x SMs) CTAs run a
// two-shot all-reduce in which rank r owns slice r -- with NVSwitch multicast (`geom_mc` != NULL) one
// multimem.ld_reduce pulls the sum of all ranks' copies through the switch and one multimem.st broadcasts the
// result to every rank; without multicast the slice is summed from / written to the peers' mapped pointers.
// The caller brackets the launch with two cross-rank barriers (inputs complete / results visible).
//
// Camera centres: PEER_CAMS = false reads view r's centre from a device [num_views,3] array (fixed when the exchange
// is built); PEER_CAMS = true from cam_pos[r], a device array of num_views pointers to 3 floats each that may be
// peer-mapped like v_rgb_views -- a trainer renders a different camera on every rank at every step, and each rank
// exposes this step's centre next to its colour gradient instead of gathering the centres with a collective.  Role A
// stages a batch's VB centres in shared memory once per CTA (3 x VB threads, one float each) so that the 128 threads
// of a CTA do not all load the same peer address, and every thread reads them into registers before the expansion:
// read inside the expansion loop instead, ptxas contracts three of the K = 16 basis' multiply-subtract pairs into
// FMAs differently from the PEER_CAMS = false kernel, and the gradients are no longer bit-identical to it.
template <bool PEER_CAMS>
using MvCamPos = typename std::conditional<PEER_CAMS, const float *const *, const float *>::type;

__device__ __forceinline__ float4 multimem_ld_reduce_add(const float *mc_ptr) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc_ptr) : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st(float *mc_ptr, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc_ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

constexpr int MV_MAX_RANKS = 16;   // peers the non-multicast all-reduce role can address

template <int K, bool PEER_CAMS>
__global__ void __launch_bounds__(SH_THREADS)
sh_backward_multiview_kernel(int n, int degrees_to_use, const float *__restrict__ means, int num_views,
                             MvCamPos<PEER_CAMS> __restrict__ cam_pos, const float *const *__restrict__ v_rgb_views,
                             float scale, float *__restrict__ v_coeffs, int vec_ok,
                             // ---- all-reduce role (geom_blocks == 0: none) ----
                             int geom_blocks, int rank, int world, long long geom_vec4,
                             float *const *__restrict__ geom_ranks, float *geom_mc) {
    constexpr int C = 3 * K;
    constexpr int S = sh_row_stride(K);
    constexpr int VB = (K > 16) ? 4 : 8;   // views staged per batch (48-KB static shared-memory budget)
    if ((int)blockIdx.x < geom_blocks) {
        // ---- role B: two-shot all-reduce of this rank's slice of the geometry gradients ----
        const long long chunk = (geom_vec4 + world - 1) / world;
        const long long lo = chunk * rank, hi = min(geom_vec4, lo + chunk);
        const long long stride = (long long)geom_blocks * SH_THREADS;
        if (geom_mc != nullptr) {
            // four independent switch reductions in flight per thread (each is a ~2-3 us NVLink round trip)
            constexpr int GU = 4;
            for (long long i0 = lo + (long long)blockIdx.x * SH_THREADS + threadIdx.x; i0 < hi; i0 += GU * stride) {
                float4 v[GU];
#pragma unroll
                for (int u = 0; u < GU; ++u)
                    if (i0 + u * stride < hi) v[u] = multimem_ld_reduce_add(geom_mc + 4 * (i0 + u * stride));
#pragma unroll
                for (int u = 0; u < GU; ++u)
                    if (i0 + u * stride < hi) {
                        v[u].x *= scale; v[u].y *= scale; v[u].z *= scale; v[u].w *= scale;
                        multimem_st(geom_mc + 4 * (i0 + u * stride), v[u]);
                    }
            }
        } else {
            for (long long i = lo + (long long)blockIdx.x * SH_THREADS + threadIdx.x; i < hi; i += stride) {
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                float4 part[MV_MAX_RANKS];
#pragma unroll
                for (int r = 0; r < MV_MAX_RANKS; ++r)
                    if (r < world) part[r] = *(reinterpret_cast<const float4 *>(geom_ranks[r]) + i);
#pragma unroll
                for (int r = 0; r < MV_MAX_RANKS; ++r)
                    if (r < world) { acc.x += part[r].x; acc.y += part[r].y; acc.z += part[r].z; acc.w += part[r].w; }
                acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
#pragma unroll
                for (int r = 0; r < MV_MAX_RANKS; ++r)
                    if (r < world) *(reinterpret_cast<float4 *>(geom_ranks[r]) + i) = acc;
            }
        }
        return;
    }
    // ---- role A: multi-view SH VJP with peer pulls ----
    __shared__ __align__(16) float tile[SH_THREADS * S];
    __shared__ float stage[VB][3 * SH_THREADS];
    __shared__ float cam_stage[3 * VB];          // PEER_CAMS: this batch's camera centres
    const int blk = (int)blockIdx.x - geom_blocks;
    const int g0 = blk * SH_THREADS;
    const int ng = min(SH_THREADS, n - g0);
    const int nb = min(nb_of(degrees_to_use), K);
    const int t = threadIdx.x;
    const int g = g0 + t;
    float mx = 0.f, my = 0.f, mz = 0.f;
    if (t < ng) { mx = means[3 * g]; my = means[3 * g + 1]; mz = means[3 * g + 2]; }
    float row[S];
#pragma unroll
    for (int j = 0; j < S; ++j) row[j] = 0.f;
    const int span = 3 * ng;                     // floats of one view's colour-gradient span of this CTA
    for (int r0 = 0; r0 < num_views; r0 += VB) {
        // coalesced pull: thread t takes floats t, t+128, t+256 of every view's span; all loads of the batch are
        // issued before the first use, so the (NVLink) latency is paid once per batch
        float pull[VB][3];
#pragma unroll
        for (int u = 0; u < VB; ++u) {
            pull[u][0] = pull[u][1] = pull[u][2] = 0.f;
            if (r0 + u < num_views) {
                const float *vr = v_rgb_views[r0 + u] + (size_t)3 * g0;   // local or peer-mapped pointer
#pragma unroll
                for (int q = 0; q < 3; ++q)
                    if (t + q * SH_THREADS < span) pull[u][q] = vr[t + q * SH_THREADS];
            }
        }
        float cam_pull = 0.f;
        if constexpr (PEER_CAMS) {
            if (t < 3 * VB && r0 + t / 3 < num_views) cam_pull = cam_pos[r0 + t / 3][t % 3];   // local or peer-mapped
        }
        __syncthreads();   // the previous batch has been consumed
#pragma unroll
        for (int u = 0; u < VB; ++u)
#pragma unroll
            for (int q = 0; q < 3; ++q) stage[u][t + q * SH_THREADS] = pull[u][q];
        if constexpr (PEER_CAMS) {
            if (t < 3 * VB) cam_stage[t] = cam_pull;
        }
        __syncthreads();
        float cam_x[VB], cam_y[VB], cam_z[VB];   // PEER_CAMS: the batch's centres, read from shared memory once
        if constexpr (PEER_CAMS) {
#pragma unroll
            for (int u = 0; u < VB; ++u) {
                cam_x[u] = cam_stage[3 * u]; cam_y[u] = cam_stage[3 * u + 1]; cam_z[u] = cam_stage[3 * u + 2];
            }
        }
        if (t < ng) {
#pragma unroll
            for (int u = 0; u < VB; ++u) {
                if (r0 + u >= num_views) break;
                const float v0 = stage[u][3 * t], v1 = stage[u][3 * t + 1], v2 = stage[u][3 * t + 2];
                if (v0 == 0.f && v1 == 0.f && v2 == 0.f) continue;  // not visible in this view
                const int r = r0 + u;
                float Y[K];
                if constexpr (PEER_CAMS)
                    sh_basis(nb, mx - cam_x[u], my - cam_y[u], mz - cam_z[u], Y);
                else
                    sh_basis(nb, mx - __ldg(cam_pos + 3 * r), my - __ldg(cam_pos + 3 * r + 1),
                             mz - __ldg(cam_pos + 3 * r + 2), Y);
#pragma unroll
                for (int b = 0; b < K; ++b) {
                    if (b < nb) {
                        row[3 * b] = fmaf(Y[b], v0, row[3 * b]);
                        row[3 * b + 1] = fmaf(Y[b], v1, row[3 * b + 1]);
                        row[3 * b + 2] = fmaf(Y[b], v2, row[3 * b + 2]);
                    }
                }
            }
        }
    }
    if (t < ng) {
#pragma unroll
        for (int j = 0; j < S; j += 4)
            *reinterpret_cast<float4 *>(&tile[t * S + j]) =
                make_float4(scale * row[j], scale * row[j + 1], scale * row[j + 2], scale * row[j + 3]);
    }
    __syncthreads();
    float *dst = v_coeffs + (size_t)g0 * C;
    const int total = ng * C;
    if (vec_ok && (C % 4 == 0)) {
        float4 *dst4 = reinterpret_cast<float4 *>(dst);
        for (int f = threadIdx.x; f < total / 4; f += SH_THREADS) {
            int e = 4 * f, gg = e / C, j = e - gg * C;
            stg_stream4(dst4 + f, *reinterpret_cast<const float4 *>(&tile[gg * S + j]));
        }
    } else {
        for (int e = threadIdx.x; e < total; e += SH_THREADS) {
            int gg = e / C, j = e - gg * C;
            dst[e] = tile[gg * S + j];
        }
    }
}

__global__ void __launch_bounds__(256)
mask_rgb_grad_kernel(long long n3, const float *__restrict__ rgbs, float *__restrict__ v_rgbs) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n3 && !rgb_grad_passes(rgbs[i])) v_rgbs[i] = 0.f;
}

int bases_of_degree(int degree) {
    switch (degree) {
        case 0: return 1;
        case 1: return 4;
        case 2: return 9;
        case 3: return 16;
        case 4: return 25;
        default: return -1;
    }
}

}  // namespace

static int launch_sh_forward(int n, int degree, int degrees_to_use, const float *viewdirs, const float *coeffs,
                             float *colors, int fuse_rgb, float bias, gsb_stream_t stream, int split = 0,
                             const float *rest = nullptr, const float *cam_pos = nullptr) {
    GSB_CHECK_ARG(n >= 0 && bases_of_degree(degree) > 0 && degrees_to_use >= 0 && degrees_to_use <= degree);
    if (n == 0) return 0;
    GSB_CHECK_ARG(viewdirs && coeffs && colors);
    cudaStream_t s = (cudaStream_t)stream;
    int grid = gsb_div_up(n, SH_THREADS);
    int vec_ok = ((uintptr_t)coeffs % 16) == 0;
#define GSB_SH_F(K) sh_forward_kernel<K><<<grid, SH_THREADS, 0, s>>>(n, degrees_to_use, viewdirs, coeffs, colors, vec_ok, fuse_rgb, bias, split, rest, cam_pos)
    switch (degree) {
        case 0: GSB_SH_F(1); break;
        case 1: GSB_SH_F(4); break;
        case 2: GSB_SH_F(9); break;
        case 3: GSB_SH_F(16); break;
        default: GSB_SH_F(25); break;
    }
#undef GSB_SH_F
    GSB_LAUNCH_CHECK();
    return 0;
}

static int launch_sh_backward(int n, int degree, int degrees_to_use, const float *viewdirs, const float *v_colors,
                              float *v_coeffs, const float *rgb_mask, gsb_stream_t stream, int split = 0,
                              float *v_rest = nullptr, const float *cam_pos = nullptr) {
    GSB_CHECK_ARG(n >= 0 && bases_of_degree(degree) > 0 && degrees_to_use >= 0 && degrees_to_use <= degree);
    if (n == 0) return 0;
    GSB_CHECK_ARG(viewdirs && v_colors && v_coeffs);
    cudaStream_t s = (cudaStream_t)stream;
    int grid = gsb_div_up(n, SH_THREADS);
    int vec_ok = ((uintptr_t)v_coeffs % 16) == 0;
#define GSB_SH_B(K) sh_backward_kernel<K><<<grid, SH_THREADS, 0, s>>>(n, degrees_to_use, viewdirs, v_colors, v_coeffs, vec_ok, rgb_mask, split, v_rest, cam_pos)
    switch (degree) {
        case 0: GSB_SH_B(1); break;
        case 1: GSB_SH_B(4); break;
        case 2: GSB_SH_B(9); break;
        case 3: GSB_SH_B(16); break;
        default: GSB_SH_B(25); break;
    }
#undef GSB_SH_B
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_sh_forward(int n, int degree, int degrees_to_use, const float *viewdirs,
                              const float *coeffs, float *colors, gsb_stream_t stream) {
    return launch_sh_forward(n, degree, degrees_to_use, viewdirs, coeffs, colors, 0, 0.f, stream);
}

extern "C" int gsb_sh_backward(int n, int degree, int degrees_to_use, const float *viewdirs,
                               const float *v_colors, float *v_coeffs, gsb_stream_t stream) {
    return launch_sh_backward(n, degree, degrees_to_use, viewdirs, v_colors, v_coeffs, nullptr, stream);
}

// Fused variants (SURVEY.md 8f row 1): rgbs = clamp_min(SH(coeffs) + bias, 0) in one pass (model.cpp:188-192)
// and its VJP: v_coeffs = Y (x) (v_rgbs * [rgbs > 0 or rgbs is -0]) (D17: -0 marks an exact tie).
extern "C" int gsb_sh_forward_rgb(int n, int degree, int degrees_to_use, const float *viewdirs,
                                  const float *coeffs, float bias, float *rgbs, gsb_stream_t stream) {
    return launch_sh_forward(n, degree, degrees_to_use, viewdirs, coeffs, rgbs, 1, bias, stream);
}

extern "C" int gsb_sh_backward_rgb(int n, int degree, int degrees_to_use, const float *viewdirs,
                                   const float *rgbs, const float *v_rgbs, float *v_coeffs,
                                   gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || rgbs);
    return launch_sh_backward(n, degree, degrees_to_use, viewdirs, v_rgbs, v_coeffs, rgbs, stream);
}

// Split variants (SURVEY.md 8f row 1, the rest of it): the colour pass of Model::forward without its ATen glue --
//   viewdirs = means - cam_pos (detached; normalised inside like the reference kernel), coeffs =
//   cat(featuresDc[:,None,:], featuresRest) (model.cpp:176-177,186-188: a 12K B/Gaussian copy forward and a split
//   backward in autograd), rgbs = clamp_min(SH + bias, 0) (:192) -- reading the two feature tensors where they lie and
//   writing their two gradients directly.
extern "C" int gsb_sh_forward_split(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                                    const float *features_dc, const float *features_rest, float bias, float *rgbs,
                                    gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || (cam_pos && features_dc && (degree == 0 || features_rest)));
    return launch_sh_forward(n, degree, degrees_to_use, means, features_dc, rgbs, 1, bias, stream, 1, features_rest,
                             cam_pos);
}

extern "C" int gsb_sh_backward_split(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                                     const float *rgbs, const float *v_rgbs, float *v_features_dc,
                                     float *v_features_rest, gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || (cam_pos && rgbs && v_features_dc && (degree == 0 || v_features_rest)));
    return launch_sh_backward(n, degree, degrees_to_use, means, v_rgbs, v_features_dc, rgbs, stream, 1,
                              v_features_rest, cam_pos);
}

// Camera variants: the split variants' view directions (means - cam_pos, formed in the kernel) on the merged
// [n,K,3] coefficient block of the flat parameter layout.  Same kernels and arithmetic as the split variants; only
// the coefficient rows are moved as one span instead of two.
extern "C" int gsb_sh_forward_rgb_cam(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                                      const float *coeffs, float bias, float *rgbs, gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || cam_pos);
    return launch_sh_forward(n, degree, degrees_to_use, means, coeffs, rgbs, 1, bias, stream, 0, nullptr, cam_pos);
}

extern "C" int gsb_sh_backward_rgb_cam(int n, int degree, int degrees_to_use, const float *means,
                                       const float *cam_pos, const float *rgbs, const float *v_rgbs, float *v_coeffs,
                                       gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || (cam_pos && rgbs));
    return launch_sh_backward(n, degree, degrees_to_use, means, v_rgbs, v_coeffs, rgbs, stream, 0, nullptr, cam_pos);
}

// Several camera views at once: gsb_sh_forward_rgb_cam for each of the num_views centres of cam_positions [V,3],
// into rgbs [V,n,3], with one read of the coefficient block.
extern "C" int gsb_sh_forward_rgb_cam_multiview(int n, int degree, int degrees_to_use, const float *means,
                                                int num_views, const float *cam_positions, const float *coeffs,
                                                float bias, float *rgbs, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && num_views >= 1 && bases_of_degree(degree) > 0 && degrees_to_use >= 0 &&
                  degrees_to_use <= degree);
    if (n == 0) return 0;
    GSB_CHECK_ARG(means && cam_positions && coeffs && rgbs);
    cudaStream_t s = (cudaStream_t)stream;
    int grid = gsb_div_up(n, SH_THREADS);
    int vec_ok = ((uintptr_t)coeffs % 16) == 0;
#define GSB_SH_FM(K) sh_forward_multiview_kernel<K><<<grid, SH_THREADS, 0, s>>>(n, degrees_to_use, means, num_views, cam_positions, coeffs, bias, rgbs, vec_ok)
    switch (degree) {
        case 0: GSB_SH_FM(1); break;
        case 1: GSB_SH_FM(4); break;
        case 2: GSB_SH_FM(9); break;
        case 3: GSB_SH_FM(16); break;
        default: GSB_SH_FM(25); break;
    }
#undef GSB_SH_FM
    GSB_LAUNCH_CHECK();
    return 0;
}

// In-place gradient of clamp_min(. , 0): v_rgbs *= [rgbs > 0 or rgbs is -0] (D17; what gsb_sh_backward_rgb does
// internally; needed separately when the SH VJP runs in the fused multi-view kernel).
extern "C" int gsb_mask_rgb_grad(int n, const float *rgbs, float *v_rgbs, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(rgbs && v_rgbs);
    const long long n3 = 3ll * n;
    mask_rgb_grad_kernel<<<(unsigned)((n3 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n3, rgbs, v_rgbs);
    GSB_LAUNCH_CHECK();
    return 0;
}

template <bool PEER_CAMS>
static int launch_multiview(int n, int degree, int degrees_to_use, const float *means, int num_views,
                            MvCamPos<PEER_CAMS> cam_positions, const float *const *v_rgbs_per_view, float scale,
                            float *v_coeffs, int rank, int world, long long geom_floats, float *const *geom_per_rank,
                            float *geom_multicast, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && bases_of_degree(degree) > 0 && degrees_to_use >= 0 && degrees_to_use <= degree);
    GSB_CHECK_ARG(num_views >= 1 && geom_floats >= 0);
    int geom_blocks = 0;
    if (geom_floats > 0) {
        GSB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world && (geom_floats % 4) == 0);
        GSB_CHECK_ARG(geom_multicast || (geom_per_rank && world <= MV_MAX_RANKS));
        GSB_CHECK_ARG(((uintptr_t)geom_multicast % 16) == 0);
        // about two rounds of four 16-byte reductions per thread; between 1 and 8 CTAs per SM.  (The role is bound
        // by the switch, so fewer CTAs leave more slots to the colour half.)
        const int sms = gsb_sm_count();
        const long long slice = (geom_floats / 4 + world - 1) / world;
        const long long want = (slice + 2 * 4 * SH_THREADS - 1) / (2 * 4 * SH_THREADS);
        geom_blocks = (int)(want < sms ? sms : (want > 8LL * sms ? 8LL * sms : want));
    }
    if (n == 0 && geom_blocks == 0) return 0;
    GSB_CHECK_ARG(n == 0 || (means && cam_positions && v_rgbs_per_view && v_coeffs));
    cudaStream_t s = (cudaStream_t)stream;
    int grid = geom_blocks + gsb_div_up(n, SH_THREADS);
    int vec_ok = ((uintptr_t)v_coeffs % 16) == 0;
#define GSB_SH_M(K) sh_backward_multiview_kernel<K, PEER_CAMS><<<grid, SH_THREADS, 0, s>>>(n, degrees_to_use, means, num_views, cam_positions, v_rgbs_per_view, scale, v_coeffs, vec_ok, geom_blocks, rank, world, geom_floats / 4, geom_per_rank, geom_multicast)
    switch (degree) {
        case 0: GSB_SH_M(1); break;
        case 1: GSB_SH_M(4); break;
        case 2: GSB_SH_M(9); break;
        case 3: GSB_SH_M(16); break;
        default: GSB_SH_M(25); break;
    }
#undef GSB_SH_M
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_sh_backward_multiview(int n, int degree, int degrees_to_use, const float *means,
                                         int num_views, const float *cam_positions,
                                         const float *const *v_rgbs_per_view, float scale, float *v_coeffs,
                                         gsb_stream_t stream) {
    return launch_multiview<false>(n, degree, degrees_to_use, means, num_views, cam_positions, v_rgbs_per_view,
                                   scale, v_coeffs, 0, 1, 0, nullptr, nullptr, stream);
}

extern "C" int gsb_exchange_gradients(int n, int degree, int degrees_to_use, const float *means, int num_views,
                                      const float *cam_positions, const float *const *v_rgbs_per_view, float scale,
                                      float *v_coeffs, int rank, int world, long long geom_floats,
                                      float *const *geom_per_rank, float *geom_multicast, gsb_stream_t stream) {
    return launch_multiview<false>(n, degree, degrees_to_use, means, num_views, cam_positions, v_rgbs_per_view,
                                   scale, v_coeffs, rank, world, geom_floats, geom_per_rank, geom_multicast, stream);
}

// Per-step camera centres: the two entry points above with view r's centre read from cam_pos_per_view[r] (a device
// array of num_views device pointers to 3 floats, local or peer-mapped) instead of a [num_views,3] array.
extern "C" int gsb_sh_backward_multiview_cams(int n, int degree, int degrees_to_use, const float *means,
                                              int num_views, const float *const *cam_pos_per_view,
                                              const float *const *v_rgbs_per_view, float scale, float *v_coeffs,
                                              gsb_stream_t stream) {
    return launch_multiview<true>(n, degree, degrees_to_use, means, num_views, cam_pos_per_view, v_rgbs_per_view,
                                  scale, v_coeffs, 0, 1, 0, nullptr, nullptr, stream);
}

extern "C" int gsb_exchange_gradients_cams(int n, int degree, int degrees_to_use, const float *means, int num_views,
                                           const float *const *cam_pos_per_view,
                                           const float *const *v_rgbs_per_view, float scale, float *v_coeffs,
                                           int rank, int world, long long geom_floats, float *const *geom_per_rank,
                                           float *geom_multicast, gsb_stream_t stream) {
    return launch_multiview<true>(n, degree, degrees_to_use, means, num_views, cam_pos_per_view, v_rgbs_per_view,
                                  scale, v_coeffs, rank, world, geom_floats, geom_per_rank, geom_multicast, stream);
}
