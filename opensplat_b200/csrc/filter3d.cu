// filter3d.cu -- Mip-Splatting's 3-D smoothing filter (DESIGN D24): the per-Gaussian filter value from the training
// cameras, the bake of the filter into a stored scene, and the filter-aware opacity reset.
//
// Built with --fmad=false: the filter value is the numpy fp32 restatement's bit for bit (tests/filter3d_f64.py), its
// view-space z the same expressions as project_forward_kernel's tz.  Min and max are exact, so the result does not
// depend on the order in which blocks finish: the largest seen depth is an integer atomicMax on the bits of positive
// floats.
#include <math.h>

#include "gsb_common.cuh"

namespace {

constexpr int FT = 256;
constexpr int CAM_CHUNK = 256;   // cameras staged in shared memory per pass

struct FCam {
    float V[12];                        // viewmat rows 0..2
    float fx, fy, cx, cy;
    float xlo, xhi, ylo, yhi;           // -(margin W), (1 + margin) W, -(margin H), (1 + margin) H
};

// d[i] = min over the cameras that see Gaussian i of its view-space z (+inf if none does); ws[0] = max bits of the
// finite d, ws[1] = max bits of fx (block 0 only)
__global__ void __launch_bounds__(FT) filter3d_depth_kernel(int n, const float *__restrict__ means, int num_cams,
                                                            const float *__restrict__ cams, float near, float margin,
                                                            float *__restrict__ d_out, unsigned *__restrict__ ws) {
    __shared__ FCam sc[CAM_CHUNK];
    __shared__ unsigned wmax[FT / 32];
    const int i = blockIdx.x * FT + threadIdx.x;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (i < n) {
        px = means[3 * i];
        py = means[3 * i + 1];
        pz = means[3 * i + 2];
    }
    float d = INFINITY;
    for (int c0 = 0; c0 < num_cams; c0 += CAM_CHUNK) {
        const int cn = min(CAM_CHUNK, num_cams - c0);
        __syncthreads();
        for (int j = threadIdx.x; j < cn; j += FT) {
            const float *c = cams + (size_t)GSB_FILTER3D_CAM_FLOATS * (c0 + j);
            FCam &s = sc[j];
#pragma unroll
            for (int k = 0; k < 12; ++k) s.V[k] = c[k];
            s.fx = c[12]; s.fy = c[13]; s.cx = c[14]; s.cy = c[15];
            const float W = c[16], H = c[17];
            s.xlo = -(margin * W); s.xhi = (1.f + margin) * W;
            s.ylo = -(margin * H); s.yhi = (1.f + margin) * H;
            if (blockIdx.x == 0) atomicMax(ws + 1, __float_as_uint(s.fx));
        }
        __syncthreads();
        if (i < n) {
            for (int j = 0; j < cn; ++j) {
                const FCam &s = sc[j];
                const float *V = s.V;
                const float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
                if (tz > near && tz < d) {   // a camera no nearer than the current minimum cannot change it
                    const float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
                    const float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
                    const float u = s.fx * (tx / tz) + s.cx, v = s.fy * (ty / tz) + s.cy;
                    if (u >= s.xlo && u <= s.xhi && v >= s.ylo && v <= s.yhi) d = tz;
                }
            }
        }
    }
    if (i < n) d_out[i] = d;
    unsigned b = (i < n && d < INFINITY) ? __float_as_uint(d) : 0u;   // d > near >= 0: the bits order as the floats
    b = __reduce_max_sync(0xffffffffu, b);
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned m = 0u;
#pragma unroll
        for (int w = 0; w < FT / 32; ++w) m = max(m, wmax[w]);
        if (m) atomicMax(ws, m);
    }
}

// f[i] = (d[i] / F) * S, an unseen Gaussian taking the largest seen d; every f = 0 when no Gaussian is seen
__global__ void __launch_bounds__(FT) filter3d_finish_kernel(int n, float S, const unsigned *__restrict__ ws,
                                                             float *__restrict__ f) {
    const int i = blockIdx.x * FT + threadIdx.x;
    if (i >= n) return;
    const unsigned mb = ws[0];
    float v = 0.f;
    if (mb != 0u) {
        float d = f[i];
        if (!(d < INFINITY)) d = __uint_as_float(mb);
        v = d / __uint_as_float(ws[1]) * S;
    }
    f[i] = v;
}

// log sigmoid(l) and sigmoid(-l) in fp64, without overflow for large |l|
__device__ __forceinline__ double log_sigmoid(double l) { return l < 0.0 ? l - log1p(exp(l)) : -log1p(exp(-l)); }
__device__ __forceinline__ double sigmoid(double l) {
    return l < 0.0 ? exp(l) / (1.0 + exp(l)) : 1.0 / (1.0 + exp(-l));
}

// a' = a + log1p((f / e)^2) / 2 = log(e^2 + f^2) / 2; l' = logit(sigmoid(l) c3) with log c3 = -sum log1p((f / e_k)^2) / 2,
// as log p - log(1 - p), 1 - p = sigmoid(-l) + sigmoid(l) (-expm1(log c3)); all in fp64, each rounded once.  In place
// is allowed (each element is read before it is written).
__global__ void __launch_bounds__(FT) filter3d_bake_kernel(int n, const float *log_scales, const float *logits,
                                                           const float *__restrict__ filter3d, float *out_log_scales,
                                                           float *out_logits) {
    const int i = blockIdx.x * FT + threadIdx.x;
    if (i >= n) return;
    const double f = filter3d[i];
    double lc = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double a = log_scales[3 * i + k];
        const double t = f * exp(-a), h = 0.5 * log1p(t * t);
        lc -= h;
        out_log_scales[3 * i + k] = (float)(a + h);
    }
    const double l = logits[i];
    const double logp = log_sigmoid(l) + lc;
    const double q = sigmoid(-l) + sigmoid(l) * -expm1(lc);
    out_logits[i] = (float)(logp - log(q));
}

// l' = min(l, logit(r / c3)) where r / c3 < 1 (logit in fp64, rounded once), l where r / c3 >= 1, and
// min(l, max_logit) -- gsb_reset_opacity's result -- where c3 == 1.  c3 is the projection's fp32 value at glob_scale 1.
__global__ void __launch_bounds__(FT) reset_opacity_filter3d_kernel(int n, float max_logit, float reset_value,
                                                                    const float *__restrict__ log_scales,
                                                                    const float *__restrict__ filter3d,
                                                                    float *__restrict__ opac, float *__restrict__ m,
                                                                    float *__restrict__ v) {
    const int i = blockIdx.x * FT + threadIdx.x;
    if (i >= n) return;
    const float f = filter3d[i], ff = f * f;
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float e = expf(log_scales[3 * i + k]);
        r[k] = e / sqrtf(e * e + ff);
    }
    const float c3 = r[0] * r[1] * r[2];
    const float l = opac[i];
    if (c3 == 1.f) {
        opac[i] = fminf(l, max_logit);
    } else {
        const double q = (double)reset_value / (double)c3;
        if (q < 1.0) opac[i] = fminf(l, (float)(log(q) - log1p(-q)));
    }
    if (m) m[i] = 0.f;
    if (v) v[i] = 0.f;
}

}  // namespace

extern "C" size_t gsb_filter3d_workspace_bytes(void) { return 2 * sizeof(unsigned); }

extern "C" int gsb_filter3d_compute(int n, const float *means, int num_cameras, const float *cameras, float near,
                                    float margin, float variance, void *workspace, size_t workspace_bytes,
                                    float *filter3d, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && num_cameras >= 1);
    GSB_CHECK_ARG(near >= 0.f && near < INFINITY && margin >= 0.f && margin < INFINITY && variance >= 0.f &&
                  variance < INFINITY);
    if (n == 0) return 0;
    GSB_CHECK_ARG(means && cameras && filter3d && workspace && workspace_bytes >= gsb_filter3d_workspace_bytes());
    GSB_CHECK_ARG(((uintptr_t)workspace % 4) == 0);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned *ws = static_cast<unsigned *>(workspace);
    GSB_CUDA(cudaMemsetAsync(ws, 0, gsb_filter3d_workspace_bytes(), st));
    const int blocks = gsb_div_up(n, FT);
    filter3d_depth_kernel<<<blocks, FT, 0, st>>>(n, means, num_cameras, cameras, near, margin, filter3d, ws);
    GSB_LAUNCH_CHECK();
    const float S = (float)sqrt((double)variance);
    filter3d_finish_kernel<<<blocks, FT, 0, st>>>(n, S, ws, filter3d);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_filter3d_bake(int n, const float *log_scales, const float *opacity_logits, const float *filter3d,
                                 float *out_log_scales, float *out_opacity_logits, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(log_scales && opacity_logits && filter3d && out_log_scales && out_opacity_logits);
    filter3d_bake_kernel<<<gsb_div_up(n, FT), FT, 0, (cudaStream_t)stream>>>(n, log_scales, opacity_logits, filter3d,
                                                                             out_log_scales, out_opacity_logits);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_reset_opacity_filter3d(int n, float max_logit, float reset_value, const float *log_scales,
                                          const float *filter3d, float *opacities, float *exp_avg, float *exp_avg_sq,
                                          gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(log_scales && filter3d && opacities);
    reset_opacity_filter3d_kernel<<<gsb_div_up(n, FT), FT, 0, (cudaStream_t)stream>>>(
        n, max_logit, reset_value, log_scales, filter3d, opacities, exp_avg, exp_avg_sq);
    GSB_LAUNCH_CHECK();
    return 0;
}
