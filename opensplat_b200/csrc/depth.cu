// depth.cu -- supervision of the rendered inverse depth by a per-image prior (DESIGN D23; graphdeco 3DGS's depth
// regularisation, gsplat's depth_loss): the per-Gaussian value stream 1/z the depth blend renders, the masked L1
// against the prior with its gradient, the chain back to the projection's depth, and the mean-pool levels of a prior.
//
// Every rounding is spelled out (__fdiv_rn, __fmul_rn, __fadd_rn) and the file is built with --fmad=false, so the
// results are the numpy fp32 restatement's bit for bit, except the loss value: a fixed-order fp64 reduction rounded
// once (the same inputs give the same bits; no float atomics).  A prior sample p is valid iff it is finite and > 0.
#include "gsb_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int L1_MAX_BLOCKS = 1024;   // the loss's partial sums: one per block, summed in block order

__device__ __forceinline__ bool valid_prior(float p) { return p > 0.f && p <= 3.402823466e38f; }

__global__ void inverse_depths_kernel(int n, const float *__restrict__ depths, const int32_t *__restrict__ radii,
                                      float *__restrict__ inv) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    if (i >= n) return;
    inv[i] = radii[i] > 0 ? __fdiv_rn(1.f, depths[i]) : 0.f;
}

// inv = 1/z: d inv / dz = -inv^2, taken as -((v_inv * inv) * inv) with inv recomputed as in the forward
__global__ void inverse_depths_backward_kernel(int n, const float *__restrict__ depths,
                                               const int32_t *__restrict__ radii, const float *__restrict__ v_inv,
                                               float *__restrict__ v_z) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    if (i >= n) return;
    float g = 0.f;
    if (radii[i] > 0) {
        const float inv = __fdiv_rn(1.f, depths[i]);
        g = -__fmul_rn(__fmul_rn(v_inv[i], inv), inv);
    }
    v_z[i] = g;
}

// fixed-order block sum of one double per thread: shuffle tree per warp, then the warps in order
__device__ double block_sum(double v, double *smem) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) smem[w] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int k = 0; k < THREADS / 32; ++k) s += smem[k];
    return s;
}

// v_rendered = g sgn(R - P) on valid pixels (sgn(0) = 0), 0 elsewhere; partials[block] = sum |R - P| over its
// valid pixels (|R - P| rounded to fp32, summed in fp64 in a fixed order)
__global__ void __launch_bounds__(THREADS) inverse_depth_l1_kernel(int count, const float *__restrict__ rendered,
                                                                   const float *__restrict__ prior, float g,
                                                                   float *__restrict__ v_rendered,
                                                                   double *__restrict__ partials) {
    __shared__ double smem[THREADS / 32];
    double acc = 0.0;
    for (int i = blockIdx.x * THREADS + threadIdx.x; i < count; i += gridDim.x * THREADS) {
        const float r = rendered[i], p = prior[i];
        float v = 0.f;
        if (valid_prior(p)) {
            acc += (double)fabsf(__fsub_rn(r, p));
            v = r > p ? g : (r < p ? -g : 0.f);
        }
        v_rendered[i] = v;
    }
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(THREADS) inverse_depth_l1_finish_kernel(int nblocks,
                                                                          const double *__restrict__ partials,
                                                                          double count, float *__restrict__ loss_out) {
    __shared__ double smem[THREADS / 32];
    double acc = 0.0;
    for (int k = threadIdx.x; k < nblocks; k += THREADS) acc += partials[k];
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) *loss_out = (float)(s / count);
}

// dst[y, x] = the mean of the valid samples of src's factor x factor block at (y, x): summed in fp32 in row-major
// order, divided by their count; 0 when the block has none
__global__ void depth_downscale_mean_kernel(int w, int factor, int dw, long long total, const float *__restrict__ src,
                                            float *__restrict__ dst) {
    const long long o = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (o >= total) return;
    const long long y = o / dw, x = o - y * dw;
    float s = 0.f;
    int c = 0;
    for (int j = 0; j < factor; ++j) {
        const float *row = src + (y * factor + j) * (long long)w + x * factor;
        for (int i = 0; i < factor; ++i) {
            const float p = row[i];
            if (valid_prior(p)) {
                s = __fadd_rn(s, p);
                ++c;
            }
        }
    }
    dst[o] = c > 0 ? __fdiv_rn(s, (float)c) : 0.f;
}

int l1_blocks(int count) { return min(gsb_div_up(count, THREADS), L1_MAX_BLOCKS); }

}  // namespace

extern "C" int gsb_inverse_depths(int n, const float *depths, const int32_t *radii, float *inv, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(depths && radii && inv);
    inverse_depths_kernel<<<gsb_div_up(n, THREADS), THREADS, 0, (cudaStream_t)stream>>>(n, depths, radii, inv);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_inverse_depths_backward(int n, const float *depths, const int32_t *radii, const float *v_inv,
                                           float *v_z, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(depths && radii && v_inv && v_z);
    inverse_depths_backward_kernel<<<gsb_div_up(n, THREADS), THREADS, 0, (cudaStream_t)stream>>>(n, depths, radii,
                                                                                                  v_inv, v_z);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t gsb_inverse_depth_l1_workspace_bytes(int img_h, int img_w) {
    if (img_h < 1 || img_w < 1 || (long long)img_h * img_w > 0x7fffffffLL) return 0;
    return gsb_align_up(sizeof(double) * (size_t)l1_blocks(img_h * img_w), 256);
}

extern "C" int gsb_inverse_depth_l1(int img_h, int img_w, const float *rendered, const float *prior, float scale_g,
                                    float *v_rendered, float *loss_out, void *workspace, size_t workspace_bytes,
                                    gsb_stream_t stream) {
    GSB_CHECK_ARG(img_h >= 1 && img_w >= 1 && (long long)img_h * img_w <= 0x7fffffffLL);
    GSB_CHECK_ARG(rendered && prior && v_rendered && loss_out && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace & 7) == 0);
    const int count = img_h * img_w, nb = l1_blocks(count);
    GSB_CHECK_ARG(workspace_bytes >= sizeof(double) * (size_t)nb);
    double *partials = (double *)workspace;
    inverse_depth_l1_kernel<<<nb, THREADS, 0, (cudaStream_t)stream>>>(count, rendered, prior, scale_g, v_rendered,
                                                                      partials);
    GSB_LAUNCH_CHECK();
    inverse_depth_l1_finish_kernel<<<1, THREADS, 0, (cudaStream_t)stream>>>(nb, partials, (double)count, loss_out);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_depth_downscale_mean(int h, int w, int factor, const float *src, float *dst, gsb_stream_t stream) {
    GSB_CHECK_ARG(factor >= 1 && h >= factor && w >= factor);
    GSB_CHECK_ARG(src && dst);
    const int dh = h / factor, dw = w / factor;
    const long long total = (long long)dh * dw;
    const long long blocks = (total + THREADS - 1) / THREADS;
    GSB_CHECK_ARG(blocks <= 0x7fffffffLL);
    depth_downscale_mean_kernel<<<(unsigned)blocks, THREADS, 0, (cudaStream_t)stream>>>(w, factor, dw, total, src,
                                                                                         dst);
    GSB_LAUNCH_CHECK();
    return 0;
}
