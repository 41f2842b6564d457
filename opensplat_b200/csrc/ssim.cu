// ssim.cu -- fused training loss (1-w) L1 + w (1 - SSIM) with its gradient w.r.t. the rendered image
// ("next" row 2 of SURVEY.md section 8f).
//
// Replaces, for the loss of Model::mainLoss (reference model.cpp:780-784): SSIM::eval (ssim.cpp:8-32 --
// five grouped 11x11 conv2d + ~15 elementwise ATen kernels), torch::l1_loss, and the autograd backward of
// all of them (~40 kernel launches, every intermediate a full [1,3,H,W] tensor in HBM) by TWO kernels:
//   ssim_forward_kernel : per 16x16 tile, both images' 26x26 halo -> shared memory, separable 11-tap
//                         window -> mu, sigma terms -> SSIM map; accumulates sum(SSIM) and sum|r - g|,
//                         writes the three partial-derivative maps dS/d(G*y), dS/d(G*y^2), dS/d(G*xy)
//   ssim_backward_kernel: per tile, the three maps' halo -> separable TRANSPOSED window ->
//                         v_rendered = -w/count (..) + (1-w)/count sign(r - g)
// Semantics follow the reference exactly, including its window: gaussian(1.5) evaluated at
// floor((i - 11)/2), i = 0..10 (ssim.cpp:41-47) -- an asymmetric staircase, NOT a centred Gaussian --
// zero padding of 5 (conv2d padding = windowSize/2), C1 = 0.01^2, C2 = 0.03^2, mean over [1,3,H,W].
// Images are [H,W,3] channels-last as the rasterizer produces them (the reference permutes, ssim.cpp:9-10);
// the kernels treat a row as 3W interleaved floats with horizontal taps 3 floats apart.
// HBM-bound by construction: reads 2 images + writes 3 maps (fwd), reads 3 maps + 2 images + writes 1 (bwd).
//
// gsb_ssim_l1_loss_masked (DESIGN D26) runs the same two kernels with MASK = true: a u8 [H,W] mask (nonzero = used)
// selects both images' halos (ignored content reads as 0, so nothing from it -- NaN or inf included -- reaches a used
// pixel's window), the forward keeps S, |y - x| and the three maps only on used pixels and counts them (N, an
// integer), the finalize kernel turns N into the two gradient scales on the device, and the backward reads them
// there and writes 0 on ignored pixels.  With MASK = false the kernels are the unmasked ones, instruction for
// instruction.
#include "gsb_common.cuh"

namespace {

constexpr int SS_T = 16;           // tile edge (pixels)
constexpr int SS_R = 5;            // window radius (windowSize 11)
constexpr int SS_H = SS_T + 2 * SS_R;   // halo edge = 26
constexpr int SS_ROW = SS_H * 3;        // floats per halo row (3 channels interleaved) = 78
constexpr int SS_OUT = SS_T * 3;        // floats per output row = 48

struct SsimWindow {
    float w[11];
};

__device__ __forceinline__ float block_sum_256(float v, float *sm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    if (threadIdx.x < 8) {
        r = sm[threadIdx.x];
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) r += __shfl_xor_sync(0xffu, r, o);
    }
    __syncthreads();
    return r;  // valid in thread 0
}

// loads the (zero padded) halo of an [H,W,3] image around tile (tx,ty) into sm[SS_H][SS_ROW]
__device__ __forceinline__ void load_halo(const float *__restrict__ img, int H, int W, int x0, int y0, float *sm) {
    for (int i = threadIdx.x; i < SS_H * SS_ROW; i += 256) {
        const int r = i / SS_ROW, cflt = i - r * SS_ROW;
        const int y = y0 - SS_R + r;
        const int xf = (x0 - SS_R) * 3 + cflt;   // float index inside the image row
        float v = 0.f;
        if (y >= 0 && y < H && xf >= 0 && xf < W * 3) v = __ldg(img + (size_t)y * W * 3 + xf);
        sm[i] = v;
    }
}

// load_halo with the ignored pixels (mask == 0) read as 0 as well: a select, so their content never enters
__device__ __forceinline__ void load_halo_masked(const float *__restrict__ img, const uint8_t *__restrict__ mask, int H,
                                                 int W, int x0, int y0, float *sm) {
    for (int i = threadIdx.x; i < SS_H * SS_ROW; i += 256) {
        const int r = i / SS_ROW, cflt = i - r * SS_ROW;
        const int y = y0 - SS_R + r;
        const int xf = (x0 - SS_R) * 3 + cflt;
        float v = 0.f;
        if (y >= 0 && y < H && xf >= 0 && xf < W * 3 && __ldg(mask + (size_t)y * W + xf / 3) != 0)
            v = __ldg(img + (size_t)y * W * 3 + xf);
        sm[i] = v;
    }
}

__device__ __forceinline__ unsigned block_count_256(unsigned v, unsigned *sm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned r = 0;
    if (threadIdx.x < 8) {
        r = sm[threadIdx.x];
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) r += __shfl_xor_sync(0xffu, r, o);
    }
    __syncthreads();
    return r;  // valid in thread 0
}

// MASK: mask [H,W] u8 (nonzero = used) and count (the number of used pixels, added per tile); unused otherwise
template <bool MASK>
__global__ void __launch_bounds__(256)
ssim_forward_kernel(int H, int W, const float *__restrict__ rendered, const float *__restrict__ gt,
                    SsimWindow win, float *__restrict__ d_mu, float *__restrict__ d_e22,
                    float *__restrict__ d_e12, float *__restrict__ sums /* [0] sum SSIM, [1] sum |r-g| */,
                    const uint8_t *__restrict__ mask, unsigned *__restrict__ count) {
    __shared__ float sx[SS_H * SS_ROW];            // gt      (img1 = x)
    __shared__ float sy[SS_H * SS_ROW];            // rendered (img2 = y)
    __shared__ float hz[5][SS_H][SS_OUT];          // horizontally filtered x, y, xx, yy, xy
    __shared__ float red[8];
    const int x0 = blockIdx.x * SS_T, y0 = blockIdx.y * SS_T;
    if constexpr (MASK) {
        load_halo_masked(gt, mask, H, W, x0, y0, sx);
        load_halo_masked(rendered, mask, H, W, x0, y0, sy);
    } else {
        load_halo(gt, H, W, x0, y0, sx);
        load_halo(rendered, H, W, x0, y0, sy);
    }
    __syncthreads();
    // horizontal pass: SS_H rows x SS_OUT floats
    for (int i = threadIdx.x; i < SS_H * SS_OUT; i += 256) {
        const int r = i / SS_OUT, c = i - r * SS_OUT;   // c = 3*px + channel
        float ax = 0.f, ay = 0.f, axx = 0.f, ayy = 0.f, axy = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float xv = sx[r * SS_ROW + c + 3 * k], yv = sy[r * SS_ROW + c + 3 * k], w = win.w[k];
            ax = fmaf(w, xv, ax);
            ay = fmaf(w, yv, ay);
            axx = fmaf(w, xv * xv, axx);
            ayy = fmaf(w, yv * yv, ayy);
            axy = fmaf(w, xv * yv, axy);
        }
        hz[0][r][c] = ax; hz[1][r][c] = ay; hz[2][r][c] = axx; hz[3][r][c] = ayy; hz[4][r][c] = axy;
    }
    __syncthreads();
    // vertical pass + SSIM map: thread = pixel (ty*16+tx), 3 channels
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int X = x0 + tx, Y = y0 + ty;
    float ssim_sum = 0.f, l1_sum = 0.f;
    unsigned used = 0;
    if (X < W && Y < H) {
        bool m = true;
        if constexpr (MASK) {
            m = __ldg(mask + (size_t)Y * W + X) != 0;
            used = m ? 1u : 0u;
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const int c = 3 * tx + ch;
            float mx = 0.f, my = 0.f, exx = 0.f, eyy = 0.f, exy = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float w = win.w[k];
                mx = fmaf(w, hz[0][ty + k][c], mx);
                my = fmaf(w, hz[1][ty + k][c], my);
                exx = fmaf(w, hz[2][ty + k][c], exx);
                eyy = fmaf(w, hz[3][ty + k][c], eyy);
                exy = fmaf(w, hz[4][ty + k][c], exy);
            }
            const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
            const float sxx = exx - mx * mx, syy = eyy - my * my, sxy = exy - mx * my;
            const float A1 = 2.f * mx * my + C1, A2 = 2.f * sxy + C2;
            const float B1 = mx * mx + my * my + C1, B2 = sxx + syy + C2;
            const float inv = 1.f / (B1 * B2);
            const float S = A1 * A2 * inv;
            if (m) ssim_sum += S;
            // partials of S w.r.t. the three filtered quantities that depend on y = rendered
            const float dS_e12 = 2.f * A1 * inv;
            const float dS_e22 = -S / B2;
            const float dS_mu = 2.f * mx * (A2 - A1) * inv - 2.f * my * S / B1 + 2.f * my * S / B2;
            const size_t o = ((size_t)Y * W + X) * 3 + ch;
            d_mu[o] = m ? dS_mu : 0.f;
            d_e22[o] = m ? dS_e22 : 0.f;
            d_e12[o] = m ? dS_e12 : 0.f;
            const float xv = sx[(ty + SS_R) * SS_ROW + 3 * (tx + SS_R) + ch];
            const float yv = sy[(ty + SS_R) * SS_ROW + 3 * (tx + SS_R) + ch];
            l1_sum += fabsf(yv - xv);   // MASK: an ignored pixel's halo values are both 0
        }
    }
    const float s0 = block_sum_256(ssim_sum, red);
    const float s1 = block_sum_256(l1_sum, red);
    if (threadIdx.x == 0) {
        atomicAdd(&sums[0], s0);
        atomicAdd(&sums[1], s1);
    }
    if constexpr (MASK) {
        const unsigned n = block_count_256(used, reinterpret_cast<unsigned *>(red));
        if (threadIdx.x == 0 && n) atomicAdd(count, n);
    }
}

// MASK: the scales are read from scales[0..1] (the finalize kernel's) in place of the two arguments, and ignored
// pixels get 0; the maps are already 0 there
template <bool MASK>
__global__ void __launch_bounds__(256)
ssim_backward_kernel(int H, int W, const float *__restrict__ rendered, const float *__restrict__ gt,
                     SsimWindow win, const float *__restrict__ d_mu, const float *__restrict__ d_e22,
                     const float *__restrict__ d_e12, float ssim_scale /* -w/count */,
                     float l1_scale /* (1-w)/count */, float *__restrict__ v_rendered,
                     const uint8_t *__restrict__ mask, const float *__restrict__ scales) {
    __shared__ float sm[SS_H * SS_ROW];
    __shared__ float hz[SS_H][SS_OUT];
    const int x0 = blockIdx.x * SS_T, y0 = blockIdx.y * SS_T;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int X = x0 + tx, Y = y0 + ty;
    float acc[3][3];   // [map][channel]: transposed-window filtered maps at this pixel
    const float *maps[3] = {d_mu, d_e22, d_e12};
#pragma unroll
    for (int m = 0; m < 3; ++m) {
        load_halo(maps[m], H, W, x0, y0, sm);
        __syncthreads();
        // transposed filter: grad_in(p) = sum_q w(p - q + R) D(q) = sum_k w(10 - k) D(p - R + k)
        for (int i = threadIdx.x; i < SS_H * SS_OUT; i += 256) {
            const int r = i / SS_OUT, c = i - r * SS_OUT;
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) a = fmaf(win.w[10 - k], sm[r * SS_ROW + c + 3 * k], a);
            hz[r][c] = a;
        }
        __syncthreads();
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) a = fmaf(win.w[10 - k], hz[ty + k][3 * tx + ch], a);
            acc[m][ch] = a;
        }
        __syncthreads();
    }
    if (X < W && Y < H) {
        if constexpr (MASK) {
            if (__ldg(mask + (size_t)Y * W + X) == 0) {
                const size_t o = ((size_t)Y * W + X) * 3;
                v_rendered[o] = v_rendered[o + 1] = v_rendered[o + 2] = 0.f;
                return;
            }
            ssim_scale = scales[0];
            l1_scale = scales[1];
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const size_t o = ((size_t)Y * W + X) * 3 + ch;
            const float xv = __ldg(gt + o), yv = __ldg(rendered + o);
            const float dssim = acc[0][ch] + 2.f * yv * acc[1][ch] + xv * acc[2][ch];
            const float d = yv - xv;
            const float sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
            v_rendered[o] = ssim_scale * dssim + l1_scale * sgn;
        }
    }
}

// combines the two sums into {total, l1, ssim}
__global__ void ssim_finalize_kernel(const float *sums, float inv_count, float w, float *loss_out) {
    const float ssim = sums[0] * inv_count, l1 = sums[1] * inv_count;
    loss_out[0] = (1.f - w) * l1 + w * (1.f - ssim);
    loss_out[1] = l1;
    loss_out[2] = ssim;
}

// the masked finalize: N = count used pixels, the count 3N formed as the host forms H W 3 for the unmasked loss, and
// the backward's two scales; N = 0 gives {0, 0, 1} and zero scales
__global__ void ssim_finalize_masked_kernel(const float *sums, const unsigned *count, float w, float *loss_out,
                                            float *scales) {
    const unsigned n = *count;
    if (n == 0) {
        loss_out[0] = 0.f;
        loss_out[1] = 0.f;
        loss_out[2] = 1.f;
        scales[0] = scales[1] = 0.f;
        return;
    }
    const float cnt = (float)n * 3.f;
    const float inv_count = 1.f / cnt;
    const float ssim = sums[0] * inv_count, l1 = sums[1] * inv_count;
    loss_out[0] = (1.f - w) * l1 + w * (1.f - ssim);
    loss_out[1] = l1;
    loss_out[2] = ssim;
    scales[0] = -w / cnt;
    scales[1] = (1.f - w) / cnt;
}

// the reference's window (ssim.cpp:41-47): exp(-floor((i - 11)/2)^2 / (2 sigma^2)), sigma = 1.5, normalised
SsimWindow reference_window() {
    SsimWindow win;
    double sum = 0.0;
    for (int i = 0; i < 11; ++i) {
        const float d = floorf((float)(i - 11) / 2.0f);
        win.w[i] = expf(-(d * d) / (2.0f * 1.5f * 1.5f));
        sum += win.w[i];
    }
    for (int i = 0; i < 11; ++i) win.w[i] = (float)(win.w[i] / sum);
    return win;
}

}  // namespace

extern "C" size_t gsb_ssim_workspace_bytes(int img_h, int img_w) {
    const size_t map = gsb_align_up((size_t)img_h * img_w * 3 * 4, 256);
    return 3 * map + 256;
}

// loss_out: device float[3] = { (1-w) L1 + w (1 - SSIM), L1, SSIM }.  v_rendered [H,W,3] = d loss / d rendered.
extern "C" int gsb_ssim_l1_loss(int img_h, int img_w, const float *rendered, const float *gt, float ssim_weight,
                                float *v_rendered, float *loss_out, void *workspace, size_t workspace_bytes,
                                gsb_stream_t stream) {
    GSB_CHECK_ARG(img_h > 0 && img_w > 0 && rendered && gt && v_rendered && loss_out && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0);
    if (workspace_bytes < gsb_ssim_workspace_bytes(img_h, img_w)) {
        gsb_set_error(GSB_ERR_WORKSPACE, "ssim workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const SsimWindow win = reference_window();
    const size_t map = gsb_align_up((size_t)img_h * img_w * 3 * 4, 256);
    char *ws = (char *)workspace;
    float *d_mu = (float *)ws, *d_e22 = (float *)(ws + map), *d_e12 = (float *)(ws + 2 * map);
    float *sums = (float *)(ws + 3 * map);
    GSB_CUDA(cudaMemsetAsync(sums, 0, 8, s));
    const dim3 grid(gsb_div_up(img_w, SS_T), gsb_div_up(img_h, SS_T));
    const float count = (float)img_h * (float)img_w * 3.f;
    ssim_forward_kernel<false><<<grid, 256, 0, s>>>(img_h, img_w, rendered, gt, win, d_mu, d_e22, d_e12, sums,
                                                    nullptr, nullptr);
    ssim_finalize_kernel<<<1, 1, 0, s>>>(sums, 1.f / count, ssim_weight, loss_out);
    ssim_backward_kernel<false><<<grid, 256, 0, s>>>(img_h, img_w, rendered, gt, win, d_mu, d_e22, d_e12,
                                                     -ssim_weight / count, (1.f - ssim_weight) / count, v_rendered,
                                                     nullptr, nullptr);
    GSB_LAUNCH_CHECK();
    return 0;
}

// DESIGN D26: the loss over the used pixels of mask [H,W] u8 (nonzero = used); the workspace of the unmasked loss.
// Nothing is read back to the host: N, the loss and the backward's scales stay on the device.
extern "C" int gsb_ssim_l1_loss_masked(int img_h, int img_w, const float *rendered, const float *gt,
                                       const uint8_t *mask, float ssim_weight, float *v_rendered, float *loss_out,
                                       void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(img_h > 0 && img_w > 0 && rendered && gt && mask && v_rendered && loss_out && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0);
    if (workspace_bytes < gsb_ssim_workspace_bytes(img_h, img_w)) {
        gsb_set_error(GSB_ERR_WORKSPACE, "ssim workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const SsimWindow win = reference_window();
    const size_t map = gsb_align_up((size_t)img_h * img_w * 3 * 4, 256);
    char *ws = (char *)workspace;
    float *d_mu = (float *)ws, *d_e22 = (float *)(ws + map), *d_e12 = (float *)(ws + 2 * map);
    // the tail: sums [0..1], the used-pixel count [2] (unsigned), the backward's scales [4..5]
    float *sums = (float *)(ws + 3 * map);
    unsigned *count = (unsigned *)(sums + 2);
    float *scales = sums + 4;
    GSB_CUDA(cudaMemsetAsync(sums, 0, 12, s));
    const dim3 grid(gsb_div_up(img_w, SS_T), gsb_div_up(img_h, SS_T));
    ssim_forward_kernel<true><<<grid, 256, 0, s>>>(img_h, img_w, rendered, gt, win, d_mu, d_e22, d_e12, sums, mask,
                                                   count);
    ssim_finalize_masked_kernel<<<1, 1, 0, s>>>(sums, count, ssim_weight, loss_out, scales);
    ssim_backward_kernel<true><<<grid, 256, 0, s>>>(img_h, img_w, rendered, gt, win, d_mu, d_e22, d_e12, 0.f, 0.f,
                                                    v_rendered, mask, scales);
    GSB_LAUNCH_CHECK();
    return 0;
}
