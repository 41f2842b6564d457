// fused.cu -- small streaming kernels around the hot path ("next" rows of SURVEY.md section 8f):
//   gsb_mse_loss_grad : loss = mean((img - target)^2) and v_img = 2 (img - target) / count in one pass
//                       (simple_trainer.cpp:199-201 does this with torch::nn::MSELoss + autograd)
//   gsb_adam_step     : one fused Adam update over a flat parameter buffer
//                       (simple_trainer.cpp:146,202 torch::optim::Adam; model.cpp:236-243 runs six of them)
//   gsb_adam_step_segments : the same update with a learning rate per segment (and per row position inside it),
//                       i.e. the six optimizers of model.cpp:58-70 over one flat buffer in one launch
// Both are HBM-bound elementwise passes: 128-bit accesses, grid = multiple of the SM count.
#include "gsb_common.cuh"

namespace {

__global__ void __launch_bounds__(256)
mse_loss_grad_kernel(long long n4, long long n, const float *__restrict__ img,
                     const float *__restrict__ target, float *__restrict__ v_img,
                     float *__restrict__ loss_out, float inv_count) {
    float acc = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 a = reinterpret_cast<const float4 *>(img)[i];
        const float4 b = reinterpret_cast<const float4 *>(target)[i];
        const float4 d = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
        acc += d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
        const float s = 2.f * inv_count;
        reinterpret_cast<float4 *>(v_img)[i] = make_float4(s * d.x, s * d.y, s * d.z, s * d.w);
    }
    // tail (n not a multiple of 4)
    for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float d = img[i] - target[i];
        acc += d * d;
        v_img[i] = 2.f * inv_count * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ float sm[8];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 8) {
        float v = sm[threadIdx.x];
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
        if (threadIdx.x == 0) atomicAdd(loss_out, v * inv_count);
    }
}

// One Adam update of one element with its roundings spelled out: FFMA for m, v and the denominator, the parameter
// step as FMUL + FSUB.  Left to the compiler, the contraction of the step depends on the surrounding code (it once
// fused it into one FFMA on some vector lanes and not others), so every path of both Adam kernels calls this one
// function: an element's result does not depend on the kernel, the path or the lane it falls on.
__device__ __forceinline__ void adam_update(float &pp, float gg, float &mm, float &vv, float lr, float b1, float b2,
                                            float eps, float inv_bc1, float inv_sqrt_bc2) {
    mm = __fmaf_rn(1.f - b1, gg, b1 * mm);
    vv = __fmaf_rn(gg, (1.f - b2) * gg, b2 * vv);
    // torch.optim.Adam: p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
    pp = __fsub_rn(pp, __fmul_rn(lr * inv_bc1, __fdividef(mm, __fmaf_rn(sqrtf(vv), inv_sqrt_bc2, eps))));
}

__global__ void __launch_bounds__(256)
adam_kernel(long long n4, long long n, float *__restrict__ p, const float *__restrict__ g,
            float *__restrict__ m, float *__restrict__ v, float lr, float b1, float b2, float eps,
            float inv_bc1, float inv_sqrt_bc2) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    auto upd = [&](float &pp, float gg, float &mm, float &vv) {
        adam_update(pp, gg, mm, vv, lr, b1, b2, eps, inv_bc1, inv_sqrt_bc2);
    };
    // two float4 per thread per trip: 8 independent 128-bit loads in flight before the first use
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + stride < n4; i += 2 * stride) {
        const long long j = i + stride;
        float4 P0 = reinterpret_cast<float4 *>(p)[i], P1 = reinterpret_cast<float4 *>(p)[j];
        const float4 G0 = ldg_stream4(reinterpret_cast<const float4 *>(g) + i);
        const float4 G1 = ldg_stream4(reinterpret_cast<const float4 *>(g) + j);
        float4 M0 = reinterpret_cast<float4 *>(m)[i], M1 = reinterpret_cast<float4 *>(m)[j];
        float4 V0 = reinterpret_cast<float4 *>(v)[i], V1 = reinterpret_cast<float4 *>(v)[j];
        upd(P0.x, G0.x, M0.x, V0.x); upd(P0.y, G0.y, M0.y, V0.y); upd(P0.z, G0.z, M0.z, V0.z); upd(P0.w, G0.w, M0.w, V0.w);
        upd(P1.x, G1.x, M1.x, V1.x); upd(P1.y, G1.y, M1.y, V1.y); upd(P1.z, G1.z, M1.z, V1.z); upd(P1.w, G1.w, M1.w, V1.w);
        reinterpret_cast<float4 *>(p)[i] = P0; reinterpret_cast<float4 *>(p)[j] = P1;
        reinterpret_cast<float4 *>(m)[i] = M0; reinterpret_cast<float4 *>(m)[j] = M1;
        reinterpret_cast<float4 *>(v)[i] = V0; reinterpret_cast<float4 *>(v)[j] = V1;
    }
    for (; i < n4; i += stride) {
        float4 P = reinterpret_cast<float4 *>(p)[i];
        const float4 G = ldg_stream4(reinterpret_cast<const float4 *>(g) + i);
        float4 M = reinterpret_cast<float4 *>(m)[i];
        float4 V = reinterpret_cast<float4 *>(v)[i];
        upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
        reinterpret_cast<float4 *>(p)[i] = P;
        reinterpret_cast<float4 *>(m)[i] = M;
        reinterpret_cast<float4 *>(v)[i] = V;
    }
    for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        upd(p[i], g[i], m[i], v[i]);
}

// The segment table travels by value in the kernel's parameter space (8 x 32 B).
struct AdamSegments {
    gsb_adam_segment s[GSB_ADAM_MAX_SEGMENTS];
    int count;
};

// Adam over the segments of a flat buffer in one launch: element e of segment s takes lr_head when
// e % row_floats < head_floats and lr_rest otherwise.  Segments start on 16-byte boundaries; the floats between
// them (padding) are never touched.
__global__ void __launch_bounds__(256)
adam_segments_kernel(AdamSegments segs, float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                     float *__restrict__ v, float b1, float b2, float eps, float inv_bc1, float inv_sqrt_bc2) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (int k = 0; k < segs.count; ++k) {
        const gsb_adam_segment sg = segs.s[k];
        float *ps = p + sg.offset, *ms = m + sg.offset, *vs = v + sg.offset;
        const float *gs = g + sg.offset;
        const long long n4 = sg.count / 4;
        for (long long i = t0; i < n4; i += stride) {
            float4 P = reinterpret_cast<float4 *>(ps)[i];
            const float4 G = ldg_stream4(reinterpret_cast<const float4 *>(gs) + i);
            float4 M = reinterpret_cast<float4 *>(ms)[i];
            float4 V = reinterpret_cast<float4 *>(vs)[i];
            // a float4 may straddle a head / rest boundary: the rate is chosen per component
            int j = (int)((4 * i) % sg.row_floats);
            float lr[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                lr[c] = j < sg.head_floats ? sg.lr_head : sg.lr_rest;
                if (++j == sg.row_floats) j = 0;
            }
            adam_update(P.x, G.x, M.x, V.x, lr[0], b1, b2, eps, inv_bc1, inv_sqrt_bc2);
            adam_update(P.y, G.y, M.y, V.y, lr[1], b1, b2, eps, inv_bc1, inv_sqrt_bc2);
            adam_update(P.z, G.z, M.z, V.z, lr[2], b1, b2, eps, inv_bc1, inv_sqrt_bc2);
            adam_update(P.w, G.w, M.w, V.w, lr[3], b1, b2, eps, inv_bc1, inv_sqrt_bc2);
            reinterpret_cast<float4 *>(ps)[i] = P;
            reinterpret_cast<float4 *>(ms)[i] = M;
            reinterpret_cast<float4 *>(vs)[i] = V;
        }
        for (long long e = 4 * n4 + t0; e < sg.count; e += stride) {
            const float lr = (int)(e % sg.row_floats) < sg.head_floats ? sg.lr_head : sg.lr_rest;
            adam_update(ps[e], gs[e], ms[e], vs[e], lr, b1, b2, eps, inv_bc1, inv_sqrt_bc2);
        }
    }
}

// ---- parameter activations of Model::forward (model.cpp:114,148-150,176-177,200), one pass each way ----
__global__ void __launch_bounds__(256)
activate_forward_kernel(int n, const float *__restrict__ means, const float *__restrict__ log_scales,
                        const float *__restrict__ raw_quats, const float *__restrict__ opacity_logits,
                        const float *__restrict__ cam_pos, float *__restrict__ scales,
                        float4 *__restrict__ quats, float *__restrict__ opacities, float *__restrict__ viewdirs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    scales[3 * i] = expf(log_scales[3 * i]);
    scales[3 * i + 1] = expf(log_scales[3 * i + 1]);
    scales[3 * i + 2] = expf(log_scales[3 * i + 2]);
    const float4 q = reinterpret_cast<const float4 *>(raw_quats)[i];
    const float inv = 1.f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    quats[i] = make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
    opacities[i] = 1.f / (1.f + expf(-opacity_logits[i]));
    const float dx = means[3 * i] - __ldg(cam_pos), dy = means[3 * i + 1] - __ldg(cam_pos + 1),
                dz = means[3 * i + 2] - __ldg(cam_pos + 2);
    const float dn = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
    viewdirs[3 * i] = dx * dn; viewdirs[3 * i + 1] = dy * dn; viewdirs[3 * i + 2] = dz * dn;
}

__global__ void __launch_bounds__(256)
activate_backward_kernel(int n, const float *__restrict__ scales, const float *__restrict__ raw_quats,
                         const float *__restrict__ opacities, const float *__restrict__ v_scales,
                         const float4 *__restrict__ v_quats, const float *__restrict__ v_opacities,
                         float *__restrict__ v_log_scales, float4 *__restrict__ v_raw_quats,
                         float *__restrict__ v_opacity_logits) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // d exp(s) = exp(s)
    v_log_scales[3 * i] = v_scales[3 * i] * scales[3 * i];
    v_log_scales[3 * i + 1] = v_scales[3 * i + 1] * scales[3 * i + 1];
    v_log_scales[3 * i + 2] = v_scales[3 * i + 2] * scales[3 * i + 2];
    // d (q / |q|) : (I - q^ q^T) / |q|
    const float4 q = reinterpret_cast<const float4 *>(raw_quats)[i];
    const float inv = 1.f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float4 h = make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv), g = v_quats[i];
    const float dot = h.x * g.x + h.y * g.y + h.z * g.z + h.w * g.w;
    v_raw_quats[i] = make_float4((g.x - h.x * dot) * inv, (g.y - h.y * dot) * inv, (g.z - h.z * dot) * inv,
                                 (g.w - h.w * dot) * inv);
    // d sigmoid = o (1 - o)
    const float o = opacities[i];
    v_opacity_logits[i] = v_opacities[i] * o * (1.f - o);
}

// ---- densification statistics of Model::afterTrain (model.cpp:317-337), one pass, no boolean-mask indexing ----
__global__ void __launch_bounds__(256)
densify_stats_kernel(int n, const float2 *__restrict__ v_xy, const int *__restrict__ radii, float max_hw,
                     float *__restrict__ xys_grad_norm, float *__restrict__ vis_counts,
                     float *__restrict__ max_2d_size) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = radii[i];
    if (r <= 0) return;  // visibleMask = radii > 0
    const float2 g = v_xy[i];
    xys_grad_norm[i] += sqrtf(g.x * g.x + g.y * g.y);
    vis_counts[i] += 1.f;
    max_2d_size[i] = fmaxf(max_2d_size[i], (float)r / max_hw);
}

// first step after a refinement (model.cpp:321-323,328-330): xysGradNorm = |v_xy| and visCounts = 1 for EVERY
// Gaussian (visible or not), max2DSize = 0 then the visible update
__global__ void __launch_bounds__(256)
densify_stats_init_kernel(int n, const float2 *__restrict__ v_xy, const int *__restrict__ radii, float max_hw,
                          float *__restrict__ xys_grad_norm, float *__restrict__ vis_counts,
                          float *__restrict__ max_2d_size) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = radii[i];
    const float2 g = v_xy[i];
    xys_grad_norm[i] = sqrtf(g.x * g.x + g.y * g.y);
    vis_counts[i] = 1.f;
    max_2d_size[i] = r > 0 ? fmaxf(0.f, (float)r / max_hw) : 0.f;
}

int sm_count() {
    static thread_local int cached = 0;
    if (!cached) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
        if (cached <= 0) cached = 132;
    }
    return cached;
}

}  // namespace

// loss_out (device float) is zeroed here (stream-ordered) and then accumulated into by the kernel.
extern "C" int gsb_mse_loss_grad(long long n, const float *img, const float *target, float *v_img,
                                 float *loss_out, float inv_count, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && loss_out && (n == 0 || (img && target && v_img)));
    GSB_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), (cudaStream_t)stream));
    if (n == 0) return 0;     // an empty image has loss 0
    const bool vec = (((uintptr_t)img | (uintptr_t)target | (uintptr_t)v_img) % 16) == 0;
    const long long n4 = vec ? n / 4 : 0;
    mse_loss_grad_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(n4, n, img, target, v_img, loss_out,
                                                                        inv_count);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_adam_step(long long n, float *param, const float *grad, float *exp_avg,
                             float *exp_avg_sq, float lr, float beta1, float beta2, float eps,
                             float bias_correction1, float bias_correction2, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && bias_correction1 > 0.f && bias_correction2 > 0.f);
    if (n == 0) return 0;
    GSB_CHECK_ARG(param && grad && exp_avg && exp_avg_sq);
    const bool vec = (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) % 16) == 0;
    const long long n4 = vec ? n / 4 : 0;
    adam_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(n4, n, param, grad, exp_avg, exp_avg_sq, lr, beta1,
                                                               beta2, eps, 1.f / bias_correction1,
                                                               1.f / sqrtf(bias_correction2));
    GSB_LAUNCH_CHECK();
    return 0;
}

// The six optimizers of Model::setupOptimizers (model.cpp:58-70) over one flat buffer in one launch: one segment
// per parameter slice, the merged SH block as one segment with two rates (featuresDc on the first 3 floats of
// every 3K-float row, featuresRest on the rest).  Same update as gsb_adam_step.
extern "C" int gsb_adam_step_segments(int num_segments, const gsb_adam_segment *segments, float *param,
                                      const float *grad, float *exp_avg, float *exp_avg_sq, float beta1, float beta2,
                                      float eps, float bias_correction1, float bias_correction2,
                                      gsb_stream_t stream) {
    GSB_CHECK_ARG(num_segments >= 0 && num_segments <= GSB_ADAM_MAX_SEGMENTS && (num_segments == 0 || segments));
    GSB_CHECK_ARG(bias_correction1 > 0.f && bias_correction2 > 0.f);
    AdamSegments segs = {};
    long long total = 0;
    for (int k = 0; k < num_segments; ++k) {
        const gsb_adam_segment &sg = segments[k];
        GSB_CHECK_ARG(sg.offset >= 0 && sg.offset % 4 == 0 && sg.count >= 0);
        GSB_CHECK_ARG(sg.row_floats > 0 && sg.head_floats >= 0 && sg.head_floats <= sg.row_floats);
        segs.s[k] = sg;
        total += sg.count;
    }
    segs.count = num_segments;
    if (total == 0) return 0;
    GSB_CHECK_ARG(param && grad && exp_avg && exp_avg_sq);
    GSB_CHECK_ARG((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) % 16) == 0);
    adam_segments_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(
        segs, param, grad, exp_avg, exp_avg_sq, beta1, beta2, eps, 1.f / bias_correction1,
        1.f / sqrtf(bias_correction2));
    GSB_LAUNCH_CHECK();
    return 0;
}

// Parameter activations of Model::forward fused into one pass (SURVEY.md 8f row 1): scales = exp(log_scales)
// (model.cpp:148), quats = raw / |raw| (:150), opacities = sigmoid(logits) (:200), viewdirs =
// normalize(means - cam_pos) (:176-177; detached, no gradient).  cam_pos is a device float[3].
extern "C" int gsb_activate_forward(int n, const float *means, const float *log_scales, const float *raw_quats,
                                    const float *opacity_logits, const float *cam_pos, float *scales, float *quats,
                                    float *opacities, float *viewdirs, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(means && log_scales && raw_quats && opacity_logits && cam_pos && scales && quats && opacities &&
                  viewdirs);
    GSB_CHECK_ARG(((uintptr_t)raw_quats % 16) == 0 && ((uintptr_t)quats % 16) == 0);
    activate_forward_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, means, log_scales, raw_quats, opacity_logits, cam_pos, scales, reinterpret_cast<float4 *>(quats), opacities,
        viewdirs);
    GSB_LAUNCH_CHECK();
    return 0;
}

// VJP of gsb_activate_forward: takes the forward OUTPUTS scales / opacities and the raw quaternions.
extern "C" int gsb_activate_backward(int n, const float *scales, const float *raw_quats, const float *opacities,
                                     const float *v_scales, const float *v_quats, const float *v_opacities,
                                     float *v_log_scales, float *v_raw_quats, float *v_opacity_logits,
                                     gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(scales && raw_quats && opacities && v_scales && v_quats && v_opacities && v_log_scales &&
                  v_raw_quats && v_opacity_logits);
    GSB_CHECK_ARG(((uintptr_t)raw_quats % 16) == 0 && ((uintptr_t)v_quats % 16) == 0 &&
                  ((uintptr_t)v_raw_quats % 16) == 0);
    activate_backward_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, scales, raw_quats, opacities, v_scales, reinterpret_cast<const float4 *>(v_quats), v_opacities, v_log_scales,
        reinterpret_cast<float4 *>(v_raw_quats), v_opacity_logits);
    GSB_LAUNCH_CHECK();
    return 0;
}

// Densification statistics (SURVEY.md 8f row 3; Model::afterTrain model.cpp:317-337): for visible Gaussians
// (radii > 0): xys_grad_norm += |v_xy|, vis_counts += 1, max_2d_size = max(max_2d_size, radii / max(H, W)).
// The reference does this with boolean-mask index / index_put (each a host-synchronising nonzero()).
extern "C" int gsb_densify_stats_update(int n, const float *v_xy, const int32_t *radii, int img_h, int img_w,
                                        float *xys_grad_norm, float *vis_counts, float *max_2d_size,
                                        gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && img_h > 0 && img_w > 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(v_xy && radii && xys_grad_norm && vis_counts && max_2d_size && ((uintptr_t)v_xy % 8) == 0);
    const float max_hw = (float)(img_h > img_w ? img_h : img_w);
    densify_stats_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, reinterpret_cast<const float2 *>(v_xy), radii, max_hw, xys_grad_norm, vis_counts, max_2d_size);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_densify_stats_init(int n, const float *v_xy, const int32_t *radii, int img_h, int img_w,
                                      float *xys_grad_norm, float *vis_counts, float *max_2d_size,
                                      gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && img_h > 0 && img_w > 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(v_xy && radii && xys_grad_norm && vis_counts && max_2d_size && ((uintptr_t)v_xy % 8) == 0);
    const float max_hw = (float)(img_h > img_w ? img_h : img_w);
    densify_stats_init_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, reinterpret_cast<const float2 *>(v_xy), radii, max_hw, xys_grad_norm, vis_counts, max_2d_size);
    GSB_LAUNCH_CHECK();
    return 0;
}
