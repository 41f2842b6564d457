// project.cu -- per-Gaussian 3D->2D projection, forward (P1) and exact VJP (P2).
//
// Forward replaces project_gaussians_forward_kernel (reference rasterizer/gsplat/forward.cu:19-103
// with helpers.cuh:13-74,91-122,145-167,225-233 and forward.cu:381-470).  Backward replaces
// project_gaussians_backward_kernel (backward.cu:357-542, helpers.cuh:77-88,125-143,169-213).
//
// This translation unit is compiled with --fmad=false: radii, num_tiles_hit (and through them the
// intersection count M, the sort keys and the tile bins) are integer functions of this fp32 chain and
// must be reproducible bit-for-bit by a host restatement (oracle/gsplat_oracle.c, built with
// -ffp-contract=off).  Only correctly-rounded operations are used, in a fixed order: IEEE div/sqrt,
// 1/sqrtf instead of the reference's 2-ulp rsqrtf (helpers.cuh:147).  The kernels are HBM-bound
// (96 B / 144 B per Gaussian), so the lost FMA contraction is free.
//
// Gradient conventions (DESIGN.md): the backward is the exact VJP of the forward map, i.e. what the
// reference's CPU back end obtains from torch autograd (gsplat_cpu.cpp:48-131) -- it keeps the
// perspective-divide term, the quaternion-normalisation Jacobian, glob_scale in v_scale and the fov
// clamp sub-gradient, which the reference's hand-written CUDA VJP drops (SURVEY.md 8c D8/D11/D12).
#include "gsb_common.cuh"

namespace {

constexpr int PJ_THREADS = 256;

struct Cam {
    float V[12];  // viewmat rows 0..2
    float P[16];  // projmat
};

__device__ __forceinline__ void quat_to_rotmat(float qw, float qx, float qy, float qz, float R[3][3]) {
    float s = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
    float w = qw * s, x = qx * s, y = qy * s, z = qz * s;
    R[0][0] = 1.f - 2.f * (y * y + z * z);
    R[0][1] = 2.f * (x * y - w * z);
    R[0][2] = 2.f * (x * z + w * y);
    R[1][0] = 2.f * (x * y + w * z);
    R[1][1] = 1.f - 2.f * (x * x + z * z);
    R[1][2] = 2.f * (y * z - w * x);
    R[2][0] = 2.f * (x * z - w * y);
    R[2][1] = 2.f * (y * z + w * x);
    R[2][2] = 1.f - 2.f * (x * x + y * y);
}

__device__ __forceinline__ void load_cam(const float *__restrict__ viewmat,
                                         const float *__restrict__ projmat, Cam &c) {
#pragma unroll
    for (int i = 0; i < 12; ++i) c.V[i] = __ldg(viewmat + i);
#pragma unroll
    for (int i = 0; i < 16; ++i) c.P[i] = __ldg(projmat + i);
}

// ACT: the parameter activations of Model::forward (model.cpp:148-150,176-177,200) as this kernel's prologue --
// `scales` holds log-scales (exp here), `quats` the raw quaternions (quat_to_rotmat normalises, as the reference's
// does, so `quats / quats.norm()` needs no pass of its own), and sigmoid(opacity_logits) is written beside the
// projection outputs for the rasterizer.
template <bool ACT>
__global__ void __launch_bounds__(PJ_THREADS)
project_forward_kernel(int n, const float *__restrict__ means3d, const float *__restrict__ scales,
                       float glob_scale, const float *__restrict__ quats,
                       const float *__restrict__ viewmat, const float *__restrict__ projmat, float fx,
                       float fy, float cx, float cy, float tan_fovx, float tan_fovy, int img_h, int img_w,
                       int tiles_x, int tiles_y, float clip_thresh, float *__restrict__ cov3d,
                       float2 *__restrict__ xys, float *__restrict__ depths, int *__restrict__ radii,
                       float *__restrict__ conics, int *__restrict__ num_tiles_hit,
                       const float *__restrict__ opacity_logits, float *__restrict__ opacities) {
    const int i = blockIdx.x * PJ_THREADS + threadIdx.x;
    if (i >= n) return;
    if (ACT) opacities[i] = 1.f / (1.f + expf(-opacity_logits[i]));
    Cam cam;
    load_cam(viewmat, projmat, cam);
    const float *V = cam.V, *P = cam.P;

    float c3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float conic0 = 0.f, conic1 = 0.f, conic2 = 0.f;
    float ux = 0.f, uy = 0.f, depth = 0.f;
    int radius_i = 0, area = 0;

    const float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];
    // clip_near_plane / transform_4x3 (helpers.cuh:91-98,225-233)
    const float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
    const float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
    const float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
    if (tz > clip_thresh) {
        // scale_rot_to_cov3d (forward.cu:450-470): M = R*S, cov3d = M M^T
        const float4 q = reinterpret_cast<const float4 *>(quats)[i];  // (w,x,y,z)
        float R[3][3], M[3][3];
        quat_to_rotmat(q.x, q.y, q.z, q.w, R);
        const float a0 = scales[3 * i], a1 = scales[3 * i + 1], a2 = scales[3 * i + 2];
        const float s0 = glob_scale * (ACT ? expf(a0) : a0), s1 = glob_scale * (ACT ? expf(a1) : a1),
                    s2 = glob_scale * (ACT ? expf(a2) : a2);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            M[r][0] = R[r][0] * s0;
            M[r][1] = R[r][1] * s1;
            M[r][2] = R[r][2] * s2;
        }
        float C[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                C[r][c] = M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2];
        c3[0] = C[0][0]; c3[1] = C[0][1]; c3[2] = C[0][2];
        c3[3] = C[1][1]; c3[4] = C[1][2]; c3[5] = C[2][2];

        // project_cov3d_ewa (forward.cu:381-447)
        const float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
        const float ttx = tz * fminf(lim_x, fmaxf(-lim_x, tx / tz));
        const float tty = tz * fminf(lim_y, fmaxf(-lim_y, ty / tz));
        const float rz = 1.f / tz, rz2 = rz * rz;
        const float J00 = fx * rz, J02 = -fx * ttx * rz2, J11 = fy * rz, J12 = -fy * tty * rz2;
        float T[2][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            T[0][c] = J00 * V[c] + J02 * V[8 + c];
            T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
        }
        const float Cs[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        float TV[2][3];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                TV[r][c] = T[r][0] * Cs[0][c] + T[r][1] * Cs[1][c] + T[r][2] * Cs[2][c];
        const float cxx = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2] + 0.3f;
        const float cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2];
        const float cyy = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2] + 0.3f;

        // compute_cov2d_bounds (helpers.cuh:51-74)
        const float det = cxx * cyy - cxy * cxy;
        if (det != 0.f) {
            const float inv_det = 1.f / det;
            conic0 = cyy * inv_det;
            conic1 = -cxy * inv_det;
            conic2 = cxx * inv_det;
            const float b = 0.5f * (cxx + cyy);
            const float sq = sqrtf(fmaxf(0.1f, b * b - det));
            const float v1 = b + sq, v2 = b - sq;
            const float radius = ceilf(3.f * sqrtf(fmaxf(v1, v2)));

            // project_pix (helpers.cuh:112-122), ndc2pix (:13-15)
            const float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
            const float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
            const float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
            const float rw = 1.f / (hw + 1e-6f);
            const float ndcx = hx * rw, ndcy = hy * rw;
            const float pxc = 0.5f * (float)img_w * ndcx + cx - 0.5f;
            const float pyc = 0.5f * (float)img_h * ndcy + cy - 0.5f;

            int x0, x1, y0, y1;
            gsb_tile_bbox(pxc, pyc, radius, tiles_x, tiles_y, x0, x1, y0, y1);
            const int a = (x1 - x0) * (y1 - y0);
            if (a > 0) {
                area = a;
                depth = tz;
                radius_i = (int)radius;
                ux = pxc;
                uy = pyc;
            }
        }
    }
    float *c3o = cov3d + 6 * (size_t)i;
#pragma unroll
    for (int k = 0; k < 6; ++k) c3o[k] = c3[k];
    xys[i] = make_float2(ux, uy);
    depths[i] = depth;
    radii[i] = radius_i;
    conics[3 * i] = conic0;
    conics[3 * i + 1] = conic1;
    conics[3 * i + 2] = conic2;
    num_tiles_hit[i] = area;
}

// ACT: VJP of the activating forward -- v_scale comes out w.r.t. the LOG-scales (x exp), the quaternion gradient
// is w.r.t. the raw quaternion as always (the normalisation is inside quat_to_rotmat), and the rasterizer's opacity
// gradient is taken through the sigmoid (x o (1 - o), from the saved activated opacity).
// ACC: add this view's VJP to the four outputs (prev + vjp, one rounding each) instead of writing it -- the sum
// over a trainer's views of one step, in view order.
template <bool ACT, bool ACC>
__global__ void __launch_bounds__(PJ_THREADS)
project_backward_kernel(int n, const float *__restrict__ means3d, const float *__restrict__ scales,
                        float glob_scale, const float *__restrict__ quats,
                        const float *__restrict__ viewmat, const float *__restrict__ projmat, float fx,
                        float fy, float tan_fovx, float tan_fovy, int img_h, int img_w,
                        const int *__restrict__ radii, const float *__restrict__ conics,
                        const float2 *__restrict__ v_xy, const float *__restrict__ v_depth,
                        const float *__restrict__ v_conic, float *__restrict__ v_mean3d,
                        float *__restrict__ v_scale, float4 *__restrict__ v_quat,
                        const float *__restrict__ opacities, const float *__restrict__ v_opacity,
                        float *__restrict__ v_opacity_logits) {
    const int i = blockIdx.x * PJ_THREADS + threadIdx.x;
    if (i >= n) return;
    if (ACT) {
        const float o = opacities[i];
        if constexpr (ACC)
            v_opacity_logits[i] = v_opacity_logits[i] + (v_opacity ? v_opacity[i] * o * (1.f - o) : 0.f);
        else
            v_opacity_logits[i] = v_opacity ? v_opacity[i] * o * (1.f - o) : 0.f;
    }
    float vm[3] = {0.f, 0.f, 0.f}, vs[3] = {0.f, 0.f, 0.f};
    float4 vq = make_float4(0.f, 0.f, 0.f, 0.f);
    if (radii[i] > 0) {
        Cam cam;
        load_cam(viewmat, projmat, cam);
        const float *V = cam.V, *P = cam.P;
        const float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];

        // pixel centre: xy = 0.5*W*(h.x*rw) + cx - 0.5, rw = 1/(h.w + 1e-6)
        const float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
        const float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
        const float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
        const float rw = 1.f / (hw + 1e-6f);
        const float2 vxy = v_xy[i];
        const float vndcx = 0.5f * (float)img_w * vxy.x, vndcy = 0.5f * (float)img_h * vxy.y;
        const float vhx = vndcx * rw, vhy = vndcy * rw;
        const float vhw = -(vndcx * hx + vndcy * hy) * rw * rw;
        vm[0] = P[0] * vhx + P[4] * vhy + P[12] * vhw;
        vm[1] = P[1] * vhx + P[5] * vhy + P[13] * vhw;
        vm[2] = P[2] * vhx + P[6] * vhy + P[14] * vhw;

        const float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
        const float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
        const float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
        float vtx = 0.f, vty = 0.f, vtz = v_depth ? v_depth[i] : 0.f;

        // conic = inverse(cov2d):  v_Sigma = -X G X,  G = [[vA, vB/2],[vB/2, vC]]
        const float A = conics[3 * i], B = conics[3 * i + 1], Cc = conics[3 * i + 2];
        const float gA = v_conic[3 * i], gB = 0.5f * v_conic[3 * i + 1], gC = v_conic[3 * i + 2];
        const float xg00 = A * gA + B * gB, xg01 = A * gB + B * gC;
        const float xg10 = B * gA + Cc * gB, xg11 = B * gB + Cc * gC;
        const float vS00 = -(xg00 * A + xg01 * B);
        const float vS01 = -(xg00 * B + xg01 * Cc);
        const float vS11 = -(xg10 * B + xg11 * Cc);

        // recompute forward intermediates
        const float4 q = reinterpret_cast<const float4 *>(quats)[i];
        float R[3][3], M[3][3];
        quat_to_rotmat(q.x, q.y, q.z, q.w, R);
        const float a[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
        const float e[3] = {ACT ? expf(a[0]) : a[0], ACT ? expf(a[1]) : a[1], ACT ? expf(a[2]) : a[2]};
        const float s[3] = {glob_scale * e[0], glob_scale * e[1], glob_scale * e[2]};
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) M[r][c] = R[r][c] * s[c];
        float Cs[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                Cs[r][c] = M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2];
        const float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
        const float qx = tx / tz, qy = ty / tz;
        const bool clamp_x = !(qx > -lim_x && qx < lim_x), clamp_y = !(qy > -lim_y && qy < lim_y);
        const float cqx = fminf(lim_x, fmaxf(-lim_x, qx)), cqy = fminf(lim_y, fmaxf(-lim_y, qy));
        const float ttx = tz * cqx, tty = tz * cqy;
        const float rz = 1.f / tz, rz2 = rz * rz, rz3 = rz2 * rz;
        const float J00 = fx * rz, J02 = -fx * ttx * rz2, J11 = fy * rz, J12 = -fy * tty * rz2;
        float T[2][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            T[0][c] = J00 * V[c] + J02 * V[8 + c];
            T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
        }
        float vST[2][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            vST[0][c] = vS00 * T[0][c] + vS01 * T[1][c];
            vST[1][c] = vS01 * T[0][c] + vS11 * T[1][c];
        }
        float vV[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) vV[r][c] = T[0][r] * vST[0][c] + T[1][r] * vST[1][c];
        float vT[2][3];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                vT[r][c] = 2.f * (vST[r][0] * Cs[0][c] + vST[r][1] * Cs[1][c] + vST[r][2] * Cs[2][c]);
        const float vJ00 = vT[0][0] * V[0] + vT[0][1] * V[1] + vT[0][2] * V[2];
        const float vJ02 = vT[0][0] * V[8] + vT[0][1] * V[9] + vT[0][2] * V[10];
        const float vJ11 = vT[1][0] * V[4] + vT[1][1] * V[5] + vT[1][2] * V[6];
        const float vJ12 = vT[1][0] * V[8] + vT[1][1] * V[9] + vT[1][2] * V[10];
        const float vttx = -fx * rz2 * vJ02, vtty = -fy * rz2 * vJ12;
        vtz += -fx * rz2 * vJ00 + 2.f * fx * ttx * rz3 * vJ02 - fy * rz2 * vJ11 +
               2.f * fy * tty * rz3 * vJ12;
        // D16: exactly on +-lim the reference's min(lim, max(-lim, q)) splits the gradient in half between the
        // branches: half to t.x, and 0.5 cq to t.z
        if (qx == lim_x || qx == -lim_x) { const float h = 0.5f * vttx; vtx += h; vtz += cqx * h; }
        else if (clamp_x) vtz += cqx * vttx; else vtx += vttx;
        if (qy == lim_y || qy == -lim_y) { const float h = 0.5f * vtty; vty += h; vtz += cqy * h; }
        else if (clamp_y) vtz += cqy * vtty; else vty += vtty;
        vm[0] += V[0] * vtx + V[4] * vty + V[8] * vtz;
        vm[1] += V[1] * vtx + V[5] * vty + V[9] * vtz;
        vm[2] += V[2] * vtx + V[6] * vty + V[10] * vtz;

        // cov3d = M M^T, M = R S
        float vM[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                vM[r][c] = 2.f * (vV[r][0] * M[0][c] + vV[r][1] * M[1][c] + vV[r][2] * M[2][c]);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            vs[c] = glob_scale * (R[0][c] * vM[0][c] + R[1][c] * vM[1][c] + R[2][c] * vM[2][c]);
            if (ACT) vs[c] = vs[c] * e[c];   // d exp(a) = exp(a)
        }
        float vR[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) vR[r][c] = vM[r][c] * s[c];
        const float nq = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
        const float inv = 1.0f / nq;
        const float w = q.x * inv, x = q.y * inv, y = q.z * inv, z = q.w * inv;
        const float gw = 2.f * (x * (vR[2][1] - vR[1][2]) + y * (vR[0][2] - vR[2][0]) + z * (vR[1][0] - vR[0][1]));
        const float gx = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[1][0] + vR[0][1]) +
                                z * (vR[2][0] + vR[0][2]) + w * (vR[2][1] - vR[1][2]));
        const float gy = 2.f * (x * (vR[1][0] + vR[0][1]) - 2.f * y * (vR[0][0] + vR[2][2]) +
                                z * (vR[2][1] + vR[1][2]) + w * (vR[0][2] - vR[2][0]));
        const float gz = 2.f * (x * (vR[2][0] + vR[0][2]) + y * (vR[2][1] + vR[1][2]) -
                                2.f * z * (vR[0][0] + vR[1][1]) + w * (vR[1][0] - vR[0][1]));
        const float dot = w * gw + x * gx + y * gy + z * gz;
        vq = make_float4((gw - w * dot) * inv, (gx - x * dot) * inv, (gy - y * dot) * inv,
                         (gz - z * dot) * inv);
    }
    if constexpr (ACC) {
        const float4 pq = v_quat[i];
        v_mean3d[3 * i] += vm[0]; v_mean3d[3 * i + 1] += vm[1]; v_mean3d[3 * i + 2] += vm[2];
        v_scale[3 * i] += vs[0]; v_scale[3 * i + 1] += vs[1]; v_scale[3 * i + 2] += vs[2];
        v_quat[i] = make_float4(pq.x + vq.x, pq.y + vq.y, pq.z + vq.z, pq.w + vq.w);
    } else {
        v_mean3d[3 * i] = vm[0]; v_mean3d[3 * i + 1] = vm[1]; v_mean3d[3 * i + 2] = vm[2];
        v_scale[3 * i] = vs[0]; v_scale[3 * i + 1] = vs[1]; v_scale[3 * i + 2] = vs[2];
        v_quat[i] = vq;
    }
}

}  // namespace

static int project_forward_impl(bool act, int n, const float *means3d, const float *scales, float glob_scale,
                                const float *quats, const float *opacity_logits, const float *viewmat,
                                const float *projmat, float fx, float fy, float cx, float cy, int img_h, int img_w,
                                int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys, float *depths,
                                int32_t *radii, float *conics, int32_t *num_tiles_hit, float *opacities,
                                gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && img_h > 0 && img_w > 0 && tiles_x > 0 && tiles_y > 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(means3d && scales && quats && viewmat && projmat && cov3d && xys && depths && radii &&
                  conics && num_tiles_hit);
    GSB_CHECK_ARG(!act || (opacity_logits && opacities));
    GSB_CHECK_ARG(((uintptr_t)quats % 16) == 0 && ((uintptr_t)xys % 8) == 0);
    // forward.cu:69-70 evaluates `0.5 * img_size.x / fx` in double and narrows
    const float tan_fovx = (float)(0.5 * (double)img_w / (double)fx);
    const float tan_fovy = (float)(0.5 * (double)img_h / (double)fy);
#define GSB_PJ_F(A) project_forward_kernel<A><<<gsb_div_up(n, PJ_THREADS), PJ_THREADS, 0, (cudaStream_t)stream>>>( \
        n, means3d, scales, glob_scale, quats, viewmat, projmat, fx, fy, cx, cy, tan_fovx, tan_fovy, img_h, img_w,   \
        tiles_x, tiles_y, clip_thresh, cov3d, reinterpret_cast<float2 *>(xys), depths, radii, conics, num_tiles_hit, \
        opacity_logits, opacities)
    if (act) GSB_PJ_F(true); else GSB_PJ_F(false);
#undef GSB_PJ_F
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_project_forward(int n, const float *means3d, const float *scales, float glob_scale,
                                   const float *quats, const float *viewmat, const float *projmat,
                                   float fx, float fy, float cx, float cy, int img_h, int img_w,
                                   int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                   float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                   gsb_stream_t stream) {
    return project_forward_impl(false, n, means3d, scales, glob_scale, quats, nullptr, viewmat, projmat, fx, fy, cx,
                                cy, img_h, img_w, tiles_x, tiles_y, clip_thresh, cov3d, xys, depths, radii, conics,
                                num_tiles_hit, nullptr, stream);
}

extern "C" int gsb_project_forward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                             const float *raw_quats, const float *opacity_logits,
                                             const float *viewmat, const float *projmat, float fx, float fy,
                                             float cx, float cy, int img_h, int img_w, int tiles_x, int tiles_y,
                                             float clip_thresh, float *cov3d, float *xys, float *depths,
                                             int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                             float *opacities, gsb_stream_t stream) {
    return project_forward_impl(true, n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, viewmat, projmat,
                                fx, fy, cx, cy, img_h, img_w, tiles_x, tiles_y, clip_thresh, cov3d, xys, depths, radii,
                                conics, num_tiles_hit, opacities, stream);
}

static int project_backward_impl(bool act, bool acc, int n, const float *means3d, const float *scales, float glob_scale,
                                 const float *quats, const float *opacities, const float *viewmat,
                                 const float *projmat, float fx, float fy, int img_h, int img_w,
                                 const int32_t *radii, const float *conics, const float *v_xy, const float *v_depth,
                                 const float *v_conic, const float *v_opacity, float *v_mean3d, float *v_scale,
                                 float *v_quat, float *v_opacity_logits, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && img_h > 0 && img_w > 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(means3d && scales && quats && viewmat && projmat && radii && conics && v_xy && v_conic &&
                  v_mean3d && v_scale && v_quat);
    GSB_CHECK_ARG(!act || (opacities && v_opacity_logits));
    GSB_CHECK_ARG(((uintptr_t)quats % 16) == 0 && ((uintptr_t)v_quat % 16) == 0 && ((uintptr_t)v_xy % 8) == 0);
    const float tan_fovx = (float)(0.5 * (double)img_w / (double)fx);
    const float tan_fovy = (float)(0.5 * (double)img_h / (double)fy);
#define GSB_PJ_B(A, ACC) project_backward_kernel<A, ACC><<<gsb_div_up(n, PJ_THREADS), PJ_THREADS, 0, (cudaStream_t)stream>>>( \
        n, means3d, scales, glob_scale, quats, viewmat, projmat, fx, fy, tan_fovx, tan_fovy, img_h, img_w, radii,     \
        conics, reinterpret_cast<const float2 *>(v_xy), v_depth, v_conic, v_mean3d, v_scale,                          \
        reinterpret_cast<float4 *>(v_quat), opacities, v_opacity, v_opacity_logits)
    if (acc) GSB_PJ_B(true, true); else if (act) GSB_PJ_B(true, false); else GSB_PJ_B(false, false);
#undef GSB_PJ_B
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_project_backward(int n, const float *means3d, const float *scales, float glob_scale,
                                    const float *quats, const float *viewmat, const float *projmat,
                                    float fx, float fy, float cx, float cy, int img_h, int img_w,
                                    const float *cov3d, const int32_t *radii, const float *conics,
                                    const float *v_xy, const float *v_depth, const float *v_conic,
                                    float *v_mean3d, float *v_scale, float *v_quat, gsb_stream_t stream) {
    (void)cov3d; (void)cx; (void)cy;
    return project_backward_impl(false, false, n, means3d, scales, glob_scale, quats, nullptr, viewmat, projmat, fx,
                                 fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, nullptr, v_mean3d, v_scale,
                                 v_quat, nullptr, stream);
}

extern "C" int gsb_project_backward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                              const float *raw_quats, const float *opacities, const float *viewmat,
                                              const float *projmat, float fx, float fy, int img_h, int img_w,
                                              const int32_t *radii, const float *conics, const float *v_xy,
                                              const float *v_depth, const float *v_conic, const float *v_opacity,
                                              float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                              float *v_opacity_logits, gsb_stream_t stream) {
    return project_backward_impl(true, false, n, means3d, log_scales, glob_scale, raw_quats, opacities, viewmat,
                                 projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity,
                                 v_mean3d, v_log_scales, v_raw_quats, v_opacity_logits, stream);
}

// The same VJP added into the four outputs (v += vjp): a trainer's several views of one step summed in place.
extern "C" int gsb_project_backward_activated_acc(int n, const float *means3d, const float *log_scales,
                                                  float glob_scale, const float *raw_quats, const float *opacities,
                                                  const float *viewmat, const float *projmat, float fx, float fy,
                                                  int img_h, int img_w, const int32_t *radii, const float *conics,
                                                  const float *v_xy, const float *v_depth, const float *v_conic,
                                                  const float *v_opacity, float *v_mean3d, float *v_log_scales,
                                                  float *v_raw_quats, float *v_opacity_logits, gsb_stream_t stream) {
    return project_backward_impl(true, true, n, means3d, log_scales, glob_scale, raw_quats, opacities, viewmat,
                                 projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity,
                                 v_mean3d, v_log_scales, v_raw_quats, v_opacity_logits, stream);
}
