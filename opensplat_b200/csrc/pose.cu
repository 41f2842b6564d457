// pose.cu -- per-image camera pose corrections (DESIGN D22; gsplat's pose optimisation): apply one image's learned
// correction to a view's camera, and take the camera gradient of the projection back to the correction.
//
// A correction is e = (t, d) in R^9: a translation t = e[0:3] and a 6-D rotation offset d = e[3:9].  With
// d' = d + (1,0,0,0,1,0), a1 = d'[0:3], a2 = d'[3:6]: b1 = a1/|a1|, b2 = normalize(a2 - (b1.a2) b1), b3 = b1 x b2, and
// Rd has the ROWS (b1, b2, b3).  The corrected camera-to-world is [R|T] Delta, Delta = [[Rd, t], [0, 1]] (Delta acts
// in the camera's own frame), so the view matrix becomes Delta^-1 view, Delta^-1 = [Rd^T | -Rd^T t], and the camera
// centre T + R t, R = view[0:3,0:3]^T.  Everything is computed in fp64 and rounded once; e = 0 returns the base
// camera unchanged, bit for bit.  One thread per call: a view is 9 parameters.
#include "gsb_common.cuh"

namespace {

struct Rot6d {
    double a1[3], a2[3], b1[3], b2[3], b3[3], w[3], n1, nw, s;   // s = b1.a2, w = a2 - s b1
};

__device__ void rot6d(const float *e, Rot6d &r) {
    for (int k = 0; k < 3; ++k) {
        r.a1[k] = (double)e[3 + k] + (k == 0 ? 1.0 : 0.0);
        r.a2[k] = (double)e[6 + k] + (k == 1 ? 1.0 : 0.0);
    }
    r.n1 = sqrt(r.a1[0] * r.a1[0] + r.a1[1] * r.a1[1] + r.a1[2] * r.a1[2]);
    for (int k = 0; k < 3; ++k) r.b1[k] = r.a1[k] / r.n1;
    r.s = r.b1[0] * r.a2[0] + r.b1[1] * r.a2[1] + r.b1[2] * r.a2[2];
    for (int k = 0; k < 3; ++k) r.w[k] = r.a2[k] - r.s * r.b1[k];
    r.nw = sqrt(r.w[0] * r.w[0] + r.w[1] * r.w[1] + r.w[2] * r.w[2]);
    for (int k = 0; k < 3; ++k) r.b2[k] = r.w[k] / r.nw;
    r.b3[0] = r.b1[1] * r.b2[2] - r.b1[2] * r.b2[1];
    r.b3[1] = r.b1[2] * r.b2[0] - r.b1[0] * r.b2[2];
    r.b3[2] = r.b1[0] * r.b2[1] - r.b1[1] * r.b2[0];
}

__device__ bool is_zero(const float *e) {
    bool z = true;
    for (int k = 0; k < GSB_POSE_FLOATS; ++k) z = z && e[k] == 0.f;
    return z;
}

// Delta^-1 = [A | u], A = Rd^T (A[r][k] = row k of Rd, column r), u = -A t
__device__ void inverse_delta(const float *e, const Rot6d &r, double A[3][3], double u[3]) {
    const double *rows[3] = {r.b1, r.b2, r.b3};
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) A[i][k] = rows[k][i];
    for (int i = 0; i < 3; ++i) u[i] = -(A[i][0] * (double)e[0] + A[i][1] * (double)e[1] + A[i][2] * (double)e[2]);
}

__global__ void pose_apply_kernel(const float *__restrict__ e, const float *__restrict__ view,
                                  const float *__restrict__ centre, float *__restrict__ view_out,
                                  float *__restrict__ centre_out) {
    if (threadIdx.x != 0) return;
    if (is_zero(e)) {
        for (int k = 0; k < 16; ++k) view_out[k] = view[k];
        for (int k = 0; k < 3; ++k) centre_out[k] = centre[k];
        return;
    }
    Rot6d r;
    rot6d(e, r);
    double A[3][3], u[3];
    inverse_delta(e, r, A, u);
    for (int i = 0; i < 3; ++i)
        for (int c = 0; c < 4; ++c) {
            double v = u[i] * (double)view[12 + c];
            for (int k = 0; k < 3; ++k) v += A[i][k] * (double)view[4 * k + c];
            view_out[4 * i + c] = (float)v;
        }
    for (int c = 0; c < 4; ++c) view_out[12 + c] = view[12 + c];
    // T' = T + R t, R = view[0:3,0:3]^T
    for (int i = 0; i < 3; ++i) {
        double v = (double)centre[i];
        for (int k = 0; k < 3; ++k) v += (double)view[4 * k + i] * (double)e[k];
        centre_out[i] = (float)v;
    }
}

__global__ void pose_backward_kernel(const float *__restrict__ e, const float *__restrict__ view,
                                     const float *__restrict__ proj, const float *__restrict__ v_viewmat,
                                     const float *__restrict__ v_projmat, float scale, float *__restrict__ grad) {
    if (threadIdx.x != 0) return;
    // G = dL/dview' = G_V + proj^T G_P (projmat' = proj view')
    double G[4][4];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            double v = (double)v_viewmat[4 * r + c];
            for (int k = 0; k < 4; ++k) v += (double)proj[4 * k + r] * (double)v_projmat[4 * k + c];
            G[r][c] = v;
        }
    // dL/dDelta^-1 = G view^T (view' = Delta^-1 view); only its rows 0..2 depend on e
    double GW[3][4];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) {
            double v = 0.0;
            for (int k = 0; k < 4; ++k) v += G[r][k] * (double)view[4 * c + k];
            GW[r][c] = v;
        }
    Rot6d r;
    rot6d(e, r);
    double A[3][3], u[3];
    inverse_delta(e, r, A, u);
    // u = -A t: dA[i][k] += -gu_i t_k, dt_k = -sum_i A[i][k] gu_i
    double gA[3][3], gt[3];
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) gA[i][k] = GW[i][k] - GW[i][3] * (double)e[k];
    for (int k = 0; k < 3; ++k) gt[k] = -(A[0][k] * GW[0][3] + A[1][k] * GW[1][3] + A[2][k] * GW[2][3]);
    // A = Rd^T: the gradient of row k of Rd is column k of gA
    double gb1[3], gb2[3], gb3[3];
    for (int i = 0; i < 3; ++i) {
        gb1[i] = gA[i][0];
        gb2[i] = gA[i][1];
        gb3[i] = gA[i][2];
    }
    // b3 = b1 x b2
    gb1[0] += r.b2[1] * gb3[2] - r.b2[2] * gb3[1];
    gb1[1] += r.b2[2] * gb3[0] - r.b2[0] * gb3[2];
    gb1[2] += r.b2[0] * gb3[1] - r.b2[1] * gb3[0];
    gb2[0] += gb3[1] * r.b1[2] - gb3[2] * r.b1[1];
    gb2[1] += gb3[2] * r.b1[0] - gb3[0] * r.b1[2];
    gb2[2] += gb3[0] * r.b1[1] - gb3[1] * r.b1[0];
    // b2 = w / |w|
    const double d2 = r.b2[0] * gb2[0] + r.b2[1] * gb2[1] + r.b2[2] * gb2[2];
    double gw[3];
    for (int k = 0; k < 3; ++k) gw[k] = (gb2[k] - r.b2[k] * d2) / r.nw;
    // w = a2 - (b1.a2) b1
    const double gwb1 = gw[0] * r.b1[0] + gw[1] * r.b1[1] + gw[2] * r.b1[2];
    double ga2[3];
    for (int k = 0; k < 3; ++k) {
        ga2[k] = gw[k] - gwb1 * r.b1[k];
        gb1[k] += -gwb1 * r.a2[k] - r.s * gw[k];
    }
    // b1 = a1 / |a1|
    const double d1 = r.b1[0] * gb1[0] + r.b1[1] * gb1[1] + r.b1[2] * gb1[2];
    double g[GSB_POSE_FLOATS];
    for (int k = 0; k < 3; ++k) {
        g[k] = gt[k];
        g[3 + k] = (gb1[k] - r.b1[k] * d1) / r.n1;
        g[6 + k] = ga2[k];
    }
    for (int k = 0; k < GSB_POSE_FLOATS; ++k) grad[k] = grad[k] + (float)((double)scale * g[k]);
}

}  // namespace

extern "C" int gsb_pose_apply(const float *pose, const float *view, const float *centre, float *view_out,
                              float *centre_out, gsb_stream_t stream) {
    GSB_CHECK_ARG(pose && view && centre && view_out && centre_out);
    pose_apply_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(pose, view, centre, view_out, centre_out);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_pose_backward(const float *pose, const float *view, const float *proj, const float *v_viewmat,
                                 const float *v_projmat, float scale, float *grad, gsb_stream_t stream) {
    GSB_CHECK_ARG(pose && view && proj && v_viewmat && v_projmat && grad);
    pose_backward_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(pose, view, proj, v_viewmat, v_projmat, scale, grad);
    GSB_LAUNCH_CHECK();
    return 0;
}
