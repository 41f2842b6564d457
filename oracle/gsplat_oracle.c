/*
 * oracle/gsplat_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C, single-threaded CPU restatement of the reference's differentiable Gaussian-splat
 * render path, with the *tile semantics* of the reference CUDA back end (which the reference
 * CPU back end, rasterizer/gsplat-cpu, does not have).  It exists to CHECK the sm_90a kernels
 * in opensplat_b200/csrc; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg
 * may load it.  The product path never links or calls it.
 *
 * Pinning: the reference ships no tests/golden vectors for this path (SURVEY.md section 4), so
 * this restatement is pinned against outputs of the reference itself: oracle/_ref (the unmodified
 * gsplat_cpu.cpp + operator .cpp files compiled from /root/reference) run by
 * tests/golden/make_golden.py, whose vectors are committed under tests/golden/.  See
 * tests/test_oracle_vs_golden.py.
 *
 * Each function cites the reference file:line it follows (paths relative to /root/reference).
 * All arithmetic is fp32, evaluated in the written order with NO fused multiply-add
 * (compile with -ffp-contract=off) so that integer artefacts (radii, num_tiles_hit, keys,
 * tile bins) can be reproduced bit-for-bit by the CUDA kernels (built with --fmad=false for the
 * projection translation unit).
 *
 * Decision rule where the reference's CUDA and CPU back ends disagree (SURVEY.md section 8c):
 *   - tile structure, depth key (view-space z), cx/cy handling, near clip, radius/num_tiles_hit
 *     rules                                    -> CUDA reference (forward.cu / helpers.cuh)
 *   - gradient mathematics (quat normalisation Jacobian, perspective divide, glob_scale,
 *     fov clamp sub-gradient, conic off-diagonal convention) -> exact VJP of the forward map,
 *     which is what the CPU reference obtains through torch autograd (gsplat_cpu.cpp:48-131).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_BLOCK_X 16 /* rasterizer/gsplat/config.h:1 */
#define ORC_BLOCK_Y 16 /* rasterizer/gsplat/config.h:2 */

/* CUDA cvt.rzi.s32.f32 semantics for (int)float: truncate, saturate, NaN -> 0. */
static int f2i_rz(float x) {
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (-2147483647 - 1);
    return (int)x;
}
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }
static float fminf_(float a, float b) { return a < b ? a : b; }
static float fmaxf_(float a, float b) { return a > b ? a : b; }

/* ------------------------------------------------------------------------------------------
 * Spherical harmonics.  rasterizer/gsplat/sh.cuh:12-37 (constants), :52-124 (forward),
 * :126-216 (vjp), :218-260 (kernels).  coeffs [N,K,3], viewdirs [N,3], colors [N,3].
 * The CUDA reference normalises viewdirs inside (sh.cuh:67-72); gsplat_cpu.cpp:438 does not
 * (callers pass unit vectors, model.cpp:177), so they agree on unit input.
 * ---------------------------------------------------------------------------------------- */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};
static const float SH_C4[9] = {2.5033429417967046f,  -1.7701307697799304f, 0.9461746957575601f,
                               -0.6690465435572892f, 0.10578554691520431f, -0.6690465435572892f,
                               0.47308734787878004f, -1.7701307697799304f, 0.6258357354491761f};

int orc_num_sh_bases(int degree) { /* sh.cuh:40-50 */
    if (degree == 0) return 1;
    if (degree == 1) return 4;
    if (degree == 2) return 9;
    if (degree == 3) return 16;
    return 25;
}

/* basis values Y[0..nb) for a (to-be-normalised) direction; sh.cuh:59-123 */
static void sh_basis(int degrees_to_use, const float *vd, float *Y) {
    Y[0] = SH_C0;
    if (degrees_to_use < 1) return;
    float norm = sqrtf(vd[0] * vd[0] + vd[1] * vd[1] + vd[2] * vd[2]);
    float x = vd[0] / norm, y = vd[1] / norm, z = vd[2] / norm;
    float xx = x * x, xy = x * y, xz = x * z, yy = y * y, yz = y * z, zz = z * z;
    Y[1] = -SH_C1 * y;
    Y[2] = SH_C1 * z;
    Y[3] = -SH_C1 * x;
    if (degrees_to_use < 2) return;
    Y[4] = SH_C2[0] * xy;
    Y[5] = SH_C2[1] * yz;
    Y[6] = SH_C2[2] * (2.f * zz - xx - yy);
    Y[7] = SH_C2[3] * xz;
    Y[8] = SH_C2[4] * (xx - yy);
    if (degrees_to_use < 3) return;
    Y[9] = SH_C3[0] * y * (3.f * xx - yy);
    Y[10] = SH_C3[1] * xy * z;
    Y[11] = SH_C3[2] * y * (4.f * zz - xx - yy);
    Y[12] = SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
    Y[13] = SH_C3[4] * x * (4.f * zz - xx - yy);
    Y[14] = SH_C3[5] * z * (xx - yy);
    Y[15] = SH_C3[6] * x * (xx - 3.f * yy);
    if (degrees_to_use < 4) return;
    Y[16] = SH_C4[0] * xy * (xx - yy);
    Y[17] = SH_C4[1] * yz * (3.f * xx - yy);
    Y[18] = SH_C4[2] * xy * (7.f * zz - 1.f);
    Y[19] = SH_C4[3] * yz * (7.f * zz - 3.f);
    Y[20] = SH_C4[4] * (zz * (35.f * zz - 30.f) + 3.f);
    Y[21] = SH_C4[5] * xz * (7.f * zz - 3.f);
    Y[22] = SH_C4[6] * (xx - yy) * (7.f * zz - 1.f);
    Y[23] = SH_C4[7] * xz * (xx - 3.f * yy);
    Y[24] = SH_C4[8] * (xx * (xx - 3.f * yy) - yy * (3.f * xx - yy));
}

/* compute_sh_forward_kernel sh.cuh:218-238 ; host compute_sh_forward_tensor bindings.cu:68-92 */
void orc_sh_forward(int n, int degree, int degrees_to_use, const float *viewdirs,
                    const float *coeffs, float *colors) {
    int K = orc_num_sh_bases(degree);
    int nb = orc_num_sh_bases(degrees_to_use);
    if (nb > K) nb = K;
    for (int i = 0; i < n; ++i) {
        float Y[25];
        sh_basis(degrees_to_use, viewdirs + 3 * i, Y);
        const float *c = coeffs + (size_t)i * K * 3;
        for (int ch = 0; ch < 3; ++ch) {
            float acc = 0.f;
            for (int b = 0; b < nb; ++b) acc += Y[b] * c[b * 3 + ch];
            colors[3 * i + ch] = acc;
        }
    }
}

/* compute_sh_backward_kernel sh.cuh:240-260 ; bases above degrees_to_use stay 0 (bindings.cu:110);
 * no gradient to viewdirs (spherical_harmonics.cpp:57-61) */
void orc_sh_backward(int n, int degree, int degrees_to_use, const float *viewdirs,
                     const float *v_colors, float *v_coeffs) {
    int K = orc_num_sh_bases(degree);
    int nb = orc_num_sh_bases(degrees_to_use);
    if (nb > K) nb = K;
    for (int i = 0; i < n; ++i) {
        float Y[25];
        sh_basis(degrees_to_use, viewdirs + 3 * i, Y);
        float *vc = v_coeffs + (size_t)i * K * 3;
        for (int b = 0; b < K; ++b)
            for (int ch = 0; ch < 3; ++ch)
                vc[b * 3 + ch] = (b < nb) ? Y[b] * v_colors[3 * i + ch] : 0.f;
    }
}

/* ------------------------------------------------------------------------------------------
 * Projection forward.  project_gaussians_forward_kernel forward.cu:19-103 with
 *   clip_near_plane helpers.cuh:225-233, transform_4x3 :91-98, scale_rot_to_cov3d forward.cu:450-470,
 *   quat_to_rotmat helpers.cuh:145-167 (quat stored w,x,y,z; rsqrtf replaced by 1/sqrtf, SURVEY 8c),
 *   project_cov3d_ewa forward.cu:381-447, compute_cov2d_bounds helpers.cuh:51-74,
 *   project_pix helpers.cuh:112-122, ndc2pix :13-15, get_tile_bbox :33-49, get_bbox :17-31.
 * Outputs are zero-initialised by the host binding (bindings.cu:162-173).
 * ---------------------------------------------------------------------------------------- */
static void quat_to_rotmat(const float *q, float R[3][3]) {
    /* helpers.cuh:145-167; R is row-major here: R[row][col] */
    float s = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
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

static void tile_bbox(float cx, float cy, float radius, int tiles_x, int tiles_y, int *x0, int *y0,
                      int *x1, int *y1) {
    /* helpers.cuh:33-49 + :17-31 */
    float tcx = cx / (float)ORC_BLOCK_X, tcy = cy / (float)ORC_BLOCK_Y;
    float trx = radius / (float)ORC_BLOCK_X, try_ = radius / (float)ORC_BLOCK_Y;
    *x0 = imin(imax(0, f2i_rz(tcx - trx)), tiles_x);
    *x1 = imin(imax(0, f2i_rz(tcx + trx + 1.f)), tiles_x);
    *y0 = imin(imax(0, f2i_rz(tcy - try_)), tiles_y);
    *y1 = imin(imax(0, f2i_rz(tcy + try_ + 1.f)), tiles_y);
}

void orc_project_forward(int n, const float *means3d, const float *scales, float glob_scale,
                         const float *quats, const float *viewmat, const float *projmat, float fx,
                         float fy, float cx, float cy, int img_h, int img_w, int tiles_x,
                         int tiles_y, float clip_thresh, float *cov3d, float *xys, float *depths,
                         int32_t *radii, float *conics, int32_t *num_tiles_hit) {
    /* forward.cu:69-70: `0.5 * img_size.x / fx` is evaluated in double, then narrowed */
    float tan_fovx = (float)(0.5 * (double)img_w / (double)fx);
    float tan_fovy = (float)(0.5 * (double)img_h / (double)fy);
    const float *V = viewmat, *P = projmat;
    for (int i = 0; i < n; ++i) {
        radii[i] = 0; /* forward.cu:42-43 */
        num_tiles_hit[i] = 0;
        float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];
        /* clip_near_plane / transform_4x3 */
        float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
        float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
        float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
        if (tz <= clip_thresh) continue;

        /* scale_rot_to_cov3d: M = R*S ; cov = M M^T */
        float R[3][3], M[3][3];
        quat_to_rotmat(quats + 4 * i, R);
        float s0 = glob_scale * scales[3 * i], s1 = glob_scale * scales[3 * i + 1],
              s2 = glob_scale * scales[3 * i + 2];
        for (int r = 0; r < 3; ++r) {
            M[r][0] = R[r][0] * s0;
            M[r][1] = R[r][1] * s1;
            M[r][2] = R[r][2] * s2;
        }
        float C[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                C[r][c] = M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2];
        float *c3 = cov3d + 6 * i;
        c3[0] = C[0][0]; c3[1] = C[0][1]; c3[2] = C[0][2];
        c3[3] = C[1][1]; c3[4] = C[1][2]; c3[5] = C[2][2];

        /* project_cov3d_ewa forward.cu:381-447 (t == view-space point, same op order) */
        float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
        float ttx = tz * fminf_(lim_x, fmaxf_(-lim_x, tx / tz));
        float tty = tz * fminf_(lim_y, fmaxf_(-lim_y, ty / tz));
        float rz = 1.f / tz, rz2 = rz * rz;
        float J00 = fx * rz, J02 = -fx * ttx * rz2, J11 = fy * rz, J12 = -fy * tty * rz2;
        /* T = J * W  (2x3) */
        float T[2][3];
        for (int c = 0; c < 3; ++c) {
            T[0][c] = J00 * V[c] + J02 * V[8 + c];
            T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
        }
        /* cov = T * Vcov * T^T */
        float Cs[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        float TV[2][3];
        for (int r = 0; r < 2; ++r)
            for (int c = 0; c < 3; ++c)
                TV[r][c] = T[r][0] * Cs[0][c] + T[r][1] * Cs[1][c] + T[r][2] * Cs[2][c];
        float cxx = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2] + 0.3f;
        float cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2];
        float cyy = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2] + 0.3f;

        /* compute_cov2d_bounds helpers.cuh:51-74 */
        float det = cxx * cyy - cxy * cxy;
        if (det == 0.f) continue;
        float inv_det = 1.f / det;
        float conic0 = cyy * inv_det, conic1 = -cxy * inv_det, conic2 = cxx * inv_det;
        float b = 0.5f * (cxx + cyy);
        float sq = sqrtf(fmaxf_(0.1f, b * b - det));
        float v1 = b + sq, v2 = b - sq;
        float radius = ceilf(3.f * sqrtf(fmaxf_(v1, v2)));
        conics[3 * i] = conic0; /* forward.cu:82 -- written before the bbox cull */
        conics[3 * i + 1] = conic1;
        conics[3 * i + 2] = conic2;

        /* project_pix helpers.cuh:112-122 */
        float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
        float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
        float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
        float rw = 1.f / (hw + 1e-6f);
        float ndcx = hx * rw, ndcy = hy * rw;
        float ux = 0.5f * (float)img_w * ndcx + cx - 0.5f;
        float uy = 0.5f * (float)img_h * ndcy + cy - 0.5f;

        int x0, y0, x1, y1;
        tile_bbox(ux, uy, radius, tiles_x, tiles_y, &x0, &y0, &x1, &y1);
        int32_t area = (x1 - x0) * (y1 - y0);
        if (area <= 0) continue;
        num_tiles_hit[i] = area; /* forward.cu:94-97 */
        depths[i] = tz;
        radii[i] = f2i_rz(radius);
        xys[2 * i] = ux;
        xys[2 * i + 1] = uy;
    }
}

/* ------------------------------------------------------------------------------------------
 * Projection backward: exact VJP of orc_project_forward w.r.t. (means3d, scales, quats) for
 * cotangents (v_xy, v_depth, v_conic).  Structure follows project_gaussians_backward_kernel
 * backward.cu:357-421 (skip radii<=0 :380; project_pix_vjp helpers.cuh:125-143;
 * cov2d_to_conic_vjp :77-88; project_cov3d_ewa_vjp backward.cu:424-502;
 * scale_rot_to_cov3d_vjp :506-542; quat_to_rotmat_vjp helpers.cuh:169-213) but, where that
 * hand VJP deviates from the true gradient, follows what the CPU reference gets from torch
 * autograd through gsplat_cpu.cpp:64-130 (SURVEY 8c D8, D11, D12):
 *   - perspective-divide term d rw/d mean kept (D12);
 *   - quaternion-normalisation Jacobian (I - qq^T)/|q| applied (D11);
 *   - v_scale multiplied by glob_scale, fov clamp sub-gradient honoured (D8);
 *   - v_conic[1] is the cotangent of the single stored off-diagonal conic entry (autograd
 *     convention of gsplat_cpu.cpp:105-109), i.e. G = [[vA, vB/2],[vB/2, vC]].
 * Accumulates in double internally? No: fp32, like the kernels; tests use tolerances.
 * ---------------------------------------------------------------------------------------- */
void orc_project_backward(int n, const float *means3d, const float *scales, float glob_scale,
                          const float *quats, const float *viewmat, const float *projmat, float fx,
                          float fy, float cx, float cy, int img_h, int img_w,
                          const int32_t *radii, const float *conics, const float *v_xy,
                          const float *v_depth, const float *v_conic, float *v_mean3d,
                          float *v_scale, float *v_quat) {
    (void)cx; (void)cy;
    float tan_fovx = (float)(0.5 * (double)img_w / (double)fx);
    float tan_fovy = (float)(0.5 * (double)img_h / (double)fy);
    const float *V = viewmat, *P = projmat;
    for (int i = 0; i < n; ++i) {
        v_mean3d[3 * i] = v_mean3d[3 * i + 1] = v_mean3d[3 * i + 2] = 0.f;
        v_scale[3 * i] = v_scale[3 * i + 1] = v_scale[3 * i + 2] = 0.f;
        v_quat[4 * i] = v_quat[4 * i + 1] = v_quat[4 * i + 2] = v_quat[4 * i + 3] = 0.f;
        if (radii[i] <= 0) continue;
        float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];
        float vmx = 0.f, vmy = 0.f, vmz = 0.f;

        /* --- pixel centre (project_pix) --- */
        float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
        float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
        float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
        float rw = 1.f / (hw + 1e-6f);
        float vndcx = 0.5f * (float)img_w * v_xy[2 * i];
        float vndcy = 0.5f * (float)img_h * v_xy[2 * i + 1];
        float vhx = vndcx * rw, vhy = vndcy * rw;
        float vhw = -(vndcx * hx + vndcy * hy) * rw * rw;
        vmx += P[0] * vhx + P[4] * vhy + P[12] * vhw;
        vmy += P[1] * vhx + P[5] * vhy + P[13] * vhw;
        vmz += P[2] * vhx + P[6] * vhy + P[14] * vhw;

        /* --- view-space point --- */
        float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
        float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
        float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
        float vtx = 0.f, vty = 0.f, vtz = v_depth ? v_depth[i] : 0.f;

        /* --- conic -> cov2d:  v_Sigma = -X G X --- */
        float A = conics[3 * i], B = conics[3 * i + 1], Cc = conics[3 * i + 2];
        float gA = v_conic[3 * i], gB = 0.5f * v_conic[3 * i + 1], gC = v_conic[3 * i + 2];
        /* XG = X*G */
        float xg00 = A * gA + B * gB, xg01 = A * gB + B * gC;
        float xg10 = B * gA + Cc * gB, xg11 = B * gB + Cc * gC;
        float vS00 = -(xg00 * A + xg01 * B);
        float vS01 = -(xg00 * B + xg01 * Cc);
        float vS11 = -(xg10 * B + xg11 * Cc);

        /* --- recompute forward intermediates --- */
        float R[3][3], M[3][3];
        quat_to_rotmat(quats + 4 * i, R);
        float s[3] = {glob_scale * scales[3 * i], glob_scale * scales[3 * i + 1],
                      glob_scale * scales[3 * i + 2]};
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) M[r][c] = R[r][c] * s[c];
        float Cs[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                Cs[r][c] = M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2];
        float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
        float qx = tx / tz, qy = ty / tz;
        int clamp_x = !(qx > -lim_x && qx < lim_x), clamp_y = !(qy > -lim_y && qy < lim_y);
        float cqx = fminf_(lim_x, fmaxf_(-lim_x, qx)), cqy = fminf_(lim_y, fmaxf_(-lim_y, qy));
        float ttx = tz * cqx, tty = tz * cqy;
        float rz = 1.f / tz, rz2 = rz * rz, rz3 = rz2 * rz;
        float J00 = fx * rz, J02 = -fx * ttx * rz2, J11 = fy * rz, J12 = -fy * tty * rz2;
        float T[2][3];
        for (int c = 0; c < 3; ++c) {
            T[0][c] = J00 * V[c] + J02 * V[8 + c];
            T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
        }
        /* v_V = T^T vS T  (3x3 symmetric) ; v_T = 2 vS T V */
        float vST[2][3];
        for (int c = 0; c < 3; ++c) {
            vST[0][c] = vS00 * T[0][c] + vS01 * T[1][c];
            vST[1][c] = vS01 * T[0][c] + vS11 * T[1][c];
        }
        float vV[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) vV[r][c] = T[0][r] * vST[0][c] + T[1][r] * vST[1][c];
        float vT[2][3];
        for (int r = 0; r < 2; ++r)
            for (int c = 0; c < 3; ++c)
                vT[r][c] = 2.f * (vST[r][0] * Cs[0][c] + vST[r][1] * Cs[1][c] + vST[r][2] * Cs[2][c]);
        /* v_J = v_T W^T */
        float vJ00 = vT[0][0] * V[0] + vT[0][1] * V[1] + vT[0][2] * V[2];
        float vJ02 = vT[0][0] * V[8] + vT[0][1] * V[9] + vT[0][2] * V[10];
        float vJ11 = vT[1][0] * V[4] + vT[1][1] * V[5] + vT[1][2] * V[6];
        float vJ12 = vT[1][0] * V[8] + vT[1][1] * V[9] + vT[1][2] * V[10];
        float vttx = -fx * rz2 * vJ02, vtty = -fy * rz2 * vJ12;
        vtz += -fx * rz2 * vJ00 + 2.f * fx * ttx * rz3 * vJ02 - fy * rz2 * vJ11 +
               2.f * fy * tty * rz3 * vJ12;
        /* exactly on +-lim torch's min/max split the gradient in half between the branches (D16) */
        if (qx == lim_x || qx == -lim_x) { float h = 0.5f * vttx; vtx += h; vtz += cqx * h; }
        else if (clamp_x) vtz += cqx * vttx; else vtx += vttx;
        if (qy == lim_y || qy == -lim_y) { float h = 0.5f * vtty; vty += h; vtz += cqy * h; }
        else if (clamp_y) vtz += cqy * vtty; else vty += vtty;
        vmx += V[0] * vtx + V[4] * vty + V[8] * vtz;
        vmy += V[1] * vtx + V[5] * vty + V[9] * vtz;
        vmz += V[2] * vtx + V[6] * vty + V[10] * vtz;
        v_mean3d[3 * i] = vmx; v_mean3d[3 * i + 1] = vmy; v_mean3d[3 * i + 2] = vmz;

        /* --- cov3d = M M^T :  v_M = 2 v_V M ; v_s_j = sum_i R_ij vM_ij ; v_R = v_M S --- */
        float vM[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                vM[r][c] = 2.f * (vV[r][0] * M[0][c] + vV[r][1] * M[1][c] + vV[r][2] * M[2][c]);
        for (int c = 0; c < 3; ++c)
            v_scale[3 * i + c] =
                glob_scale * (R[0][c] * vM[0][c] + R[1][c] * vM[1][c] + R[2][c] * vM[2][c]);
        float vR[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) vR[r][c] = vM[r][c] * s[c];
        /* R(q^) -> v_q^ ; then normalisation Jacobian */
        const float *q = quats + 4 * i;
        float nq = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        float inv = 1.0f / nq;
        float w = q[0] * inv, x = q[1] * inv, y = q[2] * inv, z = q[3] * inv;
        float gw = 2.f * (x * (vR[2][1] - vR[1][2]) + y * (vR[0][2] - vR[2][0]) + z * (vR[1][0] - vR[0][1]));
        float gx = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[1][0] + vR[0][1]) +
                          z * (vR[2][0] + vR[0][2]) + w * (vR[2][1] - vR[1][2]));
        float gy = 2.f * (x * (vR[1][0] + vR[0][1]) - 2.f * y * (vR[0][0] + vR[2][2]) +
                          z * (vR[2][1] + vR[1][2]) + w * (vR[0][2] - vR[2][0]));
        float gz = 2.f * (x * (vR[2][0] + vR[0][2]) + y * (vR[2][1] + vR[1][2]) -
                          2.f * z * (vR[0][0] + vR[1][1]) + w * (vR[1][0] - vR[0][1]));
        float dot = w * gw + x * gx + y * gy + z * gz;
        v_quat[4 * i] = (gw - w * dot) * inv;
        v_quat[4 * i + 1] = (gx - x * dot) * inv;
        v_quat[4 * i + 2] = (gy - y * dot) * inv;
        v_quat[4 * i + 3] = (gz - z * dot) * inv;
    }
}

/* ------------------------------------------------------------------------------------------
 * Binning.  torch::cumsum rasterize_gaussians.cpp:62 ; map_gaussian_to_intersects forward.cu:107-143 ;
 * torch::sort + gather rasterize_gaussians.cpp:25-32 ; get_tile_bin_edges forward.cu:148-169.
 * ---------------------------------------------------------------------------------------- */
int64_t orc_cumsum_i32(int n, const int32_t *in, int32_t *out) {
    int64_t acc = 0;
    for (int i = 0; i < n; ++i) {
        acc += in[i];
        out[i] = (int32_t)acc;
    }
    return acc;
}

void orc_map_gaussian_to_intersects(int n, const float *xys, const float *depths,
                                    const int32_t *radii, const int32_t *cum_tiles_hit, int tiles_x,
                                    int tiles_y, int64_t *isect_ids, int32_t *gaussian_ids) {
    for (int i = 0; i < n; ++i) {
        if (radii[i] <= 0) continue;
        int x0, y0, x1, y1;
        tile_bbox(xys[2 * i], xys[2 * i + 1], (float)radii[i], tiles_x, tiles_y, &x0, &y0, &x1, &y1);
        int32_t cur = (i == 0) ? 0 : cum_tiles_hit[i - 1];
        int32_t dbits;
        memcpy(&dbits, &depths[i], 4);
        int64_t depth_id = (int64_t)dbits; /* forward.cu:132 (sign-extending cast) */
        for (int ty = y0; ty < y1; ++ty)
            for (int tx = x0; tx < x1; ++tx) {
                int64_t tile_id = (int64_t)ty * tiles_x + tx;
                isect_ids[cur] = (tile_id << 32) | depth_id;
                gaussian_ids[cur] = i;
                ++cur;
            }
    }
}

/* stable ascending sort of (key, original index): bottom-up merge sort.  The reference's
 * torch::sort on CUDA is a CUB radix sort (stable in practice); ties resolve to ascending
 * original index == ascending gaussian id (SURVEY 8a row B3). */
void orc_sort_isects(int64_t m, const int64_t *keys, int64_t *keys_sorted, int32_t *index_sorted) {
    if (m <= 0) return;
    int64_t *ka = (int64_t *)malloc(sizeof(int64_t) * (size_t)m);
    int64_t *kb = (int64_t *)malloc(sizeof(int64_t) * (size_t)m);
    int32_t *ia = (int32_t *)malloc(sizeof(int32_t) * (size_t)m);
    int32_t *ib = (int32_t *)malloc(sizeof(int32_t) * (size_t)m);
    for (int64_t i = 0; i < m; ++i) { ka[i] = keys[i]; ia[i] = (int32_t)i; }
    for (int64_t w = 1; w < m; w *= 2) {
        for (int64_t lo = 0; lo < m; lo += 2 * w) {
            int64_t mid = lo + w < m ? lo + w : m, hi = lo + 2 * w < m ? lo + 2 * w : m;
            int64_t a = lo, b = mid, o = lo;
            while (a < mid && b < hi) {
                if (ka[b] < ka[a]) { kb[o] = ka[b]; ib[o++] = ia[b++]; }
                else               { kb[o] = ka[a]; ib[o++] = ia[a++]; }
            }
            while (a < mid) { kb[o] = ka[a]; ib[o++] = ia[a++]; }
            while (b < hi)  { kb[o] = ka[b]; ib[o++] = ia[b++]; }
        }
        int64_t *tk = ka; ka = kb; kb = tk;
        int32_t *ti = ia; ia = ib; ib = ti;
    }
    memcpy(keys_sorted, ka, sizeof(int64_t) * (size_t)m);
    memcpy(index_sorted, ia, sizeof(int32_t) * (size_t)m);
    free(ka); free(kb); free(ia); free(ib);
}

/* get_tile_bin_edges forward.cu:148-169.  tile_bins is [num_tiles,2], zero-initialised here
 * (the reference allocates [M,2] zeros, bindings.cu:324 -- indexed by tile id all the same). */
void orc_tile_bin_edges(int64_t m, int num_tiles, const int64_t *keys_sorted, int32_t *tile_bins) {
    memset(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)num_tiles);
    for (int64_t i = 0; i < m; ++i) {
        int32_t cur = (int32_t)(keys_sorted[i] >> 32);
        if (i == 0) tile_bins[2 * cur] = 0;
        if (i == m - 1) tile_bins[2 * cur + 1] = (int32_t)m;
        if (i > 0) {
            int32_t prev = (int32_t)(keys_sorted[i - 1] >> 32);
            if (prev != cur) {
                tile_bins[2 * prev + 1] = (int32_t)i;
                tile_bins[2 * cur] = (int32_t)i;
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Rasterize forward.  rasterize_forward forward.cu:256-378 (per pixel semantics; the 256-wide
 * shared-memory batching does not change results).  `exp_mode`: 0 = libm expf (as
 * gsplat_cpu.cpp:220 std::exp), 1 = exp2f(x*log2e) like __expf (forward.cu:343).
 * ---------------------------------------------------------------------------------------- */
static float orc_exp(float x, int exp_mode) {
    if (exp_mode == 1) return exp2f(x * 1.4426950408889634f);
    return expf(x);
}

void orc_rasterize_forward(int img_h, int img_w, int tiles_x, int tiles_y,
                           const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                           const float *xys, const float *conics, const float *colors,
                           const float *opacities, const float *background, int exp_mode,
                           float *out_img, float *final_Ts, int32_t *final_idx) {
    (void)tiles_y;
    for (int i = 0; i < img_h; ++i)
        for (int j = 0; j < img_w; ++j) {
            int tile_id = (i / ORC_BLOCK_Y) * tiles_x + (j / ORC_BLOCK_X);
            int r0 = tile_bins[2 * tile_id], r1 = tile_bins[2 * tile_id + 1];
            float px = (float)j, py = (float)i; /* forward.cu:281-282 : no half-pixel offset */
            float T = 1.f, o0 = 0.f, o1 = 0.f, o2 = 0.f;
            int cur_idx = 0; /* forward.cu:303 */
            for (int idx = r0; idx < r1; ++idx) {
                int g = gaussian_ids_sorted[idx];
                float a = conics[3 * g], b = conics[3 * g + 1], c = conics[3 * g + 2];
                float dx = xys[2 * g] - px, dy = xys[2 * g + 1] - py;
                float sigma = 0.5f * (a * dx * dx + c * dy * dy) + b * dx * dy;
                float alpha = fminf_(0.999f, opacities[g] * orc_exp(-sigma, exp_mode));
                if (sigma < 0.f || alpha < 1.f / 255.f) continue;
                float next_T = T * (1.f - alpha);
                if (next_T <= 1e-4f) break; /* terminate BEFORE blending (forward.cu:349-354) */
                float vis = alpha * T;
                o0 = o0 + colors[3 * g] * vis;
                o1 = o1 + colors[3 * g + 1] * vis;
                o2 = o2 + colors[3 * g + 2] * vis;
                T = next_T;
                cur_idx = idx;
            }
            size_t p = (size_t)i * img_w + j;
            final_Ts[p] = T;
            final_idx[p] = cur_idx;
            out_img[3 * p] = o0 + T * background[0];
            out_img[3 * p + 1] = o1 + T * background[1];
            out_img[3 * p + 2] = o2 + T * background[2];
        }
}

/* ------------------------------------------------------------------------------------------
 * Rasterize backward.  rasterize_backward_kernel backward.cu:161-355: per pixel, back to front
 * from final_idx, alpha clamp 0.99 (backward.cu:272; forward uses 0.999 -- reproduced, SURVEY R3).
 * Per-Gaussian sums are accumulated in pixel raster order in fp32 like gsplat_cpu.cpp:313-371.
 * v_output_alpha may be NULL (== zeros, rasterize_gaussians.cpp:108).
 * ---------------------------------------------------------------------------------------- */
void orc_rasterize_backward(int img_h, int img_w, int tiles_x, int tiles_y,
                            const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                            const float *xys, const float *conics, const float *colors,
                            const float *opacities, const float *background,
                            const float *final_Ts, const int32_t *final_idx,
                            const float *v_output, const float *v_output_alpha, int exp_mode,
                            int n, float *v_xy, float *v_conic, float *v_colors, float *v_opacity) {
    (void)tiles_y;
    memset(v_xy, 0, sizeof(float) * 2 * (size_t)n);
    memset(v_conic, 0, sizeof(float) * 3 * (size_t)n);
    memset(v_colors, 0, sizeof(float) * 3 * (size_t)n);
    memset(v_opacity, 0, sizeof(float) * (size_t)n);
    for (int i = 0; i < img_h; ++i)
        for (int j = 0; j < img_w; ++j) {
            int tile_id = (i / ORC_BLOCK_Y) * tiles_x + (j / ORC_BLOCK_X);
            int r0 = tile_bins[2 * tile_id], r1 = tile_bins[2 * tile_id + 1];
            if (r1 <= r0) continue;
            size_t p = (size_t)i * img_w + j;
            float px = (float)j, py = (float)i;
            float T_final = final_Ts[p], T = T_final;
            float buf0 = 0.f, buf1 = 0.f, buf2 = 0.f;
            int bin_final = final_idx[p];
            float vo0 = v_output[3 * p], vo1 = v_output[3 * p + 1], vo2 = v_output[3 * p + 2];
            float voa = v_output_alpha ? v_output_alpha[p] : 0.f;
            int start = bin_final < r1 - 1 ? bin_final : r1 - 1;
            for (int idx = start; idx >= r0; --idx) {
                int g = gaussian_ids_sorted[idx];
                float a = conics[3 * g], b = conics[3 * g + 1], c = conics[3 * g + 2];
                float dx = xys[2 * g] - px, dy = xys[2 * g + 1] - py;
                float sigma = 0.5f * (a * dx * dx + c * dy * dy) + b * dx * dy;
                float vis = orc_exp(-sigma, exp_mode);
                float opac = opacities[g];
                float alpha = fminf_(0.99f, opac * vis);
                if (sigma < 0.f || alpha < 1.f / 255.f) continue;
                float ra = 1.f / (1.f - alpha);
                T *= ra;
                float fac = alpha * T;
                float r = colors[3 * g], gg = colors[3 * g + 1], bb = colors[3 * g + 2];
                v_colors[3 * g] += fac * vo0;
                v_colors[3 * g + 1] += fac * vo1;
                v_colors[3 * g + 2] += fac * vo2;
                float v_alpha = 0.f;
                v_alpha += (r * T - buf0 * ra) * vo0;
                v_alpha += (gg * T - buf1 * ra) * vo1;
                v_alpha += (bb * T - buf2 * ra) * vo2;
                v_alpha += T_final * ra * voa;
                v_alpha += -T_final * ra * background[0] * vo0;
                v_alpha += -T_final * ra * background[1] * vo1;
                v_alpha += -T_final * ra * background[2] * vo2;
                buf0 += r * fac; buf1 += gg * fac; buf2 += bb * fac;
                float v_sigma = -opac * vis * v_alpha;
                v_conic[3 * g] += 0.5f * v_sigma * dx * dx;
                v_conic[3 * g + 1] += 0.5f * v_sigma * dx * dy;
                v_conic[3 * g + 2] += 0.5f * v_sigma * dy * dy;
                v_xy[2 * g] += v_sigma * (a * dx + b * dy);
                v_xy[2 * g + 1] += v_sigma * (b * dx + c * dy);
                v_opacity[g] += vis * v_alpha;
            }
        }
}
