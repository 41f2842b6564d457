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

#include <type_traits>

namespace {

constexpr int PJ_THREADS = 256;
// D22: the camera gradient of one view, per Gaussian: d/dviewmat rows 0..2 (12 floats), then d/dprojmat rows 0, 1
// and 3 (12 floats); row 3 of the viewmat and row 2 of the projmat are not read by the projection
constexpr int CG_TERMS = 24;

// The block's sum of each of the CG_TERMS terms, in a fixed tree: a shuffle tree within each warp, then the 8 warp
// sums added in warp order; one fp32 row per block.  Every thread of the block must call it.
__device__ __forceinline__ void camgrad_block_sum(const float (&cg)[CG_TERMS], float *__restrict__ out) {
    __shared__ float red[PJ_THREADS / 32][CG_TERMS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < CG_TERMS; ++k) {
        float v = cg[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = v + __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < CG_TERMS) {
        float v = red[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < PJ_THREADS / 32; ++w) v = v + red[w][threadIdx.x];
        out[threadIdx.x] = v;
    }
}

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

template <bool LOADP = true>
__device__ __forceinline__ void load_cam(const float *__restrict__ viewmat,
                                         const float *__restrict__ projmat, Cam &c) {
#pragma unroll
    for (int i = 0; i < 12; ++i) c.V[i] = __ldg(viewmat + i);
    if constexpr (LOADP) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c.P[i] = __ldg(projmat + i);
    }
}

// FISH (DESIGN D27): the OpenCV fisheye (Kannala-Brandt) camera.  theta = atan2(r, t.z), r = |t.xy|,
// theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8), (u, v) = f theta_d / r t.xy + c - 0.5.
// theta_lim is the host's float64 limit of the monotone part of theta_d (model.fisheye_theta_limit).
struct FishK {
    float k1, k2, k3, k4, theta_lim;
};

// Below rho = r / t.z = FISH_RHO the map is evaluated by its series in rho^2 (through rho^8: the first dropped terms
// of G and H are below fp32 rounding there; that of W, 80 c5 rho^6, is about 1e-6 of W at rho = 0.1, and w enters
// only as x^2 w beside h), which is finite and smooth at r = 0; above it by the closed form, whose cancellation in h
// and w is bounded by 1 / rho^2 and 1 / rho^4 there.
constexpr float FISH_RHO = 0.1f;

// The fisheye map's scalars at t, with g = theta_d / r (dg/dr = r h, dg/dt.z = -q): u = fx g t.x + cx - 0.5 and
// J = [[fx (g + x^2 h), fx x y h, -fx x q], [fy x y h, fy (g + y^2 h), -fy y q]].  SECOND: also w = (dh/dr) / r,
// m = (dq/dr) / r = -dh/dt.z and qz = dq/dt.z, the second derivatives the exact VJP of J needs.
struct FishT {
    float r2, theta, g, h, q, w, m, qz;
};

template <bool SECOND>
__device__ __forceinline__ FishT fisheye_terms(float tx, float ty, float tz, const FishK &k) {
    FishT f;
    f.r2 = tx * tx + ty * ty;
    const float r = sqrtf(f.r2);
    f.theta = atan2f(r, tz);
    const float t2 = f.theta * f.theta;
    const float D = 1.f + t2 * (3.f * k.k1 + t2 * (5.f * k.k2 + t2 * (7.f * k.k3 + t2 * (9.f * k.k4))));
    const float n2 = f.r2 + tz * tz;
    f.q = D / n2;
    if (r < FISH_RHO * tz) {
        // G(rho) = t.z g = 1 + c1 rho^2 + .. + c4 rho^8, H = G' / rho = t.z^3 h, W = H' / rho = t.z^5 w
        const float c1 = k.k1 - 1.f / 3.f;
        const float c2 = k.k2 - k.k1 + 0.2f;
        const float c3 = k.k3 - (5.f / 3.f) * k.k2 + (14.f / 15.f) * k.k1 - 1.f / 7.f;
        const float c4 = k.k4 - (7.f / 3.f) * k.k3 + (19.f / 9.f) * k.k2 - (818.f / 945.f) * k.k1 + 1.f / 9.f;
        const float iz = 1.f / tz, iz2 = iz * iz, p2 = f.r2 * iz2;
        const float G = 1.f + p2 * (c1 + p2 * (c2 + p2 * (c3 + p2 * c4)));
        const float H = 2.f * c1 + p2 * (4.f * c2 + p2 * (6.f * c3 + p2 * (8.f * c4)));
        f.g = G * iz;
        f.h = H * (iz2 * iz);
        if constexpr (SECOND) {
            const float W = 8.f * c2 + p2 * (24.f * c3 + p2 * (48.f * c4));
            f.w = W * ((iz2 * iz2) * iz);
            f.m = (3.f * f.h + f.r2 * f.w) / tz;
        }
    } else {
        const float td = f.theta * (1.f + t2 * (k.k1 + t2 * (k.k2 + t2 * (k.k3 + t2 * k.k4))));
        f.g = td / r;
        f.h = (tz * f.q - f.g) / f.r2;
        if constexpr (SECOND) {
            // dD/dtheta = theta E
            const float E = 6.f * k.k1 + t2 * (20.f * k.k2 + t2 * (42.f * k.k3 + t2 * (72.f * k.k4)));
            f.m = (E * tz * (f.theta / r) - 2.f * D) / (n2 * n2);
            f.w = (tz * f.m - 3.f * f.h) / f.r2;
        }
    }
    if constexpr (SECOND) f.qz = -(2.f * f.q + f.r2 * f.m) / tz;     // q is homogeneous of degree -2 in t
    return f;
}

// T = J V[0:3, 0:3] for the fisheye's full 2x3 J
__device__ __forceinline__ void fisheye_jacobian(float tx, float ty, const FishT &f, float fx, float fy,
                                                 float (&J)[2][3]) {
    const float xy = tx * ty;
    J[0][0] = fx * (f.g + (tx * tx) * f.h);
    J[0][1] = fx * (xy * f.h);
    J[0][2] = -(fx * (tx * f.q));
    J[1][0] = fy * (xy * f.h);
    J[1][1] = fy * (f.g + (ty * ty) * f.h);
    J[1][2] = -(fy * (ty * f.q));
}

// F3D (D24): sigma_k = sqrtf(s_k s_k + f f) from s_k = glob_scale e_k (e_k = expf(a_k)), r_k = s_k / sigma_k and
// c3 = (r_0 r_1) r_2 -- the one fp32 order of the forward and the backward, so that f = 0 gives sigma = s, r = 1, c3 = 1
__device__ __forceinline__ void filter3d_scales(float glob_scale, const float (&e)[3], float f, float (&sig)[3],
                                                float (&r)[3], float &c3) {
    const float ff = f * f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float s = glob_scale * e[k];
        sig[k] = sqrtf(s * s + ff);
        r[k] = s / sig[k];
    }
    c3 = r[0] * r[1] * r[2];
}

// ACT: the parameter activations of Model::forward (model.cpp:148-150,176-177,200) as this kernel's prologue --
// `scales` holds log-scales (exp here), `quats` the raw quaternions (quat_to_rotmat normalises, as the reference's
// does, so `quats / quats.norm()` needs no pass of its own), and sigmoid(opacity_logits) is written beside the
// projection outputs for the rasterizer.
// AA (with ACT only; DESIGN D19): the anti-aliased opacity -- sigmoid(logit) * comp, comp = sqrt(max(0, det0 / det)),
// det0 the determinant of the screen covariance before the 0.3 px^2 blur and det the one after it, so the blurred
// Gaussian carries the light of the unblurred one; comp = 0 where radii == 0.  Every other output is the ACT one.
// F3D (with ACT; DESIGN D24): Mip-Splatting's 3-D smoothing filter, f = filter3d[i] -- the covariance is built from
// sigma_k = sqrtf(s_k s_k + f f) in place of s_k = glob_scale exp(a_k), and the opacity is sigmoid(logit) * c3 (then
// x comp under AA), c3 = (r_0 r_1) r_2, r_k = s_k / sigma_k.  At f = 0, sigma = s, r = 1 and c3 = 1 exactly.
// FISH (with ACT; DESIGN D27): the fisheye camera of `fk` in place of projmat -- a Gaussian is also culled where
// theta > theta_lim, and J is the fisheye's full 2x3 Jacobian at the mean; the rest is the pinhole's.
template <bool ACT, bool AA = false, bool F3D = false, bool FISH = false>
__global__ void __launch_bounds__(PJ_THREADS)
project_forward_kernel(int n, const float *__restrict__ means3d, const float *__restrict__ scales,
                       float glob_scale, const float *__restrict__ quats,
                       const float *__restrict__ viewmat, const float *__restrict__ projmat, float fx,
                       float fy, float cx, float cy, float tan_fovx, float tan_fovy, int img_h, int img_w,
                       int tiles_x, int tiles_y, float clip_thresh, float *__restrict__ cov3d,
                       float2 *__restrict__ xys, float *__restrict__ depths, int *__restrict__ radii,
                       float *__restrict__ conics, int *__restrict__ num_tiles_hit,
                       const float *__restrict__ opacity_logits, float *__restrict__ opacities,
                       const float *__restrict__ filter3d = nullptr, FishK fk = {}) {
    static_assert(ACT || !AA, "the anti-aliased opacity needs the activated projection");
    static_assert(ACT || !F3D, "the 3-D filter needs the activated projection");
    static_assert((ACT && !F3D) || !FISH, "the fisheye camera takes the activated projection without the 3-D filter");
    const int i = blockIdx.x * PJ_THREADS + threadIdx.x;
    if (i >= n) return;
    if (ACT && !AA && !F3D) opacities[i] = 1.f / (1.f + expf(-opacity_logits[i]));
    float fsig[3] = {0.f, 0.f, 0.f}, fc3 = 1.f;    // F3D: the filtered scales sigma_k and c3
    if constexpr (F3D) {
        const float e[3] = {expf(scales[3 * i]), expf(scales[3 * i + 1]), expf(scales[3 * i + 2])};
        float r[3];
        filter3d_scales(glob_scale, e, filter3d[i], fsig, r, fc3);
        if (!AA) opacities[i] = 1.f / (1.f + expf(-opacity_logits[i])) * fc3;
    }
    float comp = 0.f;
    Cam cam;
    load_cam<!FISH>(viewmat, projmat, cam);
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
    FishT ft;
    if (tz > clip_thresh && (!FISH || (ft = fisheye_terms<false>(tx, ty, tz, fk)).theta <= fk.theta_lim)) {
        // scale_rot_to_cov3d (forward.cu:450-470): M = R*S, cov3d = M M^T
        const float4 q = reinterpret_cast<const float4 *>(quats)[i];  // (w,x,y,z)
        float R[3][3], M[3][3];
        quat_to_rotmat(q.x, q.y, q.z, q.w, R);
        const float a0 = scales[3 * i], a1 = scales[3 * i + 1], a2 = scales[3 * i + 2];
        const float s0 = F3D ? fsig[0] : glob_scale * (ACT ? expf(a0) : a0),
                    s1 = F3D ? fsig[1] : glob_scale * (ACT ? expf(a1) : a1),
                    s2 = F3D ? fsig[2] : glob_scale * (ACT ? expf(a2) : a2);
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

        float T[2][3];
        if constexpr (FISH) {
            float J[2][3];
            fisheye_jacobian(tx, ty, ft, fx, fy, J);
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) T[r][c] = J[r][0] * V[c] + J[r][1] * V[4 + c] + J[r][2] * V[8 + c];
        } else {
            // project_cov3d_ewa (forward.cu:381-447)
            const float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
            const float ttx = tz * fminf(lim_x, fmaxf(-lim_x, tx / tz));
            const float tty = tz * fminf(lim_y, fmaxf(-lim_y, ty / tz));
            const float rz = 1.f / tz, rz2 = rz * rz;
            const float J00 = fx * rz, J02 = -fx * ttx * rz2, J11 = fy * rz, J12 = -fy * tty * rz2;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                T[0][c] = J00 * V[c] + J02 * V[8 + c];
                T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
            }
        }
        const float Cs[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        float TV[2][3];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                TV[r][c] = T[r][0] * Cs[0][c] + T[r][1] * Cs[1][c] + T[r][2] * Cs[2][c];
        const float cxx0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2];
        const float cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2];
        const float cyy0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2];
        const float cxx = cxx0 + 0.3f, cyy = cyy0 + 0.3f;

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

            float pxc, pyc;
            if constexpr (FISH) {
                pxc = fx * (ft.g * tx) + cx - 0.5f;
                pyc = fy * (ft.g * ty) + cy - 0.5f;
            } else {
                // project_pix (helpers.cuh:112-122), ndc2pix (:13-15)
                const float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
                const float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
                const float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
                const float rw = 1.f / (hw + 1e-6f);
                const float ndcx = hx * rw, ndcy = hy * rw;
                pxc = 0.5f * (float)img_w * ndcx + cx - 0.5f;
                pyc = 0.5f * (float)img_h * ndcy + cy - 0.5f;
            }

            int x0, x1, y0, y1;
            gsb_tile_bbox(pxc, pyc, radius, tiles_x, tiles_y, x0, x1, y0, y1);
            const int a = (x1 - x0) * (y1 - y0);
            if (a > 0) {
                area = a;
                depth = tz;
                radius_i = (int)radius;
                ux = pxc;
                uy = pyc;
                if (AA && radius_i > 0) comp = sqrtf(fmaxf(0.f, (cxx0 * cyy0 - cxy * cxy) / det));
            }
        }
    }
    if constexpr (AA && F3D) opacities[i] = 1.f / (1.f + expf(-opacity_logits[i])) * fc3 * comp;
    else if (AA) opacities[i] = 1.f / (1.f + expf(-opacity_logits[i])) * comp;
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
// AA: VJP of the anti-aliased forward (D19).  `opacities` holds the opacity LOGITS (o and comp are recomputed with the
// forward's expressions, bit for bit); v_logit = v_opacity * comp * o (1 - o), and where comp > 0 the cotangent
// v_opacity * o of comp is taken to the blurred covariance and added to vS before the T / J / clamp chain.
// CAMGRAD (with ACT; DESIGN D22): also the exact VJP w.r.t. viewmat and projmat, summed over the block's Gaussians
// (camgrad_block_sum) into row blockIdx.x of cam_partials; every other output is the one without CAMGRAD, bit for bit.
// F3D (with ACT; DESIGN D24): VJP of the filtered forward with f = filter3d[i] held constant.  `opacities` holds the
// logits, as under AA.  d sigma_k / d a_k = s_k r_k, so v_scale gains the factor r_k; the opacity (o c3 [comp]) adds
// v_opacity * o_eff * (f / sigma_k)^2 to v_scale (written in that form, not 1 - r_k^2, which cancels for the small
// Gaussians the filter is for), and v_logit = v_opacity * c3 [* comp] * o (1 - o).
// FISH (with ACT, not F3D; DESIGN D27): VJP of the fisheye forward.  `opacities` holds the logits in every mode.  The
// pixel centre's gradient reaches the mean through t, and J's own dependence on t (through g, h, q and their second
// derivatives w, m, qz) is taken in full; under CAMGRAD the three projmat rows of the partial row are 0.
template <bool ACT, bool ACC, bool AA = false, bool CAMGRAD = false, bool F3D = false, bool FISH = false>
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
                        float *__restrict__ v_opacity_logits, float *__restrict__ cam_partials = nullptr,
                        const float *__restrict__ filter3d = nullptr, FishK fk = {}) {
    static_assert(ACT || !AA, "the anti-aliased opacity needs the activated projection");
    static_assert(ACT || !F3D, "the 3-D filter needs the activated projection");
    static_assert(ACT || !CAMGRAD, "the camera gradient is taken with the activated projection");
    static_assert((ACT && !F3D) || !FISH, "the fisheye camera takes the activated projection without the 3-D filter");
    const int i = blockIdx.x * PJ_THREADS + threadIdx.x;
    // CAMGRAD: every thread of the block takes part in the reduction, so none returns early
    if (!CAMGRAD && i >= n) return;
    float cg[CG_TERMS];    // CAMGRAD: this Gaussian's camera-gradient terms (0 past n and where radii == 0)
#pragma unroll
    for (int k = 0; k < CG_TERMS; ++k) cg[k] = 0.f;
    if (!CAMGRAD || i < n) {
        float comp = 0.f;
        // F3D: f, r_k and c3 as in the forward, and (f / sigma_k)^2 for the opacity's share of v_scale; computed
        // inside the radii > 0 branch from its exp(a), or on their own where radii == 0
        float f3 = 0.f, fr[3] = {1.f, 1.f, 1.f}, fc3 = 1.f, fsh[3] = {0.f, 0.f, 0.f};
        if constexpr (F3D) f3 = filter3d[i];
        if (ACT && !AA && !F3D) {
            const float o = FISH ? 1.f / (1.f + expf(-opacities[i])) : opacities[i];
            if constexpr (ACC)
                v_opacity_logits[i] = v_opacity_logits[i] + (v_opacity ? v_opacity[i] * o * (1.f - o) : 0.f);
            else
                v_opacity_logits[i] = v_opacity ? v_opacity[i] * o * (1.f - o) : 0.f;
        }
        float vm[3] = {0.f, 0.f, 0.f}, vs[3] = {0.f, 0.f, 0.f};
        float4 vq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (radii[i] > 0) {
            Cam cam;
            load_cam<!FISH>(viewmat, projmat, cam);
            const float *V = cam.V, *P = cam.P;
            const float px = means3d[3 * i], py = means3d[3 * i + 1], pz = means3d[3 * i + 2];

            float vhx = 0.f, vhy = 0.f, vhw = 0.f;
            if constexpr (!FISH) {
                // pixel centre: xy = 0.5*W*(h.x*rw) + cx - 0.5, rw = 1/(h.w + 1e-6)
                const float hx = P[0] * px + P[1] * py + P[2] * pz + P[3];
                const float hy = P[4] * px + P[5] * py + P[6] * pz + P[7];
                const float hw = P[12] * px + P[13] * py + P[14] * pz + P[15];
                const float rw = 1.f / (hw + 1e-6f);
                const float2 vxy = v_xy[i];
                const float vndcx = 0.5f * (float)img_w * vxy.x, vndcy = 0.5f * (float)img_h * vxy.y;
                vhx = vndcx * rw;
                vhy = vndcy * rw;
                vhw = -(vndcx * hx + vndcy * hy) * rw * rw;
                vm[0] = P[0] * vhx + P[4] * vhy + P[12] * vhw;
                vm[1] = P[1] * vhx + P[5] * vhy + P[13] * vhw;
                vm[2] = P[2] * vhx + P[6] * vhy + P[14] * vhw;
            }

            const float tx = V[0] * px + V[1] * py + V[2] * pz + V[3];
            const float ty = V[4] * px + V[5] * py + V[6] * pz + V[7];
            const float tz = V[8] * px + V[9] * py + V[10] * pz + V[11];
            float vtx = 0.f, vty = 0.f, vtz = v_depth ? v_depth[i] : 0.f;

            // conic = inverse(cov2d):  v_Sigma = -X G X,  G = [[vA, vB/2],[vB/2, vC]]
            const float A = conics[3 * i], B = conics[3 * i + 1], Cc = conics[3 * i + 2];
            const float gA = v_conic[3 * i], gB = 0.5f * v_conic[3 * i + 1], gC = v_conic[3 * i + 2];
            const float xg00 = A * gA + B * gB, xg01 = A * gB + B * gC;
            const float xg10 = B * gA + Cc * gB, xg11 = B * gB + Cc * gC;
            float vS00 = -(xg00 * A + xg01 * B);
            float vS01 = -(xg00 * B + xg01 * Cc);
            float vS11 = -(xg10 * B + xg11 * Cc);

            // recompute forward intermediates
            const float4 q = reinterpret_cast<const float4 *>(quats)[i];
            float R[3][3], M[3][3];
            quat_to_rotmat(q.x, q.y, q.z, q.w, R);
            const float a[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
            const float e[3] = {ACT ? expf(a[0]) : a[0], ACT ? expf(a[1]) : a[1], ACT ? expf(a[2]) : a[2]};
            float s[3] = {glob_scale * e[0], glob_scale * e[1], glob_scale * e[2]};
            if constexpr (F3D) filter3d_scales(glob_scale, e, f3, s, fr, fc3);
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
            // FISH: the fisheye's terms and J; the pinhole's clamp and J above are then unused
            FishT ft;
            float Jf[2][3];
            if constexpr (FISH) {
                ft = fisheye_terms<true>(tx, ty, tz, fk);
                fisheye_jacobian(tx, ty, ft, fx, fy, Jf);
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int c = 0; c < 3; ++c) T[r][c] = Jf[r][0] * V[c] + Jf[r][1] * V[4 + c] + Jf[r][2] * V[8 + c];
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    T[0][c] = J00 * V[c] + J02 * V[8 + c];
                    T[1][c] = J11 * V[4 + c] + J12 * V[8 + c];
                }
            }
            if constexpr (AA) {
                // the forward's cov2d sums and det, recomputed in its order
                float TV[2][3];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        TV[r][c] = T[r][0] * Cs[0][c] + T[r][1] * Cs[1][c] + T[r][2] * Cs[2][c];
                const float cxx0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2];
                const float cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2];
                const float cyy0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2];
                const float det = (cxx0 + 0.3f) * (cyy0 + 0.3f) - cxy * cxy;
                comp = sqrtf(fmaxf(0.f, (cxx0 * cyy0 - cxy * cxy) / det));
                if (v_opacity && comp > 0.f) {
                    // d comp^2 / d Sigma = ((1 - comp^2) Sigma^-1 - 0.3 det(Sigma^-1) I), per symmetric entry, written as
                    // 0.3 / det^2 [[cyy0^2 + cxy^2 + 0.3 cyy0, -cxy (cxx0 + cyy0 + 0.3)], [.., cxx0^2 + cxy^2 + 0.3 cxx0]]:
                    // the same value without the cancellation of the first form when Sigma0 is small against 0.3 I
                    const float o = 1.f / (1.f + expf(-opacities[i]));
                    const float k = 0.5f * (v_opacity[i] * (F3D ? o * fc3 : o)) / comp;
                    const float id = 1.f / det;
                    const float a = cyy0 * id, b = cxy * id, c = cxx0 * id, e = 0.3f * id;
                    vS00 = vS00 + k * (0.3f * (a * a + b * b + e * a));
                    vS01 = vS01 - k * (0.3f * (b * (a + c + e)));
                    vS11 = vS11 + k * (0.3f * (c * c + b * b + e * c));
                }
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
            if constexpr (FISH) {
                // vJ = vT V^T; A = f vJ row by row; then J^T (v_u, v_v) and sum_rc vJ_rc dJ_rc / dt, with dg = (x h, y h,
                // -q), dh = (x w, y w, -m), dq = (x m, y m, qz)
                float A[2][3];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        A[r][c] = (r == 0 ? fx : fy) *
                                  (vT[r][0] * V[4 * c] + vT[r][1] * V[4 * c + 1] + vT[r][2] * V[4 * c + 2]);
                const float2 vxy = v_xy[i];
                const float xx = tx * tx, yy = ty * ty, xy = tx * ty;
                const float hx = ft.h + xx * ft.w, hy = ft.h + yy * ft.w, S = A[0][1] + A[1][0];
                const float qxm = ft.q + xx * ft.m, qym = ft.q + yy * ft.m, xym = xy * ft.m;
                vtx = Jf[0][0] * vxy.x + Jf[1][0] * vxy.y + A[0][0] * (tx * (2.f * ft.h + hx)) + S * (ty * hx) +
                      A[1][1] * (tx * hy) - A[0][2] * qxm - A[1][2] * xym;
                vty = Jf[0][1] * vxy.x + Jf[1][1] * vxy.y + A[0][0] * (ty * hx) + S * (tx * hy) +
                      A[1][1] * (ty * (2.f * ft.h + hy)) - A[0][2] * xym - A[1][2] * qym;
                vtz = vtz + Jf[0][2] * vxy.x + Jf[1][2] * vxy.y - A[0][0] * qxm - S * xym - A[1][1] * qym -
                      (A[0][2] * tx + A[1][2] * ty) * ft.qz;
            } else {
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
            }
            vm[0] += V[0] * vtx + V[4] * vty + V[8] * vtz;
            vm[1] += V[1] * vtx + V[5] * vty + V[9] * vtz;
            vm[2] += V[2] * vtx + V[6] * vty + V[10] * vtz;
            if constexpr (CAMGRAD) {
                // D22: t = V[0:3,:] (p, 1) gives vt_r (p, 1) to row r of V, T = J V[0:3,0:3] gives J^T vT to columns
                // 0..2; (hx, hy, hw) = P rows 0, 1, 3 times (p, 1) give vh (p, 1)
                const float pc[3] = {px, py, pz}, vt[3] = {vtx, vty, vtz}, vh[3] = {vhx, vhy, vhw};
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        cg[4 * r + c] = vt[r] * pc[c];
                        cg[12 + 4 * r + c] = vh[r] * pc[c];
                    }
                    cg[4 * r + 3] = vt[r];
                    cg[12 + 4 * r + 3] = vh[r];
                }
                if constexpr (FISH) {
#pragma unroll
                    for (int j = 0; j < 3; ++j)
#pragma unroll
                        for (int c = 0; c < 3; ++c) cg[4 * j + c] = cg[4 * j + c] + (Jf[0][j] * vT[0][c] + Jf[1][j] * vT[1][c]);
                } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    cg[c] = cg[c] + J00 * vT[0][c];
                    cg[4 + c] = cg[4 + c] + J11 * vT[1][c];
                    cg[8 + c] = cg[8 + c] + (J02 * vT[0][c] + J12 * vT[1][c]);
                }
                }
            }

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
                if (F3D) vs[c] = vs[c] * fr[c];  // d sigma / d s = r
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
            if constexpr (F3D) {
#pragma unroll
                for (int k = 0; k < 3; ++k) { const float t = f3 / s[k]; fsh[k] = t * t; }
            }
        } else if constexpr (F3D) {
            const float e[3] = {expf(scales[3 * i]), expf(scales[3 * i + 1]), expf(scales[3 * i + 2])};
            float sg[3];
            filter3d_scales(glob_scale, e, f3, sg, fr, fc3);
#pragma unroll
            for (int k = 0; k < 3; ++k) { const float t = f3 / sg[k]; fsh[k] = t * t; }
        }
        if constexpr (AA && !F3D) {
            float vol = 0.f;
            if (v_opacity) {
                const float o = 1.f / (1.f + expf(-opacities[i]));
                vol = v_opacity[i] * comp * o * (1.f - o);
            }
            v_opacity_logits[i] = ACC ? v_opacity_logits[i] + vol : vol;
        }
        if constexpr (F3D) {
            float vol = 0.f;
            if (v_opacity) {
                const float o = 1.f / (1.f + expf(-opacities[i]));
                vol = AA ? v_opacity[i] * fc3 * comp * o * (1.f - o) : v_opacity[i] * fc3 * o * (1.f - o);
                if (f3 > 0.f) {
                    // d c3 / d a_k = c3 (f / sigma_k)^2: the opacity's share of v_scale, for every Gaussian
                    const float vo = v_opacity[i] * (AA ? o * fc3 * comp : o * fc3);
#pragma unroll
                    for (int k = 0; k < 3; ++k) vs[k] = vs[k] + vo * fsh[k];
                }
            }
            v_opacity_logits[i] = ACC ? v_opacity_logits[i] + vol : vol;
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
    if constexpr (CAMGRAD) camgrad_block_sum(cg, cam_partials + CG_TERMS * (size_t)blockIdx.x);
}

// D22: the sum over the blocks' partial rows, one warp per term: lane l adds blocks l, l + 32, ... in fp64 in that
// order, then a fixed shuffle tree; rounded once into v_viewmat rows 0..2 and v_projmat rows 0, 1, 3 (the rows the
// projection reads), the other two rows written 0.
__global__ void __launch_bounds__(CG_TERMS * 32)
camgrad_reduce_kernel(int nblocks, const float *__restrict__ partials, float *__restrict__ v_viewmat,
                      float *__restrict__ v_projmat) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double s = 0.0;
    for (int b = lane; b < nblocks; b += 32) s += (double)partials[CG_TERMS * (size_t)b + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (lane == 0) {
        const float r = (float)s;
        if (k < 12) v_viewmat[k] = r;
        else v_projmat[k < 20 ? k - 12 : k - 8] = r;       // projmat rows 0, 1, then 3
    }
    if (threadIdx.x < 4) {
        v_viewmat[12 + threadIdx.x] = 0.f;
        v_projmat[8 + threadIdx.x] = 0.f;
    }
}

}  // namespace

// A projection mode: the kernels' template flags (ACC and CAMGRAD are the backward's only).
enum : unsigned { PJ_ACT = 1, PJ_AA = 2, PJ_F3D = 4, PJ_FISH = 8, PJ_ACC = 16, PJ_CAMGRAD = 32 };

static unsigned pj_flag(int on, unsigned flag) { return on ? flag : 0u; }

// The modes the kernels' static_asserts allow: AA, F3D, FISH, ACC and CAMGRAD need ACT, and FISH excludes F3D.  Each
// launcher checks its call's mode against it and instantiates exactly the modes it allows.
constexpr bool pj_legal(bool act, bool acc, bool aa, bool camgrad, bool f3d, bool fish) {
    return (act || !(acc || aa || camgrad || f3d || fish)) && !(f3d && fish);
}

// f(std::bool_constant<b>...) for the run-time flags b...: the one place a mode becomes template arguments.
template <class F> static void pj_with_flags(F &&f) { f(); }
template <class F, class... R> static void pj_with_flags(F &&f, bool b, R... rest) {
    if (b) pj_with_flags([&](auto... c) { f(std::true_type{}, c...); }, rest...);
    else pj_with_flags([&](auto... c) { f(std::false_type{}, c...); }, rest...);
}

// One call of project_forward_kernel as the extern "C" wrappers describe it: the mode (PJ_ACT, PJ_AA, PJ_F3D,
// PJ_FISH), then the kernel's pointers and scalars.  opacity_logits and opacities are read under ACT, filter3d under
// F3D and fk under FISH, where projmat is NULL.
struct ProjectForward {
    unsigned mode;
    int n;
    const float *means3d, *scales;
    float glob_scale;
    const float *quats, *opacity_logits, *filter3d, *viewmat, *projmat;
    float fx, fy, cx, cy;
    int img_h, img_w, tiles_x, tiles_y;
    float clip_thresh;
    float *cov3d, *xys, *depths;
    int32_t *radii;
    float *conics;
    int32_t *num_tiles_hit;
    float *opacities;
    FishK fk;
};

static int project_forward(const ProjectForward &c, gsb_stream_t stream) {
    const unsigned m = c.mode;
    GSB_CHECK_ARG(pj_legal(m & PJ_ACT, false, m & PJ_AA, false, m & PJ_F3D, m & PJ_FISH));
    GSB_CHECK_ARG(c.n >= 0 && c.img_h > 0 && c.img_w > 0 && c.tiles_x > 0 && c.tiles_y > 0);
    if (c.n == 0) return 0;
    GSB_CHECK_ARG(c.means3d && c.scales && c.quats && c.viewmat && (c.projmat || (m & PJ_FISH)) && c.cov3d && c.xys &&
                  c.depths && c.radii && c.conics && c.num_tiles_hit);
    GSB_CHECK_ARG(!(m & PJ_ACT) || (c.opacity_logits && c.opacities));
    GSB_CHECK_ARG(((uintptr_t)c.quats % 16) == 0 && ((uintptr_t)c.xys % 8) == 0);
    // forward.cu:69-70 evaluates `0.5 * img_size.x / fx` in double and narrows
    const float tan_fovx = (float)(0.5 * (double)c.img_w / (double)c.fx);
    const float tan_fovy = (float)(0.5 * (double)c.img_h / (double)c.fy);
    pj_with_flags([&](auto act, auto aa, auto f3d, auto fish) {
        if constexpr (pj_legal(act, false, aa, false, f3d, fish))
            project_forward_kernel<act, aa, f3d, fish>
                <<<gsb_div_up(c.n, PJ_THREADS), PJ_THREADS, 0, (cudaStream_t)stream>>>(
                    c.n, c.means3d, c.scales, c.glob_scale, c.quats, c.viewmat, c.projmat, c.fx, c.fy, c.cx, c.cy,
                    tan_fovx, tan_fovy, c.img_h, c.img_w, c.tiles_x, c.tiles_y, c.clip_thresh, c.cov3d,
                    reinterpret_cast<float2 *>(c.xys), c.depths, c.radii, c.conics, c.num_tiles_hit, c.opacity_logits,
                    c.opacities, c.filter3d, c.fk);
    }, m & PJ_ACT, m & PJ_AA, m & PJ_F3D, m & PJ_FISH);
    GSB_LAUNCH_CHECK();
    return 0;
}

// One call of project_backward_kernel: the mode (PJ_ACT, PJ_ACC, PJ_AA, PJ_CAMGRAD, PJ_F3D, PJ_FISH), then the
// kernel's pointers and scalars.  `opacities` holds sigmoid(logits) for ACT alone and the logits in every other
// activated mode; cam_partials is written under CAMGRAD.
struct ProjectBackward {
    unsigned mode;
    int n;
    const float *means3d, *scales;
    float glob_scale;
    const float *quats, *opacities, *filter3d, *viewmat, *projmat;
    float fx, fy;
    int img_h, img_w;
    const int32_t *radii;
    const float *conics, *v_xy, *v_depth, *v_conic, *v_opacity;
    float *v_mean3d, *v_scale, *v_quat, *v_opacity_logits, *cam_partials;
    FishK fk;
};

static int project_backward(const ProjectBackward &c, gsb_stream_t stream) {
    const unsigned m = c.mode;
    GSB_CHECK_ARG(pj_legal(m & PJ_ACT, m & PJ_ACC, m & PJ_AA, m & PJ_CAMGRAD, m & PJ_F3D, m & PJ_FISH));
    GSB_CHECK_ARG(c.n >= 0 && c.img_h > 0 && c.img_w > 0);
    if (c.n == 0) return 0;
    GSB_CHECK_ARG(c.means3d && c.scales && c.quats && c.viewmat && (c.projmat || (m & PJ_FISH)) && c.radii &&
                  c.conics && c.v_xy && c.v_conic && c.v_mean3d && c.v_scale && c.v_quat);
    GSB_CHECK_ARG(!(m & PJ_ACT) || (c.opacities && c.v_opacity_logits));
    GSB_CHECK_ARG(((uintptr_t)c.quats % 16) == 0 && ((uintptr_t)c.v_quat % 16) == 0 && ((uintptr_t)c.v_xy % 8) == 0);
    const float tan_fovx = (float)(0.5 * (double)c.img_w / (double)c.fx);
    const float tan_fovy = (float)(0.5 * (double)c.img_h / (double)c.fy);
    pj_with_flags([&](auto act, auto acc, auto aa, auto camgrad, auto f3d, auto fish) {
        if constexpr (pj_legal(act, acc, aa, camgrad, f3d, fish))
            project_backward_kernel<act, acc, aa, camgrad, f3d, fish>
                <<<gsb_div_up(c.n, PJ_THREADS), PJ_THREADS, 0, (cudaStream_t)stream>>>(
                    c.n, c.means3d, c.scales, c.glob_scale, c.quats, c.viewmat, c.projmat, c.fx, c.fy, tan_fovx,
                    tan_fovy, c.img_h, c.img_w, c.radii, c.conics, reinterpret_cast<const float2 *>(c.v_xy), c.v_depth,
                    c.v_conic, c.v_mean3d, c.v_scale, reinterpret_cast<float4 *>(c.v_quat), c.opacities, c.v_opacity,
                    c.v_opacity_logits, c.cam_partials, c.filter3d, c.fk);
    }, m & PJ_ACT, m & PJ_ACC, m & PJ_AA, m & PJ_CAMGRAD, m & PJ_F3D, m & PJ_FISH);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_project_forward(int n, const float *means3d, const float *scales, float glob_scale,
                                   const float *quats, const float *viewmat, const float *projmat,
                                   float fx, float fy, float cx, float cy, int img_h, int img_w,
                                   int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                   float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                   gsb_stream_t stream) {
    return project_forward({0, n, means3d, scales, glob_scale, quats, nullptr, nullptr, viewmat, projmat, fx, fy, cx,
                            cy, img_h, img_w, tiles_x, tiles_y, clip_thresh, cov3d, xys, depths, radii, conics,
                            num_tiles_hit, nullptr}, stream);
}

extern "C" int gsb_project_forward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                             const float *raw_quats, const float *opacity_logits,
                                             const float *viewmat, const float *projmat, float fx, float fy,
                                             float cx, float cy, int img_h, int img_w, int tiles_x, int tiles_y,
                                             float clip_thresh, float *cov3d, float *xys, float *depths,
                                             int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                             float *opacities, gsb_stream_t stream) {
    return project_forward({PJ_ACT, n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, nullptr, viewmat,
                            projmat, fx, fy, cx, cy, img_h, img_w, tiles_x, tiles_y, clip_thresh, cov3d, xys, depths,
                            radii, conics, num_tiles_hit, opacities}, stream);
}

extern "C" int gsb_project_backward(int n, const float *means3d, const float *scales, float glob_scale,
                                    const float *quats, const float *viewmat, const float *projmat,
                                    float fx, float fy, float cx, float cy, int img_h, int img_w,
                                    const float *cov3d, const int32_t *radii, const float *conics,
                                    const float *v_xy, const float *v_depth, const float *v_conic,
                                    float *v_mean3d, float *v_scale, float *v_quat, gsb_stream_t stream) {
    (void)cov3d; (void)cx; (void)cy;
    return project_backward({0, n, means3d, scales, glob_scale, quats, nullptr, nullptr, viewmat, projmat, fx, fy,
                             img_h, img_w, radii, conics, v_xy, v_depth, v_conic, nullptr, v_mean3d, v_scale, v_quat,
                             nullptr, nullptr}, stream);
}

extern "C" int gsb_project_backward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                              const float *raw_quats, const float *opacities, const float *viewmat,
                                              const float *projmat, float fx, float fy, int img_h, int img_w,
                                              const int32_t *radii, const float *conics, const float *v_xy,
                                              const float *v_depth, const float *v_conic, const float *v_opacity,
                                              float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                              float *v_opacity_logits, gsb_stream_t stream) {
    return project_backward({PJ_ACT, n, means3d, log_scales, glob_scale, raw_quats, opacities, nullptr, viewmat,
                             projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity, v_mean3d,
                             v_log_scales, v_raw_quats, v_opacity_logits, nullptr}, stream);
}

// The same VJP added into the four outputs (v += vjp): a trainer's several views of one step summed in place.
extern "C" int gsb_project_backward_activated_acc(int n, const float *means3d, const float *log_scales,
                                                  float glob_scale, const float *raw_quats, const float *opacities,
                                                  const float *viewmat, const float *projmat, float fx, float fy,
                                                  int img_h, int img_w, const int32_t *radii, const float *conics,
                                                  const float *v_xy, const float *v_depth, const float *v_conic,
                                                  const float *v_opacity, float *v_mean3d, float *v_log_scales,
                                                  float *v_raw_quats, float *v_opacity_logits, gsb_stream_t stream) {
    return project_backward({PJ_ACT | PJ_ACC, n, means3d, log_scales, glob_scale, raw_quats, opacities, nullptr,
                             viewmat, projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity,
                             v_mean3d, v_log_scales, v_raw_quats, v_opacity_logits, nullptr}, stream);
}

// D19: the activated projection with the anti-aliased opacity, opacities = sigmoid(logits) * comp.
extern "C" int gsb_project_forward_activated_aa(int n, const float *means3d, const float *log_scales,
                                                float glob_scale, const float *raw_quats, const float *opacity_logits,
                                                const float *viewmat, const float *projmat, float fx, float fy,
                                                float cx, float cy, int img_h, int img_w, int tiles_x, int tiles_y,
                                                float clip_thresh, float *cov3d, float *xys, float *depths,
                                                int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                                float *opacities, gsb_stream_t stream) {
    return project_forward({PJ_ACT | PJ_AA, n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, nullptr,
                            viewmat, projmat, fx, fy, cx, cy, img_h, img_w, tiles_x, tiles_y, clip_thresh, cov3d, xys,
                            depths, radii, conics, num_tiles_hit, opacities}, stream);
}

// Its VJP, from the opacity logits (the forward's opacities hold sigmoid * comp): written, and added in place.
extern "C" int gsb_project_backward_activated_aa(int n, const float *means3d, const float *log_scales,
                                                 float glob_scale, const float *raw_quats,
                                                 const float *opacity_logits, const float *viewmat,
                                                 const float *projmat, float fx, float fy, int img_h, int img_w,
                                                 const int32_t *radii, const float *conics, const float *v_xy,
                                                 const float *v_depth, const float *v_conic, const float *v_opacity,
                                                 float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                                 float *v_opacity_logits, gsb_stream_t stream) {
    return project_backward({PJ_ACT | PJ_AA, n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, nullptr,
                             viewmat, projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity,
                             v_mean3d, v_log_scales, v_raw_quats, v_opacity_logits, nullptr}, stream);
}

extern "C" int gsb_project_backward_activated_aa_acc(int n, const float *means3d, const float *log_scales,
                                                     float glob_scale, const float *raw_quats,
                                                     const float *opacity_logits, const float *viewmat,
                                                     const float *projmat, float fx, float fy, int img_h, int img_w,
                                                     const int32_t *radii, const float *conics, const float *v_xy,
                                                     const float *v_depth, const float *v_conic,
                                                     const float *v_opacity, float *v_mean3d, float *v_log_scales,
                                                     float *v_raw_quats, float *v_opacity_logits,
                                                     gsb_stream_t stream) {
    return project_backward({PJ_ACT | PJ_ACC | PJ_AA, n, means3d, log_scales, glob_scale, raw_quats, opacity_logits,
                             nullptr, viewmat, projmat, fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic,
                             v_opacity, v_mean3d, v_log_scales, v_raw_quats, v_opacity_logits, nullptr}, stream);
}

// D22: the activated projection backward (any of the four variants above: accumulate = the _acc form, antialiased =
// the _aa form, opacities then the logits) that also writes the view's camera gradient as one partial row per block.
extern "C" size_t gsb_project_camera_partials_floats(int n) {
    return n > 0 ? (size_t)CG_TERMS * gsb_div_up(n, PJ_THREADS) : 0;
}

extern "C" int gsb_project_backward_activated_camgrad(int n, const float *means3d, const float *log_scales,
                                                      float glob_scale, const float *raw_quats,
                                                      const float *opacities, const float *viewmat,
                                                      const float *projmat, float fx, float fy, int img_h, int img_w,
                                                      const int32_t *radii, const float *conics, const float *v_xy,
                                                      const float *v_depth, const float *v_conic,
                                                      const float *v_opacity, float *v_mean3d, float *v_log_scales,
                                                      float *v_raw_quats, float *v_opacity_logits, int accumulate,
                                                      int antialiased, float *cam_partials, gsb_stream_t stream) {
    GSB_CHECK_ARG((accumulate == 0 || accumulate == 1) && (antialiased == 0 || antialiased == 1));
    GSB_CHECK_ARG(n >= 0 && (n == 0 || cam_partials));
    return project_backward({PJ_ACT | PJ_CAMGRAD | pj_flag(accumulate, PJ_ACC) | pj_flag(antialiased, PJ_AA), n,
                             means3d, log_scales, glob_scale, raw_quats, opacities, nullptr, viewmat, projmat, fx, fy,
                             img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity, v_mean3d, v_log_scales,
                             v_raw_quats, v_opacity_logits, cam_partials}, stream);
}

extern "C" int gsb_project_camera_grad_reduce(int nblocks, const float *partials, float *v_viewmat, float *v_projmat,
                                              gsb_stream_t stream) {
    GSB_CHECK_ARG(nblocks >= 0 && (nblocks == 0 || partials) && v_viewmat && v_projmat);
    camgrad_reduce_kernel<<<1, CG_TERMS * 32, 0, (cudaStream_t)stream>>>(nblocks, partials, v_viewmat, v_projmat);
    GSB_LAUNCH_CHECK();
    return 0;
}

// D24: the activated projection with Mip-Splatting's 3-D filter (filter3d [n], one float per Gaussian), plain or
// anti-aliased.
extern "C" int gsb_project_forward_activated_filter3d(int n, const float *means3d, const float *log_scales,
                                                      float glob_scale, const float *raw_quats,
                                                      const float *opacity_logits, const float *filter3d,
                                                      const float *viewmat, const float *projmat, float fx, float fy,
                                                      float cx, float cy, int img_h, int img_w, int tiles_x,
                                                      int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                                      float *depths, int32_t *radii, float *conics,
                                                      int32_t *num_tiles_hit, float *opacities, int antialiased,
                                                      gsb_stream_t stream) {
    GSB_CHECK_ARG(antialiased == 0 || antialiased == 1);
    GSB_CHECK_ARG(n >= 0 && (n == 0 || filter3d));
    return project_forward({PJ_ACT | PJ_F3D | pj_flag(antialiased, PJ_AA), n, means3d, log_scales, glob_scale,
                            raw_quats, opacity_logits, filter3d, viewmat, projmat, fx, fy, cx, cy, img_h, img_w,
                            tiles_x, tiles_y, clip_thresh, cov3d, xys, depths, radii, conics, num_tiles_hit,
                            opacities}, stream);
}

// Its VJP with filter3d held constant, from the opacity logits: written or accumulated, plain or anti-aliased, with
// or without the camera gradient (camgrad = 1: cam_partials as gsb_project_backward_activated_camgrad's).
extern "C" int gsb_project_backward_activated_filter3d(int n, const float *means3d, const float *log_scales,
                                                       float glob_scale, const float *raw_quats,
                                                       const float *opacity_logits, const float *filter3d,
                                                       const float *viewmat, const float *projmat, float fx, float fy,
                                                       int img_h, int img_w, const int32_t *radii,
                                                       const float *conics, const float *v_xy, const float *v_depth,
                                                       const float *v_conic, const float *v_opacity, float *v_mean3d,
                                                       float *v_log_scales, float *v_raw_quats,
                                                       float *v_opacity_logits, int accumulate, int antialiased,
                                                       int camgrad, float *cam_partials, gsb_stream_t stream) {
    GSB_CHECK_ARG((accumulate == 0 || accumulate == 1) && (antialiased == 0 || antialiased == 1) &&
                  (camgrad == 0 || camgrad == 1));
    GSB_CHECK_ARG(n >= 0 && (n == 0 || (filter3d && (!camgrad || cam_partials))));
    return project_backward({PJ_ACT | PJ_F3D | pj_flag(accumulate, PJ_ACC) | pj_flag(antialiased, PJ_AA) |
                                 pj_flag(camgrad, PJ_CAMGRAD),
                             n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, filter3d, viewmat, projmat,
                             fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity, v_mean3d,
                             v_log_scales, v_raw_quats, v_opacity_logits, camgrad ? cam_partials : nullptr}, stream);
}

// D27: the activated projection through an OpenCV fisheye camera (k1..k4; theta_lim from model.fisheye_theta_limit),
// plain or anti-aliased.  No projmat: the pixel centre and J come from the fisheye map of t.
static int fisheye_check(float fx, float fy, float k1, float k2, float k3, float k4, float theta_lim) {
    GSB_CHECK_ARG(fx > 0.f && fy > 0.f);
    GSB_CHECK_ARG(isfinite(k1) && isfinite(k2) && isfinite(k3) && isfinite(k4));
    GSB_CHECK_ARG(theta_lim > 0.f && theta_lim <= (float)(0.5 * 3.14159265358979323846));
    return 0;
}

extern "C" int gsb_project_forward_fisheye(int n, const float *means3d, const float *log_scales, float glob_scale,
                                           const float *raw_quats, const float *opacity_logits,
                                           const float *viewmat, float fx, float fy, float cx, float cy, float k1,
                                           float k2, float k3, float k4, float theta_lim, int img_h, int img_w,
                                           int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                           float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                           float *opacities, int antialiased, gsb_stream_t stream) {
    GSB_CHECK_ARG(antialiased == 0 || antialiased == 1);
    if (const int e = fisheye_check(fx, fy, k1, k2, k3, k4, theta_lim)) return e;
    return project_forward({PJ_ACT | PJ_FISH | pj_flag(antialiased, PJ_AA), n, means3d, log_scales, glob_scale,
                            raw_quats, opacity_logits, nullptr, viewmat, nullptr, fx, fy, cx, cy, img_h, img_w,
                            tiles_x, tiles_y, clip_thresh, cov3d, xys, depths, radii, conics, num_tiles_hit, opacities,
                            {k1, k2, k3, k4, theta_lim}}, stream);
}

// Its VJP from the opacity logits: written or accumulated, plain or anti-aliased, and with the camera gradient when
// cam_partials is not NULL (gsb_project_camera_partials_floats(n) floats; the projmat rows are written 0).
extern "C" int gsb_project_backward_fisheye(int n, const float *means3d, const float *log_scales, float glob_scale,
                                            const float *raw_quats, const float *opacity_logits,
                                            const float *viewmat, float fx, float fy, float k1, float k2, float k3,
                                            float k4, float theta_lim, int img_h, int img_w, const int32_t *radii,
                                            const float *conics, const float *v_xy, const float *v_depth,
                                            const float *v_conic, const float *v_opacity, float *v_mean3d,
                                            float *v_log_scales, float *v_raw_quats, float *v_opacity_logits,
                                            int accumulate, int antialiased, float *cam_partials,
                                            gsb_stream_t stream) {
    GSB_CHECK_ARG((accumulate == 0 || accumulate == 1) && (antialiased == 0 || antialiased == 1));
    if (const int e = fisheye_check(fx, fy, k1, k2, k3, k4, theta_lim)) return e;
    return project_backward({PJ_ACT | PJ_FISH | pj_flag(accumulate, PJ_ACC) | pj_flag(antialiased, PJ_AA) |
                                 pj_flag(cam_partials != nullptr, PJ_CAMGRAD),
                             n, means3d, log_scales, glob_scale, raw_quats, opacity_logits, nullptr, viewmat, nullptr,
                             fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity, v_mean3d,
                             v_log_scales, v_raw_quats, v_opacity_logits, cam_partials, {k1, k2, k3, k4, theta_lim}},
                            stream);
}
