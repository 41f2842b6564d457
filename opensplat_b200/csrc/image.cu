// image.cu -- the training images of Camera::loadImage / Camera::getImage (input_data.cpp:40-117) on the device:
// OpenCV 4's CPU INTER_AREA resize and undistort of 3-channel u8 images, byte for byte, and the u8 -> float32 u/255
// conversion of imageToTensor for a batch of images in one launch.
//
// Built with --fmad=false, and every float / double operation that must round as OpenCV's CPU code does is spelled
// out with the __*_rn intrinsics (OpenCV's baseline x86 code has no FMA on these paths).
//
//   gsb_resize_area_u8 (hal::resize, INTER_AREA, scale >= 1):
//     - the integer-scale fast path (resizeAreaFast_Invoker) when both 1/inv_scale are within DBL_EPSILON of an
//       integer: full cells give (s+2)>>2 at scale 2x2 and rint(float(s) * (1.f/area)) otherwise; cells cut by the
//       right or bottom border (the 1/f path of loadImage, e.g. 51 -> 26 at f = 2) give rint(float(s) / count);
//     - otherwise the general path (computeResizeAreaTab + ResizeArea_Invoker): per-cell weights from double cell
//       edges, a float horizontal accumulation per source row, sum += beta * buf per source row, saturating rint.
//     Each output pixel walks its own cell in OpenCV's order, so the sums round exactly as OpenCV's row buffers do.
//   gsb_undistort_u8 (cv::undistort with newK, fused with the ROI crop): the map of initUndistortRectifyMap in fp64,
//     stripe by stripe as cv::undistort computes it (stripes of min(max(1, 4096/cols), rows) rows, the new principal
//     point's y shifted by the stripe's first row, cv::invert's closed-form 3x3 inverse), quantised to 1/32 pixel
//     (CV_16SC2), then remap's fixed-point bilinear (15-bit weights, BORDER_CONSTANT 0) for the ROI pixels only.
//   gsb_u8_to_f32_views: B stored images -> one float32 [B,H,W,3] at float(u) / 255.0f (IEEE division).
//   gsb_resize_area_mask_u8 / gsb_undistort_mask_u8 (DESIGN D26): a u8 [h,w] loss mask through the same geometry; an
//     output pixel is used (1) iff every source pixel with a nonzero weight in its colour is used, else 0.
#include <float.h>
#include <math.h>

#include <algorithm>

#include "gsb_common.cuh"

namespace {

constexpr int IMG_THREADS = 256;

__device__ __forceinline__ unsigned char sat_rint_u8(float v) {   // saturate_cast<uchar>(float): cvRound, clamp
    const int r = __float2int_rn(v);
    return (unsigned char)min(max(r, 0), 255);
}

// One entry range of computeResizeAreaTab for destination index d: the partial first cell, whole cells [s1, s2),
// the partial last cell.  Weights are formed exactly as OpenCV forms them (double, then rounded to float).
struct AreaCell {
    int s1, s2;
    bool head, tail;
    float a_head, a_mid, a_tail;
};

__device__ __forceinline__ AreaCell area_cell(int d, int ssize, double scale) {
    AreaCell c;
    const double fs1 = __dmul_rn((double)d, scale);
    const double fs2 = __dadd_rn(fs1, scale);
    const double cell = fmin(scale, __dsub_rn((double)ssize, fs1));
    int s1 = (int)ceil(fs1), s2 = (int)floor(fs2);
    s2 = min(s2, ssize - 1);
    s1 = min(s1, s2);
    const double h = __dsub_rn((double)s1, fs1), t = __dsub_rn(fs2, (double)s2);
    c.s1 = s1;
    c.s2 = s2;
    c.head = h > 1e-3;
    c.tail = t > 1e-3;
    c.a_head = __double2float_rn(__ddiv_rn(h, cell));
    c.a_mid = __double2float_rn(__ddiv_rn(1.0, cell));
    c.a_tail = __double2float_rn(__ddiv_rn(fmin(fmin(t, 1.0), cell), cell));
    return c;
}

// buf += S[sx] * alpha for the three channels of one source pixel
__device__ __forceinline__ void acc_px(float *buf, const unsigned char *p, float alpha) {
#pragma unroll
    for (int k = 0; k < 3; ++k) buf[k] = __fadd_rn(buf[k], __fmul_rn((float)p[k], alpha));
}

__device__ __forceinline__ void row_buf(const unsigned char *row, const AreaCell &cx, float *buf) {
    buf[0] = buf[1] = buf[2] = 0.f;
    if (cx.head) acc_px(buf, row + 3 * (cx.s1 - 1), cx.a_head);
    for (int sx = cx.s1; sx < cx.s2; ++sx) acc_px(buf, row + 3 * sx, cx.a_mid);
    if (cx.tail) acc_px(buf, row + 3 * cx.s2, cx.a_tail);
}

__global__ void __launch_bounds__(IMG_THREADS)
resize_area_general_kernel(int sh, int sw, const unsigned char *__restrict__ src, int dh, int dw,
                           unsigned char *__restrict__ dst, double scale_x, double scale_y) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dh * dw) return;
    const int dy = i / dw, dx = i - dy * dw;
    const AreaCell cx = area_cell(dx, sw, scale_x), cy = area_cell(dy, sh, scale_y);
    float sum[3] = {0.f, 0.f, 0.f}, buf[3];
    const size_t stride = (size_t)sw * 3;
    auto add_row = [&](int sy, float beta) {
        row_buf(src + (size_t)sy * stride, cx, buf);
#pragma unroll
        for (int k = 0; k < 3; ++k) sum[k] = __fadd_rn(sum[k], __fmul_rn(beta, buf[k]));
    };
    if (cy.head) add_row(cy.s1 - 1, cy.a_head);
    for (int sy = cy.s1; sy < cy.s2; ++sy) add_row(sy, cy.a_mid);
    if (cy.tail) add_row(cy.s2, cy.a_tail);
    unsigned char *o = dst + 3 * (size_t)i;
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = sat_rint_u8(sum[k]);
}

__global__ void __launch_bounds__(IMG_THREADS)
resize_area_fast_kernel(int sh, int sw, const unsigned char *__restrict__ src, int dh, int dw,
                        unsigned char *__restrict__ dst, int isx, int isy) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dh * dw) return;
    const int dy = i / dw, dx = i - dy * dw;
    const int y0 = dy * isy, x0 = dx * isx;
    unsigned char *o = dst + 3 * (size_t)i;
    if (y0 >= sh || x0 >= sw) {   // a cell wholly outside the source (OpenCV writes 0)
        o[0] = o[1] = o[2] = 0;
        return;
    }
    const int y1 = min(y0 + isy, sh), x1 = min(x0 + isx, sw);
    int s[3] = {0, 0, 0};
    for (int y = y0; y < y1; ++y) {
        const unsigned char *row = src + ((size_t)y * sw + x0) * 3;
        for (int x = 0; x < x1 - x0; ++x) {
            s[0] += row[3 * x];
            s[1] += row[3 * x + 1];
            s[2] += row[3 * x + 2];
        }
    }
    const bool full = y0 + isy <= sh && dx < sw / isx;
    if (full && isx == 2 && isy == 2) {
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = (unsigned char)((s[k] + 2) >> 2);
    } else if (full) {
        const float scale = __fdiv_rn(1.f, (float)(isx * isy));
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = sat_rint_u8(__fmul_rn((float)s[k], scale));
    } else {
        const float count = (float)((y1 - y0) * (x1 - x0));
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = sat_rint_u8(__fdiv_rn((float)s[k], count));
    }
}

struct UndistortParams {
    double fx, fy, u0, v0;          // K
    double k1, k2, p1, p2, k3;
    double a, b, c, e;              // newK: fx, fy, cx, cy
};

// saturate_cast<int>(double): round half to even, saturate
__device__ __forceinline__ int sat_round_int(double v) {
    return (int)fmin(fmax(rint(v), -2147483648.0), 2147483647.0);
}

// the CV_16SC2 map entry (iu, iv), in 1/32 pixel, of output pixel (row r, column j) of cv::undistort
__device__ __forceinline__ void undistort_map(const UndistortParams &P, int stripe, int r, int j, int &iu, int &iv) {
    const int ys = (r / stripe) * stripe, i = r - ys;
    // iR = inv(Ar) of the stripe, Ar = [[a,0,c],[0,b,e - ys],[0,0,1]]: cv::invert's closed form, d = 1/det
    const double e = __dsub_rn(P.e, (double)ys);
    const double ab = __dmul_rn(P.a, P.b);
    const double dinv = __ddiv_rn(1.0, ab);
    const double ir0 = __dmul_rn(P.b, dinv), ir2 = __dmul_rn(-__dmul_rn(P.c, P.b), dinv);
    const double ir4 = __dmul_rn(P.a, dinv), ir5 = __dmul_rn(-__dmul_rn(P.a, e), dinv);
    const double ir8 = __dmul_rn(ab, dinv);
    const double iw = __ddiv_rn(1.0, ir8);
    const double x = __dmul_rn(__dadd_rn(__dmul_rn((double)j, ir0), ir2), iw);
    const double y = __dmul_rn(__dadd_rn(__dmul_rn((double)i, ir4), ir5), iw);
    const double x2 = __dmul_rn(x, x), y2 = __dmul_rn(y, y);
    const double r2 = __dadd_rn(x2, y2);
    const double xy2 = __dmul_rn(__dmul_rn(2.0, x), y);
    const double kr = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(P.k3, r2), P.k2), r2), P.k1),
                                               r2));
    const double xd = __dadd_rn(__dadd_rn(__dmul_rn(x, kr), __dmul_rn(P.p1, xy2)),
                                __dmul_rn(P.p2, __dadd_rn(r2, __dmul_rn(2.0, x2))));
    const double yd = __dadd_rn(__dadd_rn(__dmul_rn(y, kr), __dmul_rn(P.p1, __dadd_rn(r2, __dmul_rn(2.0, y2)))),
                                __dmul_rn(P.p2, xy2));
    const double u = __dadd_rn(__dmul_rn(P.fx, xd), P.u0);
    const double v = __dadd_rn(__dmul_rn(P.fy, yd), P.v0);
    iu = sat_round_int(__dmul_rn(u, 32.0));
    iv = sat_round_int(__dmul_rn(v, 32.0));
}

__global__ void __launch_bounds__(IMG_THREADS)
undistort_kernel(int h, int w, const unsigned char *__restrict__ src, UndistortParams P, int stripe, int roi_x,
                 int roi_y, int roi_w, int roi_h, unsigned char *__restrict__ dst) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= roi_w * roi_h) return;
    const int oy = t / roi_w, ox = t - oy * roi_w;
    const int r = roi_y + oy, j = roi_x + ox;
    int iu, iv;
    undistort_map(P, stripe, r, j, iu, iv);
    const int sx = (short)(iu >> 5), sy = (short)(iv >> 5);      // CV_16SC2
    const int ax = iu & 31, ay = iv & 31;
    unsigned char *o = dst + 3 * (size_t)t;
    if (sx >= w || sx + 1 < 0 || sy >= h || sy + 1 < 0) {
        o[0] = o[1] = o[2] = 0;
        return;
    }
    // initInterTab2D's bilinear weights: products of (32 - a) / 32 and a / 32 in units of 2^-15 (exact)
    const int w00 = (32 - ay) * (32 - ax) * 32, w01 = (32 - ay) * ax * 32, w10 = ay * (32 - ax) * 32,
              w11 = ay * ax * 32;
    const bool x0in = sx >= 0, x1in = sx + 1 < w, y0in = sy >= 0, y1in = sy + 1 < h;
    const unsigned char *p00 = src + ((size_t)sy * w + sx) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int v00 = (y0in && x0in) ? p00[k] : 0;
        const int v01 = (y0in && x1in) ? p00[3 + k] : 0;
        const int v10 = (y1in && x0in) ? p00[(size_t)w * 3 + k] : 0;
        const int v11 = (y1in && x1in) ? p00[(size_t)w * 3 + 3 + k] : 0;
        const int acc = v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11;
        o[k] = (unsigned char)min(max((acc + (1 << 14)) >> 15, 0), 255);
    }
}

// blockIdx.y = view; a grid-stride loop over the view's 4-byte words (n_bytes = H*W*3, the tail done byte by byte)
__global__ void __launch_bounds__(IMG_THREADS)
u8_to_f32_kernel(const long long *__restrict__ views, size_t n_bytes, float *__restrict__ out) {
    const unsigned char *src = (const unsigned char *)views[blockIdx.y];
    float *dst = out + (size_t)blockIdx.y * n_bytes;
    const bool vec = ((uintptr_t)src % 4 == 0) && ((uintptr_t)dst % 16 == 0);
    const size_t n4 = vec ? n_bytes / 4 : 0;
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (size_t)gridDim.x * blockDim.x) {
        const uchar4 u = reinterpret_cast<const uchar4 *>(src)[q];
        reinterpret_cast<float4 *>(dst)[q] = make_float4(__fdiv_rn((float)u.x, 255.f), __fdiv_rn((float)u.y, 255.f),
                                                         __fdiv_rn((float)u.z, 255.f), __fdiv_rn((float)u.w, 255.f));
    }
    for (size_t q = 4 * n4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < n_bytes;
         q += (size_t)gridDim.x * blockDim.x)
        dst[q] = __fdiv_rn((float)src[q], 255.f);
}

// ---- loss masks (DESIGN D26): 1 byte per pixel, nonzero = used; the outputs are 0 / 1 -------------------------------
// An output pixel is used iff every source pixel INTER_AREA sums into it is used: the entries of area_cell on both
// axes (the partial first cell, the whole cells, the partial last cell, with OpenCV's 1e-3 cut-offs).
__global__ void __launch_bounds__(IMG_THREADS)
resize_area_mask_general_kernel(int sh, int sw, const unsigned char *__restrict__ src, int dh, int dw,
                                unsigned char *__restrict__ dst, double scale_x, double scale_y) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dh * dw) return;
    const int dy = i / dw, dx = i - dy * dw;
    const AreaCell cx = area_cell(dx, sw, scale_x), cy = area_cell(dy, sh, scale_y);
    const int x0 = cx.head ? cx.s1 - 1 : cx.s1, x1 = cx.tail ? cx.s2 + 1 : cx.s2;
    const int y0 = cy.head ? cy.s1 - 1 : cy.s1, y1 = cy.tail ? cy.s2 + 1 : cy.s2;
    bool used = true;
    for (int y = y0; y < y1 && used; ++y)
        for (int x = x0; x < x1; ++x) used = used && src[(size_t)y * sw + x] != 0;
    dst[i] = used ? 1 : 0;
}

// the integer-scale fast path: the cell clipped to the image; a cell wholly outside it (OpenCV writes colour 0) is
// ignored.  isx = isy = 1 is the copy of equal sizes.
__global__ void __launch_bounds__(IMG_THREADS)
resize_area_mask_fast_kernel(int sh, int sw, const unsigned char *__restrict__ src, int dh, int dw,
                             unsigned char *__restrict__ dst, int isx, int isy) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dh * dw) return;
    const int dy = i / dw, dx = i - dy * dw;
    const int y0 = dy * isy, x0 = dx * isx;
    bool used = y0 < sh && x0 < sw;
    const int y1 = min(y0 + isy, sh), x1 = min(x0 + isx, sw);
    for (int y = y0; y < y1 && used; ++y)
        for (int x = x0; x < x1; ++x) used = used && src[(size_t)y * sw + x] != 0;
    dst[i] = used ? 1 : 0;
}

// An output pixel of the ROI is used iff every bilinear tap with a nonzero fixed-point weight lies inside the image
// and is used: (sx, sy) always, the right taps iff ax > 0, the bottom taps iff ay > 0.  A pixel whose taps all fall
// outside (colour 0, BORDER_CONSTANT) is ignored.
__global__ void __launch_bounds__(IMG_THREADS)
undistort_mask_kernel(int h, int w, const unsigned char *__restrict__ src, UndistortParams P, int stripe, int roi_x,
                      int roi_y, int roi_w, int roi_h, unsigned char *__restrict__ dst) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= roi_w * roi_h) return;
    const int oy = t / roi_w, ox = t - oy * roi_w;
    int iu, iv;
    undistort_map(P, stripe, roi_y + oy, roi_x + ox, iu, iv);
    const int sx = (short)(iu >> 5), sy = (short)(iv >> 5);
    const int xe = (iu & 31) ? sx + 1 : sx, ye = (iv & 31) ? sy + 1 : sy;   // last tap column / row
    bool used = sx >= 0 && sy >= 0 && xe < w && ye < h;
    for (int y = sy; y <= ye && used; ++y)
        for (int x = sx; x <= xe; ++x) used = used && src[(size_t)y * w + x] != 0;
    dst[t] = used ? 1 : 0;
}

}  // namespace

extern "C" int gsb_resize_area_u8(int src_h, int src_w, const uint8_t *src, int dst_h, int dst_w, uint8_t *dst,
                                  float inv_scale, gsb_stream_t stream) {
    GSB_CHECK_ARG(src_h > 0 && src_w > 0 && dst_h > 0 && dst_w > 0);
    GSB_CHECK_ARG(dst_h <= src_h && dst_w <= src_w);
    GSB_CHECK_ARG((long long)src_h * src_w <= 0x7fffffffLL / 3);
    GSB_CHECK_ARG(src && dst && (const void *)src != (const void *)dst);
    GSB_CHECK_ARG(inv_scale == 0.f || (inv_scale > 0.f && inv_scale <= 1.f));
    double ix, iy;
    if (inv_scale == 0.f) {    // dsize given: cv::resize derives the scales from the sizes
        ix = (double)dst_w / src_w;
        iy = (double)dst_h / src_h;
    } else {                   // dsize empty: dsize = cvRound(ssize * inv_scale)
        ix = iy = (double)inv_scale;
        GSB_CHECK_ARG(dst_w == (int)nearbyint(src_w * ix) && dst_h == (int)nearbyint(src_h * iy));
    }
    cudaStream_t s = (cudaStream_t)stream;
    const size_t bytes = (size_t)dst_h * dst_w * 3;
    if (dst_h == src_h && dst_w == src_w) {   // cv::resize copies
        GSB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
        return 0;
    }
    const double sx = 1.0 / ix, sy = 1.0 / iy;
    const int isx = (int)nearbyint(sx), isy = (int)nearbyint(sy);
    const int blocks = gsb_div_up(dst_h * dst_w, IMG_THREADS);
    if (fabs(sx - isx) < DBL_EPSILON && fabs(sy - isy) < DBL_EPSILON)
        resize_area_fast_kernel<<<blocks, IMG_THREADS, 0, s>>>(src_h, src_w, src, dst_h, dst_w, dst, isx, isy);
    else
        resize_area_general_kernel<<<blocks, IMG_THREADS, 0, s>>>(src_h, src_w, src, dst_h, dst_w, dst, sx, sy);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_undistort_u8(int h, int w, const uint8_t *src, float fx, float fy, float cx, float cy, float k1,
                                float k2, float p1, float p2, float k3, float new_fx, float new_fy, float new_cx,
                                float new_cy, int roi_x, int roi_y, int roi_w, int roi_h, uint8_t *dst,
                                gsb_stream_t stream) {
    GSB_CHECK_ARG(h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL / 3);
    GSB_CHECK_ARG(roi_x >= 0 && roi_y >= 0 && roi_w >= 0 && roi_h >= 0 && roi_x + roi_w <= w && roi_y + roi_h <= h);
    GSB_CHECK_ARG(isfinite(fx) && isfinite(fy) && isfinite(cx) && isfinite(cy) && fx != 0.f && fy != 0.f);
    GSB_CHECK_ARG(isfinite(new_fx) && isfinite(new_fy) && isfinite(new_cx) && isfinite(new_cy) && new_fx != 0.f &&
                  new_fy != 0.f);
    GSB_CHECK_ARG(isfinite(k1) && isfinite(k2) && isfinite(p1) && isfinite(p2) && isfinite(k3));
    if (roi_w == 0 || roi_h == 0) return 0;
    GSB_CHECK_ARG(src && dst && (const void *)src != (const void *)dst);
    const UndistortParams P{fx, fy, cx, cy, k1, k2, p1, p2, k3, new_fx, new_fy, new_cx, new_cy};
    const int stripe = std::min(std::max(1, 4096 / w), h);
    undistort_kernel<<<gsb_div_up(roi_w * roi_h, IMG_THREADS), IMG_THREADS, 0, (cudaStream_t)stream>>>(
        h, w, src, P, stripe, roi_x, roi_y, roi_w, roi_h, dst);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_u8_to_f32_views(int num_views, const int64_t *views, int h, int w, float *out,
                                   gsb_stream_t stream) {
    GSB_CHECK_ARG(num_views >= 0 && num_views <= 65535 && h > 0 && w > 0);
    if (num_views == 0) return 0;
    GSB_CHECK_ARG(views && out);
    const size_t n = (size_t)h * w * 3;
    const int blocks = (int)std::min<size_t>((n / 4 + IMG_THREADS - 1) / IMG_THREADS + 1, 1024);
    u8_to_f32_kernel<<<dim3(blocks, num_views), IMG_THREADS, 0, (cudaStream_t)stream>>>(
        (const long long *)views, n, out);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_resize_area_mask_u8(int src_h, int src_w, const uint8_t *src, int dst_h, int dst_w, uint8_t *dst,
                                       float inv_scale, gsb_stream_t stream) {
    GSB_CHECK_ARG(src_h > 0 && src_w > 0 && dst_h > 0 && dst_w > 0);
    GSB_CHECK_ARG(dst_h <= src_h && dst_w <= src_w);
    GSB_CHECK_ARG((long long)src_h * src_w <= 0x7fffffffLL / 3);
    GSB_CHECK_ARG(src && dst && (const void *)src != (const void *)dst);
    GSB_CHECK_ARG(inv_scale == 0.f || (inv_scale > 0.f && inv_scale <= 1.f));
    double ix, iy;
    if (inv_scale == 0.f) {
        ix = (double)dst_w / src_w;
        iy = (double)dst_h / src_h;
    } else {
        ix = iy = (double)inv_scale;
        GSB_CHECK_ARG(dst_w == (int)nearbyint(src_w * ix) && dst_h == (int)nearbyint(src_h * iy));
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int blocks = gsb_div_up(dst_h * dst_w, IMG_THREADS);
    const double sx = 1.0 / ix, sy = 1.0 / iy;
    const int isx = (int)nearbyint(sx), isy = (int)nearbyint(sy);
    if (dst_h == src_h && dst_w == src_w)   // the colour is copied: the mask is normalised to 0 / 1
        resize_area_mask_fast_kernel<<<blocks, IMG_THREADS, 0, s>>>(src_h, src_w, src, dst_h, dst_w, dst, 1, 1);
    else if (fabs(sx - isx) < DBL_EPSILON && fabs(sy - isy) < DBL_EPSILON)
        resize_area_mask_fast_kernel<<<blocks, IMG_THREADS, 0, s>>>(src_h, src_w, src, dst_h, dst_w, dst, isx, isy);
    else
        resize_area_mask_general_kernel<<<blocks, IMG_THREADS, 0, s>>>(src_h, src_w, src, dst_h, dst_w, dst, sx, sy);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_undistort_mask_u8(int h, int w, const uint8_t *src, float fx, float fy, float cx, float cy,
                                     float k1, float k2, float p1, float p2, float k3, float new_fx, float new_fy,
                                     float new_cx, float new_cy, int roi_x, int roi_y, int roi_w, int roi_h,
                                     uint8_t *dst, gsb_stream_t stream) {
    GSB_CHECK_ARG(h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL / 3);
    GSB_CHECK_ARG(roi_x >= 0 && roi_y >= 0 && roi_w >= 0 && roi_h >= 0 && roi_x + roi_w <= w && roi_y + roi_h <= h);
    GSB_CHECK_ARG(isfinite(fx) && isfinite(fy) && isfinite(cx) && isfinite(cy) && fx != 0.f && fy != 0.f);
    GSB_CHECK_ARG(isfinite(new_fx) && isfinite(new_fy) && isfinite(new_cx) && isfinite(new_cy) && new_fx != 0.f &&
                  new_fy != 0.f);
    GSB_CHECK_ARG(isfinite(k1) && isfinite(k2) && isfinite(p1) && isfinite(p2) && isfinite(k3));
    if (roi_w == 0 || roi_h == 0) return 0;
    GSB_CHECK_ARG(src && dst && (const void *)src != (const void *)dst);
    const UndistortParams P{fx, fy, cx, cy, k1, k2, p1, p2, k3, new_fx, new_fy, new_cx, new_cy};
    const int stripe = std::min(std::max(1, 4096 / w), h);
    undistort_mask_kernel<<<gsb_div_up(roi_w * roi_h, IMG_THREADS), IMG_THREADS, 0, (cudaStream_t)stream>>>(
        h, w, src, P, stripe, roi_x, roi_y, roi_w, roi_h, dst);
    GSB_LAUNCH_CHECK();
    return 0;
}
