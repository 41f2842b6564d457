// bilagrid.cu -- learned per-image bilateral grids (Wang et al. 2024, "Bilateral Guided Radiance Field Processing";
// gsplat's bilateral-grid module), DESIGN D21: the slice that maps a rendered image to one photo's exposure and white
// balance, its backward, and the total-variation regulariser of the grids.
//
// A grid is X x Y x L cells of 12 coefficients, stored channels-last [L][Y][X][12] (a cell is three 16-byte loads);
// the 12 coefficients of a cell are the row-major 3x4 affine matrix [A | b].  At pixel (px, py) of an H x W image:
//     gx = ((px + 0.5) / W) (X - 1),  gy = ((py + 0.5) / H) (Y - 1),   z = (0.299 r + 0.587 g) + 0.114 b,
//     gz = clamp(z, 0, 1) (L - 1),   coef = trilinear(grid, gx, gy, gz),   out = A rgb + b   (not clamped)
// Every one of those fp32 operations is rounded on its own (__f*_rn: no contraction), so gx, gy, z, gz and the cell
// (x0, y0, z0) = (min(floor(g), size - 2)) are the bits a host restatement computes in numpy float32.  A corner's
// weight is (wz wy) wx, each w the fraction or one minus it; coef_k = sum over the 8 corners in (dz, dy, dx) order
// of fma(w, G, acc); out_c = fma(a_c0, r, fma(a_c1, g, fma(a_c2, b, a_c3))).
//
// Backward: v_rgb = A^T v_out + 7 (dout/dgz . v_out) (0.299, 0.587, 0.114), the luma term only where 0 < z < 1
// (z <= 0 or z >= 1 is the flat border of the clamp, ties included), with dcoef/dgz the forward difference of the
// cells z0 and z0 + 1 (at an interior integer gz = k that is cells k and k + 1).  v_grid gets the trilinear weights
// times v_out (x) (rgb, 1).  The grid reduction uses no atomics, so it is bit-deterministic: the pixels of each
// spatial cell (x0, y0) -- a pixel rectangle, since x0 and y0 are monotone in px and py -- are cut into chunks of
// CHUNK pixels; one block per (cell, chunk) sums every pixel's contribution to the cell's 2 x 2 x 8 corners x 12
// coefficients in a fixed order (pixels bucketed by z0 with a stable sort) into a workspace slot; a second kernel adds, for every grid float, its (up to 4
// cells) x (chunks) slots in (cell y, cell x, chunk) order and adds scale times that sum into v_grid.
#include <algorithm>

#include "gsb_common.cuh"

namespace {

constexpr int GX = GSB_BILAGRID_X, GY = GSB_BILAGRID_Y, GL = GSB_BILAGRID_L, NC = GSB_BILAGRID_COEFFS;
constexpr int GRID_FLOATS = GSB_BILAGRID_FLOATS;
constexpr int CELLS_X = GX - 1, CELLS_Y = GY - 1, CELLS = CELLS_X * CELLS_Y;   // spatial cells (x0, y0)
constexpr int CELL_OUT = GL * 4 * NC;       // floats a spatial cell's pixels reach: 8 levels x 2 x 2 corners x 12
constexpr int BT = CELL_OUT;                // threads of the cell kernel: one per reached float
constexpr int CHUNK = 4 * BT;               // pixels per (cell, chunk) block, staged BT at a time
constexpr int MAX_SIDE = 1 << 15;
static_assert(NC == 12 && GL >= 2 && GX >= 2 && GY >= 2, "the slice assumes 3x4 affine cells and >= 2 cells per axis");

__device__ __forceinline__ float luma(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(0.299f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// g = ((p + 0.5) / n) (cells - 1); i0 = min(floor(g), cells - 2); f = g - i0 (exact)
__device__ __forceinline__ void axis_coord(int p, int n, int cells, int &i0, float &f) {
    const float g = __fmul_rn(__fdiv_rn(__fadd_rn((float)p, 0.5f), (float)n), (float)(cells - 1));
    i0 = min((int)g, cells - 2);
    f = __fsub_rn(g, (float)i0);
}

__device__ __forceinline__ float z_coord(float z, int &z0) {
    const float gz = __fmul_rn(fminf(fmaxf(z, 0.f), 1.f), (float)(GL - 1));
    z0 = min((int)gz, GL - 2);
    return __fsub_rn(gz, (float)z0);
}

__device__ __forceinline__ const float4 *cell_ptr(const float *grid, int l, int y, int x) {
    return reinterpret_cast<const float4 *>(grid + ((l * GY + y) * GX + x) * NC);
}

// The pixel's cell and fractions, the interpolated coefficients and (with dz) their derivative in gz.
struct Slice {
    float fx, fy, fz, z;
    int x0, y0, z0;
};

template <bool DZ>
__device__ __forceinline__ void interpolate(const float *__restrict__ grid, const Slice &s, float coef[NC],
                                            float dcoef[NC]) {
#pragma unroll
    for (int k = 0; k < NC; ++k) { coef[k] = 0.f; if (DZ) dcoef[k] = 0.f; }
    const float wx[2] = {__fsub_rn(1.f, s.fx), s.fx}, wy[2] = {__fsub_rn(1.f, s.fy), s.fy},
                wz[2] = {__fsub_rn(1.f, s.fz), s.fz};
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const float w = __fmul_rn(__fmul_rn(wz[dz], wy[dy]), wx[dx]);
                const float4 *c = cell_ptr(grid, s.z0 + dz, s.y0 + dy, s.x0 + dx);
                const float4 a = __ldg(c), b = __ldg(c + 1), d = __ldg(c + 2);
                const float g[NC] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, d.x, d.y, d.z, d.w};
#pragma unroll
                for (int k = 0; k < NC; ++k) coef[k] = __fmaf_rn(w, g[k], coef[k]);
            }
    if (DZ) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const float w = __fmul_rn(wy[dy], wx[dx]);
                const float4 *c0 = cell_ptr(grid, s.z0, s.y0 + dy, s.x0 + dx);
                const float4 *c1 = cell_ptr(grid, s.z0 + 1, s.y0 + dy, s.x0 + dx);
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float4 a = __ldg(c0 + q), b = __ldg(c1 + q);
                    dcoef[4 * q + 0] = __fmaf_rn(w, __fsub_rn(b.x, a.x), dcoef[4 * q + 0]);
                    dcoef[4 * q + 1] = __fmaf_rn(w, __fsub_rn(b.y, a.y), dcoef[4 * q + 1]);
                    dcoef[4 * q + 2] = __fmaf_rn(w, __fsub_rn(b.z, a.z), dcoef[4 * q + 2]);
                    dcoef[4 * q + 3] = __fmaf_rn(w, __fsub_rn(b.w, a.w), dcoef[4 * q + 3]);
                }
            }
    }
}

__device__ __forceinline__ Slice locate(int px, int py, int H, int W, float r, float g, float b) {
    Slice s;
    axis_coord(px, W, GX, s.x0, s.fx);
    axis_coord(py, H, GY, s.y0, s.fy);
    s.z = luma(r, g, b);
    s.fz = z_coord(s.z, s.z0);
    return s;
}

__device__ __forceinline__ float affine(const float *m, float r, float g, float b) {
    return __fmaf_rn(m[0], r, __fmaf_rn(m[1], g, __fmaf_rn(m[2], b, m[3])));
}

__global__ void __launch_bounds__(256)
bilagrid_slice_forward_kernel(int H, int W, const float *__restrict__ grid, const float *__restrict__ rgb,
                              float *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const float r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
    const Slice s = locate(i % W, i / W, H, W, r, g, b);
    float coef[NC], unused[NC];
    interpolate<false>(grid, s, coef, unused);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[3 * i + c] = affine(coef + 4 * c, r, g, b);
}

// v_rgb_j = sum_c a_cj v_c (c in order 0, 1, 2, as fmas) + lw_j dz,  dz = 7 sum_c v_c (dA_c rgb + db_c) where 0 < z < 1
__global__ void __launch_bounds__(256)
bilagrid_slice_vrgb_kernel(int H, int W, const float *__restrict__ grid, const float *__restrict__ rgb,
                           const float *__restrict__ v_out, float *__restrict__ v_rgb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const float r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
    const float v[3] = {v_out[3 * i], v_out[3 * i + 1], v_out[3 * i + 2]};
    const Slice s = locate(i % W, i / W, H, W, r, g, b);
    float coef[NC], dcoef[NC];
    interpolate<true>(grid, s, coef, dcoef);
    float dz = 0.f;
    if (s.z > 0.f && s.z < 1.f) {
#pragma unroll
        for (int c = 0; c < 3; ++c) dz = __fmaf_rn(v[c], affine(dcoef + 4 * c, r, g, b), dz);
        dz = __fmul_rn(dz, (float)(GL - 1));
    }
    const float lw[3] = {0.299f, 0.587f, 0.114f};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float a = __fmul_rn(lw[j], dz);
#pragma unroll
        for (int c = 0; c < 3; ++c) a = __fmaf_rn(coef[4 * c + j], v[c], a);
        v_rgb[3 * i + j] = a;
    }
}

// The pixels with cell index c along an axis: [begin(c), begin(c + 1)), begin(c) = the first p with i0(p) >= c
// (i0 is monotone in p).  Found from an estimate by stepping, with the kernel's own axis_coord.
__device__ int axis_begin(int c, int n, int cells) {
    if (c <= 0) return 0;
    if (c >= cells - 1) return n;
    int p = max(0, min(n, (int)((float)c * (float)n / (float)(cells - 1))));
    int i0;
    float f;
    while (p > 0) { axis_coord(p - 1, n, cells, i0, f); if (i0 < c) break; --p; }
    while (p < n) { axis_coord(p, n, cells, i0, f); if (i0 >= c) break; ++p; }
    return p;
}

// One block per (spatial cell, chunk): thread t owns corner float t = (level l, corner s = 2 sy + sx, coefficient k)
// of the cell and sums (wz wy) wx (v_c x_j) over the chunk's pixels whose z0 is l - 1 or l.  The pixels are staged BT
// at a time, bucketed by z0 with a stable counting sort (warp match + popc ranks, one thread's prefix over the warps),
// so a thread walks only its two buckets: per stage, the z0 = l - 1 pixels then the z0 = l pixels, each in pixel
// order.  partial[(cell * chunks + chunk) * CELL_OUT + t] = that sum.
constexpr int BUCKETS = GL;            // z0 in [0, L - 2], plus one bucket for slots past the chunk's end
constexpr int WARPS = BT / 32;
__global__ void __launch_bounds__(BT)
bilagrid_cell_partials_kernel(int H, int W, int chunks, const float *__restrict__ rgb, const float *__restrict__ v_out,
                              float *__restrict__ partial) {
    const int cell = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
    const int cx = cell % CELLS_X, cy = cell / CELLS_X;
    __shared__ int rect[4];
    __shared__ float st_f[3][BT], st_v[3][BT], st_x[3][BT];
    __shared__ int st_z0[BT];
    __shared__ int warp_cnt[WARPS][BUCKETS], warp_off[WARPS][BUCKETS], bucket_start[BUCKETS + 1];
    if (threadIdx.x < 4) {
        const int t = threadIdx.x;
        rect[t] = t < 2 ? axis_begin(cx + t, W, GX) : axis_begin(cy + t - 2, H, GY);
    }
    __syncthreads();
    const int px0 = rect[0], nxp = rect[1] - rect[0], py0 = rect[2], nyp = rect[3] - rect[2];
    const int count = nxp * nyp, first = chunk * CHUNK, last = min(count, first + CHUNK);
    const int t = threadIdx.x, l = t / (4 * NC), sc = (t / NC) % 4, k = t % NC;
    const int sy = sc >> 1, sx = sc & 1, c = k / 4, j = k % 4;
    const int lane = t & 31, warp = t >> 5;
    float acc = 0.f;
    for (int base = first; base < last; base += BT) {
        const int q = base + t;
        int bucket = BUCKETS - 1;
        float f[3] = {0.f, 0.f, 0.f}, x[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f};
        if (q < last) {
            const int px = px0 + q % nxp, py = py0 + q / nxp, i = py * W + px;
            x[0] = rgb[3 * i]; x[1] = rgb[3 * i + 1]; x[2] = rgb[3 * i + 2];
            const Slice s = locate(px, py, H, W, x[0], x[1], x[2]);
            bucket = s.z0;
            f[0] = s.fx; f[1] = s.fy; f[2] = s.fz;
            v[0] = v_out[3 * i]; v[1] = v_out[3 * i + 1]; v[2] = v_out[3 * i + 2];
        }
        if (t < WARPS * BUCKETS) warp_cnt[t / BUCKETS][t % BUCKETS] = 0;
        __syncthreads();
        const unsigned peers = __match_any_sync(0xffffffffu, bucket);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (rank == 0) warp_cnt[warp][bucket] = __popc(peers);
        __syncthreads();
        if (t == 0) {
            int run = 0;
            for (int b = 0; b < BUCKETS; ++b) {
                bucket_start[b] = run;
                for (int w = 0; w < WARPS; ++w) { warp_off[w][b] = run; run += warp_cnt[w][b]; }
            }
            bucket_start[BUCKETS] = run;
        }
        __syncthreads();
        const int pos = warp_off[warp][bucket] + rank;
#pragma unroll
        for (int a = 0; a < 3; ++a) { st_f[a][pos] = f[a]; st_x[a][pos] = x[a]; st_v[a][pos] = v[a]; }
        st_z0[pos] = bucket;
        __syncthreads();
        const int p0 = bucket_start[max(l - 1, 0)], p1 = bucket_start[min(l + 1, BUCKETS - 1)];
        for (int p = p0; p < p1; ++p) {
            const float fx = st_f[0][p], fy = st_f[1][p], fz = st_f[2][p];
            const float wz = st_z0[p] == l ? __fsub_rn(1.f, fz) : fz;
            const float wy = sy ? fy : __fsub_rn(1.f, fy), wx = sx ? fx : __fsub_rn(1.f, fx);
            const float w = __fmul_rn(__fmul_rn(wz, wy), wx);
            const float vx = j < 3 ? __fmul_rn(st_v[c][p], st_x[j][p]) : st_v[c][p];
            acc = __fadd_rn(acc, __fmul_rn(w, vx));
        }
        __syncthreads();
    }
    partial[(size_t)blockIdx.x * CELL_OUT + t] = acc;
}

// v_grid[e] += scale * (sum of e's slots in (cell y, cell x, chunk) order), e = ((l Y + y) X + x) 12 + k
__global__ void __launch_bounds__(256)
bilagrid_reduce_kernel(int chunks, const float *__restrict__ partial, float scale, float *__restrict__ v_grid) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= GRID_FLOATS) return;
    const int k = e % NC, x = (e / NC) % GX, y = (e / (NC * GX)) % GY, l = e / (NC * GX * GY);
    float sum = 0.f;
    for (int cy = max(y - 1, 0); cy <= min(y, CELLS_Y - 1); ++cy)
        for (int cx = max(x - 1, 0); cx <= min(x, CELLS_X - 1); ++cx) {
            const int slot = (l * 4 + 2 * (y - cy) + (x - cx)) * NC + k;
            const float *p = partial + (size_t)(cy * CELLS_X + cx) * chunks * CELL_OUT + slot;
            for (int ch = 0; ch < chunks; ++ch) sum = __fadd_rn(sum, p[(size_t)ch * CELL_OUT]);
        }
    v_grid[e] = __fadd_rn(v_grid[e], __fmul_rn(scale, sum));
}

// The TV gradient of one float: weight * sum over the axes x, y, l of inv_a ((G - G_prev) - (G_next - G)), each
// existing neighbour's term added in that order (inv_a = 2 / (elements of axis a's difference tensor)).
__global__ void __launch_bounds__(256)
bilagrid_tv_grad_kernel(long long total, const float *__restrict__ g, float weight, float inv_x, float inv_y,
                        float inv_l, float *__restrict__ v) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int r = (int)(e % GRID_FLOATS);
    const int x = (r / NC) % GX, y = (r / (NC * GX)) % GY, l = r / (NC * GX * GY);
    const float G = g[e];
    float acc = 0.f;
    const int strides[3] = {NC, NC * GX, NC * GX * GY}, pos[3] = {x, y, l}, size[3] = {GX, GY, GL};
    const float inv[3] = {inv_x, inv_y, inv_l};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (pos[a] > 0) acc = __fmaf_rn(inv[a], __fsub_rn(G, g[e - strides[a]]), acc);
        if (pos[a] < size[a] - 1) acc = __fmaf_rn(-inv[a], __fsub_rn(g[e + strides[a]], G), acc);
    }
    v[e] = __fmul_rn(weight, acc);
}

// The TV value: per axis the fp32 differences squared and summed in fp64 (each thread in index order, then a fixed
// tree over the block), over the axis's element count, the three added in fp64 and rounded once.  One block.
constexpr int TV_T = 1024;
__global__ void __launch_bounds__(TV_T)
bilagrid_tv_value_kernel(long long total, const float *__restrict__ g, double cnt_x, double cnt_y, double cnt_l,
                         float *__restrict__ out) {
    __shared__ double red[3][TV_T];
    double s[3] = {0.0, 0.0, 0.0};
    const int strides[3] = {NC, NC * GX, NC * GX * GY}, size[3] = {GX, GY, GL};
    for (long long e = threadIdx.x; e < total; e += TV_T) {
        const int r = (int)(e % GRID_FLOATS);
        const int pos[3] = {(r / NC) % GX, (r / (NC * GX)) % GY, r / (NC * GX * GY)};
        const float G = g[e];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (pos[a] < size[a] - 1) {
                const double d = (double)__fsub_rn(g[e + strides[a]], G);
                s[a] += d * d;
            }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) red[a][threadIdx.x] = s[a];
    __syncthreads();
    for (int h = TV_T / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h)
#pragma unroll
            for (int a = 0; a < 3; ++a) red[a][threadIdx.x] += red[a][threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = (float)(red[0][0] / cnt_x + red[1][0] / cnt_y + red[2][0] / cnt_l);
}

// chunks per spatial cell: the most pixels a cell can hold, over CHUNK (a cell spans at most n / (cells - 1) + 2
// pixels of an axis: the fp32 coordinate can move its edges by one pixel)
int chunks_for(int H, int W) {
    const long long nx = std::min(W, W / CELLS_X + 2), ny = std::min(H, H / CELLS_Y + 2);
    return (int)((nx * ny + CHUNK - 1) / CHUNK);
}

bool aligned16(const void *p) { return ((uintptr_t)p % 16) == 0; }

}  // namespace

extern "C" int gsb_bilagrid_slice_forward(int H, int W, const float *grid, const float *rgb, float *out,
                                          gsb_stream_t stream) {
    GSB_CHECK_ARG(H >= 1 && W >= 1 && H <= MAX_SIDE && W <= MAX_SIDE);
    GSB_CHECK_ARG(grid && rgb && out && aligned16(grid));
    const int n = H * W;
    bilagrid_slice_forward_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(H, W, grid, rgb, out);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t gsb_bilagrid_workspace_bytes(int H, int W) {
    if (H < 1 || W < 1 || H > MAX_SIDE || W > MAX_SIDE) return 0;
    return (size_t)CELLS * chunks_for(H, W) * CELL_OUT * sizeof(float);
}

extern "C" int gsb_bilagrid_slice_backward(int H, int W, const float *grid, const float *rgb, const float *v_out,
                                           float scale, float *v_rgb, float *v_grid, void *workspace,
                                           size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(H >= 1 && W >= 1 && H <= MAX_SIDE && W <= MAX_SIDE);
    GSB_CHECK_ARG(grid && rgb && v_out && v_rgb && v_grid && workspace && aligned16(grid));
    GSB_CHECK_ARG(workspace_bytes >= gsb_bilagrid_workspace_bytes(H, W) && ((uintptr_t)workspace % 256) == 0);
    cudaStream_t st = (cudaStream_t)stream;
    const int n = H * W, chunks = chunks_for(H, W);
    float *partial = static_cast<float *>(workspace);
    bilagrid_slice_vrgb_kernel<<<gsb_div_up(n, 256), 256, 0, st>>>(H, W, grid, rgb, v_out, v_rgb);
    GSB_LAUNCH_CHECK();
    bilagrid_cell_partials_kernel<<<CELLS * chunks, BT, 0, st>>>(H, W, chunks, rgb, v_out, partial);
    GSB_LAUNCH_CHECK();
    bilagrid_reduce_kernel<<<gsb_div_up(GRID_FLOATS, 256), 256, 0, st>>>(chunks, partial, scale, v_grid);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_bilagrid_tv(int num_grids, const float *grids, float weight, float *v_grids, float *tv_out,
                               gsb_stream_t stream) {
    GSB_CHECK_ARG(num_grids >= 1 && num_grids <= (1 << 16));
    GSB_CHECK_ARG(grids && v_grids);
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)num_grids * GRID_FLOATS;
    const double cnt_x = (double)num_grids * NC * GL * GY * (GX - 1), cnt_y = (double)num_grids * NC * GL * (GY - 1) * GX,
                 cnt_l = (double)num_grids * NC * (GL - 1) * GY * GX;
    bilagrid_tv_grad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        total, grids, weight, (float)(2.0 / cnt_x), (float)(2.0 / cnt_y), (float)(2.0 / cnt_l), v_grids);
    GSB_LAUNCH_CHECK();
    if (tv_out) {
        bilagrid_tv_value_kernel<<<1, TV_T, 0, st>>>(total, grids, cnt_x, cnt_y, cnt_l, tv_out);
        GSB_LAUNCH_CHECK();
    }
    return 0;
}
