// raster_bwd.cu -- back-to-front replay of the blend and per-Gaussian gradient accumulation
// (R2 of SURVEY.md section 8a).
//
// Replaces rasterize_backward_kernel (reference rasterizer/gsplat/backward.cu:161-355, host
// bindings.cu:569-632).  Per-pixel mathematics are the reference's (alpha clamp 0.99 here vs 0.999 in
// the forward pass, T rebuilt by T *= 1/(1-alpha) from final_Ts, `buffer` = colour behind, v_conic
// carries the factor 1/2 on every entry, v_output_alpha term kept).
//
// Gradient accumulation is redesigned -- the reference's known bottleneck is its global float
// atomics (9 atomicAdd per (warp, Gaussian) after a 9 x 5-step shuffle reduction, backward.cu:331-352):
//  * one warp owns a whole 16x16 tile with 8 pixels per lane, so the 256 per-pixel contributions to a
//    Gaussian are first summed over 8 pixels in registers and then across the 32 lanes ONCE per
//    (tile, Gaussian) with a halving butterfly (14 shuffles instead of the reference's 8 warps x 45);
//  * per pixel only 3 moments of w = alpha_unclamped * v_alpha are accumulated (sum w, sum w dy,
//    sum w dy^2) plus the colour gradient; the x-moments follow per lane (dx is a lane constant) and
//    the linear map moments -> (v_xy, v_conic, v_opacity) is applied once per GAUSSIAN afterwards;
//  * the per-(tile, Gaussian) partial goes to a private 48-B row of `grad_rows`, indexed by the
//    intersection's slot k in the Gaussian-major (unsorted) order -- plain stores, no atomics;
//  * a second kernel sums each Gaussian's contiguous rows [cum[g-1], cum[g]) in a fixed order and
//    writes v_xy / v_conic / v_colors / v_opacity once.  Results are bit-reproducible run to run.
// Records are streamed back-to-front with the same per-warp TMA bulk-copy ring, persistent tile
// scheduling and two-level culling as the forward pass.
#include "raster_common.cuh"

int gsb_blend_grid(const void *kernel, int num_tiles);

namespace {

__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ void zero_row(float *grad_rows, int k) {
    float4 *row = reinterpret_cast<float4 *>(grad_rows + (size_t)k * GSB_GRAD_ROW_FLOATS);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    row[0] = z; row[1] = z; row[2] = z;
}

// 80 registers -> 6 CTAs per SM.  H100 SXM at 400 W, C2: 0.849 ms per launch against 0.885 ms with 5 CTAs and
// 0.891 ms with 4
constexpr int BWD_MIN_BLOCKS = 6;
// SAT: v_output is the gradient w.r.t. the CLAMPED image of the forward kernel's SAT instantiation -- channels
// marked as cut in final_idx bits 28..30 receive no gradient (clamp_max's mask, model.cpp:222).
// DEPTH: the VJP of the forward's DEPTH instantiation (D18).  The depth map is one more channel with background 0:
// per pair d += z v_depth (nothing is added to Bq's initial value) and a tenth reduced value a_z = sum alpha T v_depth
// goes to slot 9 of the gradient row.  v_output_depth may be NULL (zeros).
constexpr int BWD_DEPTH_MIN_BLOCKS = 5;
template <bool SAT, bool DEPTH>
__global__ void __launch_bounds__(RK_THREADS, DEPTH ? BWD_DEPTH_MIN_BLOCKS : BWD_MIN_BLOCKS)
rasterize_backward_kernel(int img_h, int img_w, int tiles_x, int num_tiles,
                          const int2 *__restrict__ tile_bins, const GsbRecord *__restrict__ records,
                          const float *__restrict__ background, const float *__restrict__ final_Ts,
                          const int *__restrict__ final_idx, const float *__restrict__ v_output,
                          const float *__restrict__ v_output_alpha, float *__restrict__ grad_rows,
                          unsigned *__restrict__ tile_counter, const int *__restrict__ tile_order,
                          const float *__restrict__ record_depths, const float *__restrict__ v_output_depth) {
    __shared__ WarpRing rings[RK_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    WarpRing &ring = rings[warp];
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < RK_STAGES; ++s) mbar_init(&ring.full[s], 1);
        mbar_fence_init();
    }
    __syncwarp();
    const float bg0 = __ldg(background), bg1 = __ldg(background + 1), bg2 = __ldg(background + 2);
    unsigned gchunk = 0;

    while (true) {
        int tile = 0;
        if (lane == 0) tile = (int)atomicAdd(tile_counter, 1u);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= num_tiles) break;
        if (tile_order) tile = __ldg(tile_order + tile);   // tickets are handed out longest list first
        const int2 range = tile_bins[tile];
        if (range.y <= range.x) continue;

        const int tx = tile % tiles_x, ty = tile / tiles_x;
        const int X = tx * GSB_TILE + (lane & 15);
        const int Y0 = ty * GSB_TILE + (lane >> 4);
        const float px = (float)X;
        const float tile_x0 = (float)(tx * GSB_TILE), tile_y0 = (float)(ty * GSB_TILE);

        // Per pixel only the SCALAR Bq = (colour behind) . v_out - q is tracked instead of the reference's 3-vector
        // `buffer` (backward.cu:200,319-321): v_alpha = sum_c (rgb_c T - buffer_c ra) v_out_c + ra q
        //                                            = T (rgb . v_out) - ra (buffer . v_out - q).
        float T[RK_PIX], Bq[RK_PIX];
        const float py0 = (float)Y0;
        float vor[RK_PIX], vog[RK_PIX], vob[RK_PIX];
        float vD[RK_PIX];   // DEPTH only
        int binf[RK_PIX];
        int my_max = -1;
#pragma unroll
        for (int j = 0; j < RK_PIX; ++j) {
            const int Y = Y0 + 2 * j;
            if (X < img_w && Y < img_h) {
                const size_t p = (size_t)Y * img_w + X;
                const float Tf = final_Ts[p];
                T[j] = Tf;
                vor[j] = v_output[3 * p]; vog[j] = v_output[3 * p + 1]; vob[j] = v_output[3 * p + 2];
                binf[j] = final_idx[p];
                if (SAT) {
                    const int f = binf[j];
                    if (f & GSB_SAT_BIT0) vor[j] = 0.f;
                    if (f & (GSB_SAT_BIT0 << 1)) vog[j] = 0.f;
                    if (f & (GSB_SAT_BIT0 << 2)) vob[j] = 0.f;
                    binf[j] = f & ~GSB_SAT_MASK;
                }
                if (DEPTH) vD[j] = v_output_depth ? v_output_depth[p] : 0.f;
                const float voa = v_output_alpha ? v_output_alpha[p] : 0.f;
                // backward.cu:313-317: T_final*ra*v_out_alpha - T_final*ra*(bg . v_out)  ==  ra * q
                Bq[j] = -(Tf * (voa - (bg0 * vor[j] + bg1 * vog[j] + bg2 * vob[j])));
            } else {
                T[j] = 1.f; vor[j] = vog[j] = vob[j] = 0.f; Bq[j] = 0.f;
                if (DEPTH) vD[j] = 0.f;
                binf[j] = -1;  // never valid
            }
            my_max = max(my_max, binf[j]);
        }
        const int warp_max = __reduce_max_sync(0xffffffffu, my_max);
        // last sorted index any pixel of this tile blended, clamped into the tile's OWN segment: final_idx
        // defaults to 0 for pixels that blended nothing (forward.cu:300), which is below range.x for every tile
        // but the first -- without the clamp the zero-row loop below would walk over other tiles' rows.
        const int hi = min(range.y - 1, max(warp_max, range.x - 1));

        // intersections behind every pixel's last contributor: zero rows
        for (int idx = hi + 1 + lane; idx < range.y; idx += 32)
            zero_row(grad_rows, __float_as_int(__ldg(&records[idx].q0.w)));
        const int L = hi - range.x + 1;
        if (L <= 0) continue;
        const int nchunks = (L + RK_CHUNK - 1) / RK_CHUNK;

        // chunk c (c = 0 is the farthest) covers sorted indices [lo_c, lo_c + cnt_c)
        const unsigned g0 = gchunk;
        auto stage_of = [&](int c) { return (g0 + (unsigned)c) % RK_STAGES; };
        auto parity_of = [&](int c) { return ((g0 + (unsigned)c) / RK_STAGES) & 1u; };
        auto chunk_lo = [&](int c) { return max(range.x, hi + 1 - (c + 1) * RK_CHUNK); };
        auto chunk_cnt = [&](int c) { return (hi + 1 - c * RK_CHUNK) - chunk_lo(c); };
        auto issue = [&](int c) {
            if (lane == 0) {
                const unsigned s = stage_of(c);
                const uint32_t bytes = (uint32_t)chunk_cnt(c) * (uint32_t)sizeof(GsbRecord);
                mbar_arrive_expect_tx(&ring.full[s], bytes);
                tma_load_1d(&ring.rec[s][0], records + chunk_lo(c), bytes, &ring.full[s]);
            }
        };
        const int pro = min(RK_STAGES, nchunks);
        for (int c = 0; c < pro; ++c) issue(c);
        int issued = pro;

        for (int c = 0; c < nchunks; ++c) {
            const unsigned s = stage_of(c);
            // DEPTH: lane l loads the depth of record l of the chunk before the wait (see the forward kernel)
            float zl = 0.f;
            if (DEPTH && lane < chunk_cnt(c)) zl = __ldg(record_depths + chunk_lo(c) + lane);
            mbar_wait(&ring.full[s], parity_of(c));
            const int lo = chunk_lo(c), cnt = chunk_cnt(c);
            // level-1 cull: lane l tests record l; culled records get their zero row right here
            unsigned my_mask = 0;
            if (lane < cnt) {
                my_mask = record_slot_mask(ring.rec[s][lane], tile_x0, tile_y0);
                if (my_mask == 0u) zero_row(grad_rows, __float_as_int(ring.rec[s][lane].q0.w));
            }
            unsigned live = __ballot_sync(0xffffffffu, my_mask != 0u);
            while (live) {
                const int t = 31 - __clz(live);        // back to front
                live &= ~(1u << t);
                const unsigned rm = __shfl_sync(0xffffffffu, my_mask, t);
                float z = 0.f;
                if (DEPTH) z = __shfl_sync(0xffffffffu, zl, t);
                const int idx = lo + t;
                const float4 q0 = ring.rec[s][t].q0;
                const float4 q1 = ring.rec[s][t].q1;
                const float4 q2 = ring.rec[s][t].q2;
                const float smax = fmaxf(0.f, fmaf(q0.z, GSB_LN2, GSB_SMAX_BIAS));
                const float dx = q0.x - px;
                const float adx2 = q1.x * dx * dx;   // (a/2) dx^2
                const float bdx = q1.y * dx;
                const float dy0 = q0.y - py0;
                float s0 = 0.f, s1 = 0.f, s2 = 0.f;  // sum w, sum w dy, sum w dy^2 over this lane's pixels
                float a_r = 0.f, a_g = 0.f, a_b = 0.f;
                float a_z = 0.f;   // DEPTH only
                bool any = false;
                // slots jlo..jhi inside the y-extent (contiguous); a computed jump to jlo that leaves after jhi (an
                // A/B measurement chose it over the forward kernel's straight line of per-slot bit tests)
                const int jlo = __ffs(rm) - 1, jhi = 31 - __clz(rm);
#define GSB_BWD_SLOT(j)                                                                                   \
    {                                                                                                     \
        const float dy = dy0 - (float)(2 * j);  /* centre.y - pixel row */                                                                    \
        const float sigma = fmaf(dy, fmaf(q1.z, dy, bdx), adx2);                                          \
        if (__float_as_uint(sigma) <= __float_as_uint(smax)) { /* 0 <= sigma <= smax */                   \
            const float au = ex2_approx(fmaf(sigma, -GSB_LOG2E, q0.z)); /* opac * exp(-sigma) */          \
            const float alpha = fminf(0.99f, au);                                                         \
            if (idx <= binf[j] && alpha >= (1.f / 255.f)) {                                               \
                any = true;                                                                               \
                const float ra = rcp_approx(1.f - alpha);                                                 \
                T[j] *= ra;                                                                               \
                const float fac = alpha * T[j];                                                           \
                a_r = fmaf(fac, vor[j], a_r);                                                             \
                a_g = fmaf(fac, vog[j], a_g);                                                             \
                a_b = fmaf(fac, vob[j], a_b);                                                             \
                if (DEPTH) a_z = fmaf(fac, vD[j], a_z);                                                   \
                float d = fmaf(q2.z, vob[j], fmaf(q2.y, vog[j], q2.x * vor[j])); /* rgb . v_out */        \
                if (DEPTH) d = fmaf(z, vD[j], d);                         /* + z v_depth */               \
                const float v_alpha = fmaf(d, T[j], -(ra * Bq[j]));                                       \
                Bq[j] = fmaf(d, fac, Bq[j]);                                                              \
                /* v_sigma = -opac*vis*v_alpha = -w (backward.cu:323); v_opacity += vis*v_alpha = w/opac */ \
                const float w = au * v_alpha;                                                             \
                const float wdy = w * dy;                                                                 \
                s0 += w;                                                                                  \
                s1 += wdy;                                                                                \
                s2 = fmaf(wdy, dy, s2);                                                                   \
            }                                                                                             \
        }                                                                                                 \
        if (jhi == j) break;                                                                              \
    }
                switch (jlo) {
                    case 0: GSB_BWD_SLOT(0)
                    case 1: GSB_BWD_SLOT(1)
                    case 2: GSB_BWD_SLOT(2)
                    case 3: GSB_BWD_SLOT(3)
                    case 4: GSB_BWD_SLOT(4)
                    case 5: GSB_BWD_SLOT(5)
                    case 6: GSB_BWD_SLOT(6)
                    default: GSB_BWD_SLOT(7)
                }
#undef GSB_BWD_SLOT
                const int k = __float_as_int(q0.w);
                float *row = grad_rows + (size_t)k * GSB_GRAD_ROW_FLOATS;
                if (!__any_sync(0xffffffffu, any)) {
                    if (lane < (DEPTH ? 10 : 9)) row[lane] = 0.f;
                    continue;
                }
                // ---- one cross-lane reduction per (tile, Gaussian): 8 values by halving, 1 by butterfly
                const float sx = dx * s0;
                float v0 = s0, v1 = sx, v2 = s1, v3 = dx * sx, v4 = dx * s1, v5 = s2, v6 = a_r, v7 = a_g;
                float v8 = a_b;
                {
                    const bool up = lane & 16;
                    const float t0 = up ? v0 : v4, t1 = up ? v1 : v5, t2 = up ? v2 : v6, t3 = up ? v3 : v7;
                    const float k0 = up ? v4 : v0, k1 = up ? v5 : v1, k2 = up ? v6 : v2, k3 = up ? v7 : v3;
                    v0 = k0 + __shfl_xor_sync(0xffffffffu, t0, 16);
                    v1 = k1 + __shfl_xor_sync(0xffffffffu, t1, 16);
                    v2 = k2 + __shfl_xor_sync(0xffffffffu, t2, 16);
                    v3 = k3 + __shfl_xor_sync(0xffffffffu, t3, 16);
                }
                {
                    const bool up = lane & 8;
                    const float t0 = up ? v0 : v2, t1 = up ? v1 : v3;
                    const float k0 = up ? v2 : v0, k1 = up ? v3 : v1;
                    v0 = k0 + __shfl_xor_sync(0xffffffffu, t0, 8);
                    v1 = k1 + __shfl_xor_sync(0xffffffffu, t1, 8);
                }
                {
                    const bool up = lane & 4;
                    const float t0 = up ? v0 : v1;
                    const float k0 = up ? v1 : v0;
                    v0 = k0 + __shfl_xor_sync(0xffffffffu, t0, 4);
                }
                v0 += __shfl_xor_sync(0xffffffffu, v0, 2);
                v0 += __shfl_xor_sync(0xffffffffu, v0, 1);
                if (DEPTH) {
                    // values 8 and 9 by one halving step, then a butterfly within each half: lanes 0..15 end with the
                    // total of value 8 (the same sums in the same order as the butterfly below), lanes 16..31 with 9
                    const bool up = lane & 16;
                    const float t8 = up ? v8 : a_z, k8 = up ? a_z : v8;
                    v8 = k8 + __shfl_xor_sync(0xffffffffu, t8, 16);
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) v8 += __shfl_xor_sync(0xffffffffu, v8, o);
                    // lane l holds the total of value (l >> 2); lane 1 additionally stores value 8, lane 17 value 9
                    const bool w8 = (lane == 1), w9 = (lane == 17);
                    if (((lane & 3) == 0) || w8 || w9) row[w8 ? 8 : w9 ? 9 : (lane >> 2)] = (w8 || w9) ? v8 : v0;
                } else {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v8 += __shfl_xor_sync(0xffffffffu, v8, o);
                    // lane l now holds the total of value (l >> 2); lane 1 additionally stores value 8
                    const bool w8 = (lane == 1);
                    if (((lane & 3) == 0) || w8) row[w8 ? 8 : (lane >> 2)] = w8 ? v8 : v0;
                }
            }
            __syncwarp();
            if (issued < nchunks) { issue(issued); ++issued; }
        }
        gchunk = g0 + (unsigned)issued;
        __syncwarp();
    }
}

// Sum each Gaussian's rows (contiguous in the unsorted order), apply the moment -> gradient map
// (backward.cu:323-329 restated on sums) and write the four gradient tensors:
//   v_sigma = -w:  v_conic = -1/2 (Sxx, Sxy, Syy),  v_xy = -(a Sx + b Sy, b Sx + c Sy),  v_opacity = S0/opac
// DEPTH also sums slot 9 into v_depths.
template <bool DEPTH>
__global__ void __launch_bounds__(256)
reduce_grad_rows_kernel(int n, const int *__restrict__ cum_tiles_hit, const float *__restrict__ grad_rows,
                        const float *__restrict__ conics, const float *__restrict__ opacities,
                        float2 *__restrict__ v_xy, float *__restrict__ v_conic,
                        float *__restrict__ v_colors, float *__restrict__ v_opacity, float *__restrict__ v_depths) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const int k0 = g ? cum_tiles_hit[g - 1] : 0, k1 = cum_tiles_hit[g];
    float a[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float az = 0.f;   // DEPTH only
    for (int k = k0; k < k1; ++k) {
        const float4 *row = reinterpret_cast<const float4 *>(grad_rows + (size_t)k * GSB_GRAD_ROW_FLOATS);
        const float4 r0 = row[0], r1 = row[1];
        const float r8 = reinterpret_cast<const float *>(row)[8];
        a[0] += r0.x; a[1] += r0.y; a[2] += r0.z; a[3] += r0.w;
        a[4] += r1.x; a[5] += r1.y; a[6] += r1.z; a[7] += r1.w;
        a[8] += r8;
        if (DEPTH) az += reinterpret_cast<const float *>(row)[9];
    }
    const float S0 = a[0], Sx = a[1], Sy = a[2], Sxx = a[3], Sxy = a[4], Syy = a[5];
    const float ca = conics[3 * g], cb = conics[3 * g + 1], cc = conics[3 * g + 2];
    const float op = opacities[g];
    v_xy[g] = make_float2(-(ca * Sx + cb * Sy), -(cb * Sx + cc * Sy));
    v_conic[3 * g] = -0.5f * Sxx; v_conic[3 * g + 1] = -0.5f * Sxy; v_conic[3 * g + 2] = -0.5f * Syy;
    v_colors[3 * g] = a[6]; v_colors[3 * g + 1] = a[7]; v_colors[3 * g + 2] = a[8];
    v_opacity[g] = (op > 0.f) ? S0 / op : 0.f;
    if (DEPTH) v_depths[g] = az;
}

}  // namespace

extern "C" size_t gsb_raster_grad_rows_bytes(int m) {
    return gsb_align_up((size_t)(m > 0 ? m : 0) * GSB_GRAD_ROW_FLOATS * 4 + 256, 256);
}

// Body of gsb_rasterize_backward (depth = false) and of gsb_rasterize_backward_depth.
static int backward(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m, const int32_t *tile_bins,
                    const int32_t *tile_order, const float *conics, const float *opacities, void *records,
                    const int32_t *cum_tiles_hit, const float *background, const float *final_Ts,
                    const int32_t *final_idx, const float *v_output, const float *v_output_alpha, void *grad_rows,
                    float *v_xy, float *v_conic, float *v_colors, float *v_opacity, unsigned flags, bool depth,
                    const float *record_depths, const float *v_output_depth, float *v_depths, gsb_stream_t stream) {
    GSB_CHECK_ARG(img_h > 0 && img_w > 0 && n >= 0 && m >= 0);
    GSB_CHECK_ARG((flags & ~(unsigned)GSB_RASTER_CLAMP_MAX_ONE) == 0);
    const bool sat = (flags & GSB_RASTER_CLAMP_MAX_ONE) != 0;
    GSB_CHECK_ARG(tiles_x == gsb_div_up(img_w, GSB_TILE) && tiles_y == gsb_div_up(img_h, GSB_TILE));
    if (n == 0) return 0;
    GSB_CHECK_ARG(tile_bins && conics && opacities && cum_tiles_hit && background && final_Ts && final_idx &&
                  v_output && v_xy && v_conic && v_colors && v_opacity);
    GSB_CHECK_ARG(!depth || (v_depths && (record_depths || m == 0)));
    GSB_CHECK_ARG(((uintptr_t)v_xy % 8) == 0);
    cudaStream_t s = (cudaStream_t)stream;
    if (m > 0) {
        GSB_CHECK_ARG(records && grad_rows && ((uintptr_t)records % 16) == 0 && ((uintptr_t)grad_rows % 16) == 0);
        unsigned *counters = reinterpret_cast<unsigned *>(
            reinterpret_cast<char *>(records) + gsb_raster_records_bytes(m) - 256);
        GSB_CUDA(cudaMemsetAsync(counters, 0, 256, s));
        const int num_tiles = tiles_x * tiles_y;
#define GSB_BWD_LAUNCH(S, D)                                                                                    \
    rasterize_backward_kernel<S, D><<<gsb_blend_grid((const void *)rasterize_backward_kernel<S, D>, num_tiles),  \
                                      RK_THREADS, 0, s>>>(                                                      \
        img_h, img_w, tiles_x, num_tiles, reinterpret_cast<const int2 *>(tile_bins),                            \
        reinterpret_cast<const GsbRecord *>(records), background, final_Ts, final_idx, v_output, v_output_alpha, \
        reinterpret_cast<float *>(grad_rows), counters, tile_order, record_depths, v_output_depth)
        if (depth) {
            if (sat) GSB_BWD_LAUNCH(true, true); else GSB_BWD_LAUNCH(false, true);
        } else {
            if (sat) GSB_BWD_LAUNCH(true, false); else GSB_BWD_LAUNCH(false, false);
        }
#undef GSB_BWD_LAUNCH
    }
#define GSB_REDUCE_LAUNCH(D)                                                                                    \
    reduce_grad_rows_kernel<D><<<gsb_div_up(n, 256), 256, 0, s>>>(                                              \
        n, cum_tiles_hit, reinterpret_cast<const float *>(grad_rows), conics, opacities,                        \
        reinterpret_cast<float2 *>(v_xy), v_conic, v_colors, v_opacity, v_depths)
    if (depth) GSB_REDUCE_LAUNCH(true); else GSB_REDUCE_LAUNCH(false);
#undef GSB_REDUCE_LAUNCH
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_rasterize_backward(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m,
                                      const int32_t *tile_bins, const int32_t *tile_order, const float *conics,
                                      const float *opacities, void *records, const int32_t *cum_tiles_hit,
                                      const float *background, const float *final_Ts, const int32_t *final_idx,
                                      const float *v_output, const float *v_output_alpha, void *grad_rows,
                                      float *v_xy, float *v_conic, float *v_colors, float *v_opacity, unsigned flags,
                                      gsb_stream_t stream) {
    return backward(img_h, img_w, tiles_x, tiles_y, n, m, tile_bins, tile_order, conics, opacities, records,
                    cum_tiles_hit, background, final_Ts, final_idx, v_output, v_output_alpha, grad_rows, v_xy, v_conic,
                    v_colors, v_opacity, flags, false, nullptr, nullptr, nullptr, stream);
}

extern "C" int gsb_rasterize_backward_depth(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m,
                                            const int32_t *tile_bins, const int32_t *tile_order, const float *conics,
                                            const float *opacities, void *records, const int32_t *cum_tiles_hit,
                                            const float *background, const float *final_Ts, const int32_t *final_idx,
                                            const float *v_output, const float *v_output_alpha, void *grad_rows,
                                            float *v_xy, float *v_conic, float *v_colors, float *v_opacity,
                                            unsigned flags, const float *record_depths, const float *v_output_depth,
                                            float *v_depths, gsb_stream_t stream) {
    return backward(img_h, img_w, tiles_x, tiles_y, n, m, tile_bins, tile_order, conics, opacities, records,
                    cum_tiles_hit, background, final_Ts, final_idx, v_output, v_output_alpha, grad_rows, v_xy, v_conic,
                    v_colors, v_opacity, flags, true, record_depths, v_output_depth, v_depths, stream);
}
