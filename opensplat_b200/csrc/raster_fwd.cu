// raster_fwd.cu -- record packing + front-to-back alpha compositing (R1 of SURVEY.md section 8a).
//
// Replaces rasterize_forward (reference rasterizer/gsplat/forward.cu:256-378, host bindings.cu:338-410).
// Per-pixel semantics are the reference's: integer pixel coordinates, sigma = .5(a dx^2 + c dy^2) + b dx dy,
// alpha = min(0.999, opac * exp(-sigma)), skip if sigma < 0 or alpha < 1/255, stop BEFORE blending
// once T(1-alpha) <= 1e-4, out = colour + T * background, final_idx = sorted index of the last
// blended Gaussian (0 if none).
//
// Hopper design (differs from the reference's 256-thread CTA with __syncthreads batching and
// per-pixel global colour gathers):
//  * a pack kernel turns the sorted id list into a contiguous 48-B record stream (raster_common.cuh),
//    so a tile's list is one contiguous byte range;
//  * persistent warps pull tile ids from a global counter (no wave quantisation, no tail of idle SMs);
//    one warp owns one tile and streams its range into a private 4-stage shared-memory ring with 1-D
//    TMA bulk copies (cp.async.bulk, SASS UBLKCP) completing on mbarriers -- no __syncthreads and no
//    per-thread gather instructions in the blend loop;
//  * each lane carries 8 pixels in registers; every surviving record is read once per warp with three
//    broadcast 128-bit shared loads;
//  * two levels of conservative culling before any per-pixel work: each lane tests ONE record of the
//    32-record chunk against the tile (extent boxes stored in the record) and the warp then walks only
//    the surviving records, visiting only the pixel-row pairs inside the record's y-extent; per pixel,
//    sigma <= smax is tested before the exp.
#include "raster_common.cuh"

namespace {

__global__ void __launch_bounds__(256)
pack_records_kernel(int m, const int *__restrict__ gaussian_ids_sorted,
                    const int *__restrict__ sorted_index, const float2 *__restrict__ xys,
                    const float *__restrict__ conics, const float *__restrict__ colors,
                    const float *__restrict__ opacities, GsbRecord *__restrict__ records) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int g = gaussian_ids_sorted[i];
    const int k = sorted_index ? sorted_index[i] : i;
    const GsbRecord r = make_record(__ldg(xys + g), __ldg(conics + 3 * g), __ldg(conics + 3 * g + 1),
                                    __ldg(conics + 3 * g + 2), __ldg(opacities + g), __ldg(colors + 3 * g),
                                    __ldg(colors + 3 * g + 1), __ldg(colors + 3 * g + 2), k);
    float4 *dst = reinterpret_cast<float4 *>(records + i);
    stg_stream4(dst, r.q0);
    stg_stream4(dst + 1, r.q1);
    stg_stream4(dst + 2, r.q2);
}

// record_depths[j] = depths[gaussian_ids_sorted[j]] for j < M: the per-record depth stream of the DEPTH blend
// kernels.  On the fast path the id list is sized by the capacity, not M: entries past M hold no valid id, so M is
// read from the binning stats on the device, and after an overflow (stats[2]) nothing is written.
__global__ void __launch_bounds__(256)
gather_record_depths_kernel(int m, const int *__restrict__ gaussian_ids_sorted, const float *__restrict__ depths,
                            const int *__restrict__ bin_stats, float *__restrict__ record_depths) {
    int mv = m;
    if (bin_stats) {
        if (bin_stats[2]) return;
        mv = min(m, bin_stats[0]);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= mv) return;
    record_depths[i] = __ldg(depths + gaussian_ids_sorted[i]);
}

// 64 registers -> 8 CTAs (32 warps) per SM.  H100 SXM at 400 W, C2: 0.416 ms per launch against 0.445 ms with 7 CTAs
// and 0.464 ms with 6 (which needs no spill): occupancy wins
constexpr int FWD_MIN_BLOCKS = 8;
// COUNT = true is a diagnostic instantiation (gsb_rasterize_forward_count): same arithmetic, plus per-launch
// totals of {records that pass the per-record test, slot visits, pixel pairs whose sigma is inside the
// extent (ex2 evaluated), pixel pairs blended} in pair_counts[0..3].  The production instantiation carries none
// of it.
// SAT = true fuses the caller's `clamp_max(rgb, 1)` (model.cpp:222) into the epilogue: the image is written clamped
// and, per pixel, which channels were cut (!(value <= 1), torch's clamp_max mask) goes into bits 28..30 of final_idx
// for the SAT instantiation of the backward kernel (sorted indices stay below 2^28, checked by the entry point).
// DEPTH = true also writes out_depth = sum alpha T z over the blended pairs (z = record_depths, the per-record depth
// stream in sorted order; background depth 0) and out_alpha = 1 - T_final (D18).  The colour arithmetic is the same
// and in the same order, so out_img / final_Ts / final_idx are those of the DEPTH = false kernel.
// 8 more accumulators per lane do not fit 64 registers without spilling: DEPTH takes its own minimum of CTAs per SM.
constexpr int FWD_DEPTH_MIN_BLOCKS = 6;
template <bool COUNT, bool SAT, bool DEPTH>
__global__ void __launch_bounds__(RK_THREADS, DEPTH ? FWD_DEPTH_MIN_BLOCKS : FWD_MIN_BLOCKS)
rasterize_forward_kernel(int img_h, int img_w, int tiles_x, int num_tiles,
                         const int2 *__restrict__ tile_bins, const GsbRecord *__restrict__ records,
                         const float *__restrict__ background, float *__restrict__ out_img,
                         float *__restrict__ final_Ts, int *__restrict__ final_idx,
                         unsigned *__restrict__ tile_counter, const int *__restrict__ bin_stats,
                         unsigned long long *__restrict__ pair_counts, const int *__restrict__ tile_order,
                         const float *__restrict__ record_depths, float *__restrict__ out_depth,
                         float *__restrict__ out_alpha) {
    // bin_stats (optional): stats of gsb_bucket_tile_ranges; [2] != 0 means the binning overflowed its
    // capacities and wrote nothing -- the host redoes the frame, this launch must not touch the records
    if (bin_stats && bin_stats[2]) return;
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
    unsigned gchunk = 0;  // chunks this warp has pushed through its ring so far (stage / parity bookkeeping)
    unsigned long long n_rec = 0, n_slot = 0, n_eval = 0, n_blend = 0;   // COUNT only

    while (true) {
        int tile = 0;
        if (lane == 0) tile = (int)atomicAdd(tile_counter, 1u);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= num_tiles) break;
        if (tile_order) tile = __ldg(tile_order + tile);   // tickets are handed out longest list first

        const int tx = tile % tiles_x, ty = tile / tiles_x;
        const int X = tx * GSB_TILE + (lane & 15);
        const int Y0 = ty * GSB_TILE + (lane >> 4);
        const float px = (float)X;
        const float tile_x0 = (float)(tx * GSB_TILE), tile_y0 = (float)(ty * GSB_TILE);
        const int2 range = tile_bins[tile];
        const int L = range.y - range.x;
        const int nchunks = (L + RK_CHUNK - 1) / RK_CHUNK;

        // T[j] > 0: transmittance of a live pixel.  A finished pixel keeps its final transmittance
        // NEGATED (sign bit == "done"): T*(1-alpha) <= 1e-4 then always routes it to the (rare)
        // terminate branch, which ignores pixels that are already negative.
        float T[RK_PIX], cr[RK_PIX], cg[RK_PIX], cb[RK_PIX];
        float cd[RK_PIX];   // DEPTH only
        const float py0 = (float)Y0;
        int last[RK_PIX];
        unsigned done = 0;  // bit j: pixel j finished (or outside the image)
#pragma unroll
        for (int j = 0; j < RK_PIX; ++j) {
            T[j] = 1.f; cr[j] = cg[j] = cb[j] = 0.f; last[j] = 0;
            if (DEPTH) cd[j] = 0.f;
            if (X >= img_w || Y0 + 2 * j >= img_h) { done |= 1u << j; T[j] = -1.f; }
        }

        const unsigned g0 = gchunk;  // ring position at tile start
        auto stage_of = [&](int c) { return (g0 + (unsigned)c) % RK_STAGES; };
        auto parity_of = [&](int c) { return ((g0 + (unsigned)c) / RK_STAGES) & 1u; };
        auto issue = [&](int c) {
            if (lane == 0) {
                const int cnt = min(RK_CHUNK, L - c * RK_CHUNK);
                const uint32_t bytes = (uint32_t)cnt * (uint32_t)sizeof(GsbRecord);
                const unsigned s = stage_of(c);
                mbar_arrive_expect_tx(&ring.full[s], bytes);
                tma_load_1d(&ring.rec[s][0], records + range.x + c * RK_CHUNK, bytes, &ring.full[s]);
            }
        };
        const int pro = min(RK_STAGES, nchunks);
        for (int c = 0; c < pro; ++c) issue(c);
        int issued = pro;

        int c = 0;
        for (; c < nchunks; ++c) {
            const unsigned s = stage_of(c);
            // DEPTH: lane l loads the depth of record l of the chunk (one coalesced 128-B load), issued before the
            // wait so that its latency hides behind it; the blend loop shuffles it to the record it blends
            float zl = 0.f;
            if (DEPTH) {
                const int i = range.x + c * RK_CHUNK + lane;
                if (i < range.y) zl = __ldg(record_depths + i);
            }
            mbar_wait(&ring.full[s], parity_of(c));
            const int cnt = min(RK_CHUNK, L - c * RK_CHUNK);
            const int idx0 = range.x + c * RK_CHUNK;
            // level-1 cull: lane l tests record l of the chunk against the tile
            unsigned my_mask = 0;
            if (lane < cnt) my_mask = record_slot_mask(ring.rec[s][lane], tile_x0, tile_y0);
            unsigned live = __ballot_sync(0xffffffffu, my_mask != 0u);
            if (COUNT && lane == 0) n_rec += __popc(live);
            while (live) {
                const int t = __ffs(live) - 1;
                live &= live - 1;
                const unsigned rm = __shfl_sync(0xffffffffu, my_mask, t);  // slots inside the y-extent
                float z = 0.f;
                if (DEPTH) z = __shfl_sync(0xffffffffu, zl, t);
                const float4 q0 = ring.rec[s][t].q0;
                const float4 q1 = ring.rec[s][t].q1;
                const float4 q2 = ring.rec[s][t].q2;
                const float smax = fmaxf(0.f, fmaf(q0.z, GSB_LN2, GSB_SMAX_BIAS));
                const float dx = q0.x - px;
                const float adx2 = q1.x * dx * dx;   // (a/2) dx^2
                const float bdx = q1.y * dx;
                const float dy0 = q0.y - py0;
                const int idx = idx0 + t;   // sorted index of this record (final_idx of the pixels it is the last to blend)
                // visit only the slots inside the record's y-extent (contiguous); warp-uniform control flow: a
                // straight line of per-slot bit tests that leaves after the last slot jhi (an A/B measurement
                // chose it over a computed jump to the first slot, which the backward kernel uses)
                const int jhi = 31 - __clz(rm);
#define GSB_FWD_SLOT(j)                                                                                   \
    {                                                                                                     \
        const float dy = dy0 - (float)(2 * j);  /* centre.y - pixel row */                                                                    \
        /* sigma = (a/2)dx^2 + (c/2)dy^2 + b dx dy   (forward.cu:340-342) */                              \
        const float sigma = fmaf(dy, fmaf(q1.z, dy, bdx), adx2);                                          \
        if (COUNT && lane == 0) ++n_slot;                                                                 \
        if (__float_as_uint(sigma) <= __float_as_uint(smax)) { /* 0 <= sigma <= smax, no exp */           \
            /* alpha = min(0.999, opac*exp(-sigma)) = min(0.999, 2^(log2 opac - sigma log2 e)) */         \
            const float alpha = fminf(0.999f, ex2_approx(fmaf(sigma, -GSB_LOG2E, q0.z)));                 \
            if (COUNT) ++n_eval;                                                                          \
            if (alpha >= (1.f / 255.f)) {                                                                 \
                const float next_T = T[j] * (1.f - alpha);                                                \
                if (next_T <= 1e-4f) { /* terminate BEFORE blending */                                    \
                    if (T[j] > 0.f) { T[j] = -T[j]; done |= 1u << j; }                                    \
                } else {                                                                                  \
                    const float vis = alpha * T[j];                                                       \
                    cr[j] = fmaf(q2.x, vis, cr[j]);                                                       \
                    cg[j] = fmaf(q2.y, vis, cg[j]);                                                       \
                    cb[j] = fmaf(q2.z, vis, cb[j]);                                                       \
                    if (DEPTH) cd[j] = fmaf(z, vis, cd[j]);                                               \
                    T[j] = next_T;                                                                        \
                    last[j] = idx;                                                                        \
                    if (COUNT) ++n_blend;                                                                 \
                }                                                                                         \
            }                                                                                             \
        }                                                                                                 \
        if (jhi == j) break;                                                                              \
    }
                do {   // straight-line: one warp-uniform test per slot
                    if (rm & 1u) GSB_FWD_SLOT(0)
                    if (rm & 2u) GSB_FWD_SLOT(1)
                    if (rm & 4u) GSB_FWD_SLOT(2)
                    if (rm & 8u) GSB_FWD_SLOT(3)
                    if (rm & 16u) GSB_FWD_SLOT(4)
                    if (rm & 32u) GSB_FWD_SLOT(5)
                    if (rm & 64u) GSB_FWD_SLOT(6)
                    if (rm & 128u) GSB_FWD_SLOT(7)
                } while (0);
#undef GSB_FWD_SLOT
            }
            if (__all_sync(0xffffffffu, done == 0xffu)) { ++c; break; }  // whole tile saturated
            __syncwarp();
            if (issued < nchunks) { issue(issued); ++issued; }
        }
        // drain bulk copies still in flight (early exit) so the ring can be reused by the next tile
        for (; c < issued; ++c) mbar_wait(&ring.full[stage_of(c)], parity_of(c));
        gchunk = g0 + (unsigned)issued;
        __syncwarp();

#pragma unroll
        for (int j = 0; j < RK_PIX; ++j) {
            const int Y = Y0 + 2 * j;
            if (X < img_w && Y < img_h) {
                const size_t p = (size_t)Y * img_w + X;
                const float Tf = fabsf(T[j]);
                final_Ts[p] = Tf;
                float o0 = cr[j] + Tf * bg0, o1 = cg[j] + Tf * bg1, o2 = cb[j] + Tf * bg2;
                int fi = last[j];
                if (SAT) {
                    if (!(o0 <= 1.f)) { fi |= GSB_SAT_BIT0; o0 = o0 > 1.f ? 1.f : o0; }
                    if (!(o1 <= 1.f)) { fi |= GSB_SAT_BIT0 << 1; o1 = o1 > 1.f ? 1.f : o1; }
                    if (!(o2 <= 1.f)) { fi |= GSB_SAT_BIT0 << 2; o2 = o2 > 1.f ? 1.f : o2; }
                }
                final_idx[p] = fi;
                out_img[3 * p] = o0;
                out_img[3 * p + 1] = o1;
                out_img[3 * p + 2] = o2;
                if (DEPTH) {   // never clamped
                    out_depth[p] = cd[j];
                    out_alpha[p] = 1.f - Tf;
                }
            }
        }
    }
    if (COUNT) {
        // per-lane pixel-pair counts of one persistent warp stay far below 2^27, so the 32-bit warp sums are exact
        n_eval = __reduce_add_sync(0xffffffffu, (unsigned)n_eval);
        n_blend = __reduce_add_sync(0xffffffffu, (unsigned)n_blend);
        if (lane == 0) {
            atomicAdd(pair_counts + 0, n_rec);
            atomicAdd(pair_counts + 1, n_slot);
            atomicAdd(pair_counts + 2, n_eval);
            atomicAdd(pair_counts + 3, n_blend);
        }
    }
}


}  // namespace

int gsb_sm_count();
int gsb_blend_grid(const void *kernel, int num_tiles);

extern "C" size_t gsb_raster_records_bytes(int m) {
    // + 256 B of scratch at the end: the persistent blend kernels' tile counters
    return gsb_align_up((size_t)(m > 0 ? m : 0) * sizeof(GsbRecord), 256) + 256;
}

// records <- the per-intersection 48-byte blend records of a sorted intersection list (generic binning path)
extern "C" int gsb_pack_records(int m, const int32_t *gaussian_ids_sorted, const int32_t *sorted_index,
                                const float *xys, const float *conics, const float *colors, const float *opacities,
                                void *records, gsb_stream_t stream) {
    GSB_CHECK_ARG(m >= 0);
    if (m == 0) return 0;
    GSB_CHECK_ARG(records && gaussian_ids_sorted && xys && conics && colors && opacities);
    GSB_CHECK_ARG(((uintptr_t)records % 16) == 0 && ((uintptr_t)xys % 8) == 0);
    pack_records_kernel<<<gsb_div_up(m, 256), 256, 0, (cudaStream_t)stream>>>(
        m, gaussian_ids_sorted, sorted_index, reinterpret_cast<const float2 *>(xys), conics, colors, opacities,
        reinterpret_cast<GsbRecord *>(records));
    GSB_LAUNCH_CHECK();
    return 0;
}

// Argument checks of the two blend entry points, then the persistent warps' tile counters (the 256 B of scratch
// behind the records) are zeroed on `s` and returned in *counters.
static int blend_setup(int img_h, int img_w, int tiles_x, int tiles_y, int m, const int32_t *tile_bins,
                       const float *background, void *records, float *out_img, float *final_Ts, int32_t *final_idx,
                       cudaStream_t s, unsigned **counters) {
    GSB_CHECK_ARG(img_h > 0 && img_w > 0 && m >= 0);
    GSB_CHECK_ARG(tiles_x == gsb_div_up(img_w, GSB_TILE) && tiles_y == gsb_div_up(img_h, GSB_TILE));
    GSB_CHECK_ARG(tile_bins && background && out_img && final_Ts && final_idx && records);
    GSB_CHECK_ARG(((uintptr_t)records % 16) == 0);
    *counters = reinterpret_cast<unsigned *>(reinterpret_cast<char *>(records) + gsb_raster_records_bytes(m) - 256);
    GSB_CUDA(cudaMemsetAsync(*counters, 0, 256, s));
    return 0;
}

extern "C" int gsb_gather_record_depths(int m, const int32_t *gaussian_ids_sorted, const float *depths,
                                        const int32_t *bin_stats, float *record_depths, gsb_stream_t stream) {
    GSB_CHECK_ARG(m >= 0);
    if (m == 0) return 0;
    GSB_CHECK_ARG(gaussian_ids_sorted && depths && record_depths);
    gather_record_depths_kernel<<<gsb_div_up(m, 256), 256, 0, (cudaStream_t)stream>>>(
        m, gaussian_ids_sorted, depths, bin_stats, record_depths);
    GSB_LAUNCH_CHECK();
    return 0;
}

// Body of gsb_rasterize_forward_packed (depth = false) and of gsb_rasterize_forward_packed_depth.
static int forward_packed(int img_h, int img_w, int tiles_x, int tiles_y, int m, const int32_t *tile_bins,
                          const int32_t *tile_order, const int32_t *bin_stats, const float *background, void *records,
                          float *out_img, float *final_Ts, int32_t *final_idx, unsigned flags, bool depth,
                          const float *record_depths, float *out_depth, float *out_alpha, gsb_stream_t stream) {
    GSB_CHECK_ARG((flags & ~(unsigned)GSB_RASTER_CLAMP_MAX_ONE) == 0);
    const bool sat = (flags & GSB_RASTER_CLAMP_MAX_ONE) != 0;
    GSB_CHECK_ARG(!sat || m < GSB_SAT_BIT0);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned *counters = nullptr;
    const int rc = blend_setup(img_h, img_w, tiles_x, tiles_y, m, tile_bins, background, records, out_img, final_Ts,
                               final_idx, s, &counters);
    if (rc) return rc;
    const int num_tiles = tiles_x * tiles_y;
#define GSB_FWD_LAUNCH(S, D)                                                                                     \
    rasterize_forward_kernel<false, S, D>                                                                        \
        <<<gsb_blend_grid((const void *)rasterize_forward_kernel<false, S, D>, num_tiles), RK_THREADS, 0, s>>>(  \
            img_h, img_w, tiles_x, num_tiles, reinterpret_cast<const int2 *>(tile_bins),                         \
            reinterpret_cast<const GsbRecord *>(records), background, out_img, final_Ts, final_idx, counters,    \
            bin_stats, nullptr, tile_order, record_depths, out_depth, out_alpha)
    if (depth) {
        if (sat) GSB_FWD_LAUNCH(true, true); else GSB_FWD_LAUNCH(false, true);
    } else {
        if (sat) GSB_FWD_LAUNCH(true, false); else GSB_FWD_LAUNCH(false, false);
    }
#undef GSB_FWD_LAUNCH
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_rasterize_forward_packed(int img_h, int img_w, int tiles_x, int tiles_y, int m,
                                            const int32_t *tile_bins, const int32_t *tile_order,
                                            const int32_t *bin_stats, const float *background, void *records,
                                            float *out_img, float *final_Ts, int32_t *final_idx, unsigned flags,
                                            gsb_stream_t stream) {
    return forward_packed(img_h, img_w, tiles_x, tiles_y, m, tile_bins, tile_order, bin_stats, background, records,
                          out_img, final_Ts, final_idx, flags, false, nullptr, nullptr, nullptr, stream);
}

extern "C" int gsb_rasterize_forward_packed_depth(int img_h, int img_w, int tiles_x, int tiles_y, int m,
                                                  const int32_t *tile_bins, const int32_t *tile_order,
                                                  const int32_t *bin_stats, const float *background, void *records,
                                                  float *out_img, float *final_Ts, int32_t *final_idx, unsigned flags,
                                                  const float *record_depths, float *out_depth, float *out_alpha,
                                                  gsb_stream_t stream) {
    GSB_CHECK_ARG(out_depth && out_alpha && (record_depths || m == 0));
    return forward_packed(img_h, img_w, tiles_x, tiles_y, m, tile_bins, tile_order, bin_stats, background, records,
                          out_img, final_Ts, final_idx, flags, true, record_depths, out_depth, out_alpha, stream);
}

// Diagnostic twin of gsb_rasterize_forward_packed: same outputs, plus pair_counts (device uint64[4], accumulated --
// zero it first) = {records passing the per-record test, slot visits (x 32 = pixel tests), pixel pairs evaluated
// (sigma inside the extent), pixel pairs blended}.  Used by bench.py / the profiles for pairs-per-second figures;
// never on the timed path.
extern "C" int gsb_rasterize_forward_count(int img_h, int img_w, int tiles_x, int tiles_y, int m,
                                           const int32_t *tile_bins, const float *background, void *records,
                                           float *out_img, float *final_Ts, int32_t *final_idx,
                                           unsigned long long *pair_counts, gsb_stream_t stream) {
    GSB_CHECK_ARG(pair_counts);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned *counters = nullptr;
    const int rc = blend_setup(img_h, img_w, tiles_x, tiles_y, m, tile_bins, background, records, out_img, final_Ts,
                               final_idx, s, &counters);
    if (rc) return rc;
    const int num_tiles = tiles_x * tiles_y;
    const int grid = gsb_blend_grid((const void *)rasterize_forward_kernel<true, false, false>, num_tiles);
    rasterize_forward_kernel<true, false, false><<<grid, RK_THREADS, 0, s>>>(
        img_h, img_w, tiles_x, num_tiles, reinterpret_cast<const int2 *>(tile_bins),
        reinterpret_cast<const GsbRecord *>(records), background, out_img, final_Ts, final_idx, counters, nullptr,
        pair_counts, nullptr, nullptr, nullptr, nullptr);
    GSB_LAUNCH_CHECK();
    return 0;
}

// ---- shared launch helpers (also used by raster_bwd.cu) --------------------------------------
int gsb_sm_count() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
        if (cached <= 0) cached = 132;
        cached_dev = dev;
    }
    return cached;
}

// persistent grid: SMs x resident CTAs per SM (never more CTAs than there are tile groups).  The occupancy query
// costs a few microseconds of host time per call, so its result is cached per (thread, device, kernel): 16 entries
// hold the 9 blend kernels (forward x {plain, SAT} x {colour, DEPTH} + COUNT, backward x {plain, SAT} x {colour,
// DEPTH}) on one device with room to spare.
int gsb_blend_grid(const void *kernel, int num_tiles) {
    struct Entry { const void *kernel; int dev; int per_sm; };
    static thread_local Entry cache[16] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    int per_sm = 0;
    for (const Entry &e : cache)
        if (e.kernel == kernel && e.dev == dev) per_sm = e.per_sm;
    if (per_sm == 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, RK_THREADS, 0) != cudaSuccess || per_sm < 1)
            per_sm = 1;
        for (Entry &e : cache)
            if (e.kernel == nullptr || e.kernel == kernel) { e = Entry{kernel, dev, per_sm}; break; }
    }
    const int full = gsb_sm_count() * per_sm;
    const int need = gsb_div_up(num_tiles, RK_WARPS);
    return need < full ? need : full;
}
