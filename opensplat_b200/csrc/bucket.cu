// bucket.cu -- two-level tile binning fused with record packing (fast path of B1+B2+B3+B4 + pack).
//
// The reference scans num_tiles_hit (rasterize_gaussians.cpp:62), reads M back (:63), sorts all M intersections
// globally on the 64-bit key (tile_id << 32 | depth bits) (:25-32) and then finds tile boundaries
// (forward.cu:148-169).  The same ORDER -- by tile, then depth bits, ties by ascending unsorted slot k (what a
// stable sort of the Gaussian-major emission gives) -- is produced here without a global sort and without a
// host read-back in the middle:
//   K1 bin_count      : per Gaussian, build its 48-B attribute record once and count the tiles it is binned to (one
//                       atomic per tile -> tile sizes); K1b count_scan: single-pass chained scan (decoupled look-back)
//                       of the per-Gaussian counts -> cum_tiles_hit (the gradient-row slots).  The generic path's
//                       gsb_cumsum_tiles_hit (binning.cu) is this same scan, launched through gsb_count_scan.
//   K2 tile_scan      : exclusive scan over the T tiles (chained scan over <= 32 CTAs) -> tile_bins (first, last+1),
//                       write cursors, stats = {M, longest list, overflow flag, visible count of K1}
//   K3 bucket_emit    : per Gaussian, write (depth bits << 32 | k) into its tiles' segments (atomic cursor;
//                       arrival order is arbitrary, the composite key makes the final order unique)
//   K4 tile_sort_pack : one CTA per tile sorts its segment in shared memory (64-bit composites), then gathers the
//                       Gaussian attributes and writes the 48-B record stream directly.
// Optional conservative culling (cull = 1, what RasterizeGaussians uses): a (Gaussian, tile) pair is binned only
// if the Gaussian's extent box {alpha can reach 1/255} touches the tile -- the same test, on the same floats, that
// the blend kernels apply per record (extent_slot_mask), so no pixel result changes; it removes 20-25 % of the
// intersections from the sort, the record stream and the gradient rows.  With cull = 0 tile_bins, cum_tiles_hit
// and the per-tile order are bit-identical to the reference's / the generic path's
// (tests/test_gpu_parity.py::test_bucket_binning_matches_generic_sort).
// K2-K4 and the blend kernels are sized by CAPACITIES chosen by the host from earlier frames; K2 raises
// stats[2] when M or the longest list exceeds them and everything downstream then returns immediately, so the
// host can check the read-back AFTER it has enqueued the whole forward pass (no pipeline bubble) and redo the
// frame with larger buffers in the rare overflow case.
// Integer work, L2/HBM-bound.
#include "raster_common.cuh"

namespace {

// Tile counters / write cursors are padded to one 128-B line each: the ~400 atomics a tile receives then
// serialise in their own L2 line (and the lines spread over all L2 slices) instead of 32 tiles sharing one.
constexpr int CUR_STRIDE = 32;  // ints
constexpr int BIN_THREADS = 256;
constexpr int TSCAN_THREADS = 1024;

constexpr int LEN_BUCKETS = 64;
struct BinHeader {          // 1 KB at the start of the workspace, zeroed by the call's memset
    unsigned ticket_n;      // dynamic block ids of K1b (order of the chained scan)
    unsigned ticket_t;      // ... of K2
    unsigned done_t;        // K2 blocks finished
    int max_len;            // longest tile list (atomicMax)
    int total;              // M
    int visible;            // Gaussians with radii > 0 (K1: one atomic per CTA)
    int pad0[2];
    int len_hist[LEN_BUCKETS];   // tiles per list-length bucket (K2), for the longest-first tile order (K2b)
    int len_cur[LEN_BUCKETS];    // K2b write cursors
    int pad[120];
};
static_assert(sizeof(BinHeader) == 1024, "header is 1 KB");

// list-length bucket of a tile: 64 linear buckets over [0, len_capacity]
__device__ __forceinline__ int len_bucket(int v, int len_capacity) {
    const long long b = (long long)v * LEN_BUCKETS / ((long long)max(len_capacity, 1) + 1);
    return (int)(b < LEN_BUCKETS - 1 ? b : LEN_BUCKETS - 1);
}

// ---- single-pass chained scan across blocks (decoupled look-back) ------------------------------------------
// state[b] = flag << 62 | value: flag 1 = block aggregate published, 2 = inclusive prefix published.  Blocks take
// their index from a ticket counter, so every block a look-back waits on is already running.
constexpr unsigned long long ST_AGG = 1ull << 62, ST_INC = 2ull << 62, ST_VAL = 0xffffffffull;

__device__ __forceinline__ unsigned long long ld_state(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_state(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// Called by the first warp of a block; returns (to every lane) the sum of the aggregates of blocks 0..blk-1 and
// publishes this block's inclusive prefix.
__device__ __forceinline__ int chained_scan_prefix(unsigned long long *state, int blk, int aggregate) {
    const int lane = threadIdx.x & 31;
    if (blk == 0) {
        if (lane == 0) st_state(&state[0], ST_INC | (unsigned)aggregate);
        return 0;
    }
    if (lane == 0) st_state(&state[blk], ST_AGG | (unsigned)aggregate);
    int excl = 0;
    int j = blk - 1;
    while (true) {
        const int idx = j - lane;
        unsigned long long s = ST_INC;   // virtual block -1: inclusive prefix 0
        if (idx >= 0) s = ld_state(&state[idx]);
        const unsigned flag = (unsigned)(s >> 62);
        if (__ballot_sync(0xffffffffu, flag == 0u)) continue;   // a predecessor has not published yet: poll again
        const unsigned incm = __ballot_sync(0xffffffffu, flag == 2u);
        int val = (int)(unsigned)(s & ST_VAL);
        if (incm) {
            const int first = __ffs(incm) - 1;      // nearest predecessor with an inclusive prefix
            if (lane > first) val = 0;
            excl += __reduce_add_sync(0xffffffffu, val);
            break;
        }
        excl += __reduce_add_sync(0xffffffffu, val);
        j -= 32;
    }
    if (lane == 0) st_state(&state[blk], ST_INC | (unsigned)(excl + aggregate));
    return excl;
}

// K1: attribute record + tile counting; writes the per-Gaussian count of binned tiles (scanned by K1b).  With
// `visible` given, adds the CTA's count of visible Gaussians (radii > 0, whether or not the cull leaves them in any
// tile list: the test of model.cpp:173 is radii.sum() == 0) to *visible with one atomic.
__global__ void __launch_bounds__(BIN_THREADS)
bin_count_kernel(int n, const float2 *__restrict__ xys, const int *__restrict__ radii,
                 const float *__restrict__ conics, const float *__restrict__ colors,
                 const float *__restrict__ opacities, int cull, int tiles_x, int tiles_y,
                 int *__restrict__ tile_count, GsbRecord *__restrict__ gattr, int *__restrict__ count_out,
                 int *__restrict__ visible) {
    const int i = blockIdx.x * BIN_THREADS + threadIdx.x;
    const int r = (i < n) ? radii[i] : 0;
    if (visible) {   // uniform over the grid: the barrier is reached by every thread or by none
        const int nvis = __syncthreads_count(r > 0);
        if (threadIdx.x == 0 && nvis > 0) atomicAdd(visible, nvis);
    }
    if (i >= n) return;
    int cnt = 0;
    if (r > 0) {
        const float2 c = xys[i];
        // the record of this Gaussian is built ONCE here (log2 / sqrt / extents) and only copied per intersection
        const GsbRecord rec = make_record(c, __ldg(conics + 3 * i), __ldg(conics + 3 * i + 1),
                                          __ldg(conics + 3 * i + 2), __ldg(opacities + i), __ldg(colors + 3 * i),
                                          __ldg(colors + 3 * i + 1), __ldg(colors + 3 * i + 2), 0);
        float4 *dst = reinterpret_cast<float4 *>(gattr + i);
        dst[0] = rec.q0; dst[1] = rec.q1; dst[2] = rec.q2;
        int x0, x1, y0, y1;
        gsb_tile_bbox(c.x, c.y, (float)r, tiles_x, tiles_y, x0, x1, y0, y1);
        for (int ty = y0; ty < y1; ++ty)
            for (int tx = x0; tx < x1; ++tx) {
                if (cull && !extent_slot_mask(c.x, c.y, rec.q1.w, rec.q2.w, (float)(tx * GSB_TILE),
                                              (float)(ty * GSB_TILE)))
                    continue;
                atomicAdd(&tile_count[(size_t)(ty * tiles_x + tx) * CUR_STRIDE], 1);
                ++cnt;
            }
    }
    count_out[i] = cnt;
}

// K1b: in-place inclusive scan of the per-Gaussian counts -> cum_tiles_hit (the gradient-row slots).  Single pass:
// 2048 counts per block, chained scan across blocks (decoupled look-back over ticket-ordered blocks).
constexpr int GS_IPT = 8;
__global__ void __launch_bounds__(BIN_THREADS)
count_scan_kernel(int n, int *__restrict__ counts_then_cum, unsigned *ticket, unsigned long long *state) {
    __shared__ int sm[BIN_THREADS / 32 + 1];
    __shared__ int s_blk, s_prefix;
    if (threadIdx.x == 0) s_blk = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int blk = s_blk;
    const int e0 = (blk * BIN_THREADS + threadIdx.x) * GS_IPT;
    int v[GS_IPT];
    const bool vec = (e0 + GS_IPT <= n) && ((reinterpret_cast<uintptr_t>(counts_then_cum + e0) & 15) == 0);
    if (vec) {
        const int4 a = *reinterpret_cast<const int4 *>(counts_then_cum + e0);
        const int4 b = *reinterpret_cast<const int4 *>(counts_then_cum + e0 + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int k = 0; k < GS_IPT; ++k) v[k] = (e0 + k < n) ? counts_then_cum[e0 + k] : 0;
    }
    int tsum = 0;
#pragma unroll
    for (int k = 0; k < GS_IPT; ++k) tsum += v[k];
    int total;
    int run = block_excl_scan<BIN_THREADS>(tsum, &total, sm);
    if (threadIdx.x < 32) {
        const int p = chained_scan_prefix(state, blk, total);
        if (threadIdx.x == 0) s_prefix = p;
    }
    __syncthreads();
    run += s_prefix;
#pragma unroll
    for (int k = 0; k < GS_IPT; ++k) { run += v[k]; v[k] = run; }
    if (vec) {
        *reinterpret_cast<int4 *>(counts_then_cum + e0) = make_int4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<int4 *>(counts_then_cum + e0 + 4) = make_int4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
        for (int k = 0; k < GS_IPT; ++k)
            if (e0 + k < n) counts_then_cum[e0 + k] = v[k];
    }
}

}  // namespace

// Host side of K1b, also called by gsb_cumsum_tiles_hit (binning.cu): in-place inclusive scan of n ints.  *ticket and
// state[0 .. gsb_count_scan_blocks(n)) must be zero when the kernel starts.
int gsb_count_scan_blocks(int n) { return gsb_div_up(n > 0 ? n : 1, BIN_THREADS * GS_IPT); }

void gsb_count_scan(int n, int *counts_then_cum, unsigned *ticket, unsigned long long *state, cudaStream_t s) {
    count_scan_kernel<<<gsb_count_scan_blocks(n), BIN_THREADS, 0, s>>>(n, counts_then_cum, ticket, state);
}

namespace {

// K2: exclusive scan of the tile sizes -> tile_bins, write cursors, stats = {M, longest list, overflow, visible}
__global__ void __launch_bounds__(TSCAN_THREADS)
tile_scan_kernel(int T, int nblk, int m_capacity, int len_capacity, BinHeader *hdr, unsigned long long *state,
                 int *__restrict__ tile_count_then_cursor, int2 *__restrict__ tile_bins, int *__restrict__ stats) {
    __shared__ int sm[TSCAN_THREADS / 32 + 1];
    __shared__ int s_blk, s_prefix, s_max;
    if (threadIdx.x == 0) { s_blk = (int)atomicAdd(&hdr->ticket_t, 1u); s_max = 0; }
    __syncthreads();
    const int blk = s_blk;
    const int t = blk * TSCAN_THREADS + threadIdx.x;
    const int v = (t < T) ? tile_count_then_cursor[(size_t)t * CUR_STRIDE] : 0;
    if (t < T) atomicAdd(&hdr->len_hist[len_bucket(v, len_capacity)], 1);
    int total;
    const int excl = block_excl_scan<TSCAN_THREADS>(v, &total, sm);
    const int wmax = __reduce_max_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && wmax > 0) atomicMax(&s_max, wmax);
    if (threadIdx.x < 32) {
        const int p = chained_scan_prefix(state, blk, total);
        if (threadIdx.x == 0) s_prefix = p;
    }
    __syncthreads();
    if (t < T) {
        const int e = s_prefix + excl;
        // empty tiles keep (0,0) like the reference's zero-initialised tile_bins
        tile_bins[t] = (v > 0) ? make_int2(e, e + v) : make_int2(0, 0);
        tile_count_then_cursor[(size_t)t * CUR_STRIDE] = e;   // becomes the write cursor of K3
    }
    if (threadIdx.x == 0) {
        if (s_max > 0) atomicMax(&hdr->max_len, s_max);
        if (blk == nblk - 1) atomicExch(&hdr->total, s_prefix + total);
        __threadfence();
        const unsigned done = atomicAdd(&hdr->done_t, 1u);
        if (done == (unsigned)nblk - 1u) {   // every block has published its part
            __threadfence();
            const int M = atomicAdd(&hdr->total, 0), mx = atomicAdd(&hdr->max_len, 0);
            stats[0] = M;
            stats[1] = mx;
            stats[2] = (M > m_capacity || mx > len_capacity) ? 1 : 0;
            stats[3] = hdr->visible;   // complete (K1 ran before this kernel); 0 unless counted
        }
    }
}

// K2b: tile order for the persistent blend kernels, longest list first.  A blend warp owns a tile for 1/2 .. 1/3 of
// the whole kernel's duration, so the kernel ends with a tail in which the last-started tiles run on mostly empty SMs;
// handing the tiles out longest-first makes those last ones the cheapest.
// Order inside a length bucket is arbitrary (tiles are independent: no result depends on it).
__global__ void __launch_bounds__(TSCAN_THREADS)
tile_order_kernel(int T, int len_capacity, BinHeader *hdr, const int2 *__restrict__ tile_bins,
                  int *__restrict__ tile_order) {
    __shared__ int base[LEN_BUCKETS];
    if (threadIdx.x < LEN_BUCKETS) {
        int sfx = 0;
        for (int b = LEN_BUCKETS - 1; b > (int)threadIdx.x; --b) sfx += hdr->len_hist[b];
        base[threadIdx.x] = sfx;
    }
    __syncthreads();
    const int t = blockIdx.x * TSCAN_THREADS + threadIdx.x;
    if (t >= T) return;
    const int2 r = tile_bins[t];
    const int b = len_bucket(r.y - r.x, len_capacity);
    tile_order[base[b] + atomicAdd(&hdr->len_cur[b], 1)] = t;
}

// K3: write the composites (depth bits << 32 | k) into the tiles' segments
__global__ void __launch_bounds__(256)
bucket_emit_kernel(int n, const GsbRecord *__restrict__ gattr, const float *__restrict__ depths,
                   const int *__restrict__ radii, const int *__restrict__ cum_tiles_hit, int cull, int tiles_x,
                   int tiles_y, int *__restrict__ cursor, unsigned long long *__restrict__ comp,
                   int *__restrict__ gaussian_ids, int *__restrict__ gid_at_pos, const int *__restrict__ stats) {
    if (stats[2]) return;   // capacities exceeded: the host redoes the frame
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float4 *src = reinterpret_cast<const float4 *>(gattr + i);
    const float4 q0 = src[0];
    const float hx = src[1].w, hy = src[2].w;
    int x0, x1, y0, y1;
    gsb_tile_bbox(q0.x, q0.y, (float)r, tiles_x, tiles_y, x0, x1, y0, y1);
    int k = (i == 0) ? 0 : cum_tiles_hit[i - 1];
    const unsigned long long hi = ((unsigned long long)(unsigned)__float_as_int(depths[i])) << 32;
    for (int ty = y0; ty < y1; ++ty)
        for (int tx = x0; tx < x1; ++tx) {
            if (cull && !extent_slot_mask(q0.x, q0.y, hx, hy, (float)(tx * GSB_TILE), (float)(ty * GSB_TILE)))
                continue;
            const int pos = atomicAdd(&cursor[(size_t)(ty * tiles_x + tx) * CUR_STRIDE], 1);
            comp[pos] = hi | (unsigned)k;
            if (gid_at_pos) gid_at_pos[pos] = i;   // payload of the distribution sort of LONG lists (K4a<.., true>)
            gaussian_ids[k] = i;      // slot -> Gaussian (K4b and the optional gaussian_ids_sorted output)
            ++k;
        }
}

typedef unsigned long long u64;

// distribution sort of a tile's composites (tile_sort_pack_kernel)
constexpr int DS_MIN_BINS = 64, DS_MAX_BINS = 2048;
constexpr int DS_BIN_LIMIT = 32;   // a bin above this many entries (clustered depths) sends the tile to the comparison sorts

constexpr int BITONIC_MAX = 4096;  // lists up to this (padded) length use the bitonic network (measured faster), longer ones the radix sort

__device__ __forceinline__ u64 shfl_xor_u64(u64 v, int m) {
    unsigned lo = (unsigned)v, hi = (unsigned)(v >> 32);
    lo = __shfl_xor_sync(0xffffffffu, lo, m);
    hi = __shfl_xor_sync(0xffffffffu, hi, m);
    return ((u64)hi << 32) | lo;
}

// compare-exchange across lanes at stride j (< 32): the lane keeps the min iff keep_min
__device__ __forceinline__ u64 cex_shfl(u64 v, int j, bool keep_min) {
    const u64 o = shfl_xor_u64(v, j);
    return ((v < o) == keep_min) ? v : o;
}

// Bitonic network restricted to one 64-element block held as (a = element base+lane, b = element
// base+32+lane): runs the sub-stages j = 32..1 of merge size k (direction of element i: ascending iff
// (i & k) == 0), entirely in registers / warp shuffles.
__device__ __forceinline__ void block64_substages(u64 &a, u64 &b, int base, int lane, int k, int jstart) {
    const int ia = base + lane, ib = ia + 32;
    const bool asc_a = (ia & k) == 0, asc_b = (ib & k) == 0;
    if (jstart >= 32) {  // partner of a is b (same thread); both share the direction (k >= 64)
        const bool sw = (a > b) == asc_a;
        const u64 t = sw ? b : a;
        b = sw ? a : b;
        a = t;
    }
#pragma unroll
    for (int j = 16; j >= 1; j >>= 1) {
        if (j > jstart) continue;
        const bool lower = (lane & j) == 0;
        a = cex_shfl(a, j, lower == asc_a);
        b = cex_shfl(b, j, lower == asc_b);
    }
}

// ---- CTA-wide LSD radix sort of a tile's composites, keyed on the 32 depth bits (bits 32..63) --------------
// Lists longer than 64 use this instead of a bitonic network (cost linear in L instead of L log^2 L; dense
// scenes have thousands of records per tile).  4 stable 8-bit passes; the items stay in registers between the
// rank and scatter steps, so ONE shared buffer suffices.  Depth ties (rare) come out in arrival order, which
// the bucket emission makes arbitrary: a final fix-up re-sorts every run of equal depths by k, restoring the
// reference's stable order (tile, depth, ascending unsorted slot).
template <int ITEMS>
__device__ __forceinline__ void cta_radix_sort_depth(u64 *buf, unsigned (*whist)[256], unsigned *bin_base,
                                                    unsigned *s_flag) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int wbase = w * 32 * ITEMS;  // warp w owns the contiguous range [wbase, wbase + 32*ITEMS)
    u64 key[ITEMS];
    unsigned rank[ITEMS];
#pragma unroll
    for (int r = 0; r < ITEMS; ++r) key[r] = buf[wbase + r * 32 + lane];
    const unsigned lt_mask = (1u << lane) - 1u;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 32 + 8 * pass;
#pragma unroll
        for (int k = 0; k < 8; ++k) whist[k][threadIdx.x] = 0;
        if (threadIdx.x == 0) *s_flag = 0;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < ITEMS; ++r) {
            const unsigned d = (unsigned)(key[r] >> shift) & 0xffu;
            const unsigned peers = __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            unsigned prev = 0;
            if (lane == leader) {
                prev = whist[w][d];
                whist[w][d] = prev + __popc(peers);
            }
            prev = __shfl_sync(0xffffffffu, prev, leader);
            rank[r] = prev + __popc(peers & lt_mask);
            __syncwarp();
        }
        __syncthreads();
        {   // thread d owns digit d: offsets across warps, then exclusive scan over the 256 digits
            const unsigned d = threadIdx.x;
            unsigned run = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const unsigned c = whist[k][d];
                whist[k][d] = run;
                run += c;
            }
            if (run == 256u * ITEMS) *s_flag = 1;  // every key has this digit: pass is a no-op
            unsigned inc = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (lane == 31) bin_base[256 + w] = inc;   // warp totals
            __syncthreads();
            unsigned woff = 0;
            for (int k = 0; k < w; ++k) woff += bin_base[256 + k];
            bin_base[d] = woff + inc - run;
        }
        __syncthreads();
        if (*s_flag == 0) {
#pragma unroll
            for (int r = 0; r < ITEMS; ++r) {
                const unsigned d = (unsigned)(key[r] >> shift) & 0xffu;
                buf[bin_base[d] + whist[w][d] + rank[r]] = key[r];
            }
            __syncthreads();
#pragma unroll
            for (int r = 0; r < ITEMS; ++r) key[r] = buf[wbase + r * 32 + lane];
        }
        __syncthreads();
    }
}

// Gather + pack of one tile: record i of the tile = attributes of the Gaussian behind the i-th sorted composite.
template <int U>
__device__ __forceinline__ void write_tile_records(const u64 *__restrict__ sorted, int L, int first,
                                                   const int *__restrict__ gaussian_ids,
                                                   const GsbRecord *__restrict__ gattr,
                                                   GsbRecord *__restrict__ records, int *__restrict__ sorted_index,
                                                   int *__restrict__ gaussian_ids_sorted) {
    // The chain composite -> slot k -> Gaussian id -> attribute record is three dependent (L2 / DRAM) gathers per entry;
    // U entries per thread are walked in lock-step so that U independent chains are in flight.  U = 2 pays when shared
    // memory already limits the resident CTAs (long lists, C5: 1.53 -> 1.03 ms for the stage); with short lists the
    // extra registers cost more occupancy than the second chain brings (C2: 0.144 -> 0.191 ms), so U = 1 there.
    for (int i0 = threadIdx.x; i0 < L; i0 += U * blockDim.x) {
        int k[U], g[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = i0 + u * blockDim.x;
            k[u] = (i < L) ? (int)(unsigned)(sorted[i] & 0xffffffffull) : -1;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) g[u] = (k[u] >= 0) ? __ldg(gaussian_ids + k[u]) : 0;
        float4 q0[U], q1[U], q2[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (k[u] >= 0) {
                const float4 *src = reinterpret_cast<const float4 *>(gattr + g[u]);   // 3 x 128-bit gather
                q0[u] = __ldg(src); q1[u] = __ldg(src + 1); q2[u] = __ldg(src + 2);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = i0 + u * blockDim.x;
            if (k[u] >= 0) {
                q0[u].w = __int_as_float(k[u]);
                float4 *dst = reinterpret_cast<float4 *>(records + first + i);
                stg_stream4(dst, q0[u]);
                stg_stream4(dst + 1, q1[u]);
                stg_stream4(dst + 2, q2[u]);
                if (sorted_index) sorted_index[first + i] = k[u];
                if (gaussian_ids_sorted) gaussian_ids_sorted[first + i] = g[u];
            }
        }
    }
}

// K4a: distribution sort + pack.  Depths inside a tile are spread over [dmin, dmax]: bin the composites linearly in
// depth into ~L/2 bins (the bin index is monotone in the depth bits), scatter them, let ONE thread order each (tiny)
// bin by the full composite (depth bits, k) and pack.  Work is linear in L instead of the L log^2 L of a bitonic
// network -- at C5's ~1000-entry lists an order of magnitude fewer instructions.  The result is the same total order
// as any comparison sort of the composites.  A tile whose depths cluster (some bin above DS_BIN_LIMIT entries, or all
// depths equal) is left to K4b (tile_done[tile] = 0), which also handles lists longer than this kernel's capacity.
// Pack of one tile whose sorted composites come with their Gaussian ids (the distribution sort's payload): one
// dependent gather per entry (the attribute record) instead of two.
template <int U>
__device__ __forceinline__ void write_tile_records_g(const u64 *__restrict__ sorted, const int *__restrict__ sorted_g,
                                                     int L, int first, const GsbRecord *__restrict__ gattr,
                                                     GsbRecord *__restrict__ records, int *__restrict__ sorted_index,
                                                     int *__restrict__ gaussian_ids_sorted) {
    for (int i0 = threadIdx.x; i0 < L; i0 += U * blockDim.x) {
        float4 q0[U], q1[U], q2[U];
        int k[U], g[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = i0 + u * blockDim.x;
            if (i < L) {
                k[u] = (int)(unsigned)(sorted[i] & 0xffffffffull);
                g[u] = sorted_g[i];
                const float4 *src = reinterpret_cast<const float4 *>(gattr + g[u]);   // 3 x 128-bit gather
                q0[u] = __ldg(src); q1[u] = __ldg(src + 1); q2[u] = __ldg(src + 2);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = i0 + u * blockDim.x;
            if (i < L) {
                q0[u].w = __int_as_float(k[u]);
                float4 *dst = reinterpret_cast<float4 *>(records + first + i);
                stg_stream4(dst, q0[u]);
                stg_stream4(dst + 1, q1[u]);
                stg_stream4(dst + 2, q2[u]);
                if (sorted_index) sorted_index[first + i] = k[u];
                if (gaussian_ids_sorted) gaussian_ids_sorted[first + i] = g[u];
            }
        }
    }
}

// PAYLOAD = true (long lists): the Gaussian ids written by K3 at the tile-major positions travel through the sort as
// payload, so the pack needs ONE dependent gather per entry (C5, same box: stage 1.60 -> 1.15 ms); with short lists the
// slot -> Gaussian table is L2-resident and the extra scattered store in K3 + the payload moves cost more than the
// shorter chain saves (C2: 0.142 -> 0.159 ms), so PAYLOAD = false there.
template <int U, bool PAYLOAD>
__global__ void __launch_bounds__(256)
tile_dsort_pack_kernel(int cap, const int2 *__restrict__ tile_bins, const unsigned long long *__restrict__ comp,
                       const int *__restrict__ gid_at_pos, const int *__restrict__ gaussian_ids,
                       const GsbRecord *__restrict__ gattr, GsbRecord *__restrict__ records,
                       int *__restrict__ sorted_index, int *__restrict__ gaussian_ids_sorted,
                       const int *__restrict__ stats, unsigned char *__restrict__ tile_done) {
    // [cap] staged composites, [cap] scatter target, then the same two arrays for the payload (Gaussian ids)
    extern __shared__ unsigned long long dkey[];
    __shared__ int dhist[DS_MAX_BINS];             // bin sizes, then write cursors, finally bin ends
    __shared__ int ds_scan[256 / 32 + 1];
    __shared__ unsigned ds_lo, ds_hi;
    __shared__ int ds_maxbin;
    if (stats[2]) return;      // capacities exceeded: the host redoes the frame
    const int tile = blockIdx.x;
    const int2 range = tile_bins[tile];
    const int L = range.y - range.x;
    const int lane = threadIdx.x & 31;
    if (L <= 0) { if (threadIdx.x == 0) tile_done[tile] = 1; return; }
    if (L > cap) { if (threadIdx.x == 0) tile_done[tile] = 0; return; }
    u64 *in = dkey, *out = dkey + cap;
    int *gin = reinterpret_cast<int *>(dkey + 2 * cap), *gout = gin + cap;
    if (L <= 64) {   // tiny lists: one warp, bitonic network in registers / shuffles (ids via the slot -> Gaussian table)
        if (threadIdx.x < 32) {
            u64 a = (lane < L) ? comp[range.x + lane] : ~0ull;
            u64 b = (32 + lane < L) ? comp[range.x + 32 + lane] : ~0ull;
#pragma unroll
            for (int k = 2; k <= 64; k <<= 1) block64_substages(a, b, 0, lane, k, k >> 1);
            out[lane] = a;
            out[32 + lane] = b;
        }
        __syncthreads();
        write_tile_records<1>(out, L, range.x, gaussian_ids, gattr, records, sorted_index, gaussian_ids_sorted);
        if (threadIdx.x == 0) tile_done[tile] = 1;
        return;
    }
    if (threadIdx.x == 0) { ds_lo = ~0u; ds_hi = 0u; ds_maxbin = 0; }
    int nb = DS_MIN_BINS;
    while (nb < (L >> 1) && nb < DS_MAX_BINS) nb <<= 1;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) dhist[b] = 0;
    __syncthreads();
    unsigned lo = ~0u, hi = 0u;
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const u64 c = comp[range.x + i];
        in[i] = c;
        if (PAYLOAD) gin[i] = gid_at_pos[range.x + i];
        const unsigned d = (unsigned)(c >> 32);
        lo = min(lo, d); hi = max(hi, d);
    }
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if (lane == 0) { atomicMin(&ds_lo, lo); atomicMax(&ds_hi, hi); }
    __syncthreads();
    if (ds_hi == ds_lo) { if (threadIdx.x == 0) tile_done[tile] = 0; return; }   // (uniform) one depth only
    const float fmin = __uint_as_float(ds_lo);
    const float scale = (float)nb / (__uint_as_float(ds_hi) - fmin);
    auto bin_of = [&](u64 c) {
        const int b = (int)((__uint_as_float((unsigned)(c >> 32)) - fmin) * scale);
        return min(max(b, 0), nb - 1);
    };
    for (int i = threadIdx.x; i < L; i += blockDim.x) atomicAdd(&dhist[bin_of(in[i])], 1);
    __syncthreads();
    {   // exclusive scan over the nb bins (8 consecutive bins per thread) + the largest bin
        int v[DS_MAX_BINS / 256], tsum = 0, tmax = 0;
#pragma unroll
        for (int q = 0; q < DS_MAX_BINS / 256; ++q) {
            const int b = threadIdx.x * (DS_MAX_BINS / 256) + q;
            v[q] = (b < nb) ? dhist[b] : 0;
            tsum += v[q]; tmax = max(tmax, v[q]);
        }
        int total;
        int run = block_excl_scan<256>(tsum, &total, ds_scan);
        tmax = __reduce_max_sync(0xffffffffu, tmax);
        if (lane == 0) atomicMax(&ds_maxbin, tmax);
#pragma unroll
        for (int q = 0; q < DS_MAX_BINS / 256; ++q) {
            const int b = threadIdx.x * (DS_MAX_BINS / 256) + q;
            if (b < nb) dhist[b] = run;     // write cursor of bin b; ends as the bin's end
            run += v[q];
        }
    }
    __syncthreads();
    if (ds_maxbin > DS_BIN_LIMIT) { if (threadIdx.x == 0) tile_done[tile] = 0; return; }   // (uniform) clustered depths
    for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const u64 c = in[i];
        const int p = atomicAdd(&dhist[bin_of(c)], 1);
        out[p] = c;
        if (PAYLOAD) gout[p] = gin[i];
    }
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {
        const int e = dhist[b], st = b ? dhist[b - 1] : 0;
        for (int p = st + 1; p < e; ++p) {   // insertion sort by (depth bits, k), the Gaussian id moves along
            const u64 c = out[p];
            const int cg = PAYLOAD ? gout[p] : 0;
            int q = p - 1;
            while (q >= st && out[q] > c) {
                out[q + 1] = out[q];
                if (PAYLOAD) gout[q + 1] = gout[q];
                --q;
            }
            out[q + 1] = c;
            if (PAYLOAD) gout[q + 1] = cg;
        }
    }
    __syncthreads();
    if (PAYLOAD) write_tile_records_g<U>(out, gout, L, range.x, gattr, records, sorted_index, gaussian_ids_sorted);
    else write_tile_records<U>(out, L, range.x, gaussian_ids, gattr, records, sorted_index, gaussian_ids_sorted);
    if (threadIdx.x == 0) tile_done[tile] = 1;
}

// One CTA per tile: sort the tile's composites (depth bits << 32 | k) ascending and write its records.
//  * L <= 64: one warp, bitonic network in registers / shuffles;
//  * longer:  CTA-wide LSD radix sort on the depth bits + tie fix-up (cta_radix_sort_depth).
template <int MAXI>   // largest items-per-thread instantiation compiled in (register budget): 4, 16 or 64
__global__ void __launch_bounds__(256)
tile_sort_pack_kernel(int cap, const int2 *__restrict__ tile_bins, const unsigned long long *__restrict__ comp,
                      const int *__restrict__ gaussian_ids, const GsbRecord *__restrict__ gattr,
                      GsbRecord *__restrict__ records, int *__restrict__ sorted_index,
                      int *__restrict__ gaussian_ids_sorted, const int *__restrict__ stats,
                      const unsigned char *__restrict__ tile_done) {
    extern __shared__ unsigned long long skey[];
    __shared__ unsigned whist[8][256];
    __shared__ unsigned bin_base[256 + 8];
    __shared__ unsigned s_flag;
    if (stats[2]) return;      // capacities exceeded: the host redoes the frame
    const int tile = blockIdx.x;
    if (tile_done[tile]) return;   // already ordered and packed by tile_dsort_pack_kernel
    const int2 range = tile_bins[tile];
    const int L = range.y - range.x;
    if (L <= 0) return;
    int n2 = 64;               // padded length: 64 (bitonic) or a multiple of 256 (radix), power of two
    while (n2 < L) n2 <<= 1;
    if (n2 > 64 && n2 < 256) n2 = 256;
    if (n2 > cap) return;      // cannot happen: K2 raised stats[2] if a list is longer than the capacity
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) skey[i] = (i < L) ? comp[range.x + i] : ~0ull;
    __syncthreads();
    if (L > 1) {
        if (n2 == 64) {
            if (warp == 0) {
                u64 a = skey[lane], b = skey[32 + lane];
#pragma unroll
                for (int k = 2; k <= 64; k <<= 1) block64_substages(a, b, 0, lane, k, k >> 1);
                skey[lane] = a;
                skey[32 + lane] = b;
            }
        } else if (n2 <= BITONIC_MAX) {
            // medium lists: bitonic network, <= 64-wide merges in registers / shuffles, wider strides in smem
            const int nwarps = blockDim.x >> 5, nblk = n2 >> 6;
            for (int blk = warp; blk < nblk; blk += nwarps) {
                const int base = blk << 6;
                u64 a = skey[base + lane], b = skey[base + 32 + lane];
#pragma unroll
                for (int k = 2; k <= 64; k <<= 1) block64_substages(a, b, base, lane, k, k >> 1);
                skey[base + lane] = a;
                skey[base + 32 + lane] = b;
            }
            __syncthreads();
            for (int k = 128; k <= n2; k <<= 1) {
                for (int j = k >> 1; j >= 64; j >>= 1) {
                    for (int t = threadIdx.x; t < (n2 >> 1); t += blockDim.x) {
                        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                        const int hiI = lo + j;
                        const bool asc = ((lo & k) == 0);
                        const u64 x = skey[lo], y = skey[hiI];
                        if ((x > y) == asc) {
                            skey[lo] = y;
                            skey[hiI] = x;
                        }
                    }
                    __syncthreads();
                }
                for (int blk = warp; blk < nblk; blk += nwarps) {
                    const int base = blk << 6;
                    u64 a = skey[base + lane], b = skey[base + 32 + lane];
                    block64_substages(a, b, base, lane, k, 32);
                    skey[base + lane] = a;
                    skey[base + 32 + lane] = b;
                }
                __syncthreads();
            }
        } else {
            const int items = n2 >> 8;
            if (items == 1) cta_radix_sort_depth<1>(skey, whist, bin_base, &s_flag);
            else if (items == 2) cta_radix_sort_depth<2>(skey, whist, bin_base, &s_flag);
            else if (items == 4) cta_radix_sort_depth<4>(skey, whist, bin_base, &s_flag);
            else if (MAXI >= 16 && items == 8) cta_radix_sort_depth<(MAXI >= 16 ? 8 : 1)>(skey, whist, bin_base, &s_flag);
            else if (MAXI >= 16 && items == 16) cta_radix_sort_depth<(MAXI >= 16 ? 16 : 1)>(skey, whist, bin_base, &s_flag);
            else if (MAXI >= 64 && items == 32) cta_radix_sort_depth<(MAXI >= 64 ? 32 : 1)>(skey, whist, bin_base, &s_flag);
            else if (MAXI >= 64) cta_radix_sort_depth<(MAXI >= 64 ? 64 : 1)>(skey, whist, bin_base, &s_flag);
            // tie fix-up: the thread at the start of a run of equal depths insertion-sorts the run by k
            for (int i = threadIdx.x; i < L; i += blockDim.x) {
                const unsigned dep = (unsigned)(skey[i] >> 32);
                if (i > 0 && (unsigned)(skey[i - 1] >> 32) == dep) continue;   // not a run start
                int e = i + 1;
                while (e < L && (unsigned)(skey[e] >> 32) == dep) ++e;
                for (int p = i + 1; p < e; ++p) {
                    const u64 v = skey[p];
                    int q = p - 1;
                    while (q >= i && skey[q] > v) { skey[q + 1] = skey[q]; --q; }
                    skey[q + 1] = v;
                }
            }
        }
        __syncthreads();
    }
    write_tile_records<1>(skey, L, range.x, gaussian_ids, gattr, records, sorted_index, gaussian_ids_sorted);
}

struct BucketLayout {
    size_t hdr, state_n, state_t, cursor, zero_bytes, gattr, comp, gids, gpos, done, total;
    int nblk_n, nblk_t;
};
BucketLayout bucket_layout(int n, int m, int T) {
    BucketLayout L;
    L.nblk_n = gsb_count_scan_blocks(n);
    L.nblk_t = gsb_div_up(T > 0 ? T : 1, TSCAN_THREADS);
    size_t o = 0;
    L.hdr = o; o += sizeof(BinHeader);
    L.state_n = o; o += gsb_align_up((size_t)L.nblk_n * 8, 256);
    L.state_t = o; o += gsb_align_up((size_t)L.nblk_t * 8, 256);
    L.cursor = o; o += gsb_align_up((size_t)(T > 0 ? T : 1) * CUR_STRIDE * sizeof(int), 256);
    L.zero_bytes = o;   // everything up to here is zeroed by one memset per call
    L.gattr = o; o += gsb_align_up((size_t)n * sizeof(GsbRecord), 256);
    L.comp = o; o += gsb_align_up((size_t)m * 8, 256);
    L.gids = o; o += gsb_align_up((size_t)m * 4, 256);
    L.gpos = o; o += gsb_align_up((size_t)m * 4, 256);
    L.done = o; o += gsb_align_up((size_t)(T > 0 ? T : 1), 256);   // per tile: ordered + packed by K4a
    L.total = o;
    return L;
}

constexpr int BUCKET_MAX_CAP = 16384;  // 128 KB of shared memory per CTA

int sort_cap_of(int len_capacity) {   // shared-memory capacity (power of two) of K4 for lists up to len_capacity
    int cap = 64;
    while (cap < len_capacity && cap < (1 << 30)) cap <<= 1;
    if (cap > 64 && cap < 256) cap = 256;
    return cap;
}

}  // namespace

extern "C" int gsb_bucket_max_tile_len(void) { return BUCKET_MAX_CAP; }

extern "C" size_t gsb_bucket_workspace_bytes(int n, int m_capacity, int num_tiles) {
    return bucket_layout(n > 0 ? n : 0, m_capacity > 0 ? m_capacity : 0, num_tiles).total;
}

// Phase 1: attribute records, tile sizes -> tile_bins + write cursors (inside the workspace), the scan of the
// per-Gaussian tile counts and stats = {M, longest list, overflow, visible Gaussians or 0} (device int32[4]).
// cull: bit 0 culls by the extent box; GSB_BIN_COUNT_VISIBLE asks for the visible count in stats[3].
extern "C" int gsb_bucket_tile_ranges(int n, const float *xys, const int32_t *radii, const float *conics,
                                      const float *colors, const float *opacities, int cull, int tiles_x,
                                      int tiles_y, int m_capacity, int len_capacity, void *workspace,
                                      size_t workspace_bytes, int32_t *cum_tiles_hit, int32_t *tile_bins,
                                      int32_t *tile_order, int32_t *stats, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && tiles_x > 0 && tiles_y > 0 && m_capacity >= 0 && len_capacity >= 0);
    GSB_CHECK_ARG(tile_bins && stats && workspace && ((uintptr_t)workspace % 256) == 0);
    GSB_CHECK_ARG((cull & ~(1 | GSB_BIN_COUNT_VISIBLE)) == 0);
    const bool count_visible = (cull & GSB_BIN_COUNT_VISIBLE) != 0;
    cull &= 1;
    const int T = tiles_x * tiles_y;
    const BucketLayout L = bucket_layout(n, m_capacity, T);
    if (workspace_bytes < L.total) {
        gsb_set_error(GSB_ERR_WORKSPACE, "bucket workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    BinHeader *hdr = (BinHeader *)(ws + L.hdr);
    int *cursor = (int *)(ws + L.cursor);
    GSB_CUDA(cudaMemsetAsync(ws, 0, L.zero_bytes, s));
    if (n > 0) {
        GSB_CHECK_ARG(xys && radii && conics && colors && opacities && cum_tiles_hit && ((uintptr_t)xys % 8) == 0);
        bin_count_kernel<<<gsb_div_up(n, BIN_THREADS), BIN_THREADS, 0, s>>>(
            n, reinterpret_cast<const float2 *>(xys), radii, conics, colors, opacities, cull, tiles_x, tiles_y, cursor,
            (GsbRecord *)(ws + L.gattr), cum_tiles_hit, count_visible ? &hdr->visible : nullptr);
        gsb_count_scan(n, cum_tiles_hit, &hdr->ticket_n, (unsigned long long *)(ws + L.state_n), s);
    }
    tile_scan_kernel<<<L.nblk_t, TSCAN_THREADS, 0, s>>>(T, L.nblk_t, m_capacity, len_capacity, hdr,
                                                       (unsigned long long *)(ws + L.state_t), cursor,
                                                       reinterpret_cast<int2 *>(tile_bins), stats);
    if (tile_order)
        tile_order_kernel<<<L.nblk_t, TSCAN_THREADS, 0, s>>>(T, len_capacity, hdr,
                                                            reinterpret_cast<const int2 *>(tile_bins), tile_order);
    GSB_LAUNCH_CHECK();
    return 0;
}

// Phase 2: bucket emit + per-tile sort + record pack, sized by the same capacities as phase 1 (no host read-back
// needed in between).  sorted_index / gaussian_ids_sorted are optional outputs ([m] int32, may be NULL).
extern "C" int gsb_bucket_sort_pack(int n, int m_capacity, int len_capacity, const float *depths,
                                    const int32_t *radii, const int32_t *cum_tiles_hit, int cull, int tiles_x,
                                    int tiles_y, const int32_t *tile_bins, const int32_t *stats, void *workspace,
                                    size_t workspace_bytes, void *records, int32_t *sorted_index,
                                    int32_t *gaussian_ids_sorted, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && m_capacity >= 0 && tiles_x > 0 && tiles_y > 0 && len_capacity >= 0);
    if (n == 0 || m_capacity == 0) return 0;
    GSB_CHECK_ARG(depths && radii && cum_tiles_hit && tile_bins && stats && workspace && records);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0 && ((uintptr_t)records % 16) == 0);
    const int T = tiles_x * tiles_y;
    const BucketLayout L = bucket_layout(n, m_capacity, T);
    if (workspace_bytes < L.total) {
        gsb_set_error(GSB_ERR_WORKSPACE, "bucket workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    const int cap = sort_cap_of(len_capacity);
    if (cap > BUCKET_MAX_CAP) {
        gsb_set_error(GSB_ERR_UNSUPPORTED, "tile list longer than the in-shared-memory sort capacity; "
                      "use the generic gsb_sort_intersects path", __FILE__, __LINE__);
        return GSB_ERR_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    unsigned long long *comp = (unsigned long long *)(ws + L.comp);
    int *gids = (int *)(ws + L.gids);
    GsbRecord *gattr = (GsbRecord *)(ws + L.gattr);
    const bool long_lists = cap > 1024;   // K4a then carries the Gaussian ids as sort payload
    bucket_emit_kernel<<<gsb_div_up(n, 256), 256, 0, s>>>(n, gattr, depths, radii, cum_tiles_hit, cull, tiles_x,
                                                         tiles_y, (int *)(ws + L.cursor), comp, gids,
                                                         long_lists ? (int *)(ws + L.gpos) : nullptr, stats);
    // K4a (distribution sort) stages the list twice in shared memory; lists beyond its capacity, and tiles whose
    // depths cluster, are left to K4b (comparison sorts)
    const int dcap = cap < 8192 ? cap : 8192;
    const size_t dsmem = (size_t)dcap * (long_lists ? 24 : 16);   // 2 x 8 B composites (+ 2 x 4 B Gaussian ids) per entry
    unsigned char *tile_done = (unsigned char *)(ws + L.done);
#define GSB_DSP(U, PAY)                                                                                         \
    do {                                                                                                        \
        if (dsmem > 32 * 1024)                                                                                  \
            GSB_CUDA(cudaFuncSetAttribute(tile_dsort_pack_kernel<U, PAY>,                                       \
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsmem));            \
        tile_dsort_pack_kernel<U, PAY><<<T, 256, dsmem, s>>>(dcap, reinterpret_cast<const int2 *>(tile_bins), comp, \
                                                            (const int *)(ws + L.gpos), gids, gattr,            \
                                                            reinterpret_cast<GsbRecord *>(records), sorted_index, \
                                                            gaussian_ids_sorted, stats, tile_done);             \
    } while (0)
    if (long_lists) GSB_DSP(2, true);
    else GSB_DSP(1, false);
#undef GSB_DSP
    const size_t smem = (size_t)cap * 8;
#define GSB_TSP(MAXI)                                                                                           \
    do {                                                                                                        \
        if (smem > 38 * 1024)                                                                                   \
            GSB_CUDA(cudaFuncSetAttribute(tile_sort_pack_kernel<MAXI>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                          (int)smem));                                                          \
        tile_sort_pack_kernel<MAXI><<<T, 256, smem, s>>>(                                                       \
            cap, reinterpret_cast<const int2 *>(tile_bins), comp, gids, gattr,                                  \
            reinterpret_cast<GsbRecord *>(records), sorted_index, gaussian_ids_sorted, stats, tile_done);       \
    } while (0)
    if (cap <= 1024) GSB_TSP(4);
    else if (cap <= 4096) GSB_TSP(16);
    else GSB_TSP(64);
#undef GSB_TSP
    GSB_LAUNCH_CHECK();
    return 0;
}
