// binning.cu -- generic tile binning: scan (B1), intersection emit (B2), 64-bit key radix sort (B3),
// gather + tile bin edges (B4).  SURVEY.md section 8a.
//
// Replaces, in the reference: torch::cumsum (rasterize_gaussians.cpp:62), map_gaussian_to_intersects
// (forward.cu:107-143), torch::sort + torch::gather (rasterize_gaussians.cpp:25-32; CUB inside
// libtorch) and get_tile_bin_edges (forward.cu:148-169).
//
// B1 is the fast path's single-pass chained scan (bucket.cu, K1b, launched through gsb_count_scan), so
// both paths produce cum_tiles_hit with the same kernel.  Both also take each Gaussian's tile box from
// gsb_tile_bbox (gsb_common.cuh), the function the projection computes num_tiles_hit with.
//
// The sort is a hand-written single-pass-per-digit LSD radix sort ("onesweep" organisation: one
// up-front histogram of every digit, then per digit ONE kernel that ranks a tile of keys, publishes
// its per-digit counts and resolves its global offsets by decoupled look-back over the preceding
// tiles).  Keys are (tile_id << 32 | depth bits); only the 32 + ceil(log2(tiles)) significant bits
// are sorted (6 digit passes at 1080p/1440p/4K instead of the 8 a generic 64-bit sort needs), and the
// payload is the 32-bit original index generated on the fly in the first pass.  Integer/byte work,
// HBM/L2-bound: per pass 12 B read + 12 B written per intersection; the whole ping-pong working set
// (24 B x M) stays inside the 50 MB L2 up to M ~ 2M.
#include "gsb_common.cuh"

int gsb_count_scan_blocks(int n);
void gsb_count_scan(int n, int *counts_then_cum, unsigned *ticket, unsigned long long *state, cudaStream_t s);

namespace {

// ------------------------------------------------------------------------------------------------
// B2: emit (tile|depth) keys
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
map_intersects_kernel(int n, const float2 *__restrict__ xys, const float *__restrict__ depths,
                      const int *__restrict__ radii, const int *__restrict__ cum_tiles_hit, int tiles_x,
                      int tiles_y, long long *__restrict__ isect_ids, int *__restrict__ gaussian_ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float2 c = xys[i];
    int x0, x1, y0, y1;
    gsb_tile_bbox(c.x, c.y, (float)r, tiles_x, tiles_y, x0, x1, y0, y1);
    int cur = (i == 0) ? 0 : cum_tiles_hit[i - 1];
    const long long depth_id = (long long)__float_as_int(depths[i]);  // forward.cu:132
    for (int ty = y0; ty < y1; ++ty)
        for (int tx = x0; tx < x1; ++tx) {
            const long long tile_id = (long long)ty * tiles_x + tx;
            isect_ids[cur] = (tile_id << 32) | depth_id;
            gaussian_ids[cur] = i;
            ++cur;
        }
}

// ------------------------------------------------------------------------------------------------
// B3: onesweep LSD radix sort, 8-bit digits, 64-bit keys + 32-bit index payload
// ------------------------------------------------------------------------------------------------
constexpr int RS_THREADS = 256;
constexpr int RS_KPT = 8;                        // keys per thread
constexpr int RS_TILE = RS_THREADS * RS_KPT;     // 2048 keys per CTA
constexpr int RS_MAX_PASSES = 8;
constexpr unsigned FLAG_AGG = 1u << 30;
constexpr unsigned FLAG_PREFIX = 2u << 30;
constexpr unsigned FLAG_MASK = 3u << 30;

struct SortLayout {  // workspace carve-up (all offsets 256-B aligned)
    size_t keys_tmp, idx_tmp, digit_base, tile_counter, status, total;
    int ntiles;
};

SortLayout sort_layout(int m) {
    SortLayout L;
    L.ntiles = gsb_div_up(m > 0 ? m : 1, RS_TILE);
    size_t o = 0;
    L.keys_tmp = o; o += gsb_align_up((size_t)m * 8, 256);
    L.idx_tmp = o; o += gsb_align_up((size_t)m * 4, 256);
    L.digit_base = o; o += gsb_align_up((size_t)RS_MAX_PASSES * 256 * 4, 256);
    L.tile_counter = o; o += 256;
    L.status = o; o += gsb_align_up((size_t)RS_MAX_PASSES * L.ntiles * 256 * 4, 256);
    L.total = o;
    return L;
}

// all-digit histogram: hist[pass][digit]
__global__ void __launch_bounds__(RS_THREADS)
radix_hist_kernel(int m, int passes, const unsigned long long *__restrict__ keys,
                  unsigned *__restrict__ hist) {
    __shared__ unsigned sh[RS_MAX_PASSES * 256];
    for (int i = threadIdx.x; i < passes * 256; i += RS_THREADS) sh[i] = 0;
    __syncthreads();
    const int base = blockIdx.x * RS_TILE;
#pragma unroll
    for (int r = 0; r < RS_KPT; ++r) {
        const int i = base + r * RS_THREADS + threadIdx.x;
        if (i < m) {
            const unsigned long long k = keys[i];
            for (int p = 0; p < passes; ++p) atomicAdd(&sh[p * 256 + (unsigned)((k >> (8 * p)) & 0xff)], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < passes * 256; i += RS_THREADS)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// exclusive scan over the 256 digits of each pass (one block per pass)
__global__ void __launch_bounds__(256)
radix_digit_scan_kernel(unsigned *__restrict__ hist) {
    __shared__ int sm[256 / 32 + 1];
    unsigned *h = hist + blockIdx.x * 256;
    int v = (int)h[threadIdx.x];
    int total;
    int ex = block_excl_scan<256>(v, &total, sm);
    h[threadIdx.x] = (unsigned)ex;
}

__device__ __forceinline__ unsigned ld_relaxed(const unsigned *p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(unsigned *p, unsigned v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

template <bool FIRST>
__global__ void __launch_bounds__(RS_THREADS)
radix_onesweep_kernel(int m, int shift, const unsigned long long *__restrict__ keys_in,
                      const int *__restrict__ idx_in, unsigned long long *__restrict__ keys_out,
                      int *__restrict__ idx_out, const unsigned *__restrict__ digit_base,
                      unsigned *__restrict__ tile_counter, unsigned *__restrict__ status) {
    __shared__ unsigned whist[RS_THREADS / 32][256];  // per-warp digit counts -> per-warp offsets
    __shared__ unsigned gbase[256];                   // global position of this tile's digit run
    __shared__ unsigned s_tile;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);  // tiles are processed in ticket order
#pragma unroll
    for (int k = 0; k < RS_THREADS / 32; ++k) whist[k][threadIdx.x] = 0;
    __syncthreads();
    const unsigned tile = s_tile;
    const int base = (int)tile * RS_TILE + w * (32 * RS_KPT);

    unsigned long long key[RS_KPT];
    unsigned rank[RS_KPT];
#pragma unroll
    for (int r = 0; r < RS_KPT; ++r) {
        const int i = base + r * 32 + lane;
        key[r] = (i < m) ? keys_in[i] : ~0ull;  // padding sorts last inside the (final) tile
    }
    const unsigned lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < RS_KPT; ++r) {
        const unsigned d = (unsigned)((key[r] >> shift) & 0xff);
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

    // thread d owns digit d: exclusive scan across warps, publish, look back
    {
        const unsigned d = threadIdx.x;
        unsigned run = 0;
#pragma unroll
        for (int k = 0; k < RS_THREADS / 32; ++k) {
            unsigned c = whist[k][d];
            whist[k][d] = run;
            run += c;
        }
        const unsigned count = run;
        unsigned *st = status + (size_t)tile * 256 + d;
        unsigned excl = 0;
        if (tile == 0) {
            st_relaxed(st, count | FLAG_PREFIX);
        } else {
            st_relaxed(st, count | FLAG_AGG);
            int t = (int)tile - 1;
            while (true) {
                unsigned v = ld_relaxed(status + (size_t)t * 256 + d);
                if ((v & FLAG_MASK) == 0) continue;  // predecessor not published yet
                excl += v & ~FLAG_MASK;
                if ((v & FLAG_MASK) == FLAG_PREFIX) break;
                --t;
            }
            st_relaxed(st, (excl + count) | FLAG_PREFIX);
        }
        gbase[d] = digit_base[d] + excl;
    }
    __syncthreads();

#pragma unroll
    for (int r = 0; r < RS_KPT; ++r) {
        const int i = base + r * 32 + lane;
        if (i < m) {
            const unsigned d = (unsigned)((key[r] >> shift) & 0xff);
            const unsigned pos = gbase[d] + whist[w][d] + rank[r];
            keys_out[pos] = key[r];
            idx_out[pos] = FIRST ? i : idx_in[i];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// B4: gather ids through the permutation + tile bin edges
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gather_bin_edges_kernel(int m, const long long *__restrict__ keys_sorted,
                        const int *__restrict__ sorted_index, const int *__restrict__ gaussian_ids,
                        int *__restrict__ gaussian_ids_sorted, int2 *__restrict__ tile_bins) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    gaussian_ids_sorted[i] = gaussian_ids[sorted_index[i]];
    const int cur = (int)(keys_sorted[i] >> 32);
    if (i == 0) tile_bins[cur].x = 0;
    if (i == m - 1) tile_bins[cur].y = m;
    if (i > 0) {
        const int prev = (int)(keys_sorted[i - 1] >> 32);
        if (prev != cur) {
            tile_bins[prev].y = i;
            tile_bins[cur].x = i;
        }
    }
}

}  // namespace

// =================================================================================================
// workspace: the block ticket (256 B), then the look-back state word of every block of the chained scan
extern "C" size_t gsb_cumsum_workspace_bytes(int n) {
    return 256 + gsb_align_up((size_t)gsb_count_scan_blocks(n) * 8, 256);
}

extern "C" int gsb_cumsum_tiles_hit(int n, const int32_t *num_tiles_hit, int32_t *cum_tiles_hit,
                                    void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(num_tiles_hit && cum_tiles_hit && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0);
    const size_t ws_bytes = gsb_cumsum_workspace_bytes(n);
    if (workspace_bytes < ws_bytes) {
        gsb_set_error(GSB_ERR_WORKSPACE, "cumsum workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    GSB_CUDA(cudaMemsetAsync(ws, 0, ws_bytes, s));
    if (cum_tiles_hit != num_tiles_hit)
        GSB_CUDA(cudaMemcpyAsync(cum_tiles_hit, num_tiles_hit, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToDevice,
                                 s));
    gsb_count_scan(n, cum_tiles_hit, (unsigned *)ws, (unsigned long long *)(ws + 256), s);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_map_gaussian_to_intersects(int n, int m, const float *xys, const float *depths,
                                              const int32_t *radii, const int32_t *cum_tiles_hit,
                                              int tiles_x, int tiles_y, int64_t *isect_ids,
                                              int32_t *gaussian_ids, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && m >= 0 && tiles_x > 0 && tiles_y > 0);
    if (n == 0 || m == 0) return 0;
    GSB_CHECK_ARG(xys && depths && radii && cum_tiles_hit && isect_ids && gaussian_ids);
    map_intersects_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, reinterpret_cast<const float2 *>(xys), depths, radii, cum_tiles_hit, tiles_x, tiles_y,
        reinterpret_cast<long long *>(isect_ids), gaussian_ids);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t gsb_sort_workspace_bytes(int m) { return sort_layout(m > 0 ? m : 0).total + 256; }

extern "C" int gsb_sort_intersects(int m, int num_tiles, const int64_t *isect_ids,
                                   int64_t *isect_ids_sorted, int32_t *sorted_index, void *workspace,
                                   size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(m >= 0 && num_tiles > 0);
    if (m == 0) return 0;
    GSB_CHECK_ARG(isect_ids && isect_ids_sorted && sorted_index && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0);
    if (workspace_bytes < gsb_sort_workspace_bytes(m)) {
        gsb_set_error(GSB_ERR_WORKSPACE, "sort workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int tile_bits = 0;
    while ((1ll << tile_bits) < (long long)num_tiles) ++tile_bits;
    const int key_bits = 32 + tile_bits;
    const int passes = (key_bits + 7) / 8;
    GSB_CHECK_ARG(passes <= RS_MAX_PASSES);
    const SortLayout L = sort_layout(m);
    char *ws = (char *)workspace;
    unsigned long long *keys_tmp = (unsigned long long *)(ws + L.keys_tmp);
    int *idx_tmp = (int *)(ws + L.idx_tmp);
    unsigned *digit_base = (unsigned *)(ws + L.digit_base);
    unsigned *tile_counter = (unsigned *)(ws + L.tile_counter);
    unsigned *status = (unsigned *)(ws + L.status);
    // one memset covers digit histograms, tile tickets and look-back status words
    GSB_CUDA(cudaMemsetAsync(ws + L.digit_base, 0, L.total - L.digit_base, s));
    radix_hist_kernel<<<L.ntiles, RS_THREADS, 0, s>>>(m, passes, (const unsigned long long *)isect_ids,
                                                     digit_base);
    radix_digit_scan_kernel<<<passes, 256, 0, s>>>(digit_base);
    const unsigned long long *kin = (const unsigned long long *)isect_ids;
    const int *iin = nullptr;
    for (int p = 0; p < passes; ++p) {
        const bool to_out = ((passes - 1 - p) % 2) == 0;
        unsigned long long *kout = to_out ? (unsigned long long *)isect_ids_sorted : keys_tmp;
        int *iout = to_out ? sorted_index : idx_tmp;
        unsigned *st = status + (size_t)p * L.ntiles * 256;
        if (p == 0)
            radix_onesweep_kernel<true><<<L.ntiles, RS_THREADS, 0, s>>>(
                m, 8 * p, kin, iin, kout, iout, digit_base + p * 256, tile_counter + p, st);
        else
            radix_onesweep_kernel<false><<<L.ntiles, RS_THREADS, 0, s>>>(
                m, 8 * p, kin, iin, kout, iout, digit_base + p * 256, tile_counter + p, st);
        kin = kout;
        iin = iout;
    }
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_gather_bin_edges(int m, int num_tiles, const int64_t *isect_ids_sorted,
                                    const int32_t *sorted_index, const int32_t *gaussian_ids,
                                    int32_t *gaussian_ids_sorted, int32_t *tile_bins,
                                    gsb_stream_t stream) {
    GSB_CHECK_ARG(m >= 0 && num_tiles > 0 && tile_bins);
    cudaStream_t s = (cudaStream_t)stream;
    GSB_CUDA(cudaMemsetAsync(tile_bins, 0, (size_t)num_tiles * 8, s));
    if (m == 0) return 0;
    GSB_CHECK_ARG(isect_ids_sorted && sorted_index && gaussian_ids && gaussian_ids_sorted);
    gather_bin_edges_kernel<<<gsb_div_up(m, 256), 256, 0, s>>>(
        m, reinterpret_cast<const long long *>(isect_ids_sorted), sorted_index, gaussian_ids,
        gaussian_ids_sorted, reinterpret_cast<int2 *>(tile_bins));
    GSB_LAUNCH_CHECK();
    return 0;
}
