// mcmc.cu -- the 3DGS-MCMC refinement strategy (Kheradmand et al. 2024; gsplat's MCMCStrategy) on the flat
// parameter / Adam buffers, DESIGN D20.
//
// Gaussians are never culled: dead ones (sigmoid(logit) <= min_opacity) are moved onto live ones drawn in
// proportion to their opacity, with the opacity and scale of the drawn rows changed so the rendered image is kept;
// growth appends copies of drawn rows; every training step adds opacity-gated noise shaped by the covariance to the
// means, and L1 penalties on opacity and scale to the gradient.
//
// Every random number comes from Philox4x32-10 keyed by the 64-bit seed, counter (index, step, tag, 0), so data-
// parallel replicas draw the same numbers without a collective and a test can restate every draw.  Draws replace
// torch.multinomial: an inclusive fp64 scan of the weights and a binary search.  The scan is built so that it is
// monotone whatever the weights (a weight-0 index can never be drawn): every partial sum is formed left to right --
// within a thread's chunk, over the chunk totals of a block (one thread), over the block totals (one thread) -- and
// c_i = fl(block prefix + fl(chunk prefix + running chunk sum)); rounding to nearest is monotone in each operand.
#include "gsb_common.cuh"

namespace {

constexpr int MT = 256;             // threads per block of the scan kernels
constexpr int CHUNK = 16;           // consecutive Gaussians per thread in the scan
constexpr int MB = MT * CHUNK;      // Gaussians per scan block
constexpr int RATIO_MAX = 51;       // gsplat's n_max: the largest ratio of the relocation table

struct Segments {                   // the flat layout, by value: slice s covers [offset, offset + n * row_floats)
    long long offset[GSB_MCMC_MAX_SEGMENTS];
    int row_floats[GSB_MCMC_MAX_SEGMENTS];
    int num;
};

__device__ __forceinline__ float sigmoid_f(float logit) { return 1.f / (1.f + expf(-logit)); }

// Philox4x32-10 (Salmon et al. 2011, the Random123 constants)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k.x += W0; k.y += W1; }
        const uint32_t lo0 = M0 * c.x, hi0 = __umulhi(M0, c.x), lo1 = M1 * c.z, hi1 = __umulhi(M1, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

__device__ __forceinline__ uint4 draw(uint2 key, int index, int step, int tag) {
    return philox4x32_10(make_uint4((uint32_t)index, (uint32_t)step, (uint32_t)tag, 0u), key);
}

// u = ((x0 >> 5) 2^26 + (x1 >> 6)) 2^-53: exact in fp64, in [0, 1)
__device__ __forceinline__ double uniform53(uint32_t x0, uint32_t x1) {
    return ((double)(x0 >> 5) * 67108864.0 + (double)(x1 >> 6)) * 0x1p-53;
}

// Box-Muller on exact fp32 uniforms u1 = ((a >> 8) + 1) 2^-24 in (0, 1], u2 = (b >> 8) 2^-24 in [0, 1):
// sqrt(-2 ln u1) (cos 2 pi u2, sin 2 pi u2).  sincospif takes 2 u2 exactly, so no rounding of 2 pi u2 enters.
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b) {
    const float u1 = (float)((a >> 8) + 1u) * 0x1p-24f, u2 = (float)(b >> 8) * 0x1p-24f;
    const float rad = sqrtf(-2.f * logf(u1));
    float s, c;
    sincospif(2.f * u2, &s, &c);
    return make_float2(rad * c, rad * s);
}

__device__ __forceinline__ float3 normals3(uint4 x) {
    const float2 z01 = box_muller(x.x, x.y), z23 = box_muller(x.z, x.w);
    return make_float3(z01.x, z01.y, z23.x);
}

// ---- planning: weights, the monotone fp64 scan, the dead set --------------------------------------------------

__device__ __forceinline__ bool is_dead(float o, float min_opacity, int mask_dead) {
    return mask_dead && o <= min_opacity;
}

// Per block: chunk-local running sums, chunk prefixes (one thread, left to right) -> cdf holds the in-block sums;
// the block's total, dead count and whether any opacity is > 0.
__global__ void __launch_bounds__(MT)
mcmc_scan_local_kernel(int n, const float *__restrict__ logits, float min_opacity, int mask_dead,
                       double *__restrict__ cdf, double *__restrict__ blk_sum, int *__restrict__ blk_dead,
                       int *__restrict__ blk_any) {
    __shared__ double chunk[MT];
    const int base = blockIdx.x * MB + threadIdx.x * CHUNK;
    double run = 0.0;
    int dead = 0, any = 0;
    double loc[CHUNK];
#pragma unroll
    for (int k = 0; k < CHUNK; ++k) {
        const int i = base + k;
        loc[k] = 0.0;
        if (i < n) {
            const float o = sigmoid_f(logits[i]);
            const bool d = is_dead(o, min_opacity, mask_dead);
            run += d ? 0.0 : (double)o;
            loc[k] = run;
            dead += d;
            any |= o > 0.f;
        }
    }
    __shared__ int block_dead;
    chunk[threadIdx.x] = run;
    __syncthreads();
    if (threadIdx.x == 0) {
        double p = 0.0;
        for (int t = 0; t < MT; ++t) {
            const double l = chunk[t];
            chunk[t] = p;
            p += l;
        }
        blk_sum[blockIdx.x] = p;
        block_dead = 0;
    }
    __syncthreads();
    const double pre = chunk[threadIdx.x];
#pragma unroll
    for (int k = 0; k < CHUNK; ++k)
        if (base + k < n) cdf[base + k] = pre + loc[k];
    if (dead) atomicAdd(&block_dead, dead);
    const int block_any = __syncthreads_or(any);
    if (threadIdx.x == 0) { blk_dead[blockIdx.x] = block_dead; blk_any[blockIdx.x] = block_any; }
}

// One thread, left to right over the blocks: block prefixes of the sums and dead counts, and the 16-byte result
// {n_dead, T > 0, any opacity > 0, 0} (T = the last block prefix + the last block's sum = cdf[n - 1]).
__global__ void mcmc_scan_blocks_kernel(int nb, const double *__restrict__ blk_sum, const int *__restrict__ blk_dead,
                                        const int *__restrict__ blk_any, double *__restrict__ blk_pre,
                                        int *__restrict__ blk_dead_off, int32_t *__restrict__ result) {
    if (threadIdx.x != 0) return;
    double p = 0.0;
    int d = 0, any = 0;
    for (int b = 0; b < nb; ++b) {
        blk_pre[b] = p;
        blk_dead_off[b] = d;
        p += blk_sum[b];
        d += blk_dead[b];
        any |= blk_any[b];
    }
    result[0] = d;
    result[1] = p > 0.0;
    result[2] = any;
    result[3] = 0;
}

// c_i = fl(block prefix + in-block sum); dead indices scattered in ascending order.
__global__ void __launch_bounds__(MT)
mcmc_scan_finish_kernel(int n, const float *__restrict__ logits, float min_opacity, int mask_dead,
                        const double *__restrict__ blk_pre, const int *__restrict__ blk_dead_off,
                        double *__restrict__ cdf, int32_t *__restrict__ dead) {
    __shared__ int smem[MT / 32 + 1];
    const int base = blockIdx.x * MB + threadIdx.x * CHUNK;
    const double pre = blk_pre[blockIdx.x];
    int nd = 0;
#pragma unroll
    for (int k = 0; k < CHUNK; ++k) {
        const int i = base + k;
        if (i < n) {
            if (blockIdx.x > 0) cdf[i] = pre + cdf[i];
            nd += is_dead(sigmoid_f(logits[i]), min_opacity, mask_dead);
        }
    }
    if (!mask_dead) return;
    int total;
    int at = blk_dead_off[blockIdx.x] + block_excl_scan<MT>(nd, &total, smem);
    if (nd == 0) return;
    for (int k = 0; k < CHUNK; ++k) {
        const int i = base + k;
        if (i < n && is_dead(sigmoid_f(logits[i]), min_opacity, mask_dead)) dead[at++] = i;
    }
}

// ---- sampling -------------------------------------------------------------------------------------------------

// sample j = the smallest i with cdf[i] > u_j T; counts[i] += 1 (integer atomics: the counts are deterministic)
__global__ void __launch_bounds__(256)
mcmc_sample_kernel(int m, int n, const double *__restrict__ cdf, uint2 key, int step, int tag,
                   int32_t *__restrict__ samples, int32_t *__restrict__ counts) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint4 x = draw(key, j, step, tag);
    const double target = uniform53(x.x, x.y) * cdf[n - 1];
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cdf[mid] > target) hi = mid; else lo = mid + 1;
    }
    samples[j] = lo;
    atomicAdd(&counts[lo], 1);
}

// ---- the relocation update ------------------------------------------------------------------------------------

// Rows drawn c > 0 times: r = min(c + 1, 51), alpha = -expm1(log1p(-o) / r),
// D = sum_{k=0}^{r-1} (-1)^k C(r, k+1) alpha^(k+1) / sqrt(k+1)  (the table's double sum over i, k summed over i:
// sum_{i=k+1}^{r} C(i-1, k) = C(r, k+1)), logit <- logit(clamp(alpha, min_opacity, 1 - 2^-23)),
// log-scales <- s + log(o / D); fp64, rounded once to fp32.  C(r, k+1) and every product on its way are integers
// below 2^53, so the binomials are exact.  With zero_moments, the row's Adam moments in every slice are zeroed.
__global__ void __launch_bounds__(256)
mcmc_relocate_kernel(int n, const int32_t *__restrict__ counts, float min_opacity, float *__restrict__ logits,
                     float *__restrict__ log_scales, int zero_moments, Segments seg, float *__restrict__ exp_avg,
                     float *__restrict__ exp_avg_sq) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = counts[i];
    if (c == 0) return;
    const int r = min(c + 1, RATIO_MAX);
    const double o = (double)sigmoid_f(logits[i]);
    const double alpha = -expm1(log1p(-o) / (double)r);
    double D = 0.0, ap = alpha, binom = (double)r;
    for (int k = 0; k < r; ++k) {
        const double t = binom * ap / sqrt((double)(k + 1));
        D += (k & 1) ? -t : t;
        ap *= alpha;
        binom = binom * (double)(r - k - 1) / (double)(k + 2);
    }
    const double a = fmin(fmax(alpha, (double)min_opacity), 1.0 - 0x1p-23);
    logits[i] = (float)(log(a) - log1p(-a));
    const double ds = log(o / D);
#pragma unroll
    for (int k = 0; k < 3; ++k) log_scales[3 * i + k] = (float)((double)log_scales[3 * i + k] + ds);
    if (zero_moments) {
        for (int s = 0; s < seg.num; ++s) {
            const long long o0 = seg.offset[s] + (long long)i * seg.row_floats[s];
            for (int e = 0; e < seg.row_floats[s]; ++e) {
                exp_avg[o0 + e] = 0.f;
                exp_avg_sq[o0 + e] = 0.f;
            }
        }
    }
}

// row dst[j] <- row src[j] in every slice (blockIdx.y = slice)
__global__ void __launch_bounds__(256)
mcmc_copy_rows_kernel(int m, const int32_t *__restrict__ dst_rows, const int32_t *__restrict__ src_rows, Segments seg,
                      float *__restrict__ param) {
    const int s = blockIdx.y, rf = seg.row_floats[s];
    const long long total = (long long)m * rf;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long j = e / rf;
        const int c = (int)(e - j * rf);
        param[seg.offset[s] + (long long)dst_rows[j] * rf + c] = param[seg.offset[s] + (long long)src_rows[j] * rf + c];
    }
}

// ---- per step: the regulariser gradient and the position noise ------------------------------------------------

__global__ void __launch_bounds__(256)
mcmc_regularize_kernel(int n, const float *__restrict__ logits, const float *__restrict__ log_scales,
                       float opacity_coef, float scale_coef, float *__restrict__ grad_logits,
                       float *__restrict__ grad_log_scales) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float o = sigmoid_f(logits[i]);
    grad_logits[i] += opacity_coef * (o * (1.f - o));
#pragma unroll
    for (int k = 0; k < 3; ++k) grad_log_scales[3 * i + k] += scale_coef * expf(log_scales[3 * i + k]);
}

// means += Sigma (z sigma_100(1 - o - 0.995) noise_scale), Sigma = R diag(exp(2 s)) R^T, R from q / |q|
__global__ void __launch_bounds__(256)
mcmc_noise_kernel(int n, const float *__restrict__ logits, const float *__restrict__ log_scales,
                  const float *__restrict__ quats, uint2 key, int step, float noise_scale, float *__restrict__ means) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float o = sigmoid_f(logits[i]);
    const float gate = 1.f / (1.f + expf(-100.f * ((1.f - o) - 0.995f)));
    const float cz = gate * noise_scale;
    const float3 z = normals3(draw(key, i, step, 0));
    const float v0 = z.x * cz, v1 = z.y * cz, v2 = z.z * cz;
    const float4 q = reinterpret_cast<const float4 *>(quats)[i];
    const float nrm = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float w = q.x / nrm, x = q.y / nrm, y = q.z / nrm, zq = q.w / nrm;
    const float R[3][3] = {{1.f - 2.f * (y * y + zq * zq), 2.f * (x * y - w * zq), 2.f * (x * zq + w * y)},
                           {2.f * (x * y + w * zq), 1.f - 2.f * (x * x + zq * zq), 2.f * (y * zq - w * x)},
                           {2.f * (x * zq - w * y), 2.f * (y * zq + w * x), 1.f - 2.f * (x * x + y * y)}};
    const float e[3] = {expf(2.f * log_scales[3 * i]), expf(2.f * log_scales[3 * i + 1]),
                        expf(2.f * log_scales[3 * i + 2])};
    // Sigma v = R (e * (R^T v))
    float t[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = e[k] * (R[0][k] * v0 + R[1][k] * v1 + R[2][k] * v2);
#pragma unroll
    for (int a = 0; a < 3; ++a) means[3 * i + a] += R[a][0] * t[0] + R[a][1] * t[1] + R[a][2] * t[2];
}

__global__ void __launch_bounds__(256)
mcmc_draws_kernel(int count, uint2 key, int step, int tag, uint32_t *__restrict__ words, float *__restrict__ normals) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const uint4 x = draw(key, j, step, tag);
    if (words) reinterpret_cast<uint4 *>(words)[j] = x;
    if (normals) {
        const float3 z = normals3(x);
        normals[3 * j] = z.x; normals[3 * j + 1] = z.y; normals[3 * j + 2] = z.z;
    }
}

int load_segments(int num_segments, const gsb_row_segment *segments, Segments &seg) {
    GSB_CHECK_ARG(num_segments >= 0 && num_segments <= GSB_MCMC_MAX_SEGMENTS);
    GSB_CHECK_ARG(num_segments == 0 || segments != nullptr);
    seg.num = num_segments;
    for (int s = 0; s < num_segments; ++s) {
        GSB_CHECK_ARG(segments[s].offset >= 0 && segments[s].row_floats > 0);
        seg.offset[s] = segments[s].offset;
        seg.row_floats[s] = segments[s].row_floats;
    }
    return 0;
}

constexpr int N_MAX = 1 << 29;      // growth appends sample | 3 << 30 to the gather row map

}  // namespace

extern "C" size_t gsb_mcmc_workspace_bytes(int n) {
    if (n < 0) return 0;
    const size_t nb = (size_t)gsb_div_up(n > 0 ? n : 1, MB);
    return 2 * gsb_align_up(nb * sizeof(double), 256) + 3 * gsb_align_up(nb * sizeof(int), 256);
}

extern "C" int gsb_mcmc_plan(int n, const float *logits, float min_opacity, int mask_dead, void *workspace,
                             size_t workspace_bytes, double *cdf, int32_t *dead, int32_t *result,
                             gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && n < N_MAX);
    GSB_CHECK_ARG(result != nullptr);
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        GSB_CUDA(cudaMemsetAsync(result, 0, 4 * sizeof(int32_t), st));
        return 0;
    }
    GSB_CHECK_ARG(logits && cdf && workspace && (!mask_dead || dead));
    GSB_CHECK_ARG(workspace_bytes >= gsb_mcmc_workspace_bytes(n) && ((uintptr_t)workspace % 256) == 0);
    const int nb = gsb_div_up(n, MB);
    uint8_t *w = static_cast<uint8_t *>(workspace);
    const size_t dbytes = gsb_align_up((size_t)nb * sizeof(double), 256), ibytes = gsb_align_up((size_t)nb * sizeof(int), 256);
    double *blk_sum = reinterpret_cast<double *>(w), *blk_pre = reinterpret_cast<double *>(w + dbytes);
    int *blk_dead = reinterpret_cast<int *>(w + 2 * dbytes), *blk_any = reinterpret_cast<int *>(w + 2 * dbytes + ibytes),
        *blk_dead_off = reinterpret_cast<int *>(w + 2 * dbytes + 2 * ibytes);
    mcmc_scan_local_kernel<<<nb, MT, 0, st>>>(n, logits, min_opacity, mask_dead, cdf, blk_sum, blk_dead, blk_any);
    GSB_LAUNCH_CHECK();
    mcmc_scan_blocks_kernel<<<1, 32, 0, st>>>(nb, blk_sum, blk_dead, blk_any, blk_pre, blk_dead_off, result);
    GSB_LAUNCH_CHECK();
    mcmc_scan_finish_kernel<<<nb, MT, 0, st>>>(n, logits, min_opacity, mask_dead, blk_pre, blk_dead_off, cdf, dead);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_sample(int num_samples, int n, const double *cdf, unsigned key0, unsigned key1, int step,
                               int tag, int32_t *samples, int32_t *counts, gsb_stream_t stream) {
    GSB_CHECK_ARG(num_samples >= 0 && n >= 0 && n < N_MAX);
    GSB_CHECK_ARG(num_samples == 0 || n > 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(cdf && counts && (num_samples == 0 || samples));
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CUDA(cudaMemsetAsync(counts, 0, (size_t)n * sizeof(int32_t), st));
    if (num_samples == 0) return 0;
    mcmc_sample_kernel<<<gsb_div_up(num_samples, 256), 256, 0, st>>>(num_samples, n, cdf, make_uint2(key0, key1), step,
                                                                     tag, samples, counts);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_relocate(int n, const int32_t *counts, float min_opacity, float *logits, float *log_scales,
                                 int zero_moments, int num_segments, const gsb_row_segment *segments, float *exp_avg,
                                 float *exp_avg_sq, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0 && n < N_MAX);
    Segments seg;
    if (int e = load_segments(num_segments, segments, seg)) return e;
    if (n == 0) return 0;
    GSB_CHECK_ARG(counts && logits && log_scales);
    GSB_CHECK_ARG(!zero_moments || (exp_avg && exp_avg_sq));
    mcmc_relocate_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, counts, min_opacity, logits, log_scales, zero_moments, seg, exp_avg, exp_avg_sq);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_copy_rows(int num_rows, const int32_t *dst_rows, const int32_t *src_rows, int num_segments,
                                  const gsb_row_segment *segments, float *param, gsb_stream_t stream) {
    GSB_CHECK_ARG(num_rows >= 0);
    Segments seg;
    if (int e = load_segments(num_segments, segments, seg)) return e;
    if (num_rows == 0 || num_segments == 0) return 0;
    GSB_CHECK_ARG(dst_rows && src_rows && param);
    int max_rf = 0;
    for (int s = 0; s < seg.num; ++s) max_rf = max(max_rf, seg.row_floats[s]);
    long long blocks = ((long long)num_rows * max_rf + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    mcmc_copy_rows_kernel<<<dim3((unsigned)blocks, (unsigned)seg.num), 256, 0, (cudaStream_t)stream>>>(
        num_rows, dst_rows, src_rows, seg, param);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_regularize(int n, const float *logits, const float *log_scales, float opacity_coef,
                                   float scale_coef, float *grad_logits, float *grad_log_scales, gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(logits && log_scales && grad_logits && grad_log_scales);
    mcmc_regularize_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, logits, log_scales, opacity_coef, scale_coef, grad_logits, grad_log_scales);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_add_noise(int n, const float *logits, const float *log_scales, const float *raw_quats,
                                  unsigned key0, unsigned key1, int step, float noise_scale, float *means,
                                  gsb_stream_t stream) {
    GSB_CHECK_ARG(n >= 0);
    if (n == 0) return 0;
    GSB_CHECK_ARG(logits && log_scales && raw_quats && means && ((uintptr_t)raw_quats % 16) == 0);
    mcmc_noise_kernel<<<gsb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(
        n, logits, log_scales, raw_quats, make_uint2(key0, key1), step, noise_scale, means);
    GSB_LAUNCH_CHECK();
    return 0;
}

extern "C" int gsb_mcmc_draws(int count, unsigned key0, unsigned key1, int step, int tag, int32_t *words,
                              float *normals, gsb_stream_t stream) {
    GSB_CHECK_ARG(count >= 0);
    if (count == 0) return 0;
    GSB_CHECK_ARG((words || normals) && ((uintptr_t)words % 16) == 0);
    mcmc_draws_kernel<<<gsb_div_up(count, 256), 256, 0, (cudaStream_t)stream>>>(
        count, make_uint2(key0, key1), step, tag, reinterpret_cast<uint32_t *>(words), normals);
    GSB_LAUNCH_CHECK();
    return 0;
}
