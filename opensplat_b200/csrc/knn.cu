// knn.cu -- the initial scales of Model's constructor (model.hpp:40): PointsTensor::scales (kdtree_tensor.cpp:4-22),
// the mean distance from every point of the input cloud to its 3 nearest neighbours, exactly, on the device.
//
//   d(i,j)       = ((dx*dx) + (dy*dy)) + (dz*dz),  dx = x_i - x_j in fp32, every operation rounded separately
//                  (nanoflann's L2_Simple_Adaptor::evalMetric; this file is built with --fmad=false and spells the
//                  roundings out with __f*_rn anyway)
//   d0<=d1<=d2<=d3 the four smallest d(i,j) over all j, i itself included
//   mean_dist[i] = ((sqrtf(d1) + sqrtf(d2)) + sqrtf(d3)) / 3.0f
// The result depends only on the sorted values, so it needs no tie-breaking: it is deterministic, and permuting the
// input permutes the output.
//
// Shape: bounding box -> 63-bit Morton keys (21 bits per axis) -> gsb_sort_intersects -> points gathered into key
// order -> leaves of 32 consecutive points with boxes of their member coordinates -> a complete binary tree of boxes
// over the leaves (heap layout, padded to a power of two with empty boxes) -> one thread per query in key order:
// seed the 4-best from the query's own leaf, then traverse nearest child first with the 4 best in registers, and
// scatter the result to input order.
//
// Two rules keep the pruning exact:
//   - a candidate enters only if strictly smaller than the current 4th value, and a box is pruned when its lower
//     bound is >= the current 4th value once 4 values are held: an equal value cannot change the sorted values, and
//     a group of k duplicate points then costs nothing extra;
//   - the box bound is formed with the distance's own roundings: per axis fl(q - face) with the face a member
//     coordinate, squared, summed x -> y -> z.  Rounding is monotone, so the bound never exceeds the rounded distance
//     of any member.
#include <algorithm>

#include "gsb_common.cuh"

namespace {

constexpr int KNN_LEAF = 32;
constexpr int KNN_STACK = 32;     // the tree has at most 2^26 leaves (n < 2^31): depth <= 26
constexpr int KNN_THREADS = 256;

// float <-> unsigned with the order of the floats (for atomicMin / atomicMax)
__device__ __forceinline__ unsigned f2ord(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// bbox[0..2] = ordered min, bbox[3..5] = ordered max (pre-set to 0xffffffff / 0 by the host)
__global__ void __launch_bounds__(KNN_THREADS)
knn_bbox_kernel(int n, const float *__restrict__ xyz, unsigned *__restrict__ bbox) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n; i += (size_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = xyz[3 * i + c];
            lo[c] = fminf(lo[c], v);
            hi[c] = fmaxf(hi[c], v);
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
            hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            atomicMin(bbox + c, f2ord(lo[c]));
            atomicMax(bbox + 3 + c, f2ord(hi[c]));
        }
    }
}

__device__ __forceinline__ unsigned long long spread21(unsigned v) {   // bit b of v -> bit 3b
    unsigned long long x = v & 0x1fffffu;
    x = (x | (x << 32)) & 0x1f00000000ffffull;
    x = (x | (x << 16)) & 0x1f0000ff0000ffull;
    x = (x | (x << 8)) & 0x100f00f00f00f00full;
    x = (x | (x << 4)) & 0x10c30c30c30c30c3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}

__device__ __forceinline__ unsigned quantize21(float v, float lo, float scale) {
    // NaN-safe clamp to [0, 2^21 - 1]; an axis of zero (or non-finite) extent has scale 0 and maps to 0
    const float q = fminf(fmaxf(__fmul_rn(__fsub_rn(v, lo), scale), 0.f), 2097151.f);
    return (unsigned)q;
}

__global__ void __launch_bounds__(KNN_THREADS)
knn_morton_kernel(int n, const float *__restrict__ xyz, const unsigned *__restrict__ bbox,
                  long long *__restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long key = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float lo = ord2f(bbox[c]), hi = ord2f(bbox[3 + c]);
        const float ext = __fsub_rn(hi, lo);
        const float scale = (ext > 0.f && ext < INFINITY) ? __fdiv_rn(2097152.f, ext) : 0.f;
        key |= spread21(quantize21(xyz[3 * (size_t)i + c], lo, scale)) << (2 - c);
    }
    keys[i] = (long long)key;
}

__global__ void __launch_bounds__(KNN_THREADS)
knn_gather_kernel(int n, const float *__restrict__ xyz, const int *__restrict__ order, float4 *__restrict__ pts) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const size_t i = (size_t)order[j];
    pts[j] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 0.f);
}

// node boxes in heap layout: root 1, children 2v / 2v+1, leaf l at num_pow2 + l.  Empty boxes are (+inf, -inf).
__global__ void __launch_bounds__(KNN_THREADS)
knn_leaf_boxes_kernel(int n, int num_leaves, int num_pow2, const float4 *__restrict__ pts, float4 *__restrict__ lo,
                      float4 *__restrict__ hi) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= num_pow2) return;
    float4 a = make_float4(INFINITY, INFINITY, INFINITY, 0.f), b = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    if (l < num_leaves) {
        const int end = min(n, (l + 1) * KNN_LEAF);
        for (int j = l * KNN_LEAF; j < end; ++j) {
            const float4 p = pts[j];
            a.x = fminf(a.x, p.x); a.y = fminf(a.y, p.y); a.z = fminf(a.z, p.z);
            b.x = fmaxf(b.x, p.x); b.y = fmaxf(b.y, p.y); b.z = fmaxf(b.z, p.z);
        }
    }
    lo[num_pow2 + l] = a;
    hi[num_pow2 + l] = b;
}

__device__ __forceinline__ void merge_node(int v, float4 *__restrict__ lo, float4 *__restrict__ hi) {
    const float4 a0 = lo[2 * v], a1 = lo[2 * v + 1], b0 = hi[2 * v], b1 = hi[2 * v + 1];
    lo[v] = make_float4(fminf(a0.x, a1.x), fminf(a0.y, a1.y), fminf(a0.z, a1.z), 0.f);
    hi[v] = make_float4(fmaxf(b0.x, b1.x), fmaxf(b0.y, b1.y), fmaxf(b0.z, b1.z), 0.f);
}

// one level of internal nodes [first, 2*first)
__global__ void __launch_bounds__(KNN_THREADS)
knn_level_kernel(int first, float4 *__restrict__ lo, float4 *__restrict__ hi) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < first) merge_node(first + t, lo, hi);
}

// the levels with at most KNN_THREADS nodes, in one CTA: nodes [1, top)
__global__ void __launch_bounds__(KNN_THREADS)
knn_top_levels_kernel(int top, float4 *__restrict__ lo, float4 *__restrict__ hi) {
    for (int first = top >> 1; first >= 1; first >>= 1) {
        if ((int)threadIdx.x < first) merge_node(first + threadIdx.x, lo, hi);
        __syncthreads();
    }
}

__device__ __forceinline__ float dist2(float qx, float qy, float qz, float4 p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// the gap to the nearer face of [l, h] along one axis, rounded as the distance's difference is
__device__ __forceinline__ float face_gap(float q, float l, float h) {
    return q < l ? __fsub_rn(q, l) : (q > h ? __fsub_rn(q, h) : 0.f);
}

__device__ __forceinline__ float box_bound(float qx, float qy, float qz, float4 l, float4 h) {
    const float gx = face_gap(qx, l.x, h.x), gy = face_gap(qy, l.y, h.y), gz = face_gap(qz, l.z, h.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz));
}

struct Best4 {
    float d0, d1, d2, d3;
    int held;
    // strictly smaller than the 4th (or a slot still empty)
    __device__ __forceinline__ void insert(float d) {
        if (!(d < d3) && held >= 4) return;
        held += held < 4;
        d3 = d;
        if (d3 < d2) { const float t = d2; d2 = d3; d3 = t; }
        if (d2 < d1) { const float t = d1; d1 = d2; d2 = t; }
        if (d1 < d0) { const float t = d0; d0 = d1; d1 = t; }
    }
    __device__ __forceinline__ bool prunes(float bound) const { return held >= 4 && bound >= d3; }
};

__device__ __forceinline__ void scan_leaf(int leaf, int n, const float4 *__restrict__ pts, float qx, float qy,
                                          float qz, Best4 &b) {
    const int begin = leaf * KNN_LEAF, end = min(n, begin + KNN_LEAF);
    for (int j = begin; j < end; ++j) b.insert(dist2(qx, qy, qz, pts[j]));
}

__global__ void __launch_bounds__(KNN_THREADS)
knn_query_kernel(int n, int num_leaves, int num_pow2, const float4 *__restrict__ pts, const int *__restrict__ order,
                 const float4 *__restrict__ lo, const float4 *__restrict__ hi, float *__restrict__ mean_dist) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const float4 q = pts[j];
    const int own = j / KNN_LEAF;
    Best4 b{INFINITY, INFINITY, INFINITY, INFINITY, 0};
    scan_leaf(own, n, pts, q.x, q.y, q.z, b);

    int stack_node[KNN_STACK];
    float stack_bound[KNN_STACK];
    int sp = 0;
    int v = 1;
    while (true) {
        if (v >= num_pow2) {
            const int leaf = v - num_pow2;
            if (leaf != own && leaf < num_leaves) scan_leaf(leaf, n, pts, q.x, q.y, q.z, b);
        } else {
            const int c = 2 * v;
            const float b0 = box_bound(q.x, q.y, q.z, lo[c], hi[c]);
            const float b1 = box_bound(q.x, q.y, q.z, lo[c + 1], hi[c + 1]);
            const bool first0 = b0 <= b1;
            const int near = first0 ? c : c + 1, far = first0 ? c + 1 : c;
            const float bn = first0 ? b0 : b1, bf = first0 ? b1 : b0;
            if (!b.prunes(bf)) {
                stack_node[sp] = far;
                stack_bound[sp] = bf;
                ++sp;
            }
            if (!b.prunes(bn)) {
                v = near;
                continue;
            }
        }
        // next stacked subtree that the current 4th value does not prune
        v = 0;
        while (sp > 0) {
            --sp;
            if (!b.prunes(stack_bound[sp])) {
                v = stack_node[sp];
                break;
            }
        }
        if (v == 0) break;
    }
    const float s = __fadd_rn(__fadd_rn(__fsqrt_rn(b.d1), __fsqrt_rn(b.d2)), __fsqrt_rn(b.d3));
    mean_dist[order[j]] = __fdiv_rn(s, 3.0f);
}

struct KnnLayout {   // workspace carve-up, all offsets 256-B aligned
    size_t bbox, keys, keys_sorted, pts, order, lo, hi, sort, total;
    int num_leaves, num_pow2;
};

KnnLayout knn_layout(int n) {
    KnnLayout L;
    const size_t m = (size_t)(n > 0 ? n : 1);
    L.num_leaves = (int)((m + KNN_LEAF - 1) / KNN_LEAF);
    L.num_pow2 = 1;
    while (L.num_pow2 < L.num_leaves) L.num_pow2 <<= 1;
    size_t o = 0;
    L.bbox = o; o += 256;
    // the points in key order (16 B each) reuse the two key arrays (8 B each), which the sort no longer needs
    L.keys = o; L.pts = o; o += gsb_align_up(m * 8, 256);
    L.keys_sorted = o; o += gsb_align_up(m * 8, 256);
    o = std::max(o, L.pts + gsb_align_up(m * 16, 256));
    L.order = o; o += gsb_align_up(m * 4, 256);
    L.lo = o; o += gsb_align_up((size_t)2 * L.num_pow2 * 16, 256);
    L.hi = o; o += gsb_align_up((size_t)2 * L.num_pow2 * 16, 256);
    L.sort = o; o += gsb_sort_workspace_bytes((int)m);
    L.total = o;
    return L;
}

}  // namespace

extern "C" size_t gsb_knn_workspace_bytes(int n) { return n > 0 ? knn_layout(n).total : 0; }

extern "C" int gsb_knn_mean_dist(int n, const float *xyz, float *mean_dist, void *workspace, size_t workspace_bytes,
                                 gsb_stream_t stream) {
    GSB_CHECK_ARG(n == 0 || n >= 4);
    if (n == 0) return 0;
    GSB_CHECK_ARG(xyz && mean_dist && workspace);
    GSB_CHECK_ARG(((uintptr_t)workspace % 256) == 0);
    const KnnLayout L = knn_layout(n);
    if (workspace_bytes < L.total) {
        gsb_set_error(GSB_ERR_WORKSPACE, "knn workspace too small", __FILE__, __LINE__);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    unsigned *bbox = (unsigned *)(ws + L.bbox);
    long long *keys = (long long *)(ws + L.keys), *keys_sorted = (long long *)(ws + L.keys_sorted);
    float4 *pts = (float4 *)(ws + L.pts), *lo = (float4 *)(ws + L.lo), *hi = (float4 *)(ws + L.hi);
    int *order = (int *)(ws + L.order);

    GSB_CUDA(cudaMemsetAsync(bbox, 0xff, 3 * sizeof(unsigned), s));
    GSB_CUDA(cudaMemsetAsync(bbox + 3, 0, 3 * sizeof(unsigned), s));
    knn_bbox_kernel<<<std::min(gsb_div_up(n, KNN_THREADS), 1024), KNN_THREADS, 0, s>>>(n, xyz, bbox);
    knn_morton_kernel<<<gsb_div_up(n, KNN_THREADS), KNN_THREADS, 0, s>>>(n, xyz, bbox, keys);
    GSB_LAUNCH_CHECK();
    // num_tiles = 2^31 - 1: the sort examines key bits [0, 32 + 31) = the 63 Morton bits
    const int rc = gsb_sort_intersects(n, 0x7fffffff, (const int64_t *)keys, (int64_t *)keys_sorted, order,
                                       ws + L.sort, workspace_bytes - L.sort, stream);
    if (rc != 0) return rc;
    knn_gather_kernel<<<gsb_div_up(n, KNN_THREADS), KNN_THREADS, 0, s>>>(n, xyz, order, pts);
    knn_leaf_boxes_kernel<<<gsb_div_up(L.num_pow2, KNN_THREADS), KNN_THREADS, 0, s>>>(n, L.num_leaves, L.num_pow2,
                                                                                      pts, lo, hi);
    int first = L.num_pow2 >> 1;
    for (; first > KNN_THREADS; first >>= 1)
        knn_level_kernel<<<gsb_div_up(first, KNN_THREADS), KNN_THREADS, 0, s>>>(first, lo, hi);
    if (first >= 1) knn_top_levels_kernel<<<1, KNN_THREADS, 0, s>>>(2 * first, lo, hi);
    knn_query_kernel<<<gsb_div_up(n, KNN_THREADS), KNN_THREADS, 0, s>>>(n, L.num_leaves, L.num_pow2, pts, order, lo,
                                                                        hi, mean_dist);
    GSB_LAUNCH_CHECK();
    return 0;
}
