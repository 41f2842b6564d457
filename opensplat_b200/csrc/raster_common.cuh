// raster_common.cuh -- record stream layout, per-warp TMA ring and tile/pixel mapping shared by the
// blend kernels (raster_fwd.cu, raster_bwd.cu).
#pragma once
#include "gsb_common.cuh"

// One depth-sorted intersection = 48 bytes = three 16-byte quads, contiguous per tile, so that a
// tile's whole list is ONE contiguous range that the blend kernels pull with 1-D TMA bulk copies.
//   q0 = { x, y, log2(opacity), bits(k) }  k = slot of this intersection in the UNSORTED
//                                          (Gaussian-major) order = cum_tiles_hit[g-1] + position in
//                                          g's tile bbox; indexes the backward pass' gradient rows
//   q1 = { a/2, b, c/2, hx }               conic with the 1/2 of sigma folded in
//   q2 = { r, g, b, hy }
// (hx, hy) are CONSERVATIVE half-extents, in pixels, of the region where this Gaussian can reach
// alpha >= 1/255, i.e. of the ellipse sigma <= smax, smax = ln(255*opacity):
//   hx = sqrt(2 smax c / (ac - b^2)), hy = sqrt(2 smax a / (ac - b^2))   (+ margin).
// They let a warp skip whole records / pixel-row pairs that cannot contribute.  Culling never changes
// results: the exact alpha < 1/255 test of the reference still decides every surviving pair.
struct __align__(16) GsbRecord {
    float4 q0, q1, q2;
};
static_assert(sizeof(GsbRecord) == 48, "record must be 48 bytes");

// Blend-kernel geometry: one WARP owns one 16x16 tile at a time (persistent warps pull tile ids from
// a global counter); lane l owns column (l & 15) and the 8 rows 2*j + (l >> 4), j = 0..7 ("slot" j =
// the two pixel rows 2j, 2j+1).  No block-level synchronisation anywhere in the blend loops.
constexpr int RK_WARPS = 4;            // warps per CTA
constexpr int RK_THREADS = RK_WARPS * 32;
constexpr int RK_PIX = 8;              // pixels per lane
constexpr int RK_CHUNK = 32;           // records per TMA bulk copy (1536 B) == one record per lane
constexpr int RK_STAGES = 4;           // ring depth per warp

constexpr float GSB_LN2 = 0.6931471805599453f;
constexpr float GSB_LOG2E = 1.4426950408889634f;
// smax = ln(255*opac) + 1e-3 = log2(opac)*ln2 + (ln 255 + 1e-3); the +1e-3 keeps the pre-test
// conservative w.r.t. the rounding of sigma and of ex2.approx
constexpr float GSB_SMAX_BIAS = 5.541263545158426f + 1e-3f;

// per-intersection gradient row written by the backward blend kernel (48 B, indexed by k).  With
// w = (unclamped alpha) * v_alpha and d = centre - pixel, summed over the tile's pixels:
//   { S0 = sum w, Sx = sum w dx, Sy = sum w dy, Sxx = sum w dx^2, Sxy = sum w dx dy, Syy = sum w dy^2,
//     R, G, B = sum alpha*T*v_out, Z, 0, 0 }
// with Z = sum alpha*T*v_depth in the DEPTH instantiation (the depth map's gradient w.r.t. the Gaussian's depth, D18)
// and unused otherwise.  The (linear) map to v_xy / v_conic / v_opacity is applied once per Gaussian by the row-reduce
// kernel.
constexpr int GSB_GRAD_ROW_FLOATS = 12;

// GSB_RASTER_CLAMP_MAX_ONE (gsplat_b200.h): the forward kernel's SAT instantiation marks the colour channels of a
// pixel it cut at 1 in these bits of final_idx; the backward kernel's SAT instantiation strips them again.
constexpr int GSB_SAT_BIT0 = 1 << 28;
constexpr int GSB_SAT_MASK = 7 << 28;

struct __align__(128) WarpRing {
    GsbRecord rec[RK_STAGES][RK_CHUNK];
    uint64_t full[RK_STAGES];
};

#ifdef __CUDACC__
// Builds the 48-B record of one intersection from the per-Gaussian attributes (see layout above).
__device__ __forceinline__ GsbRecord make_record(float2 xy, float a, float b, float c, float opac, float r,
                                                 float g, float bl, int k) {
    const float lo = (opac > 0.f) ? log2f(opac) : -INFINITY;
    // extent of {sigma <= smax}: conservative (x1.001 + 0.01 px); no culling for degenerate conics
    const float smax = fmaxf(0.f, fmaf(lo, GSB_LN2, GSB_SMAX_BIAS));
    const float det = a * c - b * b;
    float hx = INFINITY, hy = INFINITY;
    if (det > 0.f && a > 0.f && c > 0.f) {
        const float s2 = 2.f * smax / det;
        hx = sqrtf(s2 * c) * 1.001f + 0.01f;
        hy = sqrtf(s2 * a) * 1.001f + 0.01f;
    }
    GsbRecord rec;
    rec.q0 = make_float4(xy.x, xy.y, lo, __int_as_float(k));
    rec.q1 = make_float4(0.5f * a, b, 0.5f * c, hx);
    rec.q2 = make_float4(r, g, bl, hy);
    return rec;
}

// Slot mask of a Gaussian with centre (cx, cy) and extent half-widths (hx, hy) against the tile whose first
// pixel is (tile_x0, tile_y0): the 8-bit mask of slots (row pairs) whose rows intersect the y-extent, or 0 if
// the extent box misses the tile.  Only additions, comparisons and exact roundings -- no multiplications, so
// every kernel that evaluates it on the same floats takes the same decision (the tile binning's cull and
// the blend kernels' per-record test must agree).
__device__ __forceinline__ unsigned extent_slot_mask(float cx, float cy, float hx, float hy, float tile_x0,
                                                     float tile_y0) {
    const float gx = cx - tile_x0, gy = cy - tile_y0;   // centre in tile-local pixel coords
    // pixel centres of the tile are 0..15 in both axes: at least one integer column and row inside the extent
    const float xlo = fmaxf(ceilf(gx - hx), 0.f), xhi = fminf(floorf(gx + hx), 15.f);
    const float ylo = fmaxf(ceilf(gy - hy), 0.f), yhi = fminf(floorf(gy + hy), 15.f);
    if (!(xlo <= xhi) || !(ylo <= yhi)) return 0u;
    const int jlo = (int)ylo >> 1, jhi = (int)yhi >> 1;
    return ((2u << jhi) - 1u) & ~((1u << jlo) - 1u);
}

// Per-lane cull of record `lane` of a chunk against this warp's tile.
__device__ __forceinline__ unsigned record_slot_mask(const GsbRecord &r, float tile_x0, float tile_y0) {
    return extent_slot_mask(r.q0.x, r.q0.y, r.q1.w, r.q2.w, tile_x0, tile_y0);
}
#endif
