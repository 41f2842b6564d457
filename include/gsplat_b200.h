/*
 * gsplat_b200.h -- C ABI of libgsplat_b200.so: the sm_90a (NVIDIA H100) implementation of the
 * differentiable Gaussian-splat render path that sits behind OpenSplat's libtorch autograd
 * operators ProjectGaussians / RasterizeGaussians / SphericalHarmonics.
 *
 * This is the drop-in boundary: every entry point replaces one `*_tensor` binding of the
 * reference's CUDA back end (rasterizer/gsplat/bindings.h, cited per function as file:line under
 * /root/reference) or one ATen call the reference operator makes between them
 * (rasterize_gaussians.cpp:25-32,62-63).  Plain pointers and sizes only -- no torch types.
 *
 * Conventions
 *  - All pointers are DEVICE pointers unless said otherwise; fp32 / int32 / int64, dense row-major.
 *  - The caller owns all memory (inputs, outputs, workspaces); the library never allocates or
 *    frees device memory and keeps no mutable global state.  Workspace sizes come from the
 *    `*_bytes` queries.  Outputs are fully written by the call (no pre-zeroing required) unless
 *    noted.
 *  - Every call is asynchronous on `stream` (a cudaStream_t passed as void*); no call
 *    synchronises the device.  Entry points are re-entrant and thread-safe (distinct streams /
 *    devices may be driven concurrently); the current CUDA device of the calling thread is used.
 *  - Return value: 0 on success, otherwise a cudaError_t (>0) or GSB_ERR_* (<0).  A description of
 *    the last error on the calling thread is available from gsb_last_error().
 *  - Tile size is fixed at 16x16 (rasterizer/gsplat/config.h:1-2; it leaks into the callers,
 *    model.cpp:144, simple_trainer.cpp:91).  tiles_x = ceil(W/16), tiles_y = ceil(H/16).
 *  - Quaternions are stored (w,x,y,z) (helpers.cuh:145-153); viewmat/projmat are row-major 4x4.
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_TILE 16
#define GSB_ERR_INVALID_ARG (-1)
#define GSB_ERR_WORKSPACE (-2)
#define GSB_ERR_UNSUPPORTED (-3)
/* flags of gsb_rasterize_forward_packed / gsb_rasterize_backward */
#define GSB_RASTER_CLAMP_MAX_ONE 1u
/* or-ed into the `cull` argument of gsb_bucket_tile_ranges: report the visible count in stats[3] */
#define GSB_BIN_COUNT_VISIBLE 2

typedef void *gsb_stream_t; /* cudaStream_t */

/* ABI version (major*100 + minor) and last error text for the calling thread. */
int gsb_version(void);
const char *gsb_last_error(void);

/* ---- Spherical harmonics ---------------------------------------------------------------------
 * gsb_sh_forward  replaces compute_sh_forward_tensor  (bindings.h:26-32, bindings.cu:68-92,
 *                 kernel sh.cuh:218-238).   viewdirs [n,3], coeffs [n,K,3] with
 *                 K = (degree+1)^2, degree in 0..4; colors [n,3].  viewdirs are normalised inside
 *                 (sh.cuh:67-72).  degrees_to_use <= degree.
 * gsb_sh_backward replaces compute_sh_backward_tensor (bindings.h:34-40, bindings.cu:94-124,
 *                 kernel sh.cuh:240-260).   v_coeffs [n,K,3] is fully written (bases above
 *                 degrees_to_use get 0, as the reference's torch::zeros).  No gradient w.r.t.
 *                 viewdirs (spherical_harmonics.cpp:57-61). */
int gsb_sh_forward(int n, int degree, int degrees_to_use, const float *viewdirs, const float *coeffs,
                   float *colors, gsb_stream_t stream);
int gsb_sh_backward(int n, int degree, int degrees_to_use, const float *viewdirs, const float *v_colors,
                    float *v_coeffs, gsb_stream_t stream);

/* Fused variants (optional, SURVEY.md 8f row 1): rgbs = clamp_min(SH(coeffs) + bias, 0) in one pass -- the
 * glue of model.cpp:188-192 -- and its VJP v_coeffs = Y (x) (v_rgbs * [rgbs > 0]). */
int gsb_sh_forward_rgb(int n, int degree, int degrees_to_use, const float *viewdirs, const float *coeffs,
                       float bias, float *rgbs, gsb_stream_t stream);
int gsb_sh_backward_rgb(int n, int degree, int degrees_to_use, const float *viewdirs, const float *rgbs,
                        const float *v_rgbs, float *v_coeffs, gsb_stream_t stream);

/* Split variants (SURVEY.md 8f row 1): the whole colour pass of Model::forward without its ATen glue --
 * viewdirs = means - cam_pos (cam_pos: device float[3]; normalised inside, no gradient, model.cpp:176-177),
 * coeffs = cat(features_dc [n,3], features_rest [n,K-1,3]) (model.cpp:186-188) read where they lie,
 * rgbs = clamp_min(SH + bias, 0) (:192); the backward writes v_features_dc / v_features_rest directly (bases above
 * degrees_to_use get 0).  features_rest / v_features_rest may be NULL at degree 0. */
int gsb_sh_forward_split(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                         const float *features_dc, const float *features_rest, float bias, float *rgbs,
                         gsb_stream_t stream);
int gsb_sh_backward_split(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                          const float *rgbs, const float *v_rgbs, float *v_features_dc, float *v_features_rest,
                          gsb_stream_t stream);
/* Camera variants: the split variants' view directions (viewdirs = means - cam_pos, cam_pos a device float[3],
 * normalised inside, no gradient) on a merged coeffs / v_coeffs [n,K,3] block, as the flat parameter layout stores
 * it.  rgbs = clamp_min(SH + bias, 0); the backward masks v_rgbs with [rgbs > 0] and fully writes v_coeffs (bases above
 * degrees_to_use get 0).  rgbs and the coefficient gradients are bit-identical to the split variants' on the same
 * data. */
int gsb_sh_forward_rgb_cam(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                           const float *coeffs, float bias, float *rgbs, gsb_stream_t stream);
int gsb_sh_backward_rgb_cam(int n, int degree, int degrees_to_use, const float *means, const float *cam_pos,
                            const float *rgbs, const float *v_rgbs, float *v_coeffs, gsb_stream_t stream);
/* Several camera views at once (a trainer's B views of one step): gsb_sh_forward_rgb_cam for every centre of
 * cam_positions (device [num_views,3]) into rgbs (device [num_views,n,3], view v at rgbs + 3*n*v).  The coefficient
 * block is read once for all views; every view's rgbs are bit-identical to a gsb_sh_forward_rgb_cam call with its
 * centre.  num_views >= 1. */
int gsb_sh_forward_rgb_cam_multiview(int n, int degree, int degrees_to_use, const float *means, int num_views,
                                     const float *cam_positions, const float *coeffs, float bias, float *rgbs,
                                     gsb_stream_t stream);

/* Data-parallel training (SURVEY.md 8e): SH VJP fused with the cross-GPU gradient exchange.
 * gsb_mask_rgb_grad: v_rgbs *= [rgbs > 0] in place (gradient of the clamp, done before exposing v_rgbs).
 * gsb_sh_backward_multiview: v_coeffs[g] = scale * sum_r Y(normalize(means[g] - cam_positions[r])) (x)
 *   v_rgbs_per_view[r][g], r < num_views.  v_rgbs_per_view is a DEVICE array of num_views device pointers
 *   ([n,3] each); entries may be peer-mapped pointers of other GPUs (CUDA IPC / symmetric memory): the
 *   kernel reads them over NVLink while it computes, replacing "sh_backward + all-reduce of 12K B/Gaussian"
 *   by an exchange of 12 B/Gaussian/view.  cam_positions is a device [num_views,3] array. */
int gsb_mask_rgb_grad(int n, const float *rgbs, float *v_rgbs, gsb_stream_t stream);
int gsb_sh_backward_multiview(int n, int degree, int degrees_to_use, const float *means, int num_views,
                              const float *cam_positions, const float *const *v_rgbs_per_view, float scale,
                              float *v_coeffs, gsb_stream_t stream);
/* gsb_exchange_gradients: the whole data-parallel exchange step as ONE launch -- gsb_sh_backward_multiview plus
 *   a two-shot all-reduce (x scale) of the remaining per-Gaussian gradients, the first geom_floats floats
 *   (multiple of 4, 16-byte aligned) of every rank's flat gradient buffer: rank r owns slice r; with NVSwitch
 *   multicast (geom_multicast = the multicast mapping of that buffer) it is one multimem.ld_reduce + one
 *   multimem.st per 16 bytes, otherwise (geom_multicast NULL) the slice is summed from and written to the
 *   peer-mapped pointers geom_per_rank[0..world) (device array; world <= 16).  The caller provides the two
 *   cross-rank barriers around the launch (all inputs written / all results visible).  Replaces the single
 *   ncclAllReduce of the flat gradient buffer the data-parallel path would otherwise need (SURVEY.md 8e). */
int gsb_exchange_gradients(int n, int degree, int degrees_to_use, const float *means, int num_views,
                           const float *cam_positions, const float *const *v_rgbs_per_view, float scale,
                           float *v_coeffs, int rank, int world, long long geom_floats,
                           float *const *geom_per_rank, float *geom_multicast, gsb_stream_t stream);
/* Per-step camera centres: gsb_sh_backward_multiview / gsb_exchange_gradients with view r's centre read from
 *   cam_pos_per_view[r] instead of cam_positions[r].  cam_pos_per_view is a DEVICE array of num_views device pointers
 *   to 3 floats each; like v_rgbs_per_view, entries may be peer-mapped, so a data-parallel trainer whose ranks render
 *   a different camera every step exposes each step's centre next to its colour gradient (written before the
 *   caller's first barrier) instead of gathering the centres with a collective.  Same arguments, checks and results
 *   otherwise: given the same centres the coefficient gradients are bit-identical to the two entry points above. */
int gsb_sh_backward_multiview_cams(int n, int degree, int degrees_to_use, const float *means, int num_views,
                                   const float *const *cam_pos_per_view, const float *const *v_rgbs_per_view,
                                   float scale, float *v_coeffs, gsb_stream_t stream);
int gsb_exchange_gradients_cams(int n, int degree, int degrees_to_use, const float *means, int num_views,
                                const float *const *cam_pos_per_view, const float *const *v_rgbs_per_view,
                                float scale, float *v_coeffs, int rank, int world, long long geom_floats,
                                float *const *geom_per_rank, float *geom_multicast, gsb_stream_t stream);

/* ---- Projection ------------------------------------------------------------------------------
 * gsb_project_forward replaces project_gaussians_forward_tensor (bindings.h:42-65,
 *   bindings.cu:133-207, kernel forward.cu:19-103).  Outputs cov3d [n,6], xys [n,2], depths [n]
 *   (view-space z), radii [n] i32 (0 == culled), conics [n,3], num_tiles_hit [n] i32; all fully
 *   written (culled Gaussians get zeros, like the reference's torch::zeros).
 * gsb_project_backward replaces project_gaussians_backward_tensor (bindings.h:67-92,
 *   bindings.cu:209-277, kernel backward.cu:357-421).  v_depth may be NULL (== zeros).  cov3d is
 *   accepted for signature parity and may be NULL (recomputed in registers).  Writes v_mean3d [n,3],
 *   v_scale [n,3], v_quat [n,4] (zeros where radii <= 0).  Computes the exact VJP of the forward
 *   map (see DESIGN.md "gradient conventions"). */
int gsb_project_forward(int n, const float *means3d, const float *scales, float glob_scale,
                        const float *quats, const float *viewmat, const float *projmat, float fx, float fy,
                        float cx, float cy, int img_h, int img_w, int tiles_x, int tiles_y,
                        float clip_thresh, float *cov3d, float *xys, float *depths, int32_t *radii,
                        float *conics, int32_t *num_tiles_hit, gsb_stream_t stream);
int gsb_project_backward(int n, const float *means3d, const float *scales, float glob_scale,
                         const float *quats, const float *viewmat, const float *projmat, float fx, float fy,
                         float cx, float cy, int img_h, int img_w, const float *cov3d,
                         const int32_t *radii, const float *conics, const float *v_xy,
                         const float *v_depth, const float *v_conic, float *v_mean3d, float *v_scale,
                         float *v_quat, gsb_stream_t stream);
/* gsb_project_forward_activated / gsb_project_backward_activated: the same two kernels with the parameter
 *   activations of Model::forward as their prologue / epilogue (model.cpp:148-150 `exp(scales)`,
 *   `quats / quats.norm()`; model.cpp:200 `sigmoid(opacities)`) -- SURVEY.md 8f row 1.  Inputs are the RAW
 *   parameters: log_scales [n,3], raw_quats [n,4] (the projection normalises the quaternion itself, as the
 *   reference's quat_to_rotmat does, so the separate normalisation pass is simply dropped), opacity_logits [n].
 *   Forward also writes opacities [n] = sigmoid(logits) for the rasterizer.  Backward takes that `opacities`
 *   array and the rasterizer's v_opacity [n] (NULL == zeros) and returns gradients w.r.t. the raw parameters:
 *   v_log_scales = v_scale * exp(log_scale), v_raw_quats, v_opacity_logits = v_opacity * o * (1 - o). */
int gsb_project_forward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                  const float *raw_quats, const float *opacity_logits, const float *viewmat,
                                  const float *projmat, float fx, float fy, float cx, float cy, int img_h,
                                  int img_w, int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                  float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                  float *opacities, gsb_stream_t stream);
int gsb_project_backward_activated(int n, const float *means3d, const float *log_scales, float glob_scale,
                                   const float *raw_quats, const float *opacities, const float *viewmat,
                                   const float *projmat, float fx, float fy, int img_h, int img_w,
                                   const int32_t *radii, const float *conics, const float *v_xy,
                                   const float *v_depth, const float *v_conic, const float *v_opacity,
                                   float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                   float *v_opacity_logits, gsb_stream_t stream);
/* gsb_project_backward_activated_acc: the same arguments and VJP, ADDED into v_mean3d, v_log_scales, v_raw_quats
 *   and v_opacity_logits (out = out + vjp, one rounding per element; the outputs must hold valid floats) -- the sum of
 *   the geometry gradients over a trainer's views of one step, in view order, without a separate add pass. */
int gsb_project_backward_activated_acc(int n, const float *means3d, const float *log_scales, float glob_scale,
                                       const float *raw_quats, const float *opacities, const float *viewmat,
                                       const float *projmat, float fx, float fy, int img_h, int img_w,
                                       const int32_t *radii, const float *conics, const float *v_xy,
                                       const float *v_depth, const float *v_conic, const float *v_opacity,
                                       float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                       float *v_opacity_logits, gsb_stream_t stream);
/* gsb_project_forward_activated_aa: gsb_project_forward_activated with the anti-aliased opacity (DESIGN D19, the
 *   "antialiased" mode of gsplat / Mip-Splatting's 2-D filter): opacities [n] = sigmoid(logits) * comp, comp =
 *   sqrt(max(0, det0 / det)) where radii > 0 and 0 elsewhere; det0 = cxx0 cyy0 - cxy^2 is the determinant of the
 *   screen covariance before the 0.3 px^2 blur, det the one after it.  Every other output is bit-identical to
 *   gsb_project_forward_activated's, so binning and blending are unchanged.
 * gsb_project_backward_activated_aa / _aa_acc: its exact VJP, written / added like gsb_project_backward_activated /
 *   _acc, with the same arguments except that they take the opacity LOGITS (opacity_logits [n]) where those take the
 *   saved opacities.  v_opacity (NULL == zeros) reaches the logits as v_opacity * comp * o (1 - o) and, where comp > 0,
 *   the geometry through comp. */
int gsb_project_forward_activated_aa(int n, const float *means3d, const float *log_scales, float glob_scale,
                                     const float *raw_quats, const float *opacity_logits, const float *viewmat,
                                     const float *projmat, float fx, float fy, float cx, float cy, int img_h,
                                     int img_w, int tiles_x, int tiles_y, float clip_thresh, float *cov3d, float *xys,
                                     float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                     float *opacities, gsb_stream_t stream);
int gsb_project_backward_activated_aa(int n, const float *means3d, const float *log_scales, float glob_scale,
                                      const float *raw_quats, const float *opacity_logits, const float *viewmat,
                                      const float *projmat, float fx, float fy, int img_h, int img_w,
                                      const int32_t *radii, const float *conics, const float *v_xy,
                                      const float *v_depth, const float *v_conic, const float *v_opacity,
                                      float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                      float *v_opacity_logits, gsb_stream_t stream);
int gsb_project_backward_activated_aa_acc(int n, const float *means3d, const float *log_scales, float glob_scale,
                                          const float *raw_quats, const float *opacity_logits, const float *viewmat,
                                          const float *projmat, float fx, float fy, int img_h, int img_w,
                                          const int32_t *radii, const float *conics, const float *v_xy,
                                          const float *v_depth, const float *v_conic, const float *v_opacity,
                                          float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                          float *v_opacity_logits, gsb_stream_t stream);

/* ---- Tile binning ----------------------------------------------------------------------------
 * gsb_cumsum_tiles_hit replaces torch::cumsum(numTilesHit, 0, kInt32) (rasterize_gaussians.cpp:62).
 *   Inclusive scan; the caller reads M = cum_tiles_hit[n-1] back (rasterize_gaussians.cpp:63).
 *   In place when cum_tiles_hit == num_tiles_hit.  The workspace (gsb_cumsum_workspace_bytes(n)
 *   bytes) must be 256-byte aligned; it is zeroed by the call.
 * gsb_map_gaussian_to_intersects replaces map_gaussian_to_intersects_tensor (bindings.h:95-103,
 *   bindings.cu:279-318, kernel forward.cu:107-143): isect_ids [m] i64 = (tile_id << 32) | depth bits,
 *   gaussian_ids [m] i32.
 * gsb_sort_intersects replaces torch::sort(isectIds) (rasterize_gaussians.cpp:25-29): STABLE
 *   ascending sort; writes sorted keys and the permutation (int32 instead of torch's int64).
 *   Only bits [0, 32 + ceil(log2(num_tiles))) of the keys are examined.
 * gsb_gather_bin_edges replaces torch::gather(gaussianIds, 0, sortedIndices)
 *   (rasterize_gaussians.cpp:32) + get_tile_bin_edges_tensor (bindings.h:105-108,
 *   bindings.cu:320-336, kernel forward.cu:148-169).  tile_bins is [num_tiles,2] i32 (x = first,
 *   y = last+1; empty tiles (0,0)), fully written. */
size_t gsb_cumsum_workspace_bytes(int n);
int gsb_cumsum_tiles_hit(int n, const int32_t *num_tiles_hit, int32_t *cum_tiles_hit, void *workspace,
                         size_t workspace_bytes, gsb_stream_t stream);
int gsb_map_gaussian_to_intersects(int n, int m, const float *xys, const float *depths,
                                   const int32_t *radii, const int32_t *cum_tiles_hit, int tiles_x,
                                   int tiles_y, int64_t *isect_ids, int32_t *gaussian_ids,
                                   gsb_stream_t stream);
size_t gsb_sort_workspace_bytes(int m);
int gsb_sort_intersects(int m, int num_tiles, const int64_t *isect_ids, int64_t *isect_ids_sorted,
                        int32_t *sorted_index, void *workspace, size_t workspace_bytes,
                        gsb_stream_t stream);
int gsb_gather_bin_edges(int m, int num_tiles, const int64_t *isect_ids_sorted,
                         const int32_t *sorted_index, const int32_t *gaussian_ids,
                         int32_t *gaussian_ids_sorted, int32_t *tile_bins, gsb_stream_t stream);

/* ---- Tile binning, fast path: two-level bucket sort fused with record packing ------------------
 * What RasterizeGaussians::forward needs between rasterize_gaussians.cpp:62 and :79 (cumsum, the M read-back,
 * emit, global sort, gather, bin edges, and gsb_pack_records) without a global sort and without a host read-back in
 * the middle of the frame.
 * cull = 0: tile_bins, cum_tiles_hit and the per-tile order (tile, then depth bits, ties by ascending unsorted
 *   slot) are bit-identical to gsb_cumsum_tiles_hit + gsb_map_gaussian_to_intersects + gsb_sort_intersects +
 *   gsb_gather_bin_edges.
 * cull = 1 (what the operator uses): a (Gaussian, tile) pair is binned only if the Gaussian's extent box
 *   {pixels where opacity * exp(-sigma) can reach 1/255} touches the tile -- exactly the test the blend kernels
 *   apply per record, so no pixel or gradient changes; M, tile_bins and cum_tiles_hit then describe the culled
 *   lists (internal to the operator: the reference's RasterizeGaussians does not return them).
 * Capacities: the caller sizes `workspace` (gsb_bucket_workspace_bytes(n, m_capacity, tiles)), `records`
 *   (gsb_raster_records_bytes(m_capacity)) and the sort's shared memory (len_capacity <= gsb_bucket_max_tile_len())
 *   from earlier frames; stats (device int32[4]) = {M, longest tile list, overflow, visible} with overflow = 1 iff
 *   M > m_capacity or longest > len_capacity.  visible is 0 unless gsb_bucket_tile_ranges gets
 *   cull | GSB_BIN_COUNT_VISIBLE; then it is the number of Gaussians with radii > 0 (counted from radii, not from the
 *   lists: with the cull a visible Gaussian may sit in no tile list; visible == 0 is the `radii.sum() == 0` test of
 *   model.cpp:173, here answered by the frame's one read-back).  On overflow gsb_bucket_sort_pack and
 *   gsb_rasterize_forward_packed (given the same stats pointer) do nothing: the host reads stats back AFTER
 *   enqueuing the whole forward pass and, on overflow, repeats the three calls with larger capacities.
 *   Exact-size use: m_capacity = M, len_capacity = longest list of a previous gsb_bucket_tile_ranges call.
 * gsb_bucket_tile_ranges: builds the per-Gaussian attribute records (in the workspace), counts and scans:
 *   cum_tiles_hit [n] (inclusive scan of the per-Gaussian binned-tile counts = the gradient-row slots of
 *   gsb_rasterize_backward), tile_bins [tiles,2] (empty tiles (0,0)), stats.
 * gsb_bucket_sort_pack: fills `records`; optional outputs sorted_index [M] / gaussian_ids_sorted [M] (NULL to
 *   skip).  Returns GSB_ERR_UNSUPPORTED if len_capacity > gsb_bucket_max_tile_len() -- take the generic path.
 * tile_order (optional, [tiles] int32): the longest-first tile order the blend calls take (see Rasterization). */
int gsb_bucket_max_tile_len(void);
size_t gsb_bucket_workspace_bytes(int n, int m_capacity, int num_tiles);
int gsb_bucket_tile_ranges(int n, const float *xys, const int32_t *radii, const float *conics, const float *colors,
                           const float *opacities, int cull, int tiles_x, int tiles_y, int m_capacity,
                           int len_capacity, void *workspace, size_t workspace_bytes, int32_t *cum_tiles_hit,
                           int32_t *tile_bins, int32_t *tile_order, int32_t *stats, gsb_stream_t stream);
int gsb_bucket_sort_pack(int n, int m_capacity, int len_capacity, const float *depths, const int32_t *radii,
                         const int32_t *cum_tiles_hit, int cull, int tiles_x, int tiles_y, const int32_t *tile_bins,
                         const int32_t *stats, void *workspace, size_t workspace_bytes, void *records,
                         int32_t *sorted_index, int32_t *gaussian_ids_sorted, gsb_stream_t stream);

/* ---- Rasterization ---------------------------------------------------------------------------
 * rasterize_forward_tensor (bindings.h:110-125, bindings.cu:338-410, kernel forward.cu:256-378) is gsb_pack_records
 * followed by gsb_rasterize_forward_packed; rasterize_backward_tensor (bindings.h:174-189, bindings.cu:569-632,
 * kernel backward.cu:161-355) is gsb_rasterize_backward.
 * gsb_raster_records_bytes: size of the `records` buffer for m intersections: the depth-sorted 48-B
 *   per-intersection records the blend kernels pull with TMA bulk copies, plus 256 B of scratch behind them that
 *   every blend call rewrites (hence `records` is non-const in the backward too).
 * gsb_raster_grad_rows_bytes: size of the backward's scratch buffer grad_rows for m intersections.
 * gsb_pack_records: fills `records` from a sorted intersection list.  Inputs as the reference's
 *   rasterize_forward_tensor (gaussian_ids_sorted [m], xys [n,2], conics [n,3], colors [n,3], opacities [n]) plus
 *   sorted_index [m] (the permutation from gsb_sort_intersects: sorted position -> unsorted intersection slot).
 *   gsb_bucket_sort_pack writes the same records on the fast path.
 * gsb_rasterize_forward_packed: the blend kernel on a packed record stream; m = the count `records` was sized with
 *   (the m_capacity on the fast path).  tile_bins [tiles,2], background [3]; writes out_img [H,W,3], final_Ts [H,W]
 *   and final_idx [H,W] i32 completely.  Keep `records` for the backward pass.
 * gsb_rasterize_forward_count: diagnostic twin of gsb_rasterize_forward_packed (same outputs, no tile order, no
 *   flags) that also ACCUMULATES into pair_counts (device uint64[4]; zero it first) {records that pass the
 *   per-record extent test, slot visits (x 32 lanes = pixel tests), pixel pairs evaluated (sigma inside the extent:
 *   one ex2), pixel pairs blended} -- the work units SURVEY.md 8(d) asks the blend kernels' throughput to be quoted
 *   in.  Never on a timed path.
 * gsb_rasterize_backward: consumes `records`, tile_bins, tile_order, final_Ts and final_idx of the forward call,
 *   conics [n,3] and opacities [n] (as the reference's signature), cum_tiles_hit [n] (the scan the records were
 *   binned with) and grad_rows.  v_output [H,W,3]; v_output_alpha [H,W] may be NULL (== zeros,
 *   rasterize_gaussians.cpp:108).  Writes v_xy [n,2], v_conic [n,3], v_colors [n,3], v_opacity [n] completely (no
 *   atomics, bit-reproducible run to run).
 * tile_order (optional, NULL = tile id order; [tiles] int32): a permutation of the tile ids, longest list first,
 *   written by gsb_bucket_tile_ranges: the persistent blend warps take tiles in that order, so the tiles still
 *   running when the kernel drains are the cheapest ones.  No result depends on it (tiles are independent).
 * bin_stats (optional): the stats of gsb_bucket_tile_ranges; if they flag an overflow, the forward does nothing.
 * flags: 0 or GSB_RASTER_CLAMP_MAX_ONE, which fuses the caller's `rgb = clamp_max(rgb, 1)` (model.cpp:222) into the
 *   blend epilogue: out_img is written clamped, the channels that were cut are remembered in bits 28..30 of
 *   final_idx (so m must stay below 2^28 and final_idx is private to the pair of calls), and the backward -- given
 *   the same flag and the gradient of the CLAMPED image -- passes no gradient through them (torch's clamp_max mask
 *   `x <= max`).
 * Depth and opacity maps (DESIGN D18): the blend's decisions are those of the colour blend; per pixel
 *   out_depth = sum alpha T z over the blended pairs (z = the projection's view-space depth of the pair's Gaussian,
 *   background depth 0, not normalised) and out_alpha = 1 - final_Ts.  Neither is ever clamped.
 * gsb_gather_record_depths: record_depths [m] = depths[gaussian_ids_sorted[j]], the per-record depth stream in sorted
 *   order.  m = the size of the id list (the m_capacity on the fast path, where gsb_bucket_sort_pack writes
 *   gaussian_ids_sorted); given the binning stats it reads M from them on the device, writes only j < M, and writes
 *   nothing after an overflow.  bin_stats may be NULL (generic path: all m ids are valid).
 * gsb_rasterize_forward_packed_depth: gsb_rasterize_forward_packed plus record_depths [m] (may be NULL if m == 0),
 *   out_depth [H,W] and out_alpha [H,W], written completely.  out_img, final_Ts and final_idx are bit-identical to
 *   gsb_rasterize_forward_packed's.
 * gsb_rasterize_backward_depth: gsb_rasterize_backward plus record_depths, v_output_depth [H,W] (NULL == zeros) and
 *   v_depths [n], written completely.  v_output_alpha is the cotangent of out_alpha.  Give it the records, final_Ts
 *   and final_idx of gsb_rasterize_forward_packed_depth (or of gsb_rasterize_forward_packed: they are the same).
 * gsb_rasterize_backward_absgrad (DESIGN D25): the arguments of gsb_rasterize_backward_depth plus v_xy_abs [n,2]
 *   (non-NULL, 8-byte aligned), written completely: per Gaussian the sum over its blended pixels of the absolute value
 *   of each pixel's contribution to v_xy, component by component (AbsGS's absolute screen-space gradient, which
 *   does not cancel across the Gaussian's centre as v_xy does).  Depth is on iff v_depths != NULL: then
 *   record_depths and v_output_depth follow gsb_rasterize_backward_depth's rules, otherwise both must be NULL.  The
 *   other outputs are bit-identical to those of gsb_rasterize_backward (without depth) or
 *   gsb_rasterize_backward_depth (with depth); v_xy_abs is bit-reproducible run to run (no atomics).  Allocates
 *   nothing. */
size_t gsb_raster_records_bytes(int m);
size_t gsb_raster_grad_rows_bytes(int m);
int gsb_pack_records(int m, const int32_t *gaussian_ids_sorted, const int32_t *sorted_index, const float *xys,
                     const float *conics, const float *colors, const float *opacities, void *records,
                     gsb_stream_t stream);
int gsb_rasterize_forward_packed(int img_h, int img_w, int tiles_x, int tiles_y, int m, const int32_t *tile_bins,
                                 const int32_t *tile_order, const int32_t *bin_stats, const float *background,
                                 void *records, float *out_img, float *final_Ts, int32_t *final_idx,
                                 unsigned flags, gsb_stream_t stream);
int gsb_rasterize_forward_count(int img_h, int img_w, int tiles_x, int tiles_y, int m, const int32_t *tile_bins,
                                const float *background, void *records, float *out_img, float *final_Ts,
                                int32_t *final_idx, unsigned long long *pair_counts, gsb_stream_t stream);
int gsb_rasterize_backward(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m, const int32_t *tile_bins,
                           const int32_t *tile_order, const float *conics, const float *opacities, void *records,
                           const int32_t *cum_tiles_hit, const float *background, const float *final_Ts,
                           const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                           void *grad_rows, float *v_xy, float *v_conic, float *v_colors, float *v_opacity,
                           unsigned flags, gsb_stream_t stream);
int gsb_gather_record_depths(int m, const int32_t *gaussian_ids_sorted, const float *depths, const int32_t *bin_stats,
                             float *record_depths, gsb_stream_t stream);
int gsb_rasterize_forward_packed_depth(int img_h, int img_w, int tiles_x, int tiles_y, int m, const int32_t *tile_bins,
                                       const int32_t *tile_order, const int32_t *bin_stats, const float *background,
                                       void *records, float *out_img, float *final_Ts, int32_t *final_idx,
                                       unsigned flags, const float *record_depths, float *out_depth, float *out_alpha,
                                       gsb_stream_t stream);
int gsb_rasterize_backward_depth(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m,
                                 const int32_t *tile_bins, const int32_t *tile_order, const float *conics,
                                 const float *opacities, void *records, const int32_t *cum_tiles_hit,
                                 const float *background, const float *final_Ts, const int32_t *final_idx,
                                 const float *v_output, const float *v_output_alpha, void *grad_rows, float *v_xy,
                                 float *v_conic, float *v_colors, float *v_opacity, unsigned flags,
                                 const float *record_depths, const float *v_output_depth, float *v_depths,
                                 gsb_stream_t stream);
int gsb_rasterize_backward_absgrad(int img_h, int img_w, int tiles_x, int tiles_y, int n, int m,
                                   const int32_t *tile_bins, const int32_t *tile_order, const float *conics,
                                   const float *opacities, void *records, const int32_t *cum_tiles_hit,
                                   const float *background, const float *final_Ts, const int32_t *final_idx,
                                   const float *v_output, const float *v_output_alpha, void *grad_rows, float *v_xy,
                                   float *v_conic, float *v_colors, float *v_opacity, unsigned flags,
                                   const float *record_depths, const float *v_output_depth, float *v_depths,
                                   float *v_xy_abs, gsb_stream_t stream);

/* ---- Streaming helpers around the path (SURVEY.md 8f "next" rows) ------------------------------
 * gsb_mse_loss_grad: loss = mean((img-target)^2) written to *loss_out (device float; zeroed by the
 *   call, then accumulated) and v_img = 2 (img-target) * inv_count, one pass (simple_trainer.cpp:199-201:
 *   torch::nn::MSELoss + autograd).  n = number of floats, inv_count = 1/n.
 * gsb_adam_step: fused Adam over a flat fp32 buffer, semantics of torch::optim::Adam without weight
 *   decay / amsgrad (simple_trainer.cpp:146,202; model.cpp:236-243): bias_correction{1,2} = 1 - beta^t. */
int gsb_mse_loss_grad(long long n, const float *img, const float *target, float *v_img, float *loss_out,
                      float inv_count, gsb_stream_t stream);
int gsb_adam_step(long long n, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float lr,
                  float beta1, float beta2, float eps, float bias_correction1, float bias_correction2,
                  gsb_stream_t stream);
/* gsb_adam_step_segments: gsb_adam_step with per-segment learning rates, in one launch (the six optimizers of
 *   model.cpp:58-70 over one flat buffer).  `segments` is a HOST array of num_segments (<= GSB_ADAM_MAX_SEGMENTS)
 *   entries; segment s covers floats [offset, offset + count) of all four buffers (offset a multiple of 4; the
 *   buffers 16-byte aligned), and its element e takes lr_head if e % row_floats < head_floats, lr_rest otherwise
 *   (a merged [n,K,3] SH block: row_floats = 3K, head_floats = 3 gives featuresDc / featuresRest their own rates).
 *   Floats outside every segment are not touched.  Same update as gsb_adam_step, rounded the same way for every
 *   float of both entry points (the parameter step's product is rounded before the subtraction), so a float gets
 *   the same bits from either call. */
#define GSB_ADAM_MAX_SEGMENTS 8
typedef struct gsb_adam_segment {
    long long offset, count;
    int row_floats, head_floats;
    float lr_head, lr_rest;
} gsb_adam_segment;
int gsb_adam_step_segments(int num_segments, const gsb_adam_segment *segments, float *param, const float *grad,
                           float *exp_avg, float *exp_avg_sq, float beta1, float beta2, float eps,
                           float bias_correction1, float bias_correction2, gsb_stream_t stream);

/* gsb_activate_forward / gsb_activate_backward: the parameter activations of Model::forward fused into one
 *   pass each way (model.cpp:148-150,176-177,200): scales = exp(log_scales), quats = raw_quats / |raw_quats|,
 *   opacities = sigmoid(opacity_logits), viewdirs = normalize(means - cam_pos) (detached: no gradient).
 *   cam_pos is a device float[3].  The backward takes the forward outputs (scales, opacities). */
int gsb_activate_forward(int n, const float *means, const float *log_scales, const float *raw_quats,
                         const float *opacity_logits, const float *cam_pos, float *scales, float *quats,
                         float *opacities, float *viewdirs, gsb_stream_t stream);
int gsb_activate_backward(int n, const float *scales, const float *raw_quats, const float *opacities,
                          const float *v_scales, const float *v_quats, const float *v_opacities,
                          float *v_log_scales, float *v_raw_quats, float *v_opacity_logits, gsb_stream_t stream);

/* gsb_densify_stats_update: the per-step densification statistics of Model::afterTrain (model.cpp:317-337) in
 *   one pass: for visible Gaussians (radii > 0) xys_grad_norm += |v_xy|, vis_counts += 1,
 *   max_2d_size = max(max_2d_size, radii / max(H, W)).  All three are [n] fp32, updated in place. */
int gsb_densify_stats_update(int n, const float *v_xy, const int32_t *radii, int img_h, int img_w,
                             float *xys_grad_norm, float *vis_counts, float *max_2d_size, gsb_stream_t stream);
/* gsb_densify_stats_init: the first step after a refinement (model.cpp:321-323,328-330, the `!numel()` branches):
 *   xys_grad_norm = |v_xy| and vis_counts = 1 for EVERY Gaussian, max_2d_size = 0 then the visible update.
 *   Overwrites the three buffers (no pre-zeroing). */
int gsb_densify_stats_init(int n, const float *v_xy, const int32_t *radii, int img_h, int img_w,
                           float *xys_grad_norm, float *vis_counts, float *max_2d_size, gsb_stream_t stream);

/* ---- Topology edits of Model::afterTrain (model.cpp:339-470; SURVEY.md 8f row 3) -----------------
 * The reference's split / duplicate / cull (boolean-mask index + cat + repeat per tensor, and the same again per
 * Adam state in addToOptimizer :253-279 / removeFromOptimizer :281-308) as one classification + compaction:
 * gsb_densify_classify decides per parent what survives and writes
 *     src_map[j] = parent | kind << 30   (j < new_n; kind 0 survivor, 1 / 2 split child of sample 0 / 1, 3 duplicate)
 *   in the reference's output order cat(originals, split sample 0, split sample 1, dups)[~culls];
 *   split_rank[i] = rank of parent i among the split parents (-1 if not split): split child `kind` of parent i
 *   uses row (kind-1) * n_splits + split_rank[i] of the [2*n_splits,3] normal samples (model.cpp:359-360);
 *   counts (device int32[8]) = {n_splits, kept originals, split parents whose children are kept, kept dups,
 *   new_n, n_dups, 0, 0} -- the one read-back of a refinement.  src_map needs room for 3n entries (a parent
 *   yields at most itself + a duplicate, or two split children + a duplicate with itself culled).
 *   Rules, evaluated as the reference does (fp32, same operation order):
 *     high  = (xys_grad_norm / vis_counts) * 0.5 * max_dim > densify_grad_thresh             (:343-344)
 *     split = (max exp(scales) > densify_size_thresh  [|| max_2d_size > split_screen_size if check_split_screen]) && high
 *     dup   = (max exp(scales) <= densify_size_thresh) && high                                (:375-376)
 *     cull  = sigmoid(opacity) < cull_alpha_thresh || split-parent ||
 *             (check_huge && (max exp(scales) > cull_scale_thresh [|| max_2d_size > cull_screen_size if check_cull_screen]))
 *     children: parent's opacity; split children scales log(exp(s)/size_fac); max_2d_size 0    (:370-372,399-403)
 *   max_2d_size may be NULL (treated as 0).  workspace: gsb_densify_workspace_bytes(n).  n < 2^29.
 * gsb_densify_means_scales builds the new means / scales (split children: mean + R(q/|q|)(exp(s) * sample),
 *   log(exp(s)/size_fac), :359-373); gsb_densify_gather_rows rebuilds any other [n,row_floats] tensor
 *   (dst[j,:] = src[parent(j),:]; zero_children = 1 writes zeros for kinds 1-3: the Adam moments of new Gaussians).
 * gsb_reset_opacity: opacities = min(opacities, max_logit) (:472-475) and, when given, zeroed Adam moments (what
 *   :477-486 intends; the reference builds the zeroed state and then drops it -- DESIGN.md D14). */
size_t gsb_densify_workspace_bytes(int n);
int gsb_densify_classify(int n, const float *scales, const float *opacities, const float *xys_grad_norm,
                         const float *vis_counts, const float *max_2d_size, float max_dim,
                         float densify_grad_thresh, float densify_size_thresh, int check_split_screen,
                         float split_screen_size, float cull_alpha_thresh, int check_huge, float cull_scale_thresh,
                         int check_cull_screen, float cull_screen_size, float size_fac, void *workspace,
                         size_t workspace_bytes, int32_t *src_map, int32_t *split_rank, int32_t *counts,
                         gsb_stream_t stream);
int gsb_densify_means_scales(int new_n, int n_splits, const int32_t *src_map, const int32_t *split_rank,
                             const float *samples, const float *means, const float *scales, const float *quats,
                             float size_fac, float *new_means, float *new_scales, gsb_stream_t stream);
int gsb_densify_gather_rows(int new_n, int row_floats, const int32_t *src_map, const float *src, float *dst,
                            int zero_children, gsb_stream_t stream);
int gsb_reset_opacity(int n, float max_logit, float *opacities, float *exp_avg, float *exp_avg_sq,
                      gsb_stream_t stream);

/* ---- 3DGS-MCMC refinement (Kheradmand et al. 2024, gsplat's MCMCStrategy; DESIGN.md D20) ----------------------
 * o = 1.f / (1.f + expf(-logit)) throughout (the raw sigmoid, as the projection forms it).  Random numbers come from
 *   Philox4x32-10 with key (key0, key1) = (seed & 0xffffffff, seed >> 32) and counter (index, step, tag, 0); tag 0 is
 *   the position noise (index = Gaussian), 1 the relocation samples, 2 the growth samples (index = sample number).
 *   A uniform is ((x0 >> 5) 2^26 + (x1 >> 6)) 2^-53; normals are Box-Muller on u1 = ((a >> 8) + 1) 2^-24,
 *   u2 = (b >> 8) 2^-24: (x0, x1) give z0 (cos) and z1 (sin), (x2, x3) give z2 (cos).
 * The flat layout is a HOST array of num_segments (<= GSB_MCMC_MAX_SEGMENTS) gsb_row_segment: slice s holds row i at
 *   floats [offset + i * row_floats, offset + (i + 1) * row_floats) of the flat buffers.
 * gsb_mcmc_plan: the weights w_i = o_i in fp64 (0 where o_i <= min_opacity when mask_dead), their inclusive scan into
 *   cdf [n] (fp64, monotone: a weight-0 index is never drawn; T = cdf[n-1]), with mask_dead the dead indices in
 *   ascending order into dead [n], and result (device int32[4]) = {n_dead, T > 0, any o > 0, 0}: the one read-back
 *   of a refinement.  workspace: gsb_mcmc_workspace_bytes(n), 256-byte aligned.  n < 2^29.
 * gsb_mcmc_sample: samples[j] = the smallest i with cdf[i] > u_j T (u_j the uniform of counter (j, step, tag, 0)),
 *   j < num_samples; counts [n] = how often each index was drawn (zeroed by the call).  Needs T > 0.
 * gsb_mcmc_relocate: every row i with counts[i] > 0, ratio r = min(counts[i] + 1, 51):
 *   alpha = -expm1(log1p(-o) / r), D = sum_{k<r} (-1)^k C(r,k+1) alpha^(k+1) / sqrt(k+1), logit <-
 *   logit(clamp(alpha, min_opacity, 1 - 2^-23)), log-scales <- s + log(o / D), in fp64 rounded once to fp32; with
 *   zero_moments its Adam moments in every slice are zeroed.
 * gsb_mcmc_copy_rows: row dst_rows[j] <- row src_rows[j] of param in every slice (the rows must not overlap).
 * gsb_mcmc_regularize: grad_logits += opacity_coef * o(1 - o), grad_log_scales += scale_coef * exp(s) (the gradients
 *   of opacity_reg mean|o| + scale_reg mean|exp s| with opacity_coef = opacity_reg / n, scale_coef = scale_reg / 3n).
 * gsb_mcmc_add_noise: means += Sigma (z * (sigma_100((1 - o) - 0.995f) * noise_scale)), z the three normals of counter
 *   (i, step, 0, 0), Sigma = R diag(exp(2 s)) R^T with R from raw_quats / |raw_quats| (16-byte aligned),
 *   sigma_100(x) = 1 / (1 + exp(-100 x)).
 * gsb_mcmc_draws: the raw Philox words [count,4] and normals [count,3] of counters (j, step, tag, 0), j < count
 *   (either output may be NULL; words 16-byte aligned). */
#define GSB_MCMC_MAX_SEGMENTS 8
typedef struct gsb_row_segment {
    long long offset;
    int row_floats, reserved;
} gsb_row_segment;
size_t gsb_mcmc_workspace_bytes(int n);
int gsb_mcmc_plan(int n, const float *logits, float min_opacity, int mask_dead, void *workspace,
                  size_t workspace_bytes, double *cdf, int32_t *dead, int32_t *result, gsb_stream_t stream);
int gsb_mcmc_sample(int num_samples, int n, const double *cdf, unsigned key0, unsigned key1, int step, int tag,
                    int32_t *samples, int32_t *counts, gsb_stream_t stream);
int gsb_mcmc_relocate(int n, const int32_t *counts, float min_opacity, float *logits, float *log_scales,
                      int zero_moments, int num_segments, const gsb_row_segment *segments, float *exp_avg,
                      float *exp_avg_sq, gsb_stream_t stream);
int gsb_mcmc_copy_rows(int num_rows, const int32_t *dst_rows, const int32_t *src_rows, int num_segments,
                       const gsb_row_segment *segments, float *param, gsb_stream_t stream);
int gsb_mcmc_regularize(int n, const float *logits, const float *log_scales, float opacity_coef, float scale_coef,
                        float *grad_logits, float *grad_log_scales, gsb_stream_t stream);
int gsb_mcmc_add_noise(int n, const float *logits, const float *log_scales, const float *raw_quats, unsigned key0,
                       unsigned key1, int step, float noise_scale, float *means, gsb_stream_t stream);
int gsb_mcmc_draws(int count, unsigned key0, unsigned key1, int step, int tag, int32_t *words, float *normals,
                   gsb_stream_t stream);

/* ---- Per-image bilateral grids (Wang et al. 2024; gsplat's bilateral-grid module; DESIGN.md D21) --------------
 * A grid is GSB_BILAGRID_L x _Y x _X cells of 12 floats, stored channels-last [L][Y][X][12] (GSB_BILAGRID_FLOATS
 *   floats, 16-byte aligned); a cell's 12 floats are the row-major 3x4 affine matrix [A | b].  Every grid starts at
 *   the identity.  rgb, out, v_out and v_rgb are [H,W,3] fp32 images, 1 <= H, W <= 32768.
 * gsb_bilagrid_slice_forward: out = A rgb + b with the coefficients trilinearly interpolated at
 *   gx = ((px + 0.5) / W)(X - 1), gy = ((py + 0.5) / H)(Y - 1), gz = clamp((0.299 r + 0.587 g) + 0.114 b, 0, 1)(L - 1)
 *   (F.grid_sample with align_corners=True and border padding, then the affine map); out is not clamped.
 * gsb_bilagrid_slice_backward: v_rgb = A^T v_out + (dout/dz . v_out)(0.299, 0.587, 0.114) (written; the luma term is
 *   0 where z <= 0 or z >= 1, and at an interior integer gz = k the derivative is the forward difference of cells k
 *   and k + 1), and v_grid += scale * (trilinear weights x v_out (x) (rgb, 1)), summed without atomics in a fixed
 *   order: the same inputs give the same bits.  workspace: gsb_bilagrid_workspace_bytes(H, W), 256-byte aligned.
 * gsb_bilagrid_tv: v_grids = weight * dTV/dG over num_grids consecutive grids (written, not added), TV(G) = the sum
 *   over the axes x, y, l of the mean of (G[i+1] - G[i])^2 over every element of that axis's difference tensor, all
 *   grids included; with tv_out (a device float) the value TV(G) through a deterministic fp64 reduction.
 * None of them allocates; bad sizes, NULL pointers and a short workspace are rejected before any launch. */
#define GSB_BILAGRID_X 16
#define GSB_BILAGRID_Y 16
#define GSB_BILAGRID_L 8
#define GSB_BILAGRID_COEFFS 12
#define GSB_BILAGRID_FLOATS (GSB_BILAGRID_L * GSB_BILAGRID_Y * GSB_BILAGRID_X * GSB_BILAGRID_COEFFS)
int gsb_bilagrid_slice_forward(int H, int W, const float *grid, const float *rgb, float *out, gsb_stream_t stream);
size_t gsb_bilagrid_workspace_bytes(int H, int W);
int gsb_bilagrid_slice_backward(int H, int W, const float *grid, const float *rgb, const float *v_out, float scale,
                                float *v_rgb, float *v_grid, void *workspace, size_t workspace_bytes,
                                gsb_stream_t stream);
int gsb_bilagrid_tv(int num_grids, const float *grids, float weight, float *v_grids, float *tv_out,
                    gsb_stream_t stream);

/* ---- Camera pose corrections (DESIGN D22; gsplat's pose optimisation) ----
 * gsb_project_backward_activated_camgrad: gsb_project_backward_activated (accumulate = 0, antialiased = 0), _acc (1, 0),
 *   _aa (0, 1) or _aa_acc (1, 1), with the same arguments (opacities = the logits when antialiased) and the same
 *   per-Gaussian outputs bit for bit, that also writes the view's camera gradient: the exact VJP w.r.t. viewmat rows
 *   0..2 and projmat rows 0, 1, 3, summed over the Gaussians with radii > 0, as one fp32 partial row of 24 floats
 *   per block of 256 Gaussians (warp shuffle tree, then the 8 warps in order) into cam_partials
 *   (gsb_project_camera_partials_floats(n) floats; n == 0 writes nothing).
 * gsb_project_camera_grad_reduce: the sum of nblocks = ceil(n / 256) partial rows, in a fixed order in fp64, rounded
 *   once into v_viewmat [4,4] and v_projmat [4,4] (row-major; row 3 of v_viewmat and row 2 of v_projmat written 0).
 *   The same inputs give the same bits.
 * A pose correction is GSB_POSE_FLOATS floats e = (t [3], d [6]); Rd = rot6d(d + (1,0,0,0,1,0)) has the rows b1, b2, b3
 *   (b1 = a1/|a1|, b2 = normalize(a2 - (b1.a2) b1), b3 = b1 x b2), and the corrected camera-to-world is [R|T] Delta,
 *   Delta = [[Rd, t], [0, 1]] (in the camera's own frame).
 * gsb_pose_apply: view_out = Delta^-1 view [4,4], centre_out = centre + view[0:3,0:3]^T t [3], in fp64, rounded once;
 *   e = 0 copies view and centre bit for bit.  The outputs must not overlap the inputs.
 * gsb_pose_backward: grad [9] += scale * d/de of the loss whose gradients w.r.t. view_out and proj @ view_out are
 *   v_viewmat and v_projmat (from gsb_project_camera_grad_reduce): G = v_viewmat + proj^T v_projmat, d/dDelta^-1 =
 *   G view^T, chained through Delta^-1 and rot6d in fp64; the added value is rounded once.
 * One thread each; none of them allocates; NULL pointers are rejected before any launch. */
#define GSB_POSE_FLOATS 9
size_t gsb_project_camera_partials_floats(int n);
int gsb_project_backward_activated_camgrad(int n, const float *means3d, const float *log_scales, float glob_scale,
                                           const float *raw_quats, const float *opacities, const float *viewmat,
                                           const float *projmat, float fx, float fy, int img_h, int img_w,
                                           const int32_t *radii, const float *conics, const float *v_xy,
                                           const float *v_depth, const float *v_conic, const float *v_opacity,
                                           float *v_mean3d, float *v_log_scales, float *v_raw_quats,
                                           float *v_opacity_logits, int accumulate, int antialiased,
                                           float *cam_partials, gsb_stream_t stream);
int gsb_project_camera_grad_reduce(int nblocks, const float *partials, float *v_viewmat, float *v_projmat,
                                   gsb_stream_t stream);
int gsb_pose_apply(const float *pose, const float *view, const float *centre, float *view_out, float *centre_out,
                   gsb_stream_t stream);
int gsb_pose_backward(const float *pose, const float *view, const float *proj, const float *v_viewmat,
                      const float *v_projmat, float scale, float *grad, gsb_stream_t stream);

/* ---- Inverse-depth priors (DESIGN D23; graphdeco 3DGS's depth regularisation, gsplat's depth_loss) ----
 * A prior sample p is valid iff it is finite and > 0 (0, negative, NaN and inf mean "no data").  Every result below
 *   but the loss value is its fp32 restatement bit for bit (IEEE division, no fused multiply-add).
 * gsb_inverse_depths: inv [n] = 1.f / depths[i] where radii[i] > 0, 0 elsewhere: the value stream the depth blend
 *   renders (gathered in place of the sort key, so the blend still sorts by depths).
 * gsb_inverse_depths_backward: v_z [n] = -((v_inv[i] * inv) * inv) where radii[i] > 0 (inv recomputed as above), 0
 *   elsewhere; v_z is the projection backward's v_depth.
 * gsb_inverse_depth_l1: over the [H,W] maps rendered R and prior P, v_rendered = scale_g * sgn(R - P) on valid pixels
 *   (sgn(0) = 0) and 0 elsewhere, written completely; *loss_out (a device float) = sum over the valid pixels of
 *   |R - P| / (H W), unweighted: each |R - P| rounded to fp32, summed in fp64 in a fixed order, divided and rounded
 *   once (the same inputs give the same bits).  workspace: gsb_inverse_depth_l1_workspace_bytes(H, W), 8-byte
 *   aligned.  1 <= H W < 2^31.
 * gsb_depth_downscale_mean: dst [h/factor, w/factor] (integer division) = the mean of the valid samples of each
 *   factor x factor block of src [h,w]: summed in fp32 in row-major order, then divided by their count, or 0 when the
 *   block has none.  factor >= 1, h, w >= factor.
 * None of them allocates; bad sizes and NULL pointers are rejected before any launch; n = 0 is a no-op. */
int gsb_inverse_depths(int n, const float *depths, const int32_t *radii, float *inv, gsb_stream_t stream);
int gsb_inverse_depths_backward(int n, const float *depths, const int32_t *radii, const float *v_inv, float *v_z,
                                gsb_stream_t stream);
size_t gsb_inverse_depth_l1_workspace_bytes(int img_h, int img_w);
int gsb_inverse_depth_l1(int img_h, int img_w, const float *rendered, const float *prior, float scale_g,
                         float *v_rendered, float *loss_out, void *workspace, size_t workspace_bytes,
                         gsb_stream_t stream);
int gsb_depth_downscale_mean(int h, int w, int factor, const float *src, float *dst, gsb_stream_t stream);

/* ---- Scene export (Model::savePly model.cpp:505-558, Model::saveSplat :560-594; SURVEY.md 8f row 4) ----
 * Packs the file BODY on the device (the caller writes the text header and copies the rows D2H, typically on a
 * side stream into pinned memory).  features_dc / features_rest take a row stride in floats so both the reference's
 * [n,3] + [n,K-1,3] tensors and a merged [n,K,3] block (dc = block, rest = block + 3, strides 3K) are accepted.
 * keep_crs mirrors Model::keepCrs: means / crs_scale + crs_translation (HOST float[3]), scales log(exp(s)/crs_scale).
 * gsb_pack_ply_rows: out_rows [n, gsb_ply_row_floats(K)] fp32 = x y z, 0 0 0, f_dc_0..2, f_rest (channel-major,
 *   "Match Inria's version" :525), opacity, scale_0..2, rot_0..3.  Byte-exact vs the reference when !keep_crs.
 * gsb_splat_order_keys + gsb_sort_intersects(n, num_tiles = 1, keys, ...) give the reference's row order
 *   (descending (sum exp(scale)) / (1 + exp(-opacity)), :571-583; ties by ascending index where std::sort is
 *   unspecified); gsb_pack_splat_rows writes the 32-B rows (mean 3 f32, exp(scale) 3 f32, rgb 3 u8, alpha u8,
 *   quat 4 u8) in that order (order == NULL: identity). */
int gsb_ply_row_floats(int sh_bases);
int gsb_pack_ply_rows(int n, int sh_bases, const float *means, const float *features_dc, int dc_stride,
                      const float *features_rest, int rest_stride, const float *opacities, const float *scales,
                      const float *quats, int keep_crs, float crs_scale, const float *crs_translation,
                      float *out_rows, gsb_stream_t stream);
/* gsb_unpack_ply_rows: the inverse (Model::loadPly's per-row reads + reshape/transpose, model.cpp:724-746): PLY
 *   vertex rows -> the six parameter tensors; with keep_crs, means = (means - translation) * scale and
 *   scales = log(scale * exp(scales)) (model.cpp:737-740).  Normals are ignored. */
int gsb_unpack_ply_rows(int n, int sh_bases, const float *rows, int keep_crs, float crs_scale,
                        const float *crs_translation, float *means, float *features_dc, int dc_stride,
                        float *features_rest, int rest_stride, float *opacities, float *scales, float *quats,
                        gsb_stream_t stream);
int gsb_splat_order_keys(int n, const float *scales, const float *opacities, int keep_crs, float crs_scale,
                         int64_t *keys, gsb_stream_t stream);
int gsb_pack_splat_rows(int n, const int32_t *order, const float *means, const float *scales,
                        const float *features_dc, int dc_stride, const float *opacities, const float *quats,
                        int keep_crs, float crs_scale, const float *crs_translation, void *out_rows,
                        gsb_stream_t stream);

/* gsb_ssim_l1_loss: the training loss of Model::mainLoss (model.cpp:780-784): (1-w) * mean|rendered - gt| +
 *   w * (1 - SSIM(rendered, gt)) with the reference's SSIM (ssim.cpp:8-47: 11x11 window gaussian(1.5) evaluated
 *   at floor((i-11)/2), zero padding 5, C1 = 1e-4, C2 = 9e-4, mean over all channels) and its gradient w.r.t.
 *   `rendered`, fused into two tile kernels.  rendered / gt / v_rendered are [H,W,3] channels-last;
 *   loss_out is a device float[3] = {total, L1, SSIM}; workspace of gsb_ssim_workspace_bytes(H, W). */
size_t gsb_ssim_workspace_bytes(int img_h, int img_w);
int gsb_ssim_l1_loss(int img_h, int img_w, const float *rendered, const float *gt, float ssim_weight,
                     float *v_rendered, float *loss_out, void *workspace, size_t workspace_bytes,
                     gsb_stream_t stream);
/* gsb_ssim_l1_loss_masked (DESIGN D26): the loss over the used pixels of mask [H,W] u8 (nonzero = used, 0 = ignored).
 *   With m the mask, N = sum m, x~ = m ? gt : 0 and y~ = m ? rendered : 0 (selected, so non-finite values in ignored
 *   pixels never reach the result) and S_c the SSIM map of x~ and y~: L1 = sum m |y - x| / 3N, SSIM = sum m S_c / 3N,
 *   total = (1-w) L1 + w (1 - SSIM); v_rendered is its gradient, exactly 0 on ignored pixels.  N = 0 gives {0, 0, 1}
 *   and a zero gradient.  With every pixel used and H W <= 2^24, v_rendered equals gsb_ssim_l1_loss's bit for bit and
 *   loss_out holds the same sums (in both entry points their per-tile float atomics make the last bits of the three
 *   scalars depend on the order the tiles finish).
 *   N, the loss and the gradient scales stay on the device (no host read-back).  The workspace is
 *   gsb_ssim_workspace_bytes(H, W), 256-byte aligned. */
int gsb_ssim_l1_loss_masked(int img_h, int img_w, const float *rendered, const float *gt, const uint8_t *mask,
                            float ssim_weight, float *v_rendered, float *loss_out, void *workspace,
                            size_t workspace_bytes, gsb_stream_t stream);

/* ---- Point-cloud initialisation (Model's constructor, model.hpp:23-57) ---------------------------
 * gsb_knn_mean_dist replaces PointsTensor::scales (kdtree_tensor.cpp:4-22, a nanoflann k-d tree on the CPU):
 *   mean_dist [n] = the mean distance from every point of xyz [n,3] to its 3 nearest neighbours, exactly.  With
 *   d(i,j) = ((dx*dx) + (dy*dy)) + (dz*dz), dx = x_i - x_j in fp32 and every operation rounded separately, and
 *   d0 <= d1 <= d2 <= d3 the four smallest d(i,j) over all j (i itself included):
 *   mean_dist[i] = ((sqrtf(d1) + sqrtf(d2)) + sqrtf(d3)) / 3.0f (IEEE sqrt and division).  The result depends only on
 *   those values: it is deterministic, and permuting the points permutes it.  n = 0 is a no-op; 1 <= n < 4 is
 *   GSB_ERR_INVALID_ARG (the reference reads unset result slots there).  Coordinates must be finite (not checked:
 *   non-finite input gives unspecified values).  The workspace (gsb_knn_workspace_bytes(n) bytes) must be 256-byte
 *   aligned. */
size_t gsb_knn_workspace_bytes(int n);
int gsb_knn_mean_dist(int n, const float *xyz, float *mean_dist, void *workspace, size_t workspace_bytes,
                      gsb_stream_t stream);

/* ---- Mip-Splatting's 3-D smoothing filter (DESIGN D24) ------------------------------------------------------------
 * gsb_project_forward_activated_filter3d: gsb_project_forward_activated (antialiased = 0) or _aa (1) with the filter
 *   f = filter3d[i] (one float per Gaussian): the covariance is built from sigma_k = sqrtf(s_k s_k + f f) in place of
 *   s_k = glob_scale expf(a_k), and opacities = sigmoid(logit) * c3 (* comp when antialiased, comp from the filtered
 *   screen covariance), c3 = (r_0 r_1) r_2, r_k = s_k / sigma_k.  At f = 0 every output equals the unfiltered
 *   entry point's bit for bit.
 * gsb_project_backward_activated_filter3d: its exact VJP with filter3d held constant.  opacity_logits are the logits
 *   (as the _aa backward takes them); accumulate = 1 adds to the four outputs (as _acc), camgrad = 1 also writes the
 *   camera-gradient partial rows into cam_partials (as gsb_project_backward_activated_camgrad).  At f = 0 the outputs
 *   equal the unfiltered variant's, up to the sign of a zero.
 * gsb_filter3d_compute: filter3d [n] from the means [n,3] and num_cameras >= 1 training cameras, a DEVICE array of
 *   GSB_FILTER3D_CAM_FLOATS floats each: viewmat rows 0..2 (12), fx, fy, cx, cy, W, H (fx > 0).  Camera j sees
 *   Gaussian i when z > near and -(margin W) <= u <= (1 + margin) W and -(margin H) <= v <= (1 + margin) H, where
 *   (x, y, z) is the projection's view-space point (tx, ty, tz), u = fx (x / z) + cx and v = fy (y / z) + cy, all fp32
 *   without contraction; d[i] = the least such z, an unseen Gaussian takes the largest d of the seen ones, and
 *   f[i] = (d[i] / F) * S with F = max_j fx_j and S = (float)sqrt((double)variance); every f is 0 when no Gaussian
 *   is seen.  The result does not depend on scheduling (min / max only).  workspace: gsb_filter3d_workspace_bytes(),
 *   4-byte aligned.  near, margin, variance >= 0 and finite.
 * gsb_filter3d_bake: the filter baked into a scene at glob_scale 1, in fp64, each output rounded once:
 *   out_log_scales = log(e^2 + f^2) / 2 with e = exp(a), out_opacity_logits = logit(sigmoid(l) c3).  In place is
 *   allowed.
 * gsb_reset_opacity_filter3d: gsb_reset_opacity on the effective opacity sigmoid(l) c3 (c3 the projection's fp32 value
 *   at glob_scale 1): l = min(l, logit(reset_value / c3)) where reset_value / c3 < 1 (the logit in fp64, rounded once),
 *   l unchanged where it is >= 1, and min(l, max_logit) -- gsb_reset_opacity's result -- where c3 == 1; the moments,
 *   when given, are zeroed as there.
 * None of them allocates; bad flags, sizes and NULL pointers are rejected before any launch; n = 0 is a no-op. */
#define GSB_FILTER3D_CAM_FLOATS 18
int gsb_project_forward_activated_filter3d(int n, const float *means3d, const float *log_scales, float glob_scale,
                                           const float *raw_quats, const float *opacity_logits, const float *filter3d,
                                           const float *viewmat, const float *projmat, float fx, float fy, float cx,
                                           float cy, int img_h, int img_w, int tiles_x, int tiles_y,
                                           float clip_thresh, float *cov3d, float *xys, float *depths, int32_t *radii,
                                           float *conics, int32_t *num_tiles_hit, float *opacities, int antialiased,
                                           gsb_stream_t stream);
int gsb_project_backward_activated_filter3d(int n, const float *means3d, const float *log_scales, float glob_scale,
                                            const float *raw_quats, const float *opacity_logits,
                                            const float *filter3d, const float *viewmat, const float *projmat,
                                            float fx, float fy, int img_h, int img_w, const int32_t *radii,
                                            const float *conics, const float *v_xy, const float *v_depth,
                                            const float *v_conic, const float *v_opacity, float *v_mean3d,
                                            float *v_log_scales, float *v_raw_quats, float *v_opacity_logits,
                                            int accumulate, int antialiased, int camgrad, float *cam_partials,
                                            gsb_stream_t stream);
size_t gsb_filter3d_workspace_bytes(void);
int gsb_filter3d_compute(int n, const float *means, int num_cameras, const float *cameras, float near, float margin,
                         float variance, void *workspace, size_t workspace_bytes, float *filter3d,
                         gsb_stream_t stream);
int gsb_filter3d_bake(int n, const float *log_scales, const float *opacity_logits, const float *filter3d,
                      float *out_log_scales, float *out_opacity_logits, gsb_stream_t stream);
int gsb_reset_opacity_filter3d(int n, float max_logit, float reset_value, const float *log_scales,
                               const float *filter3d, float *opacities, float *exp_avg, float *exp_avg_sq,
                               gsb_stream_t stream);

/* ---- Fisheye cameras (DESIGN D27) ------------------------------------------------------------------------------------
 * The activated projection through OpenCV's fisheye model (Kannala-Brandt) in the view frame (x right, y down, +z
 * forward): t = viewmat (p, 1), theta = atan2(|t.xy|, t.z), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 +
 * k4 theta^8), (u, v) = (fx, fy) theta_d / |t.xy| t.xy + (cx, cy) - 0.5.  The EWA covariance takes the full 2x3
 * Jacobian of (u, v) at t; the 0.3 blur, conic, radius, tile box and the anti-aliased opacity are the pinhole's.  A
 * Gaussian is culled (as t.z <= clip_thresh culls it) also where theta > theta_lim; theta_lim is the first zero of
 * d theta_d / d theta in (0, pi/2), else pi/2, in float64 rounded once (model.fisheye_theta_limit).
 * gsb_project_forward_fisheye: the arguments of gsb_project_forward_activated without projmat, with the distortion
 *   and theta_lim after cx, cy, and antialiased (0 / 1) before the stream; the same seven outputs.
 * gsb_project_backward_fisheye: its exact VJP.  opacity_logits are the logits in every mode; accumulate = 1 adds to
 *   the four outputs; cam_partials != NULL also writes the camera-gradient partial rows of
 *   gsb_project_backward_activated_camgrad (gsb_project_camera_partials_floats(n) floats) for
 *   gsb_project_camera_grad_reduce, whose v_projmat is then 0.
 * Both check fx, fy > 0, finite k1..k4, 0 < theta_lim <= (float)(pi / 2) and the flags. */
int gsb_project_forward_fisheye(int n, const float *means3d, const float *log_scales, float glob_scale,
                                const float *raw_quats, const float *opacity_logits, const float *viewmat, float fx,
                                float fy, float cx, float cy, float k1, float k2, float k3, float k4, float theta_lim,
                                int img_h, int img_w, int tiles_x, int tiles_y, float clip_thresh, float *cov3d,
                                float *xys, float *depths, int32_t *radii, float *conics, int32_t *num_tiles_hit,
                                float *opacities, int antialiased, gsb_stream_t stream);
int gsb_project_backward_fisheye(int n, const float *means3d, const float *log_scales, float glob_scale,
                                 const float *raw_quats, const float *opacity_logits, const float *viewmat, float fx,
                                 float fy, float k1, float k2, float k3, float k4, float theta_lim, int img_h, int img_w,
                                 const int32_t *radii, const float *conics, const float *v_xy, const float *v_depth,
                                 const float *v_conic, const float *v_opacity, float *v_mean3d, float *v_log_scales,
                                 float *v_raw_quats, float *v_opacity_logits, int accumulate, int antialiased,
                                 float *cam_partials, gsb_stream_t stream);

/* ---- Training images (Camera::loadImage / Camera::getImage, input_data.cpp:40-117) --------------------------------
 * Images are 3-channel u8, [h,w,3] row-major and dense.
 * gsb_resize_area_u8 is cv::resize(src, dst, ..., INTER_AREA) of OpenCV 4's CPU code, byte for byte, for dst_h <= src_h and
 *   dst_w <= src_w.  inv_scale = 0: the call with dsize given (getImage: the scales come from the sizes);
 *   0 < inv_scale <= 1: the call with an empty dsize and fx = fy = inv_scale (loadImage's 1/downscaleFactor), and then
 *   dst must be cvRound(src * (double)inv_scale) on both axes.  An integer scale (within DBL_EPSILON) takes OpenCV's
 *   fast path (at 2x2 full cells round as (s+2)>>2, other full cells as rint(float(s) * (1.f/area)), border cells as
 *   rint(float(s)/count)); any other scale the general path (double cell edges, float weights and row sums).  Equal
 *   sizes copy.  src and dst must not overlap.
 * gsb_undistort_u8 is cv::undistort(src, tmp, K, {k1,k2,p1,p2,k3}, newK) followed by the crop
 *   dst = tmp[roi_y:roi_y+roi_h, roi_x:roi_x+roi_w], writing only the ROI: dst is [roi_h,roi_w,3].  K and newK are
 *   (fx, fy, cx, cy) with zero skew, given as the float values of the reference's CV_32F matrices; the map is
 *   computed in fp64 stripe by stripe as cv::undistort does, quantised to 1/32 pixel, and the remap is OpenCV's
 *   fixed-point bilinear with BORDER_CONSTANT 0.  An empty ROI is a no-op.
 * gsb_u8_to_f32_views converts num_views images of [h,w,3] u8 (views: a DEVICE array of num_views device addresses,
 *   int64) into out [num_views,h,w,3] float32 = float(u) / 255.0f (IEEE division, as imageToTensor), in one launch.
 *   num_views = 0 is a no-op; at most 65535.
 * gsb_resize_area_mask_u8 / gsb_undistort_mask_u8 (DESIGN D26) take a u8 [h,w] loss mask (nonzero = used) through the
 *   geometry of gsb_resize_area_u8 / gsb_undistort_u8, with the same arguments and checks, and write 0 / 1 bytes: an
 *   output pixel is 1 iff every source pixel with a nonzero weight in the colour's output pixel is used.  Resize: the
 *   cell clipped to the image on the integer-scale path (a cell wholly outside it is 0), the entries of OpenCV's
 *   computeResizeAreaTab (with its 1e-3 cut-offs) on the general path; equal sizes normalise the mask to 0 / 1.
 *   Undistort: the tap (sx, sy) always, the right taps iff the map's x fraction is nonzero, the bottom taps iff its y
 *   fraction is; a tap outside the image makes the pixel 0. */
int gsb_resize_area_u8(int src_h, int src_w, const uint8_t *src, int dst_h, int dst_w, uint8_t *dst, float inv_scale,
                       gsb_stream_t stream);
int gsb_undistort_u8(int h, int w, const uint8_t *src, float fx, float fy, float cx, float cy, float k1, float k2,
                     float p1, float p2, float k3, float new_fx, float new_fy, float new_cx, float new_cy, int roi_x,
                     int roi_y, int roi_w, int roi_h, uint8_t *dst, gsb_stream_t stream);
int gsb_u8_to_f32_views(int num_views, const int64_t *views, int h, int w, float *out, gsb_stream_t stream);
int gsb_resize_area_mask_u8(int src_h, int src_w, const uint8_t *src, int dst_h, int dst_w, uint8_t *dst,
                            float inv_scale, gsb_stream_t stream);
int gsb_undistort_mask_u8(int h, int w, const uint8_t *src, float fx, float fy, float cx, float cy, float k1, float k2,
                          float p1, float p2, float k3, float new_fx, float new_fy, float new_cx, float new_cy,
                          int roi_x, int roi_y, int roi_w, int roi_h, uint8_t *dst, gsb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
