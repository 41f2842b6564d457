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

/* ---- Tile binning ----------------------------------------------------------------------------
 * gsb_cumsum_tiles_hit replaces torch::cumsum(numTilesHit, 0, kInt32) (rasterize_gaussians.cpp:62).
 *   Inclusive scan; the caller reads M = cum_tiles_hit[n-1] back (rasterize_gaussians.cpp:63).
 *   If total_out != NULL the total is also written there (device or mapped-pinned int32).
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
                         size_t workspace_bytes, int32_t *total_out, gsb_stream_t stream);
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
 *   from earlier frames; stats (device int32[4]) = {M, longest tile list, overflow, 0} with overflow = 1 iff
 *   M > m_capacity or longest > len_capacity, in which case gsb_bucket_sort_pack and
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
 *   `x <= max`). */
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

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
