"""Python mirror of the reference's autograd operator layer, on top of the C ABI.

Same class names, argument order/meaning and error behaviour as the reference's libtorch operators
(/root/reference):
  ProjectGaussians     project_gaussians.hpp:12-30,  project_gaussians.cpp:5-90
  RasterizeGaussians   rasterize_gaussians.hpp:22-37, rasterize_gaussians.cpp:39-140
  binAndSortGaussians  rasterize_gaussians.hpp:11-19, rasterize_gaussians.cpp:6-37
  SphericalHarmonics   spherical_harmonics.hpp:15-23, spherical_harmonics.cpp:32-63
The C++/libtorch version of this layer (the actual drop-in for model.cpp / simple_trainer.cpp) is in
opensplat_b200/csrc/ops; this module is what the parity tests and bench.py drive.

All compute happens in libgsplat_b200.so (hand-written sm_90a CUDA); torch supplies memory, streams
and the autograd graph.  CPU tensors are rejected -- there is no fallback path.
"""
import torch

from . import capi

BLOCK_X = 16  # rasterizer/gsplat/config.h:1-2
BLOCK_Y = 16


def tile_bounds(width, height):
    """TileBounds as the callers compute it (model.cpp:144, simple_trainer.cpp:91)."""
    return ((width + BLOCK_X - 1) // BLOCK_X, (height + BLOCK_Y - 1) // BLOCK_Y, 1)


def deg_from_sh(num_bases):  # spherical_harmonics.cpp:3-16
    return {1: 0, 4: 1, 9: 2, 16: 3}.get(int(num_bases), 4)


def num_sh_bases(degree):  # sh.cuh:40-50
    return {0: 1, 1: 4, 2: 9, 3: 16}.get(int(degree), 25)


def _empty(shape, dtype, like):
    return torch.empty(shape, dtype=dtype, device=like.device)


class _Workspace:
    """Grow-only device scratch buffers keyed by (device, tag): avoids a cudaMalloc per call
    (the reference pays ~20 torch::zeros allocations per iteration, SURVEY 8a O1-O3)."""

    def __init__(self):
        self.bufs = {}

    def get(self, device, tag, nbytes):
        key = (device.index if device.index is not None else torch.cuda.current_device(), tag)
        b = self.bufs.get(key)
        if b is None or b.numel() < nbytes:
            b = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=device)
            self.bufs[key] = b
        return b


_ws = _Workspace()


# ------------------------------------------------------------------------------------------------
# functional layer (one call per C-ABI entry point; mirrors bindings.h `*_tensor` functions)
# ------------------------------------------------------------------------------------------------
def compute_sh_forward(degree, degrees_to_use, viewdirs, coeffs):
    n = coeffs.shape[0]
    nb = num_sh_bases(degree)
    if coeffs.dim() != 3 or coeffs.shape[1] != nb or coeffs.shape[2] != 3:
        raise ValueError("coeffs must have dimensions (N, D, 3)")  # bindings.cu:76-79
    viewdirs, coeffs = capi.f32(viewdirs), capi.f32(coeffs)
    colors = _empty((n, 3), torch.float32, coeffs)
    capi.check(capi.lib().gsb_sh_forward(n, degree, degrees_to_use, capi.ptr(viewdirs), capi.ptr(coeffs),
                                         capi.ptr(colors), capi.stream()))
    return colors


def compute_sh_backward(degree, degrees_to_use, viewdirs, v_colors):
    n = v_colors.shape[0]
    if viewdirs.dim() != 2 or viewdirs.shape[0] != n or viewdirs.shape[1] != 3:
        raise ValueError("viewdirs must have dimensions (N, 3)")  # bindings.cu:101-104
    if v_colors.dim() != 2 or v_colors.shape[1] != 3:
        raise ValueError("v_colors must have dimensions (N, 3)")
    viewdirs, v_colors = capi.f32(viewdirs), capi.f32(v_colors)
    v_coeffs = _empty((n, num_sh_bases(degree), 3), torch.float32, v_colors)
    capi.check(capi.lib().gsb_sh_backward(n, degree, degrees_to_use, capi.ptr(viewdirs), capi.ptr(v_colors),
                                          capi.ptr(v_coeffs), capi.stream()))
    return v_coeffs


def project_gaussians_forward(means3d, scales, glob_scale, quats, viewmat, projmat, fx, fy, cx, cy,
                              img_height, img_width, tile_bounds_, clip_thresh=0.01):
    n = means3d.shape[0]
    means3d, scales, quats = capi.f32(means3d), capi.f32(scales), capi.f32(quats)
    viewmat, projmat = capi.f32(viewmat), capi.f32(projmat)
    cov3d = _empty((n, 6), torch.float32, means3d)
    xys = _empty((n, 2), torch.float32, means3d)
    depths = _empty((n,), torch.float32, means3d)
    radii = _empty((n,), torch.int32, means3d)
    conics = _empty((n, 3), torch.float32, means3d)
    nth = _empty((n,), torch.int32, means3d)
    capi.check(capi.lib().gsb_project_forward(
        n, capi.ptr(means3d), capi.ptr(scales), glob_scale, capi.ptr(quats), capi.ptr(viewmat),
        capi.ptr(projmat), fx, fy, cx, cy, img_height, img_width, tile_bounds_[0], tile_bounds_[1],
        clip_thresh, capi.ptr(cov3d), capi.ptr(xys), capi.ptr(depths), capi.ptr(radii), capi.ptr(conics),
        capi.ptr(nth), capi.stream()))
    return cov3d, xys, depths, radii, conics, nth


def project_gaussians_backward(means3d, scales, glob_scale, quats, viewmat, projmat, fx, fy, cx, cy,
                               img_height, img_width, cov3d, radii, conics, v_xy, v_depth, v_conic):
    n = means3d.shape[0]
    means3d, scales, quats = capi.f32(means3d), capi.f32(scales), capi.f32(quats)
    viewmat, projmat = capi.f32(viewmat), capi.f32(projmat)
    v_xy, v_conic = capi.f32(v_xy), capi.f32(v_conic)
    v_depth = capi.f32(v_depth) if v_depth is not None else None
    v_mean = _empty((n, 3), torch.float32, means3d)
    v_scale = _empty((n, 3), torch.float32, means3d)
    v_quat = _empty((n, 4), torch.float32, means3d)
    capi.check(capi.lib().gsb_project_backward(
        n, capi.ptr(means3d), capi.ptr(scales), glob_scale, capi.ptr(quats), capi.ptr(viewmat),
        capi.ptr(projmat), fx, fy, cx, cy, img_height, img_width, None, capi.ptr(radii.contiguous()),
        capi.ptr(capi.f32(conics)), capi.ptr(v_xy), capi.ptr(v_depth), capi.ptr(v_conic), capi.ptr(v_mean),
        capi.ptr(v_scale), capi.ptr(v_quat), capi.stream()))
    return v_mean, v_scale, v_quat


def cumsum_tiles_hit(num_tiles_hit):
    """torch::cumsum(numTilesHit, 0, kInt32) (rasterize_gaussians.cpp:62)."""
    n = num_tiles_hit.shape[0]
    num_tiles_hit = num_tiles_hit.contiguous()
    cum = _empty((n,), torch.int32, num_tiles_hit)
    L = capi.lib()
    wsb = L.gsb_cumsum_workspace_bytes(n)
    ws = _ws.get(num_tiles_hit.device, "cumsum", wsb)
    capi.check(L.gsb_cumsum_tiles_hit(n, capi.ptr(num_tiles_hit), capi.ptr(cum), capi.ptr(ws), ws.numel(),
                                      None, capi.stream()))
    return cum


def map_gaussian_to_intersects(num_points, num_intersects, xys, depths, radii, cum_tiles_hit, tile_bounds_):
    isect = _empty((num_intersects,), torch.int64, xys)
    gids = _empty((num_intersects,), torch.int32, xys)
    capi.check(capi.lib().gsb_map_gaussian_to_intersects(
        num_points, num_intersects, capi.ptr(capi.f32(xys)), capi.ptr(capi.f32(depths)),
        capi.ptr(radii.contiguous()), capi.ptr(cum_tiles_hit.contiguous()), tile_bounds_[0], tile_bounds_[1],
        capi.ptr(isect), capi.ptr(gids), capi.stream()))
    return isect, gids


def sort_intersects(isect_ids, num_tiles):
    """torch::sort(isectIds) (rasterize_gaussians.cpp:25-29): returns (sorted keys, int32 permutation)."""
    m = isect_ids.shape[0]
    ks = torch.empty_like(isect_ids)
    idx = _empty((m,), torch.int32, isect_ids)
    L = capi.lib()
    wsb = L.gsb_sort_workspace_bytes(m)
    ws = _ws.get(isect_ids.device, "sort", wsb + 256)
    off = (-ws.data_ptr()) % 256
    capi.check(L.gsb_sort_intersects(m, num_tiles, capi.ptr(isect_ids.contiguous()), capi.ptr(ks), capi.ptr(idx),
                                     ws.data_ptr() + off, ws.numel() - off, capi.stream()))
    return ks, idx


def gather_bin_edges(isect_ids_sorted, sorted_index, gaussian_ids, num_tiles):
    m = isect_ids_sorted.shape[0]
    gs = _empty((m,), torch.int32, isect_ids_sorted)
    bins = _empty((num_tiles, 2), torch.int32, isect_ids_sorted)
    capi.check(capi.lib().gsb_gather_bin_edges(m, num_tiles, capi.ptr(isect_ids_sorted), capi.ptr(sorted_index),
                                               capi.ptr(gaussian_ids), capi.ptr(gs), capi.ptr(bins),
                                               capi.stream()))
    return gs, bins


def binAndSortGaussians(numPoints, numIntersects, xys, depths, radii, cumTilesHit, tileBounds,
                        return_index=False):
    """rasterize_gaussians.cpp:6-37 -> (isectIds, gaussianIds, isectIdsSorted, gaussianIdsSorted, tileBins)."""
    isect, gids = map_gaussian_to_intersects(numPoints, numIntersects, xys, depths, radii, cumTilesHit,
                                             tileBounds)
    num_tiles = tileBounds[0] * tileBounds[1]
    ks, idx = sort_intersects(isect, num_tiles)
    gs, bins = gather_bin_edges(ks, idx, gids, num_tiles)
    if return_index:
        return isect, gids, ks, gs, bins, idx
    return isect, gids, ks, gs, bins


class BinPlan:
    """Capacities of the M-dependent buffers of the fast binning path, carried from frame to frame (grow-only
    high-water marks with headroom) so that a frame needs no host read-back before its kernels are enqueued:
    the kernels are sized by these capacities, raise stats[2] if a frame outgrows them, and the host checks the
    (asynchronous) read-back after enqueuing the whole forward pass.  One instance per device (operator layer) or
    per pipeline."""

    def __init__(self):
        self.m_cap = 0
        self.len_cap = 0
        self.host = None   # pinned int32[4]
        self.event = None

    def grow(self, m, max_len):
        if m > self.m_cap:
            self.m_cap = int(m * 1.25) + 4096
        if max_len > self.len_cap:
            want = max_len + max_len // 4
            cap = 64
            while cap < want:
                cap <<= 1
            if cap > 64 and cap < 256:
                cap = 256
            # never plan beyond what the in-shared-memory sort can take; longer lists go the generic way
            self.len_cap = min(cap, capi.lib().gsb_bucket_max_tile_len())

    def read_back(self, stats):
        """Enqueue the asynchronous D2H copy of the device stats; returns after recording the event."""
        if self.host is None:
            self.host = torch.zeros(4, dtype=torch.int32).pin_memory()
            self.event = torch.cuda.Event()
        self.host.copy_(stats, non_blocking=True)
        self.event.record()

    def wait(self):
        self.event.synchronize()
        m, max_len, overflow, _ = (int(v) for v in self.host.tolist())
        return m, max_len, bool(overflow)


_plans = {}


def _plan_for(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    p = _plans.get(key)
    if p is None:
        p = _plans[key] = BinPlan()
    return p


def bucket_tile_ranges(xys, radii, conics, colors, opacities, tile_bounds_, m_capacity, len_capacity, cull=True,
                       workspace=None):
    """Fast-path phase 1: per-Gaussian attribute records (kept in the workspace), cum_tiles_hit [n], tile_bins
    [T,2] and the device stats {M, longest tile list, overflow, 0}, without sorting and without a read-back."""
    n = xys.shape[0]
    T = tile_bounds_[0] * tile_bounds_[1]
    L = capi.lib()
    if workspace is None:
        workspace = torch.empty(L.gsb_bucket_workspace_bytes(n, m_capacity, T) + 256, dtype=torch.uint8,
                                device=xys.device)
    off = (-workspace.data_ptr()) % 256
    # tile_bins [T,2] followed by the longest-first tile order [T] in ONE tensor (rows 0..T-1 / the flat tail), so that
    # whoever holds the bins also holds the order the blend kernels should take the tiles in
    binord = _empty((3 * T,), torch.int32, xys)
    bins, order = binord[:2 * T].view(T, 2), binord[2 * T:]
    cum = _empty((n,), torch.int32, xys)
    stats = _empty((4,), torch.int32, xys)
    capi.check(L.gsb_bucket_tile_ranges(
        n, capi.ptr(capi.f32(xys)), capi.ptr(radii.contiguous()), capi.ptr(capi.f32(conics)),
        capi.ptr(capi.f32(colors)), capi.ptr(capi.f32(opacities)), 1 if cull else 0, tile_bounds_[0],
        tile_bounds_[1], m_capacity, len_capacity, workspace.data_ptr() + off, workspace.numel() - off,
        capi.ptr(cum), capi.ptr(bins), capi.ptr(order), capi.ptr(stats), capi.stream()))
    bins.tile_order = order
    return bins, cum, stats, workspace


def bucket_sort_pack(n, m_capacity, len_capacity, depths, radii, cum_tiles_hit, tile_bounds_, tile_bins, stats,
                     workspace, cull=True, want_index=False):
    """Fast-path phase 2: bucket emit + per-tile shared-memory sort + record pack -> records (+ optional
    sorted_index / gaussian_ids_sorted for inspection), sized by the capacities phase 1 was given."""
    L = capi.lib()
    off = (-workspace.data_ptr()) % 256
    records = torch.empty(L.gsb_raster_records_bytes(m_capacity), dtype=torch.uint8, device=depths.device)
    idx = _empty((m_capacity,), torch.int32, depths) if want_index else None
    gs = _empty((m_capacity,), torch.int32, depths) if want_index else None
    capi.check(L.gsb_bucket_sort_pack(
        n, m_capacity, len_capacity, capi.ptr(capi.f32(depths)), capi.ptr(radii.contiguous()),
        capi.ptr(cum_tiles_hit), 1 if cull else 0, tile_bounds_[0], tile_bounds_[1], capi.ptr(tile_bins),
        capi.ptr(stats), workspace.data_ptr() + off, workspace.numel() - off, capi.ptr(records), capi.ptr(idx),
        capi.ptr(gs), capi.stream()))
    return records, idx, gs


CLAMP_MAX_ONE = 1   # GSB_RASTER_CLAMP_MAX_ONE (include/gsplat_b200.h)


def rasterize_forward_packed(tile_bounds_, img_size, m_capacity, tile_bins, records, background, stats=None,
                             tile_order=None, flags=0):
    W, H = img_size[0], img_size[1]
    out = _empty((H, W, 3), torch.float32, records)
    fT = _empty((H, W), torch.float32, records)
    fI = _empty((H, W), torch.int32, records)
    if tile_order is None:
        tile_order = getattr(tile_bins, "tile_order", None)
    capi.check(capi.lib().gsb_rasterize_forward_packed(
        H, W, tile_bounds_[0], tile_bounds_[1], m_capacity, capi.ptr(tile_bins), capi.ptr(tile_order), capi.ptr(stats),
        capi.ptr(capi.f32(background)), capi.ptr(records), capi.ptr(out), capi.ptr(fT), capi.ptr(fI), int(flags),
        capi.stream()))
    return out, fT, fI


def rasterize_forward(tile_bounds_, img_size, gaussian_ids_sorted, sorted_index, tile_bins, xys, conics,
                      colors, opacities, background, flags=0):
    m = gaussian_ids_sorted.shape[0]
    L = capi.lib()
    records = torch.empty(L.gsb_raster_records_bytes(m), dtype=torch.uint8, device=xys.device)
    if colors.shape[-1] != 3:
        raise ValueError("only 3-channel colors are supported")  # the N-D path is dead code in OpenSplat
    capi.check(L.gsb_pack_records(
        m, capi.ptr(gaussian_ids_sorted), capi.ptr(sorted_index), capi.ptr(capi.f32(xys)),
        capi.ptr(capi.f32(conics)), capi.ptr(capi.f32(colors)), capi.ptr(capi.f32(opacities)), capi.ptr(records),
        capi.stream()))
    return rasterize_forward_packed(tile_bounds_, img_size, m, tile_bins, records, background, None, None,
                                    flags) + (records,)


def rasterize_backward(img_height, img_width, n, m, tile_bins, conics, opacities, records, cum_tiles_hit,
                       background, final_Ts, final_idx, v_output, v_output_alpha=None, tile_order=None, flags=0):
    L = capi.lib()
    tb = tile_bounds(img_width, img_height)
    rows = _ws.get(final_Ts.device, "grad_rows", L.gsb_raster_grad_rows_bytes(m) + 16)
    off = (-rows.data_ptr()) % 16
    v_xy = _empty((n, 2), torch.float32, final_Ts)
    v_conic = _empty((n, 3), torch.float32, final_Ts)
    v_colors = _empty((n, 3), torch.float32, final_Ts)
    v_opacity = _empty((n, 1), torch.float32, final_Ts)
    v_output = capi.f32(v_output)
    capi.check(L.gsb_rasterize_backward(
        img_height, img_width, tb[0], tb[1], n, m, capi.ptr(tile_bins), capi.ptr(tile_order), capi.ptr(capi.f32(conics)),
        capi.ptr(capi.f32(opacities)), capi.ptr(records), capi.ptr(cum_tiles_hit),
        capi.ptr(capi.f32(background)), capi.ptr(final_Ts), capi.ptr(final_idx),
        capi.ptr(v_output), capi.ptr(v_output_alpha) if v_output_alpha is not None else None,
        rows.data_ptr() + off, capi.ptr(v_xy), capi.ptr(v_conic), capi.ptr(v_colors), capi.ptr(v_opacity),
        int(flags), capi.stream()))
    return v_xy, v_conic, v_colors, v_opacity


# ------------------------------------------------------------------------------------------------
# autograd operators (names and slots as the reference)
# ------------------------------------------------------------------------------------------------
class ProjectGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, scales, globScale, quats, viewMat, projMat, fx, fy, cx, cy, imgHeight, imgWidth,
                tileBounds, clipThresh=0.01):
        cov3d, xys, depths, radii, conics, nth = project_gaussians_forward(
            means, scales, float(globScale), quats, viewMat, projMat, float(fx), float(fy), float(cx),
            float(cy), int(imgHeight), int(imgWidth), tileBounds, float(clipThresh))
        ctx.meta = (float(globScale), float(fx), float(fy), float(cx), float(cy), int(imgHeight), int(imgWidth))
        ctx.save_for_backward(means, scales, quats, viewMat, projMat, cov3d, radii, conics)
        ctx.mark_non_differentiable(radii, nth)
        return xys, depths, radii, conics, nth, cov3d  # project_gaussians.cpp:44

    @staticmethod
    def backward(ctx, v_xys, v_depths, v_radii, v_conics, v_numTiles, v_cov3d):
        means, scales, quats, viewMat, projMat, cov3d, radii, conics = ctx.saved_tensors
        gs, fx, fy, cx, cy, H, W = ctx.meta
        if v_xys is None:
            v_xys = torch.zeros_like(means[:, :2])
        if v_conics is None:
            v_conics = torch.zeros_like(conics)
        v_mean, v_scale, v_quat = project_gaussians_backward(
            means, scales, gs, quats, viewMat, projMat, fx, fy, cx, cy, H, W, cov3d, radii, conics, v_xys,
            v_depths, v_conics)
        # 14 slots, grads only for means(0), scales(1), quats(3)  (project_gaussians.cpp:75-89)
        return (v_mean, v_scale, None, v_quat) + (None,) * 10


class RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background):
        return RasterizeGaussians._forward(ctx, 0, xys, depths, radii, conics, numTilesHit, colors, opacity,
                                           imgHeight, imgWidth, background)

    @staticmethod
    def _forward(ctx, flags, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background):
        numPoints = xys.shape[0]
        tb = tile_bounds(imgWidth, imgHeight)
        if colors.shape[-1] != 3:
            raise ValueError("only 3-channel colors are supported")
        limit = capi.lib().gsb_bucket_max_tile_len()
        plan = _plan_for(xys.device)
        # Binning, packing and blending are enqueued with buffer capacities planned from earlier frames; the one
        # device->host read-back of the path (M, rasterize_gaussians.cpp:63) is waited for only AFTER the whole
        # forward pass has been enqueued, and a frame that outgrew the plan (or the first one) is simply redone.
        while True:
            m_cap, len_cap = plan.m_cap, plan.len_cap
            bins, cum, stats, ws = bucket_tile_ranges(xys, radii, conics, colors, opacity, tb, m_cap, len_cap)
            plan.read_back(stats)
            if m_cap > 0:
                records, _, _ = bucket_sort_pack(numPoints, m_cap, len_cap, depths, radii, cum, tb, bins, stats, ws)
                out, fT, fI = rasterize_forward_packed(tb, (imgWidth, imgHeight, 1), m_cap, bins, records,
                                                       background, stats, None, flags)
            numIntersects, max_len, overflow = plan.wait()
            if not overflow:
                if m_cap == 0:   # no plan yet and nothing on screen: background only
                    records = torch.empty(capi.lib().gsb_raster_records_bytes(0), dtype=torch.uint8,
                                          device=xys.device)
                    out, fT, fI = rasterize_forward_packed(tb, (imgWidth, imgHeight, 1), 0, bins, records, background,
                                                           None, None, flags)
                break
            if max_len <= limit:
                plan.grow(numIntersects, max_len)
                continue
            # pathological tile lists (longer than the in-shared-memory sort can take): generic global radix
            # sort (binAndSortGaussians) on the reference's own, unculled intersection lists
            cum = cumsum_tiles_hit(numTilesHit)
            m_cap = int(cum[-1])
            _, _, _, gs, bins, idx = binAndSortGaussians(numPoints, m_cap, xys, depths, radii, cum, tb,
                                                         return_index=True)
            out, fT, fI, records = rasterize_forward(tb, (imgWidth, imgHeight, 1), gs, idx, bins, xys, conics,
                                                     colors, opacity, background, flags)
            break
        ctx.meta = (int(imgHeight), int(imgWidth), numPoints, m_cap, flags)
        order = getattr(bins, "tile_order", None)
        ctx.has_order = order is not None
        ctx.save_for_backward(bins, conics, opacity, records, cum, background, fT, fI,
                              order if order is not None else bins)
        return out

    @staticmethod
    def backward(ctx, v_outImg):
        H, W, n, m, flags = ctx.meta
        bins, conics, opacity, records, cum, background, fT, fI, order = ctx.saved_tensors
        v_xy, v_conic, v_colors, v_opacity = rasterize_backward(H, W, n, m, bins, conics, opacity, records, cum,
                                                                background, fT, fI, v_outImg.contiguous(), None,
                                                                tile_order=order if ctx.has_order else None,
                                                                flags=flags)
        # 10 slots; grads for xys(0), conics(3), colors(5), opacity(6) (rasterize_gaussians.cpp:129-139)
        return v_xy, None, None, v_conic, None, v_colors, v_opacity, None, None, None


class RasterizeGaussiansClamped(RasterizeGaussians):
    """`clamp_max(RasterizeGaussians(...), 1)` (model.cpp:213-222) as ONE operator: the blend kernel's epilogue writes
    the clamped image and the backward kernel applies clamp_max's gradient mask (GSB_RASTER_CLAMP_MAX_ONE).  Same
    arguments and gradient slots as RasterizeGaussians.  C++ twin: gsb::RasterizeGaussiansClamped."""

    @staticmethod
    def forward(ctx, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background):
        return RasterizeGaussians._forward(ctx, CLAMP_MAX_ONE, xys, depths, radii, conics, numTilesHit, colors,
                                           opacity, imgHeight, imgWidth, background)


class ProjectGaussiansActivated(torch.autograd.Function):
    """ProjectGaussians on the RAW parameters of the model (model.cpp:148-150,200 + 152-165 as one operator):
    `scales` are log-scales (exp fused), `quats` un-normalised (the projection normalises), and the opacity logits
    ride along: returns (xys, depths, radii, conics, numTilesHit, cov3d, opacities [N,1] = sigmoid(logits)).
    Gradients come back w.r.t. the raw parameters.  C++ twin: gsb::ProjectGaussiansActivated."""

    @staticmethod
    def forward(ctx, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat, fx, fy, cx, cy,
                imgHeight, imgWidth, tileBounds, clipThresh=0.01):
        n = means.shape[0]
        m3, ls, rq = capi.f32(means), capi.f32(logScales), capi.f32(rawQuats)
        ol = capi.f32(opacityLogits).reshape(n)
        vm, pm = capi.f32(viewMat), capi.f32(projMat)
        cov3d = _empty((n, 6), torch.float32, m3)
        xys = _empty((n, 2), torch.float32, m3)
        depths = _empty((n,), torch.float32, m3)
        radii = _empty((n,), torch.int32, m3)
        conics = _empty((n, 3), torch.float32, m3)
        nth = _empty((n,), torch.int32, m3)
        opac = _empty((n, 1), torch.float32, m3)
        capi.check(capi.lib().gsb_project_forward_activated(
            n, capi.ptr(m3), capi.ptr(ls), float(globScale), capi.ptr(rq), capi.ptr(ol), capi.ptr(vm), capi.ptr(pm),
            float(fx), float(fy), float(cx), float(cy), int(imgHeight), int(imgWidth), tileBounds[0], tileBounds[1],
            float(clipThresh), capi.ptr(cov3d), capi.ptr(xys), capi.ptr(depths), capi.ptr(radii), capi.ptr(conics),
            capi.ptr(nth), capi.ptr(opac), capi.stream()))
        ctx.meta = (float(globScale), float(fx), float(fy), int(imgHeight), int(imgWidth), tuple(opacityLogits.shape))
        ctx.save_for_backward(m3, ls, rq, vm, pm, radii, conics, opac)
        ctx.mark_non_differentiable(radii, nth)
        return xys, depths, radii, conics, nth, cov3d, opac

    @staticmethod
    def backward(ctx, v_xys, v_depths, v_radii, v_conics, v_numTiles, v_cov3d, v_opac):
        m3, ls, rq, vm, pm, radii, conics, opac = ctx.saved_tensors
        gs, fx, fy, H, W, ol_shape = ctx.meta
        n = m3.shape[0]
        if v_xys is None:
            v_xys = torch.zeros_like(m3[:, :2])
        if v_conics is None:
            v_conics = torch.zeros_like(conics)
        v_mean = _empty((n, 3), torch.float32, m3)
        v_ls = _empty((n, 3), torch.float32, m3)
        v_rq = _empty((n, 4), torch.float32, m3)
        v_ol = _empty((n,), torch.float32, m3)
        vx, vc = capi.f32(v_xys), capi.f32(v_conics)
        vd = capi.f32(v_depths) if v_depths is not None else None
        vo = capi.f32(v_opac).reshape(n) if v_opac is not None else None
        capi.check(capi.lib().gsb_project_backward_activated(
            n, capi.ptr(m3), capi.ptr(ls), gs, capi.ptr(rq), capi.ptr(opac), capi.ptr(vm), capi.ptr(pm), fx, fy, H, W,
            capi.ptr(radii), capi.ptr(conics), capi.ptr(vx), capi.ptr(vd), capi.ptr(vc), capi.ptr(vo),
            capi.ptr(v_mean), capi.ptr(v_ls), capi.ptr(v_rq), capi.ptr(v_ol), capi.stream()))
        # 15 slots; grads for means(0), logScales(1), rawQuats(3), opacityLogits(4)
        return (v_mean, v_ls, None, v_rq, v_ol.reshape(ol_shape)) + (None,) * 10


class SphericalHarmonics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, degreesToUse, viewDirs, coeffs):
        degree = deg_from_sh(coeffs.shape[-2])
        ctx.meta = (int(degreesToUse), degree)
        ctx.save_for_backward(viewDirs)
        return compute_sh_forward(degree, int(degreesToUse), viewDirs, coeffs)

    @staticmethod
    def backward(ctx, v_colors):
        degreesToUse, degree = ctx.meta
        (viewDirs,) = ctx.saved_tensors
        return None, None, compute_sh_backward(degree, degreesToUse, viewDirs, v_colors.contiguous())


class SphericalHarmonicsRgb(torch.autograd.Function):
    """The colour pass of Model::forward without its ATen glue (model.cpp:176-177,186-192):
    rgbs = clamp_min(SH(degreesToUse, means - camPos, cat(featuresDc[:,None,:], featuresRest)) + 0.5, 0), reading the
    two feature tensors where they lie and writing their two gradients directly (gsb_sh_forward_split /
    gsb_sh_backward_split).  C++ twin: gsb::SphericalHarmonicsRgb (csrc/ops/fused_extras.hpp)."""

    @staticmethod
    def forward(ctx, degreesToUse, means, camPos, featuresDc, featuresRest):
        n = means.shape[0]
        degree = deg_from_sh(featuresRest.shape[-2] + 1)
        if featuresDc.shape != (n, 3) or featuresRest.dim() != 3 or featuresRest.shape[2] != 3:
            raise ValueError("featuresDc [N,3], featuresRest [N,K-1,3]")
        m, dc, rest = capi.f32(means), capi.f32(featuresDc), capi.f32(featuresRest)
        cp = capi.f32(torch.as_tensor(camPos).to(means.device)).reshape(3)
        rgbs = _empty((n, 3), torch.float32, m)
        capi.check(capi.lib().gsb_sh_forward_split(n, degree, int(degreesToUse), capi.ptr(m), capi.ptr(cp), capi.ptr(dc),
                                                   capi.ptr(rest), 0.5, capi.ptr(rgbs), capi.stream()))
        ctx.meta = (int(degreesToUse), degree, featuresRest.shape[-2])
        ctx.save_for_backward(m, cp, rgbs)
        return rgbs

    @staticmethod
    def backward(ctx, v_rgbs):
        use, degree, kr = ctx.meta
        m, cp, rgbs = ctx.saved_tensors
        n = m.shape[0]
        v_dc = _empty((n, 3), torch.float32, m)
        v_rest = _empty((n, kr, 3), torch.float32, m)
        capi.check(capi.lib().gsb_sh_backward_split(n, degree, use, capi.ptr(m), capi.ptr(cp), capi.ptr(rgbs),
                                                    capi.ptr(capi.f32(v_rgbs)), capi.ptr(v_dc), capi.ptr(v_rest),
                                                    capi.stream()))
        return None, None, None, v_dc, v_rest


class MainLoss(torch.autograd.Function):
    """Model::mainLoss (model.cpp:780-784): (1 - w) * L1 + w * (1 - SSIM), fused forward + gradient
    (gsb_ssim_l1_loss).  rendered, gt: [H,W,3] CUDA tensors.  Returns the scalar loss."""

    @staticmethod
    def forward(ctx, rendered, gt, ssimWeight):
        H, W = rendered.shape[0], rendered.shape[1]
        if rendered.dim() != 3 or rendered.shape[2] != 3 or gt.shape != rendered.shape:
            raise ValueError("rendered and gt must be [H,W,3]")
        L = capi.lib()
        r, g = capi.f32(rendered), capi.f32(gt)
        ws = _ws.get(r.device, "ssim", L.gsb_ssim_workspace_bytes(H, W) + 256)
        off = (-ws.data_ptr()) % 256
        v = torch.empty_like(r)
        out = torch.empty(3, dtype=torch.float32, device=r.device)
        capi.check(L.gsb_ssim_l1_loss(H, W, capi.ptr(r), capi.ptr(g), float(ssimWeight), capi.ptr(v), capi.ptr(out),
                                      ws.data_ptr() + off, ws.numel() - off, capi.stream()))
        ctx.save_for_backward(v)
        ctx.parts = out
        return out[0].clone()

    @staticmethod
    def backward(ctx, v_loss):
        (v,) = ctx.saved_tensors
        return v * v_loss, None, None


class ActivateGaussians(torch.autograd.Function):
    """Fused parameter activations of Model::forward (model.cpp:148-150,176-177,200):
    (means, log_scales, raw_quats, opacity_logits, cam_pos[3]) -> (scales, quats, opacities [N,1], viewdirs)."""

    @staticmethod
    def forward(ctx, means, log_scales, raw_quats, opacity_logits, cam_pos):
        n = means.shape[0]
        means, ls, rq = capi.f32(means), capi.f32(log_scales), capi.f32(raw_quats)
        ol = capi.f32(opacity_logits).reshape(-1)
        cp = capi.f32(torch.as_tensor(cam_pos).to(means.device)).reshape(3)   # a host tensor is accepted (as in C++)
        scales, quats = torch.empty_like(ls), torch.empty_like(rq)
        opac = torch.empty((n, 1), dtype=torch.float32, device=means.device)
        vd = torch.empty_like(means)
        capi.check(capi.lib().gsb_activate_forward(n, capi.ptr(means), capi.ptr(ls), capi.ptr(rq), capi.ptr(ol),
                                                   capi.ptr(cp), capi.ptr(scales), capi.ptr(quats), capi.ptr(opac),
                                                   capi.ptr(vd), capi.stream()))
        ctx.save_for_backward(scales, rq, opac)
        ctx.mark_non_differentiable(vd)
        return scales, quats, opac, vd

    @staticmethod
    def backward(ctx, v_scales, v_quats, v_opac, v_vd):
        scales, rq, opac = ctx.saved_tensors
        n = scales.shape[0]
        z = lambda t, like: capi.f32(t) if t is not None else torch.zeros_like(like)
        v_scales, v_quats, v_opac = z(v_scales, scales), z(v_quats, rq), z(v_opac, opac)
        v_ls, v_rq = torch.empty_like(scales), torch.empty_like(rq)
        v_ol = torch.empty_like(opac)
        capi.check(capi.lib().gsb_activate_backward(n, capi.ptr(scales), capi.ptr(rq), capi.ptr(opac),
                                                    capi.ptr(v_scales), capi.ptr(v_quats), capi.ptr(v_opac),
                                                    capi.ptr(v_ls), capi.ptr(v_rq), capi.ptr(v_ol), capi.stream()))
        return None, v_ls, v_rq, v_ol, None
