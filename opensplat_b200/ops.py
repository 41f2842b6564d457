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
from typing import NamedTuple

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
    ws = _ws.get(num_tiles_hit.device, "cumsum", wsb + 256)
    off = (-ws.data_ptr()) % 256
    capi.check(L.gsb_cumsum_tiles_hit(n, capi.ptr(num_tiles_hit), capi.ptr(cum), ws.data_ptr() + off,
                                      ws.numel() - off, capi.stream()))
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
    per pipeline.  After wait(), `visible` holds stats[3]: the frame's count of Gaussians with radii > 0 when the
    binning was asked for it (GSB_BIN_COUNT_VISIBLE), else 0."""

    def __init__(self):
        self.m_cap = 0
        self.len_cap = 0
        self.visible = 0
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
        m, max_len, overflow, self.visible = (int(v) for v in self.host.tolist())
        return m, max_len, bool(overflow)


_plans = {}


def _plan_for(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    p = _plans.get(key)
    if p is None:
        p = _plans[key] = BinPlan()
    return p


BIN_COUNT_VISIBLE = 2   # GSB_BIN_COUNT_VISIBLE (include/gsplat_b200.h)


class BinFrame:
    """The binning of one frame and the state its backward pass reads.  bin_blend() enqueues the fast path (binning,
    per-tile sort + pack, blend) with the capacities of `plan`, waits once for the stats read-back, redoes a frame that
    outgrew the plan and takes tile lists longer than gsb_bucket_max_tile_len() through the generic global sort.  Then
    the frame holds `records`, `cum`, `tile_bins`, `tile_order` (`_ordered`: only the fast path blends in that order),
    `m_raster` (the intersection count the records are laid out for) and the frame's stats `m` / `max_len`; a frame
    blended with a depth output also holds `record_depths`, the per-record depth stream its backward reads.
    SplatPipeline is one frame reused from frame to frame; RasterizeGaussians builds one per call on the device's
    plan."""

    def __init__(self, plan, device):
        self.plan, self.dev, self.L = plan, torch.device(device), capi.lib()
        self.stats_dev = torch.empty(4, dtype=torch.int32, device=self.dev)
        self.m = self.max_len = self.m_raster = 0
        self.m_cap = -1   # the buffers are built by the first frame
        self.gids_sorted = self.record_depths = None   # depth output only, allocated by the first frame asking for it
        self._ordered = False
        self._ev = []     # stage events of the current step (SplatPipeline); a redone frame drops them

    def _stage(self, name):
        """A stage boundary of the frame: SplatPipeline records its stage events and NVTX ranges here."""

    def _grow(self, m_cap, n, T):
        """(Re)allocates the frame's buffers for n Gaussians, T tiles and an intersection capacity m_cap."""
        d, i32, u8 = self.dev, torch.int32, torch.uint8
        self.cum = torch.empty((n,), dtype=i32, device=d)
        self.tile_bins = torch.empty((T, 2), dtype=i32, device=d)
        self.tile_order = torch.empty((T,), dtype=i32, device=d)   # longest list first (fast path)
        self.records = torch.empty(self.L.gsb_raster_records_bytes(m_cap), dtype=u8, device=d)
        self.bucket_ws = torch.empty(self.L.gsb_bucket_workspace_bytes(n, m_cap, T) + 256, dtype=u8, device=d)
        self.m_cap = m_cap
        self.gids_sorted = self.record_depths = None

    def _depth_buffers(self, m):
        """The sorted Gaussian ids and the per-record depth stream of a depth frame, for at least m records."""
        if self.record_depths is None or self.record_depths.numel() < m:
            self.gids_sorted = torch.empty((max(m, 1),), dtype=torch.int32, device=self.dev)
            self.record_depths = torch.empty((max(m, 1),), dtype=torch.float32, device=self.dev)

    def bin_blend(self, xys, radii, conics, depths, nth, rgbs, opacities, background, out_img, final_Ts, final_idx,
                  flags, count_visible=False, out_depth=None, out_alpha=None, depth_values=None):
        """Binning, packing and the blend kernel of one frame (after SH colour and projection) into out_img [H,W,3],
        final_Ts and final_idx [H,W], with the frame's one host wait; returns out_img.  The per-Gaussian inputs are
        contiguous float32 / int32 CUDA tensors (nth: the projection's tile counts, read by the generic path only);
        flags: gsb_rasterize_forward_packed's; count_visible: have the binning count the Gaussians with radii > 0 into
        plan.visible.  out_depth / out_alpha ([H,W] float32, both or neither): the frame also writes the depth and
        opacity maps (DESIGN D18) through the DEPTH blend kernel, from the per-record depth stream it gathers from
        `depths` (kept in `record_depths` for the backward).  depth_values ([n] float32, default `depths`): the
        per-Gaussian value the depth map blends instead (DESIGN D23: 1/z); sorting and packing still read `depths`."""
        L, P, s, plan = self.L, capi.ptr, capi.stream(), self.plan
        depth = out_depth is not None
        if depth != (out_alpha is not None):
            raise ValueError("bin_blend: out_depth and out_alpha go together")
        values = depths if depth_values is None else depth_values
        n, H, W = xys.shape[0], out_img.shape[0], out_img.shape[1]
        tb = tile_bounds(W, H)
        T = tb[0] * tb[1]
        bin_flags = 1 | (BIN_COUNT_VISIBLE if count_visible else 0)
        limit = L.gsb_bucket_max_tile_len()
        # Everything below is sized by capacities planned from earlier frames and enqueued WITHOUT waiting for the
        # path's one device->host read-back (M, rasterize_gaussians.cpp:63): the host looks at it after the blend
        # kernel has been enqueued (the GPU never idles) and redoes a frame that outgrew the plan.
        while True:
            if plan.m_cap != self.m_cap:
                self._grow(plan.m_cap, n, T)
            m_cap, len_cap = plan.m_cap, plan.len_cap
            boff = (-self.bucket_ws.data_ptr()) % 256
            wsp, wsb = self.bucket_ws.data_ptr() + boff, self.bucket_ws.numel() - boff
            self._stage("scan")
            # cull = 1: bin only (Gaussian, tile) pairs whose extent box touches the tile
            capi.check(L.gsb_bucket_tile_ranges(n, P(xys), P(radii), P(conics), P(rgbs), P(opacities), bin_flags,
                                                tb[0], tb[1], m_cap, len_cap, wsp, wsb, P(self.cum), P(self.tile_bins),
                                                P(self.tile_order), P(self.stats_dev), s))
            plan.read_back(self.stats_dev)
            if depth:
                self._depth_buffers(m_cap)
            if m_cap > 0:
                self._stage("bucket_sort_pack")
                capi.check(L.gsb_bucket_sort_pack(n, m_cap, len_cap, P(depths), P(radii), P(self.cum), 1, tb[0],
                                                  tb[1], P(self.tile_bins), P(self.stats_dev), wsp, wsb,
                                                  P(self.records), None, P(self.gids_sorted) if depth else None, s))
            self._stage("raster_fwd")
            if depth:
                # the ids past M hold nothing valid: the gather reads M from the stats (no Gaussian: M = 0)
                if n > 0:
                    capi.check(L.gsb_gather_record_depths(m_cap, P(self.gids_sorted), P(values), P(self.stats_dev),
                                                          P(self.record_depths), s))
                capi.check(L.gsb_rasterize_forward_packed_depth(
                    H, W, tb[0], tb[1], m_cap, P(self.tile_bins), P(self.tile_order), P(self.stats_dev),
                    P(background), P(self.records), P(out_img), P(final_Ts), P(final_idx), flags,
                    P(self.record_depths), P(out_depth), P(out_alpha), s))
            else:
                capi.check(L.gsb_rasterize_forward_packed(H, W, tb[0], tb[1], m_cap, P(self.tile_bins),
                                                          P(self.tile_order), P(self.stats_dev), P(background),
                                                          P(self.records), P(out_img), P(final_Ts), P(final_idx),
                                                          flags, s))
            self._stage("end_fwd")
            self.m, self.max_len, overflow = plan.wait()
            if not overflow:
                self.m_raster, self._ordered = m_cap, True
                return out_img
            self._ev = []            # the frame is redone: drop its stage events
            if self.max_len > limit:
                break                # pathological tile lists: generic path below
            plan.grow(self.m, self.max_len)
        # ---- generic path: reference-exact global sort (binAndSortGaussians) of the unculled lists, with the M
        # read-back in the middle
        self._stage("generic_bin")
        cum = cumsum_tiles_hit(nth)
        m = self.m = int(cum[-1])
        if m > self.m_cap:
            self._grow(int(m * 1.25) + 1024, n, T)
            plan.m_cap = self.m_cap
        _, _, _, gids_sorted, self.tile_bins, sorted_index = binAndSortGaussians(n, m, xys, depths, radii, cum, tb,
                                                                                 return_index=True)
        self.cum = cum
        self._stage("raster_fwd")
        capi.check(L.gsb_pack_records(m, P(gids_sorted), P(sorted_index), P(xys), P(conics), P(rgbs), P(opacities),
                                      P(self.records), s))
        if depth:
            self._depth_buffers(m)
            capi.check(L.gsb_gather_record_depths(m, P(gids_sorted), P(values), None, P(self.record_depths), s))
            capi.check(L.gsb_rasterize_forward_packed_depth(
                H, W, tb[0], tb[1], m, P(self.tile_bins), None, None, P(background), P(self.records), P(out_img),
                P(final_Ts), P(final_idx), flags, P(self.record_depths), P(out_depth), P(out_alpha), s))
        else:
            capi.check(L.gsb_rasterize_forward_packed(H, W, tb[0], tb[1], m, P(self.tile_bins), None, None,
                                                      P(background), P(self.records), P(out_img), P(final_Ts),
                                                      P(final_idx), flags, s))
        self.m_raster, self._ordered = m, False
        self._stage("end_fwd")
        return out_img


def bucket_tile_ranges(xys, radii, conics, colors, opacities, tile_bounds_, m_capacity, len_capacity, cull=True,
                       workspace=None, count_visible=False):
    """Fast-path phase 1: per-Gaussian attribute records (kept in the workspace), cum_tiles_hit [n], tile_bins
    [T,2] and the device stats {M, longest tile list, overflow, visible}, without sorting and without a read-back.
    visible (the count of radii > 0) is 0 unless count_visible."""
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
        capi.ptr(capi.f32(colors)), capi.ptr(capi.f32(opacities)),
        (1 if cull else 0) | (BIN_COUNT_VISIBLE if count_visible else 0), tile_bounds_[0],
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
                       background, final_Ts, final_idx, v_output, v_output_alpha=None, tile_order=None, flags=0,
                       record_depths=None, v_output_depth=None):
    """-> (v_xy, v_conic, v_colors, v_opacity); given the frame's record_depths (a depth frame) the backward of the
    depth and opacity maps as well (gsb_rasterize_backward_depth, v_output_depth None == zeros), and v_depths [n]
    follows."""
    L = capi.lib()
    tb = tile_bounds(img_width, img_height)
    rows = _ws.get(final_Ts.device, "grad_rows", L.gsb_raster_grad_rows_bytes(m) + 16)
    off = (-rows.data_ptr()) % 16
    v_xy = _empty((n, 2), torch.float32, final_Ts)
    v_conic = _empty((n, 3), torch.float32, final_Ts)
    v_colors = _empty((n, 3), torch.float32, final_Ts)
    v_opacity = _empty((n, 1), torch.float32, final_Ts)
    v_output = capi.f32(v_output)
    if record_depths is not None:
        v_depths = _empty((n,), torch.float32, final_Ts)
        capi.check(L.gsb_rasterize_backward_depth(
            img_height, img_width, tb[0], tb[1], n, m, capi.ptr(tile_bins), capi.ptr(tile_order),
            capi.ptr(capi.f32(conics)), capi.ptr(capi.f32(opacities)), capi.ptr(records), capi.ptr(cum_tiles_hit),
            capi.ptr(capi.f32(background)), capi.ptr(final_Ts), capi.ptr(final_idx), capi.ptr(v_output),
            capi.ptr(capi.f32(v_output_alpha)) if v_output_alpha is not None else None, rows.data_ptr() + off,
            capi.ptr(v_xy), capi.ptr(v_conic), capi.ptr(v_colors), capi.ptr(v_opacity), int(flags),
            capi.ptr(record_depths), capi.ptr(capi.f32(v_output_depth)) if v_output_depth is not None else None,
            capi.ptr(v_depths), capi.stream()))
        return v_xy, v_conic, v_colors, v_opacity, v_depths
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
    def _forward(ctx, flags, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background,
                 depth=False, depth_values=None):
        """The forward of the rasterizer operators: the image, or with depth=True (image, depth map, alpha map); the
        depth map blends depth_values ([n], default depths) when given."""
        if colors.shape[-1] != 3:
            raise ValueError("only 3-channel colors are supported")
        xys, depths, conics, colors, opacity, background = (capi.f32(t) for t in (xys, depths, conics, colors,
                                                                                   opacity, background))
        if depth_values is not None:
            depth_values = capi.f32(depth_values).reshape(-1)
            if depth_values.shape[0] != xys.shape[0]:
                raise ValueError("depthValues must hold one value per Gaussian")
        H, W = int(imgHeight), int(imgWidth)
        out = _empty((H, W, 3), torch.float32, xys)
        fT = _empty((H, W), torch.float32, xys)
        fI = _empty((H, W), torch.int32, xys)
        od = _empty((H, W), torch.float32, xys) if depth else None
        oa = _empty((H, W), torch.float32, xys) if depth else None
        # one frame per call on the device's plan; the backward gets its tensors through save_for_backward
        f = BinFrame(_plan_for(xys.device), xys.device)
        f.bin_blend(xys, radii.contiguous(), conics, depths, numTilesHit, colors, opacity, background, out, fT, fI,
                    flags, out_depth=od, out_alpha=oa, depth_values=depth_values)
        ctx.meta = (H, W, xys.shape[0], f.m_raster, flags)
        ctx.depth_values = depth_values is not None
        ctx.save_for_backward(f.tile_bins, conics, opacity, f.records, f.cum, background, fT, fI,
                              f.tile_order if f._ordered else None, f.record_depths if depth else None)
        return (out, od, oa) if depth else out

    @staticmethod
    def backward(ctx, v_outImg):
        H, W, n, m, flags = ctx.meta
        bins, conics, opacity, records, cum, background, fT, fI, order, _ = ctx.saved_tensors
        v_xy, v_conic, v_colors, v_opacity = rasterize_backward(H, W, n, m, bins, conics, opacity, records, cum,
                                                                background, fT, fI, v_outImg.contiguous(), None,
                                                                tile_order=order, flags=flags)
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


class RasterizeGaussiansDepth(torch.autograd.Function):
    """RasterizeGaussians with the depth and opacity maps (DESIGN D18): same arguments, returns (rgb [H,W,3],
    depth [H,W], alpha [H,W]) with depth = sum alpha T z over the pairs the colour blend blends (z = `depths`, the
    projection's view-space depth; background depth 0, not normalised) and alpha = 1 - T_final.  rgb is bit-identical
    to RasterizeGaussians'.  Gradients go to xys (0), depths (1), conics (3), colors (5) and opacity (6), so a depth
    loss reaches the means through ProjectGaussians' depths output.
    With the optional trailing depthValues ([n], DESIGN D23: e.g. where(radii > 0, 1 / depths, 0)) the depth map
    blends v = depthValues in place of z: depth = sum alpha T v, with the tiles still sorted by `depths`.  Its gradient
    then goes to depthValues (slot 10) and none to depths; rgb, alpha and the other gradients are unchanged.  C++
    twin (without depthValues): gsb::RasterizeGaussiansDepth."""

    @staticmethod
    def forward(ctx, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background,
                depthValues=None):
        return RasterizeGaussians._forward(ctx, 0, xys, depths, radii, conics, numTilesHit, colors, opacity,
                                           imgHeight, imgWidth, background, depth=True, depth_values=depthValues)

    @staticmethod
    def backward(ctx, v_outImg, v_depth, v_alpha):
        H, W, n, m, flags = ctx.meta
        bins, conics, opacity, records, cum, background, fT, fI, order, rd = ctx.saved_tensors
        if v_outImg is None:
            v_outImg = torch.zeros((H, W, 3), dtype=torch.float32, device=fT.device)
        v_xy, v_conic, v_colors, v_opacity, v_depths = rasterize_backward(
            H, W, n, m, bins, conics, opacity, records, cum, background, fT, fI, v_outImg.contiguous(),
            v_alpha.contiguous() if v_alpha is not None else None, tile_order=order, flags=flags, record_depths=rd,
            v_output_depth=v_depth.contiguous() if v_depth is not None else None)
        if ctx.depth_values:    # 11 slots: the depth gradient belongs to depthValues (10), not to depths (1)
            return v_xy, None, None, v_conic, None, v_colors, v_opacity, None, None, None, v_depths.reshape(n)
        return v_xy, v_depths, None, v_conic, None, v_colors, v_opacity, None, None, None, None


class RasterizeGaussiansDepthClamped(RasterizeGaussiansDepth):
    """RasterizeGaussiansDepth with rgb = clamp_max(rgb, 1) fused as in RasterizeGaussiansClamped; depth and alpha are
    never clamped.  The same optional depthValues.  C++ twin (without depthValues): gsb::RasterizeGaussiansDepthClamped."""

    @staticmethod
    def forward(ctx, xys, depths, radii, conics, numTilesHit, colors, opacity, imgHeight, imgWidth, background,
                depthValues=None):
        return RasterizeGaussians._forward(ctx, CLAMP_MAX_ONE, xys, depths, radii, conics, numTilesHit, colors,
                                           opacity, imgHeight, imgWidth, background, depth=True,
                                           depth_values=depthValues)


class ProjectionMode(NamedTuple):
    """How the activated projection runs: antialiased (D19), filter3d (D24: the [N] float32 3-D filter, held constant)
    or None, and fisheye (D27: (k1, k2, k3, k4, theta_lim)) or None for a pinhole camera."""
    antialiased: bool = False
    filter3d: "torch.Tensor | None" = None
    fisheye: "tuple | None" = None


def project_activated_forward(L, mode, n, means, log_scales, glob_scale, quats, logits, viewmat, projmat, fx, fy, cx,
                              cy, img_h, img_w, tile_bounds, clip_thresh, out, stream):
    """The activated projection in `mode` through library L into out = (cov3d, xys, depths, radii, conics,
    num_tiles_hit, opacities), every buffer a contiguous CUDA tensor.  A fisheye camera does not read projmat."""
    P = capi.ptr
    head = (n, P(means), P(log_scales), glob_scale, P(quats), P(logits))
    tail = (img_h, img_w, tile_bounds[0], tile_bounds[1], clip_thresh) + tuple(P(t) for t in out)
    if mode.fisheye is not None:
        capi.check(L.gsb_project_forward_fisheye(*head, P(viewmat), fx, fy, cx, cy, *mode.fisheye, *tail,
                                                 int(mode.antialiased), stream))
    elif mode.filter3d is not None:
        capi.check(L.gsb_project_forward_activated_filter3d(*head, P(mode.filter3d), P(viewmat), P(projmat), fx, fy,
                                                            cx, cy, *tail, int(mode.antialiased), stream))
    else:
        project = L.gsb_project_forward_activated_aa if mode.antialiased else L.gsb_project_forward_activated
        capi.check(project(*head, P(viewmat), P(projmat), fx, fy, cx, cy, *tail, stream))


def project_activated_backward(L, mode, n, means, log_scales, glob_scale, quats, logits, sigmoid, viewmat, projmat,
                               fx, fy, img_h, img_w, radii, conics, v_xy, v_depth, v_conic, v_opacity, grads, stream,
                               accumulate=False, cam_grad=None, cam_partials=None):
    """The VJP of project_activated_forward in `mode` into grads = (v_means, v_log_scales, v_quats, v_logits), written,
    or added to them under `accumulate`.  sigmoid: the forward's opacities, read only by the pinhole projection without
    AA or the 3-D filter (every other mode recomputes them from the logits).  v_depth and v_opacity may be None.
    cam_grad (D22): (v_viewmat, v_projmat), [4,4] each, to receive the camera gradient, or None; cam_partials: its
    per-block rows, gsb_project_camera_partials_floats(n) floats, allocated here when None."""
    P = capi.ptr
    if cam_grad is not None and cam_partials is None:
        cam_partials = _empty((L.gsb_project_camera_partials_floats(n),), torch.float32, means)
    part = P(cam_partials) if cam_grad is not None else None
    plain = not mode.antialiased and mode.filter3d is None and mode.fisheye is None
    head = (n, P(means), P(log_scales), glob_scale, P(quats), P(sigmoid if plain else logits))
    tail = ((img_h, img_w, P(radii), P(conics), P(v_xy), P(v_depth), P(v_conic), P(v_opacity))
            + tuple(P(t) for t in grads))
    acc, aa = int(accumulate), int(mode.antialiased)
    if mode.fisheye is not None:
        capi.check(L.gsb_project_backward_fisheye(*head, P(viewmat), fx, fy, *mode.fisheye, *tail, acc, aa, part,
                                                  stream))
    elif mode.filter3d is not None:
        capi.check(L.gsb_project_backward_activated_filter3d(*head, P(mode.filter3d), P(viewmat), P(projmat), fx, fy,
                                                             *tail, acc, aa, int(cam_grad is not None), part, stream))
    elif cam_grad is not None:
        capi.check(L.gsb_project_backward_activated_camgrad(*head, P(viewmat), P(projmat), fx, fy, *tail, acc, aa, part,
                                                            stream))
    else:
        if mode.antialiased:
            project = L.gsb_project_backward_activated_aa_acc if acc else L.gsb_project_backward_activated_aa
        else:
            project = L.gsb_project_backward_activated_acc if acc else L.gsb_project_backward_activated
        capi.check(project(*head, P(viewmat), P(projmat), fx, fy, *tail, stream))
    if cam_grad is not None:
        capi.check(L.gsb_project_camera_grad_reduce(cam_partials.numel() // capi.CAMGRAD_TERMS, part,
                                                    P(cam_grad[0]), P(cam_grad[1]), stream))


class ProjectGaussiansActivated(torch.autograd.Function):
    """ProjectGaussians on the RAW parameters of the model (model.cpp:148-150,200 + 152-165 as one operator):
    `scales` are log-scales (exp fused), `quats` un-normalised (the projection normalises), and the opacity logits
    ride along: returns (xys, depths, radii, conics, numTilesHit, cov3d, opacities [N,1] = sigmoid(logits)).
    Gradients come back w.r.t. the raw parameters, and w.r.t. viewMat and projMat when those require grad (DESIGN
    D22: the exact VJP summed over the visible Gaussians, reduced inside the projection backward; row 3 of the
    viewMat gradient and row 2 of the projMat gradient are 0, as the projection does not read them).  C++ twin:
    gsb::ProjectGaussiansActivated (without the camera gradient).  filter3D (DESIGN D24): an optional [N] float32
    3-D filter (filter3d.compute_filter3d), held constant: the covariance is built from sqrt(exp(a)^2 globScale^2 + f^2)
    and the opacity is multiplied by c3; without it the operator runs exactly as before."""

    @staticmethod
    def forward(ctx, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat, fx, fy, cx, cy,
                imgHeight, imgWidth, tileBounds, clipThresh=0.01, filter3D=None):
        return ProjectGaussiansActivated._forward(ctx, False, means, logScales, globScale, rawQuats, opacityLogits,
                                                  viewMat, projMat, fx, fy, cx, cy, imgHeight, imgWidth, tileBounds,
                                                  clipThresh, filter3D)

    @staticmethod
    def _forward(ctx, aa, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat, fx, fy, cx, cy,
                 imgHeight, imgWidth, tileBounds, clipThresh, filter3D=None, fisheye=None):
        """The forward of every activated operator: projMat is None through a fisheye camera."""
        n = means.shape[0]
        m3, ls, rq = capi.f32(means), capi.f32(logScales), capi.f32(rawQuats)
        ol = capi.f32(opacityLogits).reshape(n)
        vm, pm = capi.f32(viewMat), capi.f32(projMat) if projMat is not None else None
        f3 = None
        if filter3D is not None:
            # D24: the 3-D filter, a constant [N] float32 (no gradient)
            if filter3D.dtype != torch.float32 or tuple(filter3D.shape) != (n,) or filter3D.device != m3.device:
                raise ValueError(f"filter3D must be a float32 [{n}] tensor on the means' device")
            f3 = filter3D.detach().contiguous()
        cov3d = _empty((n, 6), torch.float32, m3)
        xys = _empty((n, 2), torch.float32, m3)
        depths = _empty((n,), torch.float32, m3)
        radii = _empty((n,), torch.int32, m3)
        conics = _empty((n, 3), torch.float32, m3)
        nth = _empty((n,), torch.int32, m3)
        opac = _empty((n, 1), torch.float32, m3)
        project_activated_forward(capi.lib(), ProjectionMode(aa, f3, fisheye), n, m3, ls, float(globScale), rq, ol, vm,
                                  pm, float(fx), float(fy), float(cx), float(cy), int(imgHeight), int(imgWidth),
                                  tileBounds, float(clipThresh), (cov3d, xys, depths, radii, conics, nth, opac),
                                  capi.stream())
        ctx.meta = (float(globScale), float(fx), float(fy), int(imgHeight), int(imgWidth), tuple(opacityLogits.shape),
                    aa, fisheye)
        ctx.save_for_backward(m3, ls, rq, ol, opac, vm, pm, radii, conics, f3)
        ctx.mark_non_differentiable(radii, nth)
        return xys, depths, radii, conics, nth, cov3d, opac

    @staticmethod
    def backward(ctx, v_xys, v_depths, v_radii, v_conics, v_numTiles, v_cov3d, v_opac):
        m3, ls, rq, ol, opac, vm, pm, radii, conics, f3 = ctx.saved_tensors
        gs, fx, fy, H, W, ol_shape, aa, fisheye = ctx.meta
        n = m3.shape[0]
        if v_xys is None:
            v_xys = torch.zeros_like(m3[:, :2])
        if v_conics is None:
            v_conics = torch.zeros_like(conics)
        v_mean = _empty((n, 3), torch.float32, m3)
        v_ls = _empty((n, 3), torch.float32, m3)
        v_rq = _empty((n, 4), torch.float32, m3)
        v_ol = _empty((n,), torch.float32, m3)
        vd = capi.f32(v_depths) if v_depths is not None else None
        vo = capi.f32(v_opac).reshape(n) if v_opac is not None else None
        want_view, want_proj = ctx.needs_input_grad[5], ctx.needs_input_grad[6]
        cam = (_empty((4, 4), torch.float32, m3), _empty((4, 4), torch.float32, m3)) if want_view or want_proj else None
        project_activated_backward(capi.lib(), ProjectionMode(aa, f3, fisheye), n, m3, ls, gs, rq, ol, opac, vm, pm, fx,
                                   fy, H, W, radii, conics, capi.f32(v_xys), vd, capi.f32(v_conics), vo,
                                   (v_mean, v_ls, v_rq, v_ol), capi.stream(), cam_grad=cam)
        v_view = cam[0].reshape(vm.shape) if want_view else None
        v_proj = cam[1].reshape(pm.shape) if want_proj else None
        # 16 slots; grads for means(0), logScales(1), rawQuats(3), opacityLogits(4), viewMat(5), projMat(6)
        return (v_mean, v_ls, None, v_rq, v_ol.reshape(ol_shape), v_view, v_proj) + (None,) * 9


class ProjectGaussiansActivatedAntialiased(ProjectGaussiansActivated):
    """ProjectGaussiansActivated with the anti-aliased opacity (DESIGN D19, gsplat's "antialiased" mode): the same
    arguments and outputs, but opacities = sigmoid(logits) * sqrt(max(0, det0 / det)), det0 / det the determinants of
    the screen covariance before / after the 0.3 px^2 blur (0 for a culled Gaussian), so that a Gaussian smaller than a
    pixel is not drawn brighter than it is.  The other six outputs are those of ProjectGaussiansActivated, bit for bit.
    C++ twin: gsb::ProjectGaussiansActivatedAntialiased."""

    @staticmethod
    def forward(ctx, means, logScales, globScale, rawQuats, opacityLogits, viewMat, projMat, fx, fy, cx, cy,
                imgHeight, imgWidth, tileBounds, clipThresh=0.01, filter3D=None):
        return ProjectGaussiansActivated._forward(ctx, True, means, logScales, globScale, rawQuats, opacityLogits,
                                                  viewMat, projMat, fx, fy, cx, cy, imgHeight, imgWidth, tileBounds,
                                                  clipThresh, filter3D)


class ProjectGaussiansFisheye(torch.autograd.Function):
    """ProjectGaussiansActivated through an OpenCV fisheye camera (DESIGN D27, gsb_project_forward_fisheye): the same
    outputs, with the pixel centre and the EWA Jacobian of the Kannala-Brandt map of the view-space mean.  k: the four
    distortion coefficients (k1, k2, k3, k4); thetaLim: model.fisheye_theta_limit(*k), beyond which a Gaussian is
    culled.  antialiased: the opacity of ProjectGaussiansActivatedAntialiased.  Gradients come back w.r.t. the raw
    parameters, and w.r.t. viewMat when it requires grad (there is no projMat)."""

    @staticmethod
    def forward(ctx, means, logScales, globScale, rawQuats, opacityLogits, viewMat, fx, fy, cx, cy, k, thetaLim,
                imgHeight, imgWidth, tileBounds, clipThresh=0.01, antialiased=False):
        k = tuple(float(x) for x in k)
        if len(k) != 4:
            raise ValueError("k takes the four fisheye coefficients (k1, k2, k3, k4)")
        return ProjectGaussiansActivated._forward(ctx, bool(antialiased), means, logScales, globScale, rawQuats,
                                                  opacityLogits, viewMat, None, fx, fy, cx, cy, imgHeight, imgWidth,
                                                  tileBounds, clipThresh, fisheye=k + (float(thetaLim),))

    @staticmethod
    def backward(ctx, *grads):
        # 17 slots; grads for means(0), logScales(1), rawQuats(3), opacityLogits(4), viewMat(5) (slot 6 is fx)
        return ProjectGaussiansActivated.backward(ctx, *grads)[:6] + (None,) * 11


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
    (gsb_ssim_l1_loss).  rendered, gt: [H,W,3] CUDA tensors.  Returns the scalar loss.  mask (DESIGN D26): an optional
    uint8 or bool [H,W] tensor on rendered's device; the loss is then taken over its nonzero (used) pixels only
    (gsb_ssim_l1_loss_masked), and the gradient is 0 on the others."""

    @staticmethod
    def forward(ctx, rendered, gt, ssimWeight, mask=None):
        H, W = rendered.shape[0], rendered.shape[1]
        if rendered.dim() != 3 or rendered.shape[2] != 3 or gt.shape != rendered.shape:
            raise ValueError("rendered and gt must be [H,W,3]")
        if mask is not None:
            if (not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.uint8, torch.bool)
                    or tuple(mask.shape) != (H, W) or mask.device != rendered.device):
                raise ValueError(f"mask must be a uint8 or bool [{H},{W}] tensor on {rendered.device}")
            mask = mask.contiguous()
            mask = mask.view(torch.uint8) if mask.dtype == torch.bool else mask
        L = capi.lib()
        r, g = capi.f32(rendered), capi.f32(gt)
        ws = _ws.get(r.device, "ssim", L.gsb_ssim_workspace_bytes(H, W) + 256)
        off = (-ws.data_ptr()) % 256
        v = torch.empty_like(r)
        out = torch.empty(3, dtype=torch.float32, device=r.device)
        if mask is None:
            capi.check(L.gsb_ssim_l1_loss(H, W, capi.ptr(r), capi.ptr(g), float(ssimWeight), capi.ptr(v),
                                          capi.ptr(out), ws.data_ptr() + off, ws.numel() - off, capi.stream()))
        else:
            capi.check(L.gsb_ssim_l1_loss_masked(H, W, capi.ptr(r), capi.ptr(g), capi.ptr(mask), float(ssimWeight),
                                                 capi.ptr(v), capi.ptr(out), ws.data_ptr() + off, ws.numel() - off,
                                                 capi.stream()))
        ctx.save_for_backward(v)
        ctx.parts = out
        return out[0].clone()

    @staticmethod
    def backward(ctx, v_loss):
        (v,) = ctx.saved_tensors
        return v * v_loss, None, None, None


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


class BilateralGridSlice(torch.autograd.Function):
    """One image's bilateral grid applied to an image (DESIGN D21; gsb_bilagrid_slice_forward / _backward):
    (grid [12,L,Y,X] in F.grid_sample's order, rgb [H,W,3]) -> out [H,W,3] = A rgb + b with the coefficients
    trilinearly interpolated at the pixel's position and luma, not clamped.  Both inputs get gradients."""

    @staticmethod
    def forward(ctx, grid, rgb):
        shape = (capi.BILAGRID_COEFFS, capi.BILAGRID_L, capi.BILAGRID_Y, capi.BILAGRID_X)
        if tuple(grid.shape) != shape or rgb.dim() != 3 or rgb.shape[2] != 3:
            raise ValueError(f"grid must be {list(shape)} and rgb [H,W,3]")
        H, W = rgb.shape[0], rgb.shape[1]
        g = capi.f32(grid).permute(1, 2, 3, 0).contiguous()
        r = capi.f32(rgb)
        out = torch.empty_like(r)
        capi.check(capi.lib().gsb_bilagrid_slice_forward(H, W, capi.ptr(g), capi.ptr(r), capi.ptr(out),
                                                         capi.stream()))
        ctx.save_for_backward(g, r)
        return out

    @staticmethod
    def backward(ctx, v_out):
        g, r = ctx.saved_tensors
        H, W = r.shape[0], r.shape[1]
        L = capi.lib()
        ws = _ws.get(r.device, "bilagrid", L.gsb_bilagrid_workspace_bytes(H, W) + 256)
        off = (-ws.data_ptr()) % 256
        v_rgb = torch.empty_like(r)
        v_grid = torch.zeros_like(g)
        capi.check(L.gsb_bilagrid_slice_backward(H, W, capi.ptr(g), capi.ptr(r), capi.ptr(capi.f32(v_out)), 1.0,
                                                 capi.ptr(v_rgb), capi.ptr(v_grid), ws.data_ptr() + off,
                                                 ws.numel() - off, capi.stream()))
        return v_grid.permute(3, 0, 1, 2), v_rgb


class BilateralGridTV(torch.autograd.Function):
    """The total variation of bilateral grids [N,12,L,Y,X] (DESIGN D21; gsb_bilagrid_tv): the sum over the axes X, Y
    and L of the mean squared difference of neighbours along that axis, each mean over all N grids.  Returns the
    scalar TV."""

    @staticmethod
    def forward(ctx, grids):
        if grids.dim() != 5 or tuple(grids.shape[1:]) != (capi.BILAGRID_COEFFS, capi.BILAGRID_L, capi.BILAGRID_Y,
                                                          capi.BILAGRID_X):
            raise ValueError("grids must be [N,12,L,Y,X]")
        g = capi.f32(grids).permute(0, 2, 3, 4, 1).contiguous()
        v = torch.empty_like(g)
        out = torch.empty((), dtype=torch.float32, device=g.device)
        capi.check(capi.lib().gsb_bilagrid_tv(g.shape[0], capi.ptr(g), 1.0, capi.ptr(v), capi.ptr(out),
                                              capi.stream()))
        ctx.save_for_backward(v)
        return out

    @staticmethod
    def backward(ctx, v_tv):
        (v,) = ctx.saved_tensors
        return v.permute(0, 4, 1, 2, 3) * v_tv
