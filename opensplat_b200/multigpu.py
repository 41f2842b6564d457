"""Data-parallel (over camera views) gradient exchange on NVLink / NVSwitch, fused with the SH backward pass.

Baseline (parallel.allreduce_gradients): every rank runs sh_backward and then ONE NCCL all-reduce over the
flat 59-float/Gaussian gradient buffer (236 MB at 1M Gaussians, SH degree 3).

Fused path (this module): the same kernel (`sh_backward_multiview_kernel`, two CTA roles) either as ONE launch per step
(`exchange()`: `gsb_exchange_gradients` between two cross-rank barriers) or, in the pipeline, as its two roles on two
streams (`start_colour()` right after rasterize-backward, `finish()` after project-backward) so that the colour pulls
overlap project_backward and the geometry all-reduce:
 * the SH VJP is rank-1 in (view basis) x (colour gradient), so instead of reducing the 48 coefficient gradients
   per Gaussian every rank exposes only its view's colour gradient v_rgb [N,3] in symmetric (peer-mapped) memory
   and the kernel forms sum_r Y_r (x) v_rgb_r itself, pulling the peers' v_rgb over NVLink with coalesced loads
   while it computes;
 * the remaining 11 floats/Gaussian (means, scales, quats, opacity -- the prefix of the flat gradient buffer, which
   lives in the same symmetric allocation so the backward kernels write it in place) are all-reduced by the first
   CTAs of the same launch: two-shot, rank r owns slice r, with NVSwitch multicast one `multimem.ld_reduce` (sum
   formed inside the switch) and one `multimem.st` (broadcast) per 16 bytes; without multicast through the peers'
   mapped pointers.
NVLink bytes per rank per step at G ranks (N Gaussians): received (G-1) x 12 N (colour gradients) + 44 N
(reduced slice + broadcasts), sent the same -- against 2(G-1)/G x 236 N each way for the flat all-reduce
(G = 8: 128 MB instead of 413 MB at 1M Gaussians), and no separate sh_backward / NCCL kernels.

Camera centres: by default every rank's centre is gathered once, when the exchange is built (a caller that renders
the same view on every step, bench.py).  A trainer renders a different camera on every rank at every step: it calls
`set_camera()` before each backward pass, which copies the step's centre into a 16-byte trailer of this rank's
symmetric allocation, and from then on the launches use the `_cams` entry points, whose kernel reads every peer's
centre through the peer mapping, as it reads the colour gradients -- no collective on the step.  `degrees_to_use`
(the SH degree schedule) is passed through to the kernel; it defaults to the pipeline's full degree.

Several views per rank (`views_per_rank=B`, a trainer's B views of one step): the allocation holds B colour slots and
B centre trailers, and the launches expand all B x G views, ordered rank-major (view r*B + b), so that every replica
sums the same views in the same order; gradients are averaged over the B x G views.  `symmetric_layout` and
`view_pointers` hold the offset and pointer arithmetic.
"""
import os

import torch
import torch.distributed as dist

from . import capi


def symmetric_layout(numel, n, views_per_rank=1):
    """Float offsets of the symmetric allocation [flat gradients (numel) | B colour slots v_rgb [n,3] | B 16-byte
    centre trailers]: (rgb_off, cam_off, total).  The B slots are one contiguous [B,n,3] block (slot b at
    rgb_off + 3 n b), so that one gsb_mask_rgb_grad over n B floats triples masks them all; the block and every
    trailer start on a 16-byte boundary.  At B = 1 this is the single-view layout."""
    if numel < 0 or n < 0 or views_per_rank < 1:
        raise ValueError("symmetric_layout: numel >= 0, n >= 0 and views_per_rank >= 1")
    rgb_off = (numel + 3) // 4 * 4
    cam_off = rgb_off + (3 * n * views_per_rank + 3) // 4 * 4
    return rgb_off, cam_off, cam_off + 4 * views_per_rank


def view_pointers(bases, n, views_per_rank, rgb_off, cam_off):
    """Device addresses of every rank's B colour slots and B centre trailers, given each rank's base address of the
    allocation (`bases`, in rank order): two lists of G x B entries, rank-major (entry r B + b is rank r's view b)."""
    rgb = [base + 4 * (rgb_off + 3 * n * b) for base in bases for b in range(views_per_rank)]
    cam = [base + 4 * (cam_off + 4 * b) for base in bases for b in range(views_per_rank)]
    return rgb, cam


class ViewParallelExchange:
    def __init__(self, pipe, cam_pos=None, group=None, views_per_rank=1):
        """cam_pos: this rank's fixed camera centre(s) ([B,3], or [3] at B = 1), gathered from every rank once here;
        None when the caller passes each step's centres to set_camera() instead (a collective either way: every rank
        passes one or none).  views_per_rank: the B views every rank contributes per step; every rank must pass the
        same B (checked here, with one small all-gather)."""
        self.pipe = pipe
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.views = int(views_per_rank)
        if self.views < 1:
            raise ValueError("views_per_rank must be >= 1")
        dev = pipe.dev
        mine = torch.tensor([self.views], dtype=torch.int64, device=dev)
        every = torch.empty(self.world, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(every, mine, group=self.group)
        if bool((every != mine).any()):
            raise ValueError(f"ViewParallelExchange: the ranks disagree on views_per_rank ({every.tolist()})")
        self.num_views = self.world * self.views      # views expanded per step, rank-major
        self.cam_positions = None
        if cam_pos is not None:
            # every rank's camera centres (tiny, exchanged once)
            cp = torch.as_tensor(cam_pos, dtype=torch.float32, device=dev).reshape(self.views, 3)
            allcp = [torch.zeros_like(cp) for _ in range(self.world)]
            dist.all_gather(allcp, cp, group=self.group)
            self.cam_positions = torch.cat(allcp, 0).contiguous()
        self.per_step_cams = False   # set_camera() switches the launches to the peers' per-step centres
        self.use_multicast = os.environ.get("GSB_EXCHANGE_MULTICAST", "1") != "0"
        self.overlap = os.environ.get("GSB_EXCHANGE_OVERLAP", "1") != "0"
        self.side = torch.cuda.Stream(device=dev)
        self._rgb_ready, self._colour_done = torch.cuda.Event(), torch.cuda.Event()
        self._alloc_symmetric(pipe)

    def _alloc_symmetric(self, pipe):
        import torch.distributed._symmetric_memory as symm_mem
        dev, n = pipe.dev, pipe.n
        # ONE symmetric allocation: [flat gradient buffer | this rank's B colour gradients v_rgb [B,n,3] | this
        # step's B camera centres (3 floats of a 16-byte trailer each, read by the peers once set_camera() is used)]
        B = self.views
        rgb_off, cam_off, total = symmetric_layout(pipe.numel, n, B)
        t = symm_mem.empty(total, dtype=torch.float32, device=dev)
        t.zero_()
        hdl = symm_mem.rendezvous(t, self.group.group_name)
        self.buf, self.hdl = t, hdl
        pipe.rebind_grad_flat(t[:pipe.numel])
        self.v_rgb_views = t[rgb_off:rgb_off + 3 * n * B].view(B, n, 3)
        self.v_rgb = self.v_rgb_views[0]
        self.cams = t[cam_off:cam_off + 4 * B].view(B, 4)[:, :3]
        base_off = int(getattr(hdl, "offset", 0) or 0)      # the tensor's offset inside its symmetric allocation block
        ptrs = [int(p) + base_off for p in hdl.buffer_ptrs]
        self.geom_ptrs = torch.tensor(ptrs, dtype=torch.int64, device=dev)              # peers' flat buffers
        rgb_ptrs, cam_ptrs = view_pointers(ptrs, n, B, rgb_off, cam_off)
        self.rgb_ptrs = torch.tensor(rgb_ptrs, dtype=torch.int64, device=dev)
        self.cam_ptrs = torch.tensor(cam_ptrs, dtype=torch.int64, device=dev)   # peers' centres
        mc = int(getattr(hdl, "multicast_ptr", 0) or 0) if self.use_multicast else 0
        mc = mc + base_off if mc else 0
        assert ptrs[self.rank] == t.data_ptr(), "symmetric-memory handle does not describe this tensor"
        self.multicast_ptr = mc                                                           # 0: no NVSwitch multicast
        self.geom_numel = pipe.geom_numel   # means, scales, quats, opacities (16-byte aligned slices)
        assert self.geom_numel % 4 == 0

    def resize(self, pipe):
        """After a refinement changed the Gaussian count (collective: every rank refines in lock-step, see
        densify.Densifier.sync_stats): new symmetric buffers + rendezvous."""
        torch.cuda.current_stream().synchronize()
        dist.barrier(group=self.group)
        self._alloc_symmetric(pipe)

    def v_rgbs_buffer(self, b=0):
        """Where this step's rasterize-backward of view b must write its colour gradient."""
        return self.v_rgb_views[b]

    def set_camera(self, cam_pos_dev, b=0):
        """This step's camera centre of view b (a device float[3]): a stream-ordered device-to-device copy into this
        rank's trailer b, no host wait, no collective.  Call it for every view before every backward pass once it is
        used (a resize() leaves new, zeroed trailers).  Safe to overwrite: the previous step closed with
        barrier(channel=2), which every rank passes only after its multi-view kernel -- the last reader of the peers'
        trailers -- finished."""
        self.cams[b].copy_(cam_pos_dev)
        self.per_step_cams = True

    def _entry_points(self):
        """(multi-view SH backward, fused exchange, camera-centre argument): the `_cams` entry points with the peers'
        per-step centres once set_camera() has been called, otherwise the fixed centres gathered at construction
        (the two pairs take the same arguments)."""
        L = capi.lib()
        if self.per_step_cams:
            return L.gsb_sh_backward_multiview_cams, L.gsb_exchange_gradients_cams, self.cam_ptrs.data_ptr()
        if self.cam_positions is None:
            raise RuntimeError("ViewParallelExchange built without cam_pos: call set_camera() before the backward pass")
        return L.gsb_sh_backward_multiview, L.gsb_exchange_gradients, capi.ptr(self.cam_positions)

    def _mask(self, rgbs):
        """The clamp's gradient on all B colour slots, one launch: rgbs are the forward colours of this rank's B views
        (one contiguous [B,n,3] block; default the pipeline's [n,3] rgbs, B = 1)."""
        p = self.pipe
        rgbs = p.rgbs if rgbs is None else rgbs
        if rgbs.numel() != 3 * p.n * self.views or not rgbs.is_contiguous():
            raise ValueError(f"rgbs must be one contiguous [{self.views},{p.n},3] block")
        capi.check(capi.lib().gsb_mask_rgb_grad(p.n * self.views, capi.ptr(rgbs), capi.ptr(self.v_rgb_views),
                                                capi.stream()))

    def start_colour(self, average=True, degrees_to_use=None, rgbs=None):
        """Call right after rasterize-backward (v_rgb is final, the geometry gradients are not yet): masks v_rgb with
        the clamp's gradient and starts the multi-view SH backward -- the part of the exchange that moves most bytes,
        (G-1) x 12 B per Gaussian -- on a side stream, so that it overlaps project_backward and, afterwards, the
        all-reduce of the geometry gradients.  degrees_to_use: the SH degree schedule's (default: the full degree).
        average: scale both halves by 1/(B G), the mean over every view of the step.  rgbs: see _mask."""
        p = self.pipe
        multiview, _, cams = self._entry_points()
        use = p.deg if degrees_to_use is None else int(degrees_to_use)
        self._scale = 1.0 / self.num_views if average else 1.0
        cur = torch.cuda.current_stream()
        self._mask(rgbs)
        self._rgb_ready.record(cur)
        with torch.cuda.stream(self.side):
            self.side.wait_event(self._rgb_ready)
            self.hdl.barrier(channel=0)          # every rank's v_rgb (and camera centres) are complete
            capi.check(multiview(
                p.n, p.deg, use, capi.ptr(p.p["means"]), self.num_views, cams,
                self.rgb_ptrs.data_ptr(), self._scale, capi.ptr(p.g["coeffs"]), self.side.cuda_stream))
            self._colour_done.record(self.side)

    def finish(self, degrees_to_use=None):
        """Call after project_backward: all-reduces the geometry gradients (two-shot; NVSwitch multimem when mapped),
        joins the colour half and closes the step with the barrier that lets every rank overwrite its buffers."""
        p = self.pipe
        _, exchange, cams = self._entry_points()
        use = p.deg if degrees_to_use is None else int(degrees_to_use)
        self.hdl.barrier(channel=1)              # every rank's geometry gradients are complete
        capi.check(exchange(
            0, p.deg, use, None, 1, cams, None, self._scale, None, self.rank, self.world,
            self.geom_numel, self.geom_ptrs.data_ptr(), self.multicast_ptr if self.multicast_ptr else None,
            capi.stream()))
        torch.cuda.current_stream().wait_event(self._colour_done)
        # every rank's slice of the reduced geometry gradients has landed everywhere, and nobody still reads the v_rgb /
        # geometry buffers / camera trailers of this step (so the next step may overwrite them)
        self.hdl.barrier(channel=2)

    def exchange(self, average=True, degrees_to_use=None, rgbs=None):
        """The whole exchange after project_backward, as ONE fused launch (gsb_exchange_gradients: both CTA roles in one
        grid) between two barriers -- no overlap with the backward kernels; what callers use that cannot split the
        step (bench.py's operator-level e2e arm).  Arguments as start_colour."""
        p = self.pipe
        _, exchange, cams = self._entry_points()
        use = p.deg if degrees_to_use is None else int(degrees_to_use)
        scale = 1.0 / self.num_views if average else 1.0
        self._mask(rgbs)
        # every rank has finished writing this step's v_rgb, camera centres and geometry gradients
        self.hdl.barrier(channel=0)
        capi.check(exchange(
            p.n, p.deg, use, capi.ptr(p.p["means"]), self.num_views, cams,
            self.rgb_ptrs.data_ptr(), scale, capi.ptr(p.g["coeffs"]), self.rank, self.world, self.geom_numel,
            self.geom_ptrs.data_ptr(), self.multicast_ptr if self.multicast_ptr else None, capi.stream()))
        self.hdl.barrier(channel=2)
