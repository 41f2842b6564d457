"""One step of the reference's training loop (opensplat.cpp:151-170: Model::forward, mainLoss, backward,
optimizersStep, schedulersStep, afterTrain) over the flat parameter / gradient / Adam-moment buffers of
pipeline.SplatPipeline, without autograd:

    trainer = SplatTrainer(params, cfg)        # the arguments of model.GaussianModel
    for step in range(1, steps + 1):
        loss = trainer.step(cam, gt, step)     # device tensor {total, L1, SSIM}; never read on the host here

It runs the kernels model.GaussianModel runs, with the same camera and learning-rate code, in the same order except
that a view's densification statistics are taken right after its backward pass (they read only the view's xys
gradient and radii, which nothing later in the step writes), so the two follow the same trajectory (same Gaussian counts, and
at one view per step without a group the same parameter and moment bits: the segmented Adam rounds every float as
gsb_adam_step does, see include/gsplat_b200.h).  What changes is the bookkeeping
around them: one segmented Adam launch instead of six, no autograd nodes, and one host wait per step (the binning read-back, whose stats[3] visible count replaces the
`radii.sum() == 0` test of model.cpp:173).  Between refinements a step allocates no device memory; a refinement
(densify.Densifier, unchanged) re-creates the flat layout through SplatPipeline.resize_gaussians.

Several views per step (`views_per_step=B`, with or without a group):

    trainer = SplatTrainer(params, cfg, views_per_step=4)
    loss = trainer.step([cam_a, cam_b, cam_c, cam_d], gts, step)   # gts: B [H,W,3] images or [B,H,W,3]; loss [B,3]

One step body serves every B; B = 1 is the default.  All B views render at the step's one resolution: one upload of
the B cameras and the SH forward for the B camera centres; then each view runs projection, binning (its own host
wait), blend, loss, rasterize-backward into its own colour slot, projection backward (the writing kernel for view 0,
gsb_project_backward_activated_acc after it, so the geometry gradients sum over the views in place) and its
densification statistics (densify.Densifier.accumulate_view, in view order); then the SH backward of the B colour
gradients, one segmented Adam launch and the rest of Model::afterTrain (Densifier.finish_step).  Adam sees the mean
over the B x G views (G ranks, 1 without a group).  The schedules (SH degree, downscale, means learning rate,
refinement, alpha reset) advance once per step, not per view, and no learning rate is scaled with B.  Between
refinements a step allocates nothing and waits on the host once per view.

At B = 1 three launches differ, so that a one-view step keeps the kernels whose results match model.GaussianModel's:
the SH forward is gsb_sh_forward_rgb_cam instead of gsb_sh_forward_rgb_cam_multiview; `proj @ view` is the 2-D matmul
GaussianModel forms (a batched matmul is a different cuBLAS call, not shown to give the same bits); and without a
group the SH backward is gsb_sh_backward_rgb_cam, whose coefficient gradients are those of the split kernels
GaussianModel runs, instead of gsb_mask_rgb_grad plus one launch of the exchange kernel, which expands the B colour
gradients with other roundings and scales the geometry prefix by 1/B.

A view that hits nothing adds zero gradients but counts in the divisor.  In one process a step whose views all hit
nothing trains nothing (model.cpp:173-174: no Adam step, no statistics), and a lone such view runs no backward pass.

Data-parallel over camera views (`group=` a process group, one process per GPU, B views per rank per step):

    trainer = SplatTrainer(params, cfg, group=dist.group.WORLD)
    loss = trainer.step(cams[(step - 1 + rank) % V], gt, step)

Every rank holds the same replica.  The backward pass runs on multigpu.ViewParallelExchange: rasterize-backward writes
each view's colour gradient into its slot of the symmetric buffer, the fused multi-view SH backward expands every
rank's colour gradients with that rank's camera centres for this step (set_camera: the centres travel through the
peer mapping too) and the geometry gradients are all-reduced by the same launch, all between symmetric-memory barriers
-- no NCCL kernel on the step.  The SH backward is the same for every B.  Every replica takes the same segmented Adam
step, so the replicas stay bit-identical; the statistics of a refinement are reduced by Densifier.sync_stats.  With
more than one rank, a rank whose views hit nothing runs the backward pass (exact zeros), contributes zero statistics
and takes every collective, as model.GaussianModel does under a group (parallel.allreduce_tensor_grads,
Densifier.after_train).  Between refinements a step still allocates nothing and waits on the host once per view (the
barriers are device-side).

Under a Gaussian budget (`cfg=mcmc.MCMCConfig(...)`, DESIGN D20) the step takes no densification statistics; the
regularisers' gradients are added after the views are averaged and exchanged, and after Adam mcmc.MCMCRefiner
relocates and grows the set on a refinement step and adds the position noise.  Every draw is keyed by (seed, step,
index), so replicas stay identical without a collective.

With per-image appearance grids (`appearance=appearance.AppearanceConfig(num_images=...)`, DESIGN D21) every step
names its views' training images (`step(cam, gt, step, image=i)`).  The step first writes the grids' TV gradient;
each view's clamped render is sliced through its image's grid before the loss, and the slice backward turns the loss
gradient into the render's gradient and adds 1/B of the grid gradient; after the Gaussians' Adam step one Adam step
updates every grid.  evaluate(), render() and `image` stay the raw render.

With per-image pose corrections (`pose=pose.PoseConfig(num_images=...)`, DESIGN D22) every step names its views'
training images the same way.  Each view's camera is corrected on the device (gsb_pose_apply) between the upload and
`proj @ view`; the step first writes reg * e into the corrections' gradient, each view's projection backward also
reduces the camera gradient (gsb_project_backward_activated_camgrad, gsb_project_camera_grad_reduce), which
gsb_pose_backward takes to 1/B of its image's correction gradient; after the Gaussians' Adam step one Adam step
updates every correction.  evaluate() and render() take image= to render at that image's corrected pose.

With per-image inverse-depth priors (`depth=depth.DepthConfig()`, DESIGN D23) a step may give each view a prior
(`step(cam, gt, step, depth=P)`).  A view with one also renders R = sum alpha T (1/z) through the depth blend (the
tiles still sorted by z; the colour is the same bits), takes the masked L1 against P after the colour loss
(gsb_inverse_depth_l1, weighted by depth.depth_weight), and its backward adds the depth term to the blend's geometry
gradients and, through gsb_inverse_depths_backward, to the projection's depth; densification statistics and a pose
correction's gradient see it too.  A view without one issues exactly the launches of a plain trainer.  The loss
returned stays the image loss; `depth_losses` holds the unweighted depth loss of each view.

With Mip-Splatting's 3-D smoothing filter (`filter3d=filter3d.Filter3DConfig(cameras=...)`, DESIGN D24) every
projection, forward and backward, in step(), evaluate() and render(), takes the per-Gaussian filter f
(gsb_project_*_activated_filter3d).  f is computed from the training cameras, uploaded once, at construction, after
every step whose refinement ran and on filter3d.recompute_due's schedule once refinement has stopped; the alpha reset
clamps the effective opacity, and save() writes the baked scene.  With pose corrections f uses the cameras as given,
uncorrected.  Under a group every rank computes the same f from the same cameras (no collective).

With AbsGS's absolute gradients (`cfg=densify.RefineConfig(absgrad=True, densify_grad_thresh=0.0008)`, DESIGN D25)
each view's rasterize-backward is gsb_rasterize_backward_absgrad, which also writes the per-Gaussian sum of each
pixel's |contribution| to the 2-D mean's gradient (v_xy_abs), and the view's densification statistics take it in
place of v_xy.  The launch count, every gradient and the Adam step are those of a plain trainer."""
import ctypes as C

import torch

from . import capi, ops
from .densify import Densifier, RefineConfig
from .export import SceneWriter
from .appearance import Appearance, to_gsplat_order
from .pose import Poses
from .depth import DepthConfig, depth_weight
from .filter3d import Filter3DConfig, bake, camera_table, compute_filter3d, recompute_due
from .mcmc import MCMCConfig, MCMCRefiner
from .model import (LEARNING_RATES, MEANS_LR_INIT, PARAM_NAMES, Camera, camera_setup, downscale_factor,
                    means_learning_rate)
from .parallel import flat_views
from .pipeline import SplatPipeline


def adam_segments(offs, lr):
    """Segment table of gsb_adam_step_segments for the flat layout `offs` (parallel.flat_layout) and the reference's
    six learning rates `lr` (keyed like model.LEARNING_RATES): one (offset, count, row_floats, head_floats, lr_head,
    lr_rest) per slice.  The merged SH block [n,K,3] gives featuresDc the first 3 floats of every 3K-float row and
    featuresRest the rest."""
    segs = []
    for name, (o, c, shp) in offs.items():
        row = 1
        for d in shp[1:]:
            row *= d
        if name == "coeffs":
            segs.append((o, c, row, 3, lr["featuresDc"], lr["featuresRest"]))
        else:
            segs.append((o, c, row, row, lr[name], lr[name]))
    return segs


def _split_coeffs(views):
    """Copies of the reference's six tensors from flat-layout views (featuresDc / featuresRest cut out of coeffs)."""
    c = views["coeffs"]
    out = {k: views[k].clone() for k in ("means", "scales", "quats", "opacities")}
    out["featuresDc"] = c[:, 0, :].clone(memory_format=torch.contiguous_format)
    out["featuresRest"] = c[:, 1:, :].clone(memory_format=torch.contiguous_format)
    return {k: out[k] for k in PARAM_NAMES}


def check_images(image, views, num_images):
    """The step's training-image indices as a list of `views` ints; raises ValueError unless image= names `views`
    images in [0, num_images).  Shared by the per-image features (appearance grids, pose corrections)."""
    if image is None:
        raise ValueError("a step with per-image appearance grids or pose corrections needs image= (the training "
                         "image of each view)")
    if isinstance(image, (list, tuple)):
        idx = list(image)
    elif views == 1:
        idx = [image]
    else:
        raise ValueError(f"image= must be a sequence of {views} training images")
    if len(idx) != views:
        raise ValueError(f"image= must name {views} training images, got {len(idx)}")
    for i in idx:
        if isinstance(i, bool) or not isinstance(i, int) or not 0 <= i < num_images:
            raise ValueError(f"image indices must be ints in [0, {num_images}), got {i!r}")
    return idx


def view_setups(cams, gts, views, downscale):
    """The camera blocks (model.camera_setup) of one step's `views` cameras at `downscale`, checked against the
    ground-truth images: returns (setups, H, W).  Raises ValueError unless there are exactly `views` cameras and
    images, all cameras render at one resolution and every image is a float32 [H,W,3] tensor of it."""
    cams = [cams] if isinstance(cams, Camera) else list(cams)
    if gts is None:      # a render without ground truth (SplatTrainer.render)
        gts = [None] * len(cams)
    if len(cams) != views or len(gts) != views:
        raise ValueError(f"a step takes {views} cameras and {views} ground-truth images (views_per_step={views}), "
                         f"got {len(cams)} and {len(gts)}")
    setups = [camera_setup(c, downscale) for c in cams]
    H, W = setups[0][0], setups[0][1]
    if any((su[0], su[1]) != (H, W) for su in setups):
        raise ValueError("all views of a step must render at the same resolution, got (W, H) "
                         f"{sorted({(su[1], su[0]) for su in setups})}")
    for gt in gts:
        if gt is None:
            continue
        if gt.dtype != torch.float32 or tuple(gt.shape) != (H, W, 3):
            raise ValueError(f"every gt must be a float32 [{H},{W},3] image (this step's render resolution)")
    return setups, H, W


class SplatTrainer:
    def __init__(self, params, cfg=None, sh_degree=None, sh_degree_interval=1000, num_downscales=0,
                 resolution_schedule=3000, background=(0.6130, 0.0101, 0.3984), device="cuda:0", generator=None,
                 ssim_weight=0.2, m_capacity=None, group=None, views_per_step=1, antialiased=False,
                 appearance=None, pose=None, depth=None, filter3d=None):
        """params: dict with the reference's six tensors (means [n,3], scales [n,3] log, quats [n,4] raw,
        featuresDc [n,3], featuresRest [n,K-1,3], opacities [n,1] logits), as model.GaussianModel takes them.
        cfg: densify.RefineConfig (the reference's refinement, the default) or mcmc.MCMCConfig (3DGS-MCMC under a
        Gaussian budget, DESIGN D20: no densification statistics are taken, the loss returned stays the image loss).
        RefineConfig(absgrad=True) (DESIGN D25) feeds the statistics AbsGS's absolute screen-space gradient, written
        by the blend backward (gsb_rasterize_backward_absgrad) in place of v_xy; nothing else in the step changes.
        m_capacity: initial intersection capacity of the binning buffers (grown on demand).
        group: a process group to train data-parallel over camera views (any size, 1 included); every rank
        constructs the trainer with the same parameters and calls step() with the same step numbers.
        views_per_step: B camera views per step (per rank under a group); step() then takes B cameras and B images.
        antialiased: train and render with the anti-aliased opacity (DESIGN D19), as model.GaussianModel(antialiased=
        True): the projection kernels are the _aa ones, and nothing else in the step changes.
        appearance: an appearance.AppearanceConfig to learn one bilateral grid per training image (DESIGN D21); step()
        then takes image=.  Not available with group=.
        pose: a pose.PoseConfig to learn one camera pose correction per training image (DESIGN D22); step() then takes
        image=, and evaluate() / render() may.  Not available with group=; with appearance=, num_images must agree.
        depth: a depth.DepthConfig to supervise the rendered inverse depth with per-image priors (DESIGN D23); step()
        then takes depth=.
        filter3d: a filter3d.Filter3DConfig to train and render with Mip-Splatting's 3-D smoothing filter (DESIGN
        D24) from its training cameras; save() then writes the baked scene."""
        import torch.distributed as dist
        self.views_per_step = B = int(views_per_step)
        if B < 1:
            raise ValueError("views_per_step must be >= 1")
        if group is None and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise RuntimeError("SplatTrainer without a group runs in one process; pass group= to train data-parallel "
                               "over camera views")
        if appearance is not None and group is not None:
            raise ValueError("appearance grids are not available with group= (data-parallel training)")
        if pose is not None and group is not None:
            raise ValueError("pose corrections are not available with group= (data-parallel training)")
        if pose is not None and appearance is not None and pose.num_images != appearance.num_images:
            raise ValueError(f"appearance= and pose= must name the same training images, got num_images "
                             f"{appearance.num_images} and {pose.num_images}")
        if depth is not None and not isinstance(depth, DepthConfig):
            raise ValueError("depth= takes a depth.DepthConfig")
        if filter3d is not None and not isinstance(filter3d, Filter3DConfig):
            raise ValueError("filter3d= takes a filter3d.Filter3DConfig")
        self.depth = depth
        self.filter3d_cfg = filter3d
        self.device = torch.device(device)
        self.cfg = cfg or RefineConfig()
        self.antialiased = bool(antialiased)
        t = {k: torch.as_tensor(params[k]).to(device=self.device, dtype=torch.float32) for k in PARAM_NAMES}
        n, k_bases = t["means"].shape[0], t["featuresRest"].shape[1] + 1
        self.sh_degree = ops.deg_from_sh(k_bases) if sh_degree is None else int(sh_degree)
        self.sh_degree_interval = int(sh_degree_interval)
        self.num_downscales, self.resolution_schedule = int(num_downscales), int(resolution_schedule)
        self.ssim_weight = float(ssim_weight)
        # the image size is known from the first camera: the pipeline starts with one-tile placeholder buffers
        self.pipe = pp = SplatPipeline(n, 16, 16, sh_degree=ops.deg_from_sh(k_bases), device=self.device,
                                       m_capacity=m_capacity)
        for k in ("means", "scales", "quats"):
            pp.p[k].copy_(t[k])
        pp.p["opacities"].copy_(t["opacities"].reshape(n, 1))
        pp.p["coeffs"][:, 0, :].copy_(t["featuresDc"])
        pp.p["coeffs"][:, 1:, :].copy_(t["featuresRest"])
        pp.adam_m = torch.zeros_like(pp.param_flat)
        pp.adam_v = torch.zeros_like(pp.param_flat)
        pp.background.copy_(torch.tensor(background, dtype=torch.float32))
        self.L = capi.lib()
        self.appearance = None if appearance is None else Appearance(appearance, self.device)
        self.poses = None if pose is None else Poses(pose, self.device)
        self.num_images = next((c.num_images for c in (appearance, pose) if c is not None), None)
        self.lr = dict(LEARNING_RATES)
        # the refinement strategy: the reference's Model::afterTrain (RefineConfig) or 3DGS-MCMC (MCMCConfig, D20)
        self.refiner = MCMCRefiner(self.cfg) if isinstance(self.cfg, MCMCConfig) else None
        self.densifier = None if self.refiner is not None else Densifier(self.cfg, generator=generator, group=group)
        self._absgrad = self.densifier is not None and getattr(self.cfg, "absgrad", False)
        # the B cameras: views [B,16] | projs [B,16] | centres [B,3], one pinned staging block, one upload per step;
        # with pose corrections (D22) the uploaded views and centres go to base views [B,16] | base centres [B,3]
        # behind them, and the corrected ones are written into the first slots
        floats = 35 * B + (19 * B if pose is not None else 0)
        self.cams_host = torch.zeros(floats, dtype=torch.float32).pin_memory()
        self.cams_dev = torch.zeros(floats, dtype=torch.float32, device=self.device)
        self.viewmats = self.cams_dev[:16 * B].view(B, 4, 4)
        self.projs = self.cams_dev[16 * B:32 * B].view(B, 4, 4)
        self.cam_positions = self.cams_dev[32 * B:35 * B].view(B, 3)
        if pose is not None:
            self.base_viewmats = self.cams_dev[35 * B:51 * B].view(B, 4, 4)
            self.base_positions = self.cams_dev[51 * B:].view(B, 3)
            self.cam_grads = torch.zeros((2, 4, 4), dtype=torch.float32, device=self.device)  # d/dview, d/dprojmat
        self.projmats = torch.zeros((B, 4, 4), dtype=torch.float32, device=self.device)
        self.losses = torch.zeros((B, 3), dtype=torch.float32, device=self.device)
        self.depth_losses = torch.zeros(B, dtype=torch.float32, device=self.device)   # D23: per view, unweighted
        self.eval_loss = torch.zeros(3, dtype=torch.float32, device=self.device)    # evaluate()'s result
        self.resolution = None
        self.render_maps = None   # render()'s outputs, sized by the resolution
        self.pixel_reallocs = 0   # resolution changes after the first step (the downscale schedule)
        self.writer = None
        self.last_info = {"refined": False}
        self.world, self.exchange = 1, None
        if group is not None:
            from .multigpu import ViewParallelExchange
            self.world = dist.get_world_size(group)
            # symmetric gradient buffer + colour slots + trailers; SplatPipeline.resize_gaussians rebuilds them after a
            # refinement
            pp.exchange = self.exchange = ViewParallelExchange(pp, group=group, views_per_rank=B)
        if filter3d is not None:   # D24: the training cameras, uploaded once, and the compute's workspace
            self.f3d_cams = camera_table(filter3d.cameras, self.device)
            self.f3d_ws = torch.empty(self.L.gsb_filter3d_workspace_bytes(), dtype=torch.uint8, device=self.device)
        self._alloc_gaussian_scratch()
        if filter3d is not None:
            self._compute_filter3d()

    def _alloc_gaussian_scratch(self):
        """The trainer's per-Gaussian buffers, (re)built at construction and after a refinement."""
        pp, n, B, d = self.pipe, self.pipe.n, self.views_per_step, self.device
        self.opac = torch.empty(n, dtype=torch.float32, device=d)     # sigmoid(logits) (x comp: D19) for the blend
        self.v_opac = torch.empty(n, dtype=torch.float32, device=d)   # blend gradient w.r.t. it
        # The B views' colours and colour gradients, [B,n,3] each.  At B = 1 they are the pipeline's own [n,3]
        # buffers; under a group the colour gradients live in the exchange's symmetric allocation.
        if B == 1:
            self.rgbs_views = pp.rgbs.view(1, n, 3)
        else:
            self.rgbs_views = torch.empty((B, n, 3), dtype=torch.float32, device=d)
        if self.exchange is not None:
            self.v_rgb_views = self.exchange.v_rgb_views
        elif B == 1:
            self.v_rgb_views = pp.v_rgbs.view(1, n, 3)
        else:
            self.v_rgb_views = torch.empty((B, n, 3), dtype=torch.float32, device=d)
            # the pointer tables of the one multi-view SH backward launch (_sh_backward)
            self.rgb_ptrs = torch.tensor([self.v_rgb_views[b].data_ptr() for b in range(B)], dtype=torch.int64,
                                         device=d)
            self.geom_ptrs = torch.tensor([pp.grad_flat.data_ptr()], dtype=torch.int64, device=d)
        if self.poses is not None:   # D22: the projection backward's per-block camera-gradient rows
            floats = self.L.gsb_project_camera_partials_floats(n)
            self.cam_blocks = floats // capi.CAMGRAD_TERMS
            self.cam_partials = torch.empty(max(floats, 1), dtype=torch.float32, device=d)
        if self.filter3d_cfg is not None:   # D24: the 3-D filter, recomputed after every refinement
            self.f3d = torch.empty(n, dtype=torch.float32, device=d)
        if self._absgrad:   # D25: the blend's absolute screen-space gradient, the statistics' input
            self.v_xy_abs = torch.empty((n, 2), dtype=torch.float32, device=d)
        if self.depth is not None:   # D23: 1/z where radii > 0, its blend gradient, and the projection's v_depth
            self.inv_depths = torch.empty(n, dtype=torch.float32, device=d)
            self.v_inv_depths = torch.empty(n, dtype=torch.float32, device=d)
            self.v_z = torch.empty(n, dtype=torch.float32, device=d)

    def _set_resolution(self, W, H):
        if self.resolution is not None:
            self.pixel_reallocs += 1
        self.resolution = (W, H)
        self.pipe._alloc_pixels(W, H)
        self.render_maps = None
        self.ssim_ws = torch.empty(self.L.gsb_ssim_workspace_bytes(H, W) + 256, dtype=torch.uint8, device=self.device)
        if self.appearance is not None:     # D21: the adjusted image, its loss gradient, the slice backward's workspace
            self.adj_img = torch.empty((H, W, 3), dtype=torch.float32, device=self.device)
            self.v_adj = torch.empty((H, W, 3), dtype=torch.float32, device=self.device)
            self.bilagrid_ws = torch.empty(self.L.gsb_bilagrid_workspace_bytes(H, W) + 256, dtype=torch.uint8,
                                           device=self.device)
        if self.depth is not None:   # D23: the rendered inverse depth, its opacity map, its gradient, the L1's workspace
            f32, d = torch.float32, self.device
            self.depth_render = torch.empty((H, W), dtype=f32, device=d)
            self.depth_alpha = torch.empty((H, W), dtype=f32, device=d)
            self.v_depth_render = torch.empty((H, W), dtype=f32, device=d)
            self.depth_ws = torch.empty(self.L.gsb_inverse_depth_l1_workspace_bytes(H, W), dtype=torch.uint8, device=d)

    @property
    def n(self):
        return self.pipe.n

    @property
    def image(self):
        """The image of the last step ([H,W,3], clamped to 1; the background where nothing was visible); with
        several views per step, the last view's."""
        return self.pipe.out_img

    def params(self):
        """Copies of the reference's six tensors."""
        return _split_coeffs(self.pipe.p)

    def adam_state(self):
        """(exp_avg, exp_avg_sq): copies keyed like params()."""
        pp = self.pipe
        return _split_coeffs(flat_views(pp.adam_m, pp.offs)), _split_coeffs(flat_views(pp.adam_v, pp.offs))

    def appearance_grids(self):
        """A copy of the appearance grids in F.grid_sample's order, [num_images, 12, L, Y, X] (D21)."""
        if self.appearance is None:
            raise ValueError("this trainer has no appearance grids")
        return to_gsplat_order(self.appearance.grids)

    def filter3d(self):
        """A copy of the 3-D filter, [n] float32 (D24)."""
        if self.filter3d_cfg is None:
            raise ValueError("this trainer has no 3-D filter")
        return self.f3d.clone()

    def _filter3d_of(self, means):
        """D24: the 3-D filter of `means` from the trainer's cameras, into a new tensor."""
        c = self.filter3d_cfg
        return compute_filter3d(means, self.f3d_cams, c.variance, c.near, c.margin)

    def _compute_filter3d(self):
        """D24: recompute the trainer's filter buffer from the current means."""
        pp, c = self.pipe, self.filter3d_cfg
        capi.check(self.L.gsb_filter3d_compute(pp.n, capi.ptr(pp.p["means"]), self.f3d_cams.shape[0],
                                               capi.ptr(self.f3d_cams), c.near, c.margin, c.variance,
                                               capi.ptr(self.f3d_ws), self.f3d_ws.numel(), capi.ptr(self.f3d),
                                               capi.stream()))

    def pose_deltas(self):
        """A copy of the pose corrections, [num_images, 9]: translation e[0:3] and 6-D rotation offset e[3:9] per
        training image (D22; pose.adjusted_camera applies one to a model.Camera)."""
        if self.poses is None:
            raise ValueError("this trainer has no pose corrections")
        return self.poses.deltas.clone()

    def _images(self, image, views):
        """The training images of `views` views (check_images), or None for each view when image is None and
        nothing requires it."""
        if self.num_images is None:
            if image is not None:
                raise ValueError("image= needs a trainer constructed with appearance= or pose=")
            return [None] * views
        return check_images(image, views, self.num_images)

    def _depth_maps(self, depth, views):
        """step()'s depth= as a list of `views` maps or Nones, each checked for type, dtype, device and rank (step()
        checks their size against the render resolution)."""
        if depth is None:
            return [None] * views
        if self.depth is None:
            raise ValueError("depth= needs a trainer constructed with depth=DepthConfig(...)")
        if isinstance(depth, torch.Tensor):
            if views == 1:
                maps = [depth]
            elif depth.dim() == 3:
                maps = list(depth.unbind(0))
            else:
                raise ValueError(f"depth= must be a [{views},H,W] tensor or a sequence of {views} maps")
        elif isinstance(depth, (list, tuple)):
            maps = list(depth)
        else:
            raise ValueError("depth= must be a float32 [H,W] CUDA tensor, a sequence of them (or None), or [B,H,W]")
        if len(maps) != views:
            raise ValueError(f"depth= must give {views} maps (None for a view without one), got {len(maps)}")
        for m in maps:
            if m is None:
                continue
            if (not isinstance(m, torch.Tensor) or m.dtype != torch.float32 or m.device != self.device
                    or m.dim() != 2 or not m.is_contiguous()):
                raise ValueError(f"every depth map must be a contiguous float32 [H,W] tensor on {self.device}")
        return maps

    def step(self, cam, gt, step, image=None, depth=None):
        """One training step at `step` (1-based, as opensplat.cpp counts).  At views_per_step = 1: cam is one
        model.Camera, gt one [H,W,3] fp32 CUDA image at this step's render resolution, and the result is the device
        tensor {total, L1, SSIM}.  At B > 1: cam is a sequence of B cameras, gt B images (a sequence or a [B,H,W,3]
        tensor), and the result is the device [B,3] tensor of the views' {total, L1, SSIM}.  The next step overwrites
        the result.  image: with appearance grids or pose corrections, the training image of the view (an int) or of
        each of the B views (a sequence of B ints); without them it must be None.  depth: with depth priors (D23), at
        B = 1 one float32 [H,W] CUDA inverse-depth map at this step's render resolution or None; at B > 1 a sequence of
        B such maps, any of which may be None, or a [B,H,W] tensor.  Raises ValueError on a wrong number of views,
        mixed resolutions, a wrong image, a wrong image= or a wrong depth=."""
        pp, B, ap, po = self.pipe, self.views_per_step, self.appearance, self.poses
        images = self._images(image, B)
        priors = self._depth_maps(depth, B)
        gts = [gt] if B == 1 else gt
        if any(m is not None for m in priors):
            _, H, W = view_setups(cam, gts, B, downscale_factor(step, self.num_downscales, self.resolution_schedule))
            if any(m is not None and tuple(m.shape) != (H, W) for m in priors):
                raise ValueError(f"every depth map must be [{H},{W}] (this step's render resolution)")
            # g = w(s) / (H W) in fp64, rounded once: the gradient of the weighted loss w.r.t. a valid pixel of R
            depth_g = float(depth_weight(self.depth, step) / (H * W))
        # ---- forward, enqueued without a host wait until each view's binning read-back ----
        setups, H, W, use = self._setup_views(cam, gts, B, step, images if po is not None else None)
        if ap is not None:
            ap.tv()                         # D21: the grids' gradient starts as tv_weight * dTV
        if po is not None:
            po.start_step()                 # D22: the corrections' gradient starts as reg * e
        visible = []
        for b in range(B):
            intr = setups[b][2]
            self._render_view(b, intr, gts[b], self.losses[b], image=images[b] if ap is not None else None,
                              prior=priors[b])
            if priors[b] is not None:
                self._depth_loss(priors[b], depth_g, self.depth_losses[b])
            elif self.depth is not None:
                self.depth_losses[b].zero_()
            visible.append(pp.plan.visible > 0)
            # model.cpp:173-174: a lone view that hits nothing trains nothing.  Next to other views, or data-parallel
            # with more than one rank, its backward pass runs and writes zero gradients (no Gaussian has radii > 0):
            # the sum over the views and the divisor B x G stay as they are, and the rank takes the exchange's
            # barriers.
            if B > 1 or visible[b] or self.world > 1:
                self._backward_view(b, use, intr[0], intr[1], image=images[b], prior=priors[b] is not None)
            # this view's densification statistics (pp.v_xy / pp.radii are overwritten by the next view); with
            # absgrad (D25) they take the absolute screen-space gradient instead
            if self.densifier is not None:
                v_xy = self.v_xy_abs if self._absgrad else pp.v_xy
                self.densifier.accumulate_view(step, v_xy if visible[b] else None, pp.radii, H, W)
        # A step whose views all hit nothing trains nothing; with more than one rank it still takes part in the step
        # (the Adam step every replica takes, the refinement's collectives; see the module docstring).
        trains = any(visible) or self.world > 1
        if trains:
            self._sh_backward(use)
            if self.refiner is not None:     # D20: the regularisers, on the averaged and exchanged gradients
                self.refiner.regularize(pp)
            self._adam_step()
            if ap is not None:
                ap.adam_step(step)
            if po is not None:
                po.adam_step(step)
        self.lr["means"] = means_learning_rate(step, self.cfg.max_steps, MEANS_LR_INIT)
        if trains and self.refiner is not None:
            # ---- D20: relocation and growth on a refinement step, then the position noise ----
            self._adopt(*self.refiner.finish_step(step, pp, self.lr["means"]))
        elif trains:
            # ---- the rest of Model::afterTrain on views into the flat buffers ----
            self._adopt(*self.densifier.finish_step(step, pp.p, flat_views(pp.adam_m, pp.offs),
                                                    flat_views(pp.adam_v, pp.offs), H, W,
                                                    filter3d=None if self.filter3d_cfg is None else self._filter3d_of))
        else:
            self.last_info = {"refined": False}
        if self.filter3d_cfg is not None and recompute_due(self.cfg, self.filter3d_cfg, step,
                                                           self.last_info["refined"]):
            self._compute_filter3d()
        return self.losses[0] if B == 1 else self.losses

    def evaluate(self, cam, gt, step, image=None):
        """The loss of one view without training on it (opensplat.cpp:203-207, the --val camera): Model::forward at
        `step`'s downscale factor and SH degree, then mainLoss against gt (a float32 [H,W,3] CUDA image at that
        resolution).  It runs the forward kernels and the loss of a one-view step() (at any views_per_step) and
        returns the device tensor {total, L1, SSIM}, overwritten by the next evaluate().  Parameters, Adam state and
        the densification statistics are left alone, and the next step() computes what it would have computed
        without this call.  Other trainer state it does change: `image` becomes the evaluated view's render; a view
        at another resolution than the last step's reallocates the pixel buffers, and the next step reallocates them
        back, each counted in `pixel_reallocs`; and the binning buffers grow if the view needs more intersections
        than they hold (a step grows them the same way, with no effect on its result).  image: with pose corrections,
        render at training image `image`'s corrected pose (D22).  Raises ValueError on a wrong image or image=."""
        setups = self._setup_views(cam, [gt], 1, step, self._view_pose(image))[0]
        self._render_view(0, setups[0][2], gt, self.eval_loss)
        return self.eval_loss

    def render(self, cam, step, normalize_depth=False, image=None):
        """Renders one view without training on it: Model::forward at `step`'s downscale factor and SH degree (the
        clamped colour, as evaluate() renders it) plus the depth and opacity maps (DESIGN D18).  Returns
        {"rgb" [H,W,3], "depth" [H,W], "alpha" [H,W]}: depth = sum alpha T z over the blended pairs (z the view-space
        depth of the Gaussian; 0 where nothing is blended), alpha = 1 - T_final; with normalize_depth, depth / alpha
        where alpha > 0 and 0 elsewhere.  The tensors are overwritten by the next render().  Like evaluate(), it leaves
        parameters, Adam state and the densification statistics alone, and the next step() computes what it would have
        computed without this call; it does not change `image`.  A view at another resolution than the last step's
        reallocates the pixel buffers, as evaluate() does.  image: as evaluate()'s."""
        setups = self._setup_views(cam, None, 1, step, self._view_pose(image))[0]
        pp = self.pipe
        H, W = pp.H, pp.W
        if self.render_maps is None:
            f32, d = torch.float32, self.device
            self.render_maps = {"rgb": torch.empty((H, W, 3), dtype=f32, device=d),
                                "depth": torch.empty((H, W), dtype=f32, device=d),
                                "alpha": torch.empty((H, W), dtype=f32, device=d),
                                "normalized": torch.empty((H, W), dtype=f32, device=d)}
        r = self.render_maps
        self._project_blend(0, setups[0][2], out_img=r["rgb"], out_depth=r["depth"], out_alpha=r["alpha"])
        depth = r["depth"]
        if normalize_depth:
            depth = r["normalized"]
            torch.div(r["depth"], r["alpha"], out=depth)
            depth.masked_fill_(r["alpha"] <= 0, 0.0)
        return {"rgb": r["rgb"], "depth": depth, "alpha": r["alpha"]}

    def _view_pose(self, image):
        """evaluate() / render()'s image= as _setup_views' `images`: None without it."""
        if image is None:
            return None
        if self.poses is None:
            raise ValueError("image= in evaluate() and render() needs a trainer constructed with pose=")
        return check_images(image, 1, self.num_images)

    def _setup_views(self, cams, gts, views, step, images=None):
        """What the forward passes of a step's `views` views share: view_setups at `step`'s downscale factor, the
        render resolution, one upload of the cameras into slots 0..views-1 of the camera block (the last host wait, a
        binning read-back, came after the block's previous upload), `proj @ view` and the SH colours.  One view takes
        the 2-D matmul and the one-view SH forward (see the module docstring).  With `images` (D22: one training image
        per view) each view's camera is uploaded into the base slots and corrected by its image's pose into the
        working slots before the matmul.  Returns (setups, H, W, use): use is the step's SH degrees_to_use."""
        setups, H, W = view_setups(cams, gts, views, downscale_factor(step, self.num_downscales,
                                                                       self.resolution_schedule))
        if (W, H) != self.resolution:
            self._set_resolution(W, H)
        pp, L, P, s = self.pipe, self.L, capi.ptr, capi.stream()
        host, B, n, p = self.cams_host, self.views_per_step, pp.n, pp.p
        for b, (_, _, _, view, proj, cam_pos) in enumerate(setups):
            vo, co = (35 * B + 16 * b, 51 * B + 3 * b) if images is not None else (16 * b, 32 * B + 3 * b)
            host[vo:vo + 16].copy_(view.reshape(16))
            host[16 * (B + b):16 * (B + b) + 16].copy_(proj.reshape(16))
            host[co:co + 3].copy_(cam_pos)
        self.cams_dev.copy_(host, non_blocking=True)
        if images is not None:
            for b in range(views):
                capi.check(L.gsb_pose_apply(P(self.poses.deltas[images[b]]), P(self.base_viewmats[b]),
                                            P(self.base_positions[b]), P(self.viewmats[b]), P(self.cam_positions[b]),
                                            s))
        use = min(step // self.sh_degree_interval, self.sh_degree)
        if views == 1:
            torch.matmul(self.projs[0], self.viewmats[0], out=self.projmats[0])
            capi.check(L.gsb_sh_forward_rgb_cam(n, pp.deg, use, P(p["means"]), P(self.cam_positions[0]),
                                                P(p["coeffs"]), 0.5, P(self.rgbs_views[0]), s))
        else:
            torch.matmul(self.projs, self.viewmats, out=self.projmats)
            capi.check(L.gsb_sh_forward_rgb_cam_multiview(n, pp.deg, use, P(p["means"]), views, P(self.cam_positions),
                                                          P(p["coeffs"]), 0.5, P(self.rgbs_views), s))
        return setups, H, W, use

    def _project_blend(self, b, intr, out_img=None, out_depth=None, out_alpha=None, prior=False):
        """View b's projection with the activations from camera slot b (intrinsics `intr`), then binning and the
        clamped blend (the view's one host wait) into the pipeline's image, or into out_img with the depth and opacity
        maps (render()).  prior (D23): also 1/z where radii > 0, blended into depth_render."""
        pp, L, P, s = self.pipe, self.L, capi.ptr, capi.stream()
        n, p, tb, H, W = pp.n, pp.p, pp.tb, pp.H, pp.W
        fx, fy, cx, cy = intr
        head = (n, P(p["means"]), P(p["scales"]), 1.0, P(p["quats"]), P(p["opacities"]))
        tail = (P(self.viewmats[b]), P(self.projmats[b]), fx, fy, cx, cy, H, W, tb[0], tb[1], 0.01, P(pp.cov3d),
                P(pp.xys), P(pp.depths), P(pp.radii), P(pp.conics), P(pp.nth), P(self.opac))
        if self.filter3d_cfg is not None:     # D24
            capi.check(L.gsb_project_forward_activated_filter3d(*head, P(self.f3d), *tail, int(self.antialiased), s))
        else:
            project = L.gsb_project_forward_activated_aa if self.antialiased else L.gsb_project_forward_activated
            capi.check(project(*head, *tail, s))
        if prior:
            capi.check(L.gsb_inverse_depths(n, P(pp.depths), P(pp.radii), P(self.inv_depths), s))
            out_depth, out_alpha = self.depth_render, self.depth_alpha
        pp._bin_blend(self.opac, ops.CLAMP_MAX_ONE, count_visible=True, rgbs=self.rgbs_views[b], out_img=out_img,
                      out_depth=out_depth, out_alpha=out_alpha, depth_values=self.inv_depths if prior else None)

    def _render_view(self, b, intr, gt, loss, image=None, prior=None):
        """View b's forward pass after _setup_views: _project_blend, then the loss against gt into `loss` ({total, L1,
        SSIM}) and its image gradient into the pipeline's v_img.  With a training image (D21) the loss is taken on
        the render sliced through that image's grid, and the slice backward writes v_img and adds 1/B of the grid
        gradient.  prior (D23): the view's depth prior; the blend also renders the inverse depth (_depth_loss takes
        its loss)."""
        pp, L, P, s = self.pipe, self.L, capi.ptr, capi.stream()
        H, W = pp.H, pp.W
        self._project_blend(b, intr, prior=prior is not None)
        off = (-self.ssim_ws.data_ptr()) % 256
        if image is None:
            capi.check(L.gsb_ssim_l1_loss(H, W, P(pp.out_img), P(gt), self.ssim_weight, P(pp.v_img), P(loss),
                                          self.ssim_ws.data_ptr() + off, self.ssim_ws.numel() - off, s))
            return
        ap = self.appearance
        capi.check(L.gsb_bilagrid_slice_forward(H, W, P(ap.grids[image]), P(pp.out_img), P(self.adj_img), s))
        capi.check(L.gsb_ssim_l1_loss(H, W, P(self.adj_img), P(gt), self.ssim_weight, P(self.v_adj), P(loss),
                                      self.ssim_ws.data_ptr() + off, self.ssim_ws.numel() - off, s))
        woff = (-self.bilagrid_ws.data_ptr()) % 256
        capi.check(L.gsb_bilagrid_slice_backward(H, W, P(ap.grids[image]), P(pp.out_img), P(self.v_adj),
                                                 1.0 / self.views_per_step, P(pp.v_img), P(ap.grad[image]),
                                                 self.bilagrid_ws.data_ptr() + woff, self.bilagrid_ws.numel() - woff,
                                                 s))

    def _depth_loss(self, prior, g, loss):
        """D23: the unweighted depth loss of the last _render_view into `loss` (a device float) and its gradient, g
        times the sign on valid pixels, into v_depth_render."""
        P = capi.ptr
        H, W = self.pipe.H, self.pipe.W
        capi.check(self.L.gsb_inverse_depth_l1(H, W, P(self.depth_render), P(prior), g, P(self.v_depth_render),
                                               P(loss), P(self.depth_ws), self.depth_ws.numel(), capi.stream()))

    def _backward_view(self, b, use, fx, fy, image=None, prior=False):
        """View b's backward pass after its forward pass: rasterize-backward into colour slot b, then projection
        backward into the geometry gradients (view 0 writes them, later views add to them).  With pose corrections
        (D22) the projection backward also reduces the view's camera gradient, which gsb_pose_backward adds, times
        1/B, to training image `image`'s correction gradient.  With a depth prior (D23) the blend backward also takes
        the depth map's gradient, and its 1/z gradient reaches the projection's v_depth.  Under a group it first
        publishes the view's camera centre, read by the peers' multi-view SH backward, and after the last view's
        rasterize-backward starts the exchange's colour half (degrees_to_use `use`).  On a view that hit nothing
        every gradient it writes is zero."""
        pp, L, P = self.pipe, self.L, capi.ptr
        n, p, g, ex = pp.n, pp.p, pp.g, self.exchange
        if ex is not None:
            ex.set_camera(self.cam_positions[b], b)
        v_depth = None
        v_xy_abs = self.v_xy_abs if self._absgrad else None   # D25
        if prior:
            pp._raster_backward_depth(self.opac, self.v_opac, self.v_rgb_views[b], ops.CLAMP_MAX_ONE,
                                      self.v_depth_render, self.v_inv_depths, v_xy_abs=v_xy_abs)
            capi.check(L.gsb_inverse_depths_backward(n, P(pp.depths), P(pp.radii), P(self.v_inv_depths), P(self.v_z),
                                                     capi.stream()))
            v_depth = self.v_z
        else:
            pp._raster_backward(self.opac, self.v_opac, self.v_rgb_views[b], ops.CLAMP_MAX_ONE, v_xy_abs=v_xy_abs)
        if ex is not None and ex.overlap and b == self.views_per_step - 1:
            # every colour slot is final: colour pulls + SH expansion start now, on a side stream
            ex.start_colour(degrees_to_use=use, rgbs=self.rgbs_views)
        if self.antialiased or self.filter3d_cfg is not None:     # D19, D24: the backward recomputes o from the logits
            pj = L.gsb_project_backward_activated_aa if b == 0 else L.gsb_project_backward_activated_aa_acc
            opac = p["opacities"]
        else:
            pj = L.gsb_project_backward_activated if b == 0 else L.gsb_project_backward_activated_acc
            opac = self.opac
        args = (n, P(p["means"]), P(p["scales"]), 1.0, P(p["quats"]), P(opac), P(self.viewmats[b]),
                P(self.projmats[b]), fx, fy, pp.H, pp.W, P(pp.radii), P(pp.conics), P(pp.v_xy), P(v_depth),
                P(pp.v_conic), P(self.v_opac), P(g["means"]), P(g["scales"]), P(g["quats"]), P(g["opacities"]))
        s, po = capi.stream(), self.poses
        if self.filter3d_cfg is not None:     # D24: the filter after the logits; accumulate, antialiased, camgrad
            capi.check(L.gsb_project_backward_activated_filter3d(
                *args[:6], P(self.f3d), *args[6:], int(b > 0), int(self.antialiased), int(po is not None),
                P(self.cam_partials) if po is not None else None, s))
        elif po is None:
            capi.check(pj(*args, s))
        else:
            capi.check(L.gsb_project_backward_activated_camgrad(*args, int(b > 0), int(self.antialiased),
                                                                P(self.cam_partials), s))
        if po is None:
            return
        cg = self.cam_grads
        capi.check(L.gsb_project_camera_grad_reduce(self.cam_blocks, P(self.cam_partials), P(cg[0]), P(cg[1]), s))
        capi.check(L.gsb_pose_backward(P(po.deltas[image]), P(self.base_viewmats[b]), P(self.projs[b]), P(cg[0]),
                                       P(cg[1]), 1.0 / self.views_per_step, P(po.grad[image]), s))

    def _sh_backward(self, use):
        """The SH backward of the step's B colour gradients (degrees_to_use `use`, the clamp's gradient included) into
        the coefficient gradients, and the geometry gradients averaged over the B x G views.  Data-parallel: the
        exchange expands every rank's colour gradients and all-reduces the geometry prefix
        (multigpu.ViewParallelExchange)."""
        pp, L, P, s = self.pipe, self.L, capi.ptr, capi.stream()
        n, p, g, B, ex = pp.n, pp.p, pp.g, self.views_per_step, self.exchange
        if ex is not None:
            if ex.overlap:
                ex.finish(degrees_to_use=use)          # all-reduce of the geometry prefix, joins the colour half
            else:
                ex.exchange(degrees_to_use=use, rgbs=self.rgbs_views)    # both halves in one launch
        elif B == 1:
            capi.check(L.gsb_sh_backward_rgb_cam(n, pp.deg, use, P(p["means"]), P(self.cam_positions[0]),
                                                 P(self.rgbs_views), P(self.v_rgb_views), P(g["coeffs"]), s))
        else:
            # The clamp's gradient on the B slots (mask = rgbs > 0 or -0, the exact tie: D17) and their expansion, plus
            # the geometry prefix times 1/B (the all-reduce role at world 1), in one launch of the data-parallel
            # exchange kernel.
            capi.check(L.gsb_mask_rgb_grad(n * B, P(self.rgbs_views), P(self.v_rgb_views), s))
            capi.check(L.gsb_exchange_gradients(
                n, pp.deg, use, P(p["means"]), B, P(self.cam_positions), self.rgb_ptrs.data_ptr(), 1.0 / B,
                P(g["coeffs"]), 0, 1, pp.geom_numel, self.geom_ptrs.data_ptr(), None, s))

    def _adam_step(self):
        """The six optimizers in one launch (torch.optim.Adam defaults, as GaussianModel.optimizers_step)."""
        pp, P = self.pipe, capi.ptr
        pp.adam_t += 1
        t = pp.adam_t
        segs = adam_segments(pp.offs, self.lr)
        table = (capi.AdamSegment * len(segs))(*[capi.AdamSegment(*sg) for sg in segs])
        capi.check(self.L.gsb_adam_step_segments(len(segs), C.addressof(table), P(pp.param_flat), P(pp.grad_flat),
                                                 P(pp.adam_m), P(pp.adam_v), 0.9, 0.999, 1e-8, 1.0 - 0.9 ** t,
                                                 1.0 - 0.999 ** t, capi.stream()))

    def _adopt(self, new_p, new_m, new_v, info):
        """The refinement's result (densify.Densifier or mcmc.MCMCRefiner): a changed Gaussian set re-creates the flat layout (the only allocations of a
        step)."""
        pp = self.pipe
        if new_p is not pp.p:
            pp.resize_gaussians(new_p, new_m, new_v)
            self._alloc_gaussian_scratch()
        self.last_info = info

    # ---- Model::save (model.cpp:496-594) -----------------------------------------------------------------------
    def save(self, filename, step=0, keep_crs=False, scale=1.0, translation=(0.0, 0.0, 0.0), wait=True):
        """Writes the scene as GaussianModel.save does, packing the rows straight from the flat buffer.  With the 3-D
        filter (D24) it writes the baked scene (filter3d.bake): log-scales log(e^2 + f^2) / 2 and logits
        logit(sigmoid(l) c3), so any 3DGS viewer renders what was trained; loading that file into a filtered trainer
        would apply the filter a second time."""
        if self.writer is None:
            self.writer = SceneWriter(self.device)
        params = dict(self.pipe.p)
        if self.filter3d_cfg is not None:
            params = bake(params, self.f3d)
        self.writer.save(filename, params, step, keep_crs, scale, translation)
        if wait:
            self.writer.wait()
