"""Host-side mirror of Model::afterTrain (reference model.cpp:311-500) over the C ABI: per-step densification
statistics, the refine schedule, split / duplicate / cull as one classification + compaction, opacity reset.

The arithmetic lives in csrc/densify.cu (+ the two statistics kernels in csrc/fused.cu); this file is the
reference's control flow: which step does what, the single counts read-back, sizing the new tensors and drawing
the normal samples with torch's generator (so a seeded run draws what the reference's torch::randn draws).
There is no CPU fallback."""
from dataclasses import dataclass

import torch

from . import capi


@dataclass
class RefineConfig:
    """Defaults are the reference CLI's (opensplat.cpp:30-43); the three cull constants are model.cpp:344,444-445."""
    refine_every: int = 100
    warmup_length: int = 500
    reset_alpha_every: int = 30
    densify_grad_thresh: float = 0.0002
    densify_size_thresh: float = 0.01
    stop_screen_size_at: int = 4000
    split_screen_size: float = 0.05
    max_steps: int = 30000
    num_cameras: int = 1
    cull_alpha_thresh: float = 0.1
    cull_scale_thresh: float = 0.5
    cull_screen_size: float = 0.15
    size_fac: float = 1.6
    n_split_samples: int = 2        # fixed by the row map (kinds 1, 2)
    # Alpha reset: the reference BUILDS a zeroed Adam state for the opacities and then drops it (model.cpp:477-486;
    # DESIGN.md D14), so its moments effectively survive.  True = the evident intent (moments zeroed), False = the
    # reference's effective behaviour (moments kept).
    reset_opacity_moments: bool = True
    # AbsGS (DESIGN D25, gsplat's DefaultStrategy(absgrad=True)): the statistics take the per-Gaussian sum of each
    # pixel's |contribution| to the 2-D mean's gradient, component by component, in place of v_xy.  Those sums are
    # larger than |v_xy|, so raise densify_grad_thresh with it (gsplat: 0.0008).  SplatTrainer only.
    absgrad: bool = False

    @property
    def stop_split_at(self):        # model.hpp:31
        return self.max_steps // 2


def classify(scales, opacities, xys_grad_norm, vis_counts, max_2d_size, max_dim, cfg, check_split_screen,
             check_huge, check_cull_screen):
    """gsb_densify_classify.  Returns (src_map [3n] i32, split_rank [n] i32, counts [8] i32 device)."""
    L = capi.lib()
    n = scales.shape[0]
    d = scales.device
    ws = torch.empty(L.gsb_densify_workspace_bytes(n), dtype=torch.uint8, device=d)
    src_map = torch.empty(max(3 * n, 1), dtype=torch.int32, device=d)
    split_rank = torch.empty(max(n, 1), dtype=torch.int32, device=d)
    counts = torch.empty(8, dtype=torch.int32, device=d)
    capi.check(L.gsb_densify_classify(
        n, capi.ptr(scales), capi.ptr(opacities), capi.ptr(xys_grad_norm), capi.ptr(vis_counts),
        capi.ptr(max_2d_size), float(max_dim), cfg.densify_grad_thresh, cfg.densify_size_thresh,
        int(check_split_screen), cfg.split_screen_size, cfg.cull_alpha_thresh, int(check_huge), cfg.cull_scale_thresh,
        int(check_cull_screen), cfg.cull_screen_size, cfg.size_fac, capi.ptr(ws), ws.numel(), capi.ptr(src_map),
        capi.ptr(split_rank), capi.ptr(counts), capi.stream()))
    return src_map, split_rank, counts


def gather_rows(src_map, new_n, src, zero_children=False):
    """dst[j] = src[parent(j)] (zeros for children when zero_children: Adam moments, model.cpp:253-279)."""
    src = src.contiguous()
    n = src.shape[0]
    row = src.numel() // max(n, 1)
    dst = torch.empty((new_n,) + tuple(src.shape[1:]), dtype=torch.float32, device=src.device)
    if new_n:
        capi.check(capi.lib().gsb_densify_gather_rows(new_n, row, capi.ptr(src_map), capi.ptr(src), capi.ptr(dst),
                                                      int(zero_children), capi.stream()))
    return dst


def means_scales(src_map, split_rank, new_n, n_splits, samples, means, scales, quats, size_fac):
    new_means = torch.empty((new_n, 3), dtype=torch.float32, device=means.device)
    new_scales = torch.empty((new_n, 3), dtype=torch.float32, device=means.device)
    if new_n:
        capi.check(capi.lib().gsb_densify_means_scales(
            new_n, n_splits, capi.ptr(src_map), capi.ptr(split_rank), capi.ptr(samples) if n_splits else None,
            capi.ptr(means), capi.ptr(scales), capi.ptr(quats), size_fac, capi.ptr(new_means), capi.ptr(new_scales),
            capi.stream()))
    return new_means, new_scales


class Densifier:
    """State and schedule of Model::afterTrain.  `params` / `adam_m` / `adam_v` are dicts of contiguous fp32 CUDA
    tensors with leading dimension n; "means", "scales" (log), "quats" (raw), "opacities" (logits, [n,1]) are
    required, anything else (featuresDc / featuresRest / a merged coeffs block) is carried along row-wise."""

    def __init__(self, cfg=None, generator=None, sample_fn=None, group=None):
        self.cfg = cfg or RefineConfig()
        self.group = group
        self.generator = generator
        # sample_fn(rows, device) -> [rows,3] normal samples; default torch.randn on the device (model.cpp:359)
        self.sample_fn = sample_fn
        self.xys_grad_norm = self.vis_counts = self.max_2d_size = None
        self.last_info = None

    # model.cpp:317-337
    def accumulate(self, v_xy, radii, img_h, img_w):
        L = capi.lib()
        n = radii.shape[0]
        first = self.xys_grad_norm is None
        if first:
            d = radii.device
            self.xys_grad_norm = torch.empty(n, dtype=torch.float32, device=d)
            self.vis_counts = torch.empty(n, dtype=torch.float32, device=d)
            self.max_2d_size = torch.empty(n, dtype=torch.float32, device=d)
        fn = L.gsb_densify_stats_init if first else L.gsb_densify_stats_update
        capi.check(fn(n, capi.ptr(v_xy), capi.ptr(radii), img_h, img_w, capi.ptr(self.xys_grad_norm),
                      capi.ptr(self.vis_counts), capi.ptr(self.max_2d_size), capi.stream()))

    def _world(self):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return 1
        return dist.get_world_size(self.group)

    def sync_stats(self, group=None):
        """Data-parallel replicas render different views, so their statistics differ; reduce them (sum of gradient
        norms and visibility counts, max of screen sizes) so that every replica classifies identically.  Device
        agnostic (NCCL on the GPUs, gloo in the CPU tests).  Not in the reference (single GPU); with one rank it is
        the identity."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) <= 1:
            return
        if self.xys_grad_norm is None:
            return
        dist.all_reduce(self.xys_grad_norm, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.vis_counts, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.max_2d_size, op=dist.ReduceOp.MAX, group=group)

    def schedule(self, step):
        """(refine?, densify?, reset_alpha?, check_split_screen, check_huge) for `step` -- model.cpp:339-341,349,441,472."""
        c = self.cfg
        refine = step % c.refine_every == 0 and step > c.warmup_length
        reset_interval = c.reset_alpha_every * c.refine_every
        densify = refine and step < c.stop_split_at and step % reset_interval > c.num_cameras + c.refine_every
        reset = refine and step < c.stop_split_at and step % reset_interval == c.refine_every
        return refine, densify, reset, step < c.stop_screen_size_at, step > c.refine_every * c.reset_alpha_every

    def after_train(self, step, params, adam_m, adam_v, v_xy, radii, img_h, img_w):
        """One call per training step, after the optimizer step (opensplat.cpp main loop).  Returns
        (params, adam_m, adam_v, info); the dicts are new objects when the Gaussian set changed.  The same as
        accumulate_view() for the step's one view followed by finish_step()."""
        if v_xy is None and self._world() <= 1:   # `!xys.grad().defined()`  (radii.sum() == 0), model.cpp:315
            info = {"refined": False, "added": 0, "culled": 0, "alpha_reset": False, "n": int(radii.shape[0])}
            return params, adam_m, adam_v, info
        self.accumulate_view(step, v_xy, radii, img_h, img_w)
        return self.finish_step(step, params, adam_m, adam_v, img_h, img_w)

    def accumulate_view(self, step, v_xy, radii, img_h, img_w):
        """The statistics update of one view (model.cpp:315-337): the first view after a clear initialises the
        statistics, later views update them.  A step with several views calls it once per view, in view order, then
        finish_step() once.  v_xy None: the view hit nothing (`!xys.grad().defined()`); in one process it adds
        nothing, under a process group it adds zero statistics, as a rank whose view hit nothing does."""
        if v_xy is None:
            if self._world() <= 1:
                return
            # Data-parallel: this rank's view saw nothing, but the other ranks will enter the collectives of a
            # refine step and change the Gaussian count -- take the same branches with zero statistics instead of
            # returning (a rank that skips would hang the all-reduce or keep a different Gaussian set).
            v_xy = torch.zeros((radii.shape[0], 2), dtype=torch.float32, device=radii.device)
            radii = torch.zeros_like(radii)
        if step < self.cfg.stop_split_at:
            self.accumulate(v_xy, radii, img_h, img_w)

    def finish_step(self, step, params, adam_m, adam_v, img_h, img_w, filter3d=None):
        """The rest of Model::afterTrain once the step's views are accumulated (model.cpp:339-492): the refine / reset
        schedule, the statistics' reduction over the group, refinement, alpha reset and the clear.  Returns
        (params, adam_m, adam_v, info) as after_train.  filter3d (DESIGN D24): a function of the means giving the 3-D
        filter of the Gaussian set; the alpha reset then clamps the effective opacity (reset_opacity)."""
        info = {"refined": False, "added": 0, "culled": 0, "alpha_reset": False, "n": int(params["means"].shape[0])}
        refine, densify, reset, chk_screen, chk_huge = self.schedule(step)
        if not refine:
            return params, adam_m, adam_v, info
        info["refined"] = True
        self.sync_stats(self.group)
        if densify:
            params, adam_m, adam_v, r = self.refine(params, adam_m, adam_v, max(img_h, img_w), chk_screen, chk_huge)
            info.update(r)
        if reset:
            zero = self.cfg.reset_opacity_moments
            m = adam_m.get("opacities") if (adam_m and zero) else None
            v = adam_v.get("opacities") if (adam_v and zero) else None
            if filter3d is None:
                self.reset_opacity(params["opacities"], m, v)
            else:
                self.reset_opacity(params["opacities"], m, v, params["scales"], filter3d(params["means"]))
            info["alpha_reset"] = True
        self.xys_grad_norm = self.vis_counts = self.max_2d_size = None   # "Clear", model.cpp:489-492
        self.last_info = info
        return params, adam_m, adam_v, info

    def refine(self, params, adam_m, adam_v, max_dim, check_split_screen, check_huge):
        c = self.cfg
        n = params["means"].shape[0]
        src_map, split_rank, counts = classify(params["scales"], params["opacities"], self.xys_grad_norm,
                                               self.vis_counts, self.max_2d_size, max_dim, c, check_split_screen,
                                               check_huge, check_split_screen)
        cnt = counts.cpu().tolist()           # the one read-back of a refinement
        n_splits, new_n, n_dups = cnt[0], cnt[4], cnt[5]
        d = params["means"].device
        if self.sample_fn is not None:
            samples = self.sample_fn(c.n_split_samples * n_splits, d).to(device=d, dtype=torch.float32).contiguous()
        else:
            samples = torch.randn((c.n_split_samples * n_splits, 3), device=d, generator=self.generator)  # model.cpp:359
            if self._world() > 1:
                # replicas must place the split children identically: rank 0's draw is the one everybody uses
                # (per-process generators are not synchronised; the reference is single-GPU)
                import torch.distributed as dist
                src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
                dist.broadcast(samples, src=src, group=self.group)
        new_p = {}
        new_p["means"], new_p["scales"] = means_scales(src_map, split_rank, new_n, n_splits, samples, params["means"],
                                                       params["scales"], params["quats"], c.size_fac)
        for k, t in params.items():
            if k not in new_p:
                new_p[k] = gather_rows(src_map, new_n, t)
        new_m = {k: gather_rows(src_map, new_n, t, zero_children=True) for k, t in (adam_m or {}).items()}
        new_v = {k: gather_rows(src_map, new_n, t, zero_children=True) for k, t in (adam_v or {}).items()}
        added = c.n_split_samples * n_splits + n_dups
        return new_p, new_m, new_v, {"n_splits": n_splits, "n_dups": n_dups, "added": added,
                                     "culled": n + added - new_n, "n": new_n, "src_map": src_map[:new_n],
                                     "samples": samples}

    def reset_opacity(self, opacities, exp_avg=None, exp_avg_sq=None, log_scales=None, filter3d=None):
        """model.cpp:472-487: clamp the logits at logit(2 * cull_alpha_thresh), zero the opacity Adam moments.  With
        the 3-D filter f (filter3d [n], DESIGN D24) and the log-scales, clamp the effective opacity sigmoid(l) c3 at
        the same value instead (Mip-Splatting's reset_opacity; gsb_reset_opacity_filter3d)."""
        reset_value = torch.tensor(self.cfg.cull_alpha_thresh * 2.0, dtype=torch.float32)
        max_logit = float(torch.logit(reset_value))
        if filter3d is not None:
            capi.check(capi.lib().gsb_reset_opacity_filter3d(
                opacities.shape[0], max_logit, float(reset_value), capi.ptr(log_scales), capi.ptr(filter3d),
                capi.ptr(opacities), capi.ptr(exp_avg), capi.ptr(exp_avg_sq), capi.stream()))
            return
        capi.check(capi.lib().gsb_reset_opacity(opacities.shape[0], max_logit, capi.ptr(opacities), capi.ptr(exp_avg),
                                                capi.ptr(exp_avg_sq), capi.stream()))
