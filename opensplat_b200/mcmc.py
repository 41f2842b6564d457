"""The 3DGS-MCMC refinement strategy (Kheradmand et al. 2024; gsplat's MCMCStrategy) for trainer.SplatTrainer, under
a fixed Gaussian budget (DESIGN.md D20):

    trainer = SplatTrainer(params, MCMCConfig(cap_max=500_000))

Gaussians are moved, never culled: on a refinement step the dead ones (opacity <= min_opacity) are relocated onto
live ones drawn in proportion to their opacity, then the set grows by 5 % up to cap_max by appending copies of drawn
Gaussians; the opacity and scale of every drawn Gaussian change so that the rendered image is kept.  Every training
step adds L1 penalties on opacity and scale to the gradient (before Adam) and opacity-gated noise shaped by each
Gaussian's covariance to the means (after Adam).  The returned loss stays the image loss: the penalties enter as
gradients only.

The arithmetic lives in csrc/mcmc.cu; this file is the control flow.  Every random number comes from Philox keyed by
(seed, step, index), so data-parallel replicas stay identical without a collective.  A refinement waits on the host
once (the 16-byte plan read-back); growth reuses gsb_densify_gather_rows and SplatPipeline.resize_gaussians.  There
is no CPU fallback."""
import ctypes as C
from dataclasses import dataclass

import torch

from . import capi
from .densify import gather_rows
from .parallel import flat_views

RELOCATE_TAG, GROW_TAG = 1, 2
_CHILD = -(1 << 30)          # 3 << 30 as an int32: a gather row-map entry whose Adam moments come out zero


@dataclass
class MCMCConfig:
    """Defaults are gsplat's MCMCStrategy's.  A step refines when refine_start < step < refine_stop and
    step % refine_every == 0.  max_steps drives the means learning-rate schedule, as RefineConfig.max_steps does."""
    cap_max: int = 1_000_000
    refine_start: int = 500
    refine_stop: int = 25_000
    refine_every: int = 100
    min_opacity: float = 0.005
    noise_lr: float = 5e5
    opacity_reg: float = 0.01
    scale_reg: float = 0.01
    seed: int = 0
    max_steps: int = 30_000

    def __post_init__(self):
        if self.cap_max < 0 or self.refine_every < 1:
            raise ValueError("cap_max must be >= 0 and refine_every >= 1")
        if not 0.0 < self.min_opacity < 1.0:
            raise ValueError("min_opacity must lie in (0, 1)")
        if self.noise_lr < 0 or self.opacity_reg < 0 or self.scale_reg < 0:
            raise ValueError("noise_lr, opacity_reg and scale_reg must be >= 0")
        if not 0 <= int(self.seed) < 1 << 64:
            raise ValueError("seed must be an unsigned 64-bit integer")


def refines(cfg, step):
    """Whether `step` (1-based) is a refinement step."""
    return cfg.refine_start < step < cfg.refine_stop and step % cfg.refine_every == 0


def grow_count(n, cap_max):
    """Gaussians a refinement appends to a set of n: 5 % up to cap_max, never a negative count (a set above the cap,
    e.g. one loaded from a file, neither grows nor shrinks)."""
    return max(0, min(cap_max, int(1.05 * n)) - n)


def seed_key(seed):
    """The Philox key (key0, key1) of a 64-bit seed."""
    seed = int(seed)
    return seed & 0xffffffff, seed >> 32


def row_segments(offs):
    """The gsb_row_segment table of a flat layout (parallel.flat_layout): one (offset, row_floats) per slice."""
    segs = []
    for o, c, shp in offs.values():
        row = 1
        for d in shp[1:]:
            row *= d
        segs.append(capi.RowSegment(o, row, 0))
    return (capi.RowSegment * len(segs))(*segs)


class MCMCRefiner:
    """Host control flow of the strategy over a SplatPipeline's flat parameter and Adam buffers."""

    def __init__(self, cfg=None):
        self.cfg = cfg or MCMCConfig()
        self.key = seed_key(self.cfg.seed)

    def regularize(self, pipe):
        """Adds the gradients of opacity_reg mean|o| + scale_reg mean|exp s| to the pipeline's gradient buffer."""
        c, n = self.cfg, pipe.n
        if n == 0 or (c.opacity_reg == 0 and c.scale_reg == 0):
            return
        p, g = pipe.p, pipe.g
        capi.check(capi.lib().gsb_mcmc_regularize(
            n, capi.ptr(p["opacities"]), capi.ptr(p["scales"]), c.opacity_reg / n, c.scale_reg / (3 * n),
            capi.ptr(g["opacities"]), capi.ptr(g["scales"]), capi.stream()))

    def add_noise(self, step, params, lr_means):
        """means += Sigma z sigma_100(1 - o - 0.995) lr_means noise_lr, in place on the dict's tensors."""
        c, n = self.cfg, params["means"].shape[0]
        if n == 0 or c.noise_lr == 0:
            return
        capi.check(capi.lib().gsb_mcmc_add_noise(
            n, capi.ptr(params["opacities"]), capi.ptr(params["scales"]), capi.ptr(params["quats"]), *self.key,
            step, lr_means * c.noise_lr, capi.ptr(params["means"]), capi.stream()))

    def finish_step(self, step, pipe, lr_means):
        """The rest of a training step after Adam: on a refinement step relocation then growth, then the noise
        (lr_means: the means learning rate after this step's update).  Returns (params, adam_m, adam_v, info) as
        densify.Densifier.finish_step does: pipe.p and the pipeline's moment views when the count is unchanged, new
        dicts of tensors after growth.  info = {refined, relocated, added, n}, plus the drawn indices
        (relocation_samples, growth_samples: device int32) of the phases that ran."""
        params = pipe.p
        adam_m, adam_v = flat_views(pipe.adam_m, pipe.offs), flat_views(pipe.adam_v, pipe.offs)
        info = {"refined": False, "relocated": 0, "added": 0, "n": pipe.n}
        if refines(self.cfg, step):
            info["refined"] = True
            params, adam_m, adam_v = self._refine(step, pipe, info)
            info["n"] = params["means"].shape[0]
        self.add_noise(step, params, lr_means)
        return params, adam_m, adam_v, info

    def _refine(self, step, pipe, info):
        L, P, s = capi.lib(), capi.ptr, capi.stream()
        c, n, p = self.cfg, pipe.n, pipe.p
        adam_m, adam_v = flat_views(pipe.adam_m, pipe.offs), flat_views(pipe.adam_v, pipe.offs)
        if n == 0:
            return p, adam_m, adam_v
        d = pipe.param_flat.device
        ws = torch.empty(L.gsb_mcmc_workspace_bytes(n), dtype=torch.uint8, device=d)
        cdf = torch.empty(n, dtype=torch.float64, device=d)
        dead = torch.empty(n, dtype=torch.int32, device=d)
        counts = torch.empty(n, dtype=torch.int32, device=d)
        result = torch.empty(4, dtype=torch.int32, device=d)
        segs = row_segments(pipe.offs)
        nseg, table = len(segs), C.addressof(segs)

        def plan(mask_dead):
            capi.check(L.gsb_mcmc_plan(n, P(p["opacities"]), c.min_opacity, int(mask_dead), P(ws), ws.numel(),
                                       P(cdf), P(dead) if mask_dead else None, P(result), s))

        def draw(m, tag, zero_moments):
            samples = torch.empty(m, dtype=torch.int32, device=d)
            capi.check(L.gsb_mcmc_sample(m, n, P(cdf), *self.key, step, tag, P(samples), P(counts), s))
            capi.check(L.gsb_mcmc_relocate(n, P(counts), c.min_opacity, P(p["opacities"]), P(p["scales"]),
                                           int(zero_moments), nseg, table, P(pipe.adam_m), P(pipe.adam_v), s))
            return samples

        plan(mask_dead=True)
        n_dead, live, any_positive, _ = result.tolist()      # the one host wait of a refinement
        if n_dead and live:
            samples = draw(n_dead, RELOCATE_TAG, zero_moments=True)
            capi.check(L.gsb_mcmc_copy_rows(n_dead, P(dead), P(samples), nseg, table, P(pipe.param_flat), s))
            info["relocated"], info["relocation_samples"] = n_dead, samples
        n_new = grow_count(n, c.cap_max)
        # After a relocation every drawn row has an opacity >= min_opacity > 0; without one the opacities are those
        # the plan saw.  So the growth weights sum to > 0 exactly when this holds, and no second read-back is needed.
        if not n_new or not (info["relocated"] or any_positive):
            return p, adam_m, adam_v
        plan(mask_dead=False)
        samples = draw(n_new, GROW_TAG, zero_moments=False)
        src_map = torch.cat([torch.arange(n, dtype=torch.int32, device=d), samples | _CHILD])
        new_n = n + n_new
        new_p = {k: gather_rows(src_map, new_n, t) for k, t in p.items()}
        new_m = {k: gather_rows(src_map, new_n, t, zero_children=True) for k, t in adam_m.items()}
        new_v = {k: gather_rows(src_map, new_n, t, zero_children=True) for k, t in adam_v.items()}
        info["added"], info["growth_samples"] = n_new, samples
        return new_p, new_m, new_v
