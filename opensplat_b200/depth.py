"""Per-image inverse-depth priors for trainer.SplatTrainer (graphdeco 3DGS's depth regularisation, gsplat's
depth_loss), DESIGN.md D23:

    maps = DepthMaps(priors, device)               # one [H,W] inverse-depth prior per training image (level 1)
    tr = SplatTrainer(params, depth=DepthConfig())
    f = downscale_factor(step, num_downscales, resolution_schedule)
    loss = tr.step(cam, images.gt(i, f), step, depth=maps.get(i, f))   # B > 1: depth=maps.get([i0, i1, ...], f)
    tr.depth_losses                                 # device [B]: the unweighted depth loss of each view

Colour says little about depth in textureless regions, sky or sparse captures; a prior there keeps the Gaussians at
the right distance.  A prior P is an INVERSE depth in the units of the trainer's cameras; a pixel is valid iff P is
finite and > 0, so 0, negative, NaN and inf mean "no data" (a sparse map from SfM points is a mostly-zero P).  Metric
depth d goes in as where(d > 0, 1 / d, 0); a monocular estimate must be aligned (scale and shift) to the SfM points
beforehand, as graphdeco's make_depth_scale.py does.

Each view with a prior adds w(s) * sum_valid |R - P| / (H W) to the loss, R = sum alpha T (1/z) the rendered inverse
depth (not normalised by alpha).  The kernels live in csrc/depth.cu; this file holds the weight schedule and the
priors' levels.  There is no CPU fallback."""
from dataclasses import dataclass

import torch

from . import capi


@dataclass
class DepthConfig:
    """The depth term's weight at trainer step s (1-based) is weight * final_weight_factor^(min(s - 1, max_steps) /
    max_steps): held at its final value past max_steps.  The defaults are graphdeco's (depth_l1_weight_init 1.0,
    depth_l1_weight_final 0.01, over 30 000 iterations)."""
    weight: float = 1.0
    final_weight_factor: float = 0.01
    max_steps: int = 30_000

    def __post_init__(self):
        if not self.weight >= 0:
            raise ValueError("weight must be >= 0")
        if not self.final_weight_factor > 0:
            raise ValueError("final_weight_factor must be > 0")
        if isinstance(self.max_steps, bool) or int(self.max_steps) != self.max_steps or self.max_steps < 1:
            raise ValueError("max_steps must be an integer >= 1")


def depth_weight(cfg, step):
    """The depth term's weight w(step) at trainer step `step` (1-based), in float64."""
    return cfg.weight * cfg.final_weight_factor ** (min(step - 1, cfg.max_steps) / cfg.max_steps)


class DepthMaps:
    """One inverse-depth prior per training image, at the size of that image's prepared level 1
    (images.ImageSet.level(i)), stored as fp32 on the device, and its downscaled levels.  Memory: 4 bytes per pixel,
    plus a quarter and a sixteenth of that for the levels of --num-downscales 2."""

    def __init__(self, maps, device="cuda:0"):
        self.device = torch.device(device)
        self._levels = []
        for i, m in enumerate(maps):
            t = torch.as_tensor(m)
            if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
                raise ValueError(f"prior {i} must be a [H,W] map, got shape {tuple(t.shape)}")
            self._levels.append({1: t.to(device=self.device, dtype=torch.float32).contiguous()})

    def __len__(self):
        return len(self._levels)

    def get(self, i, factor=1):
        """Image i's prior at downscale `factor` ([H/factor, W/factor] by integer division, as ImageSet.gt(i,
        factor)), built on first use by gsb_depth_downscale_mean and cached: a tensor for one index, a list for a list
        of indices.  i may be negative, as a list index."""
        if isinstance(i, (list, tuple)):
            return [self.get(k, factor) for k in i]
        levels = self._levels[range(len(self._levels))[int(i)]]
        factor = int(factor)
        if factor <= 1:
            return levels[1]
        if factor not in levels:
            src = levels[1]
            h, w = src.shape
            if h // factor < 1 or w // factor < 1:
                raise ValueError(f"factor {factor} leaves nothing of the {w}x{h} prior of image {i}")
            out = torch.empty((h // factor, w // factor), dtype=torch.float32, device=self.device)
            capi.check(capi.lib().gsb_depth_downscale_mean(h, w, factor, capi.ptr(src), capi.ptr(out), capi.stream()))
            levels[factor] = out
        return levels[factor]
