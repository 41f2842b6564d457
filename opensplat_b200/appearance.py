"""Per-image appearance for trainer.SplatTrainer: one learned bilateral grid per training image (Wang et al. 2024,
"Bilateral Guided Radiance Field Processing"; gsplat's bilateral-grid module), DESIGN.md D21:

    tr = SplatTrainer(params, appearance=AppearanceConfig(num_images=len(cameras)))
    loss = tr.step(cam, gt, step, image=i)         # B > 1: image=[i0, i1, ...]
    grids = tr.appearance_grids()                  # copy, [num_images, 12, 8, 16, 16]

Each grid maps the rendered colour to its photo's colour with an affine transform that varies smoothly over the image
and with brightness, so shot-to-shot exposure and white balance go into the grids instead of the Gaussians.  The grids
enter the loss only: evaluate(), render() and `image` show the raw render.  The kernels live in csrc/bilagrid.cu;
this file holds the four grid buffers (parameters, gradient, Adam m and v), the learning-rate schedule and the grids'
Adam step counter.  There is no CPU fallback."""
from dataclasses import dataclass

import torch

from . import capi


@dataclass
class AppearanceConfig:
    """num_images: the training images, one grid each.  The learning rate at trainer step s (1-based) is
    lr * final_lr_factor^((s - 1) / max_steps) * (warmup_start + (1 - warmup_start) min(s - 1, warmup_steps) /
    warmup_steps); Adam takes betas (0.9, 0.999) and eps 1e-15.  tv_weight scales the grids' total variation, which
    enters as a gradient only (the returned loss stays the image loss).  The defaults are gsplat's."""
    num_images: int
    lr: float = 2e-3
    final_lr_factor: float = 0.01
    warmup_start: float = 0.01
    warmup_steps: int = 1000
    max_steps: int = 30_000
    tv_weight: float = 10.0
    grid_x: int = capi.BILAGRID_X
    grid_y: int = capi.BILAGRID_Y
    grid_l: int = capi.BILAGRID_L

    def __post_init__(self):
        if isinstance(self.num_images, bool) or int(self.num_images) != self.num_images or self.num_images < 1:
            raise ValueError("num_images must be an integer >= 1")
        if (self.grid_x, self.grid_y, self.grid_l) != (capi.BILAGRID_X, capi.BILAGRID_Y, capi.BILAGRID_L):
            raise ValueError(f"the grid size is fixed at {capi.BILAGRID_X} x {capi.BILAGRID_Y} x {capi.BILAGRID_L}")
        if not self.lr > 0 or not self.final_lr_factor > 0:
            raise ValueError("lr and final_lr_factor must be > 0")
        if not 0.0 <= self.warmup_start <= 1.0:
            raise ValueError("warmup_start must lie in [0, 1]")
        if self.warmup_steps < 1 or self.max_steps < 1:
            raise ValueError("warmup_steps and max_steps must be >= 1")
        if not self.tv_weight >= 0:
            raise ValueError("tv_weight must be >= 0")


def learning_rate(cfg, step):
    """The grids' learning rate at trainer step `step` (1-based)."""
    s = step - 1
    decay = cfg.final_lr_factor ** (s / cfg.max_steps)
    warm = cfg.warmup_start + (1.0 - cfg.warmup_start) * min(s, cfg.warmup_steps) / cfg.warmup_steps
    return cfg.lr * decay * warm


def identity_grids(n, device):
    """n identity grids, channels-last [n, L, Y, X, 12]: A = I, b = 0 in every cell."""
    g = torch.zeros((n, capi.BILAGRID_L, capi.BILAGRID_Y, capi.BILAGRID_X, capi.BILAGRID_COEFFS), dtype=torch.float32,
                    device=device)
    g[..., 0] = g[..., 5] = g[..., 10] = 1.0
    return g


def to_gsplat_order(grids):
    """[n, L, Y, X, 12] -> [n, 12, L, Y, X] (F.grid_sample's order), a copy."""
    return grids.permute(0, 4, 1, 2, 3).contiguous()


def from_gsplat_order(grids):
    """[n, 12, L, Y, X] -> [n, L, Y, X, 12], a copy."""
    return grids.permute(0, 2, 3, 4, 1).contiguous()


class Appearance:
    """The grid buffers and their optimiser state for one trainer."""

    def __init__(self, cfg, device):
        self.cfg = cfg
        self.grids = identity_grids(cfg.num_images, device)
        self.grad = torch.zeros_like(self.grids)
        self.exp_avg = torch.zeros_like(self.grids)
        self.exp_avg_sq = torch.zeros_like(self.grids)
        self.adam_t = 0

    def tv(self):
        """Writes tv_weight * dTV into the gradient buffer: the step's first write of it."""
        capi.check(capi.lib().gsb_bilagrid_tv(self.cfg.num_images, capi.ptr(self.grids), float(self.cfg.tv_weight),
                                              capi.ptr(self.grad), None, capi.stream()))

    def adam_step(self, step):
        """One Adam step over every grid at trainer step `step`."""
        self.adam_t += 1
        t = self.adam_t
        capi.check(capi.lib().gsb_adam_step(self.grids.numel(), capi.ptr(self.grids), capi.ptr(self.grad),
                                            capi.ptr(self.exp_avg), capi.ptr(self.exp_avg_sq),
                                            learning_rate(self.cfg, step), 0.9, 0.999, 1e-15, 1.0 - 0.9 ** t,
                                            1.0 - 0.999 ** t, capi.stream()))
