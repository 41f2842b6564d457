"""Mip-Splatting's 3-D smoothing filter (DESIGN D24): one float f per Gaussian, bounding its world-space size by the
highest sampling rate any training camera has at its position, so that training at low resolution or rendering closer
than any training camera does not leave sub-sample Gaussians behind as speckle.

    cfg = Filter3DConfig(cameras=train_cams)               # the training cameras (model.Camera), full resolution
    trainer = SplatTrainer(params, filter3d=cfg)           # recomputes f, renders with it, bakes it on save

f is a constant between recomputations (no gradient).  The projection builds each Gaussian's covariance from
sigma_k = sqrt(e_k^2 + f^2) (e_k = exp(a_k), a the log-scales) and multiplies its opacity by
c3 = prod_k e_k / sigma_k; bake() writes that effective Gaussian as plain log-scales and logits, which any 3DGS viewer
renders as trained.  The arithmetic lives in csrc/filter3d.cu and csrc/project.cu; there is no CPU fallback."""
import math
from dataclasses import dataclass

import torch

from . import capi
from .model import Camera, camera_setup


@dataclass(frozen=True)
class Filter3DConfig:
    """cameras: the training cameras (a non-empty sequence of model.Camera), each taken at full resolution -- not the
    held-out view.  variance: the filter's screen-space variance in px^2 at the sharpest camera; near: the least
    view-space depth at which a camera counts as seeing a Gaussian; margin: how far outside the image (as a fraction
    of its width / height) a camera still counts; recompute_every: the recomputation period once refinement has
    stopped.  Defaults are Mip-Splatting's."""
    cameras: tuple
    variance: float = 0.2
    near: float = 0.2
    margin: float = 0.15
    recompute_every: int = 100

    def __post_init__(self):
        if isinstance(self.cameras, Camera):
            raise ValueError("cameras= takes a sequence of model.Camera (the training cameras)")
        cams = tuple(self.cameras)
        if not cams or not all(isinstance(c, Camera) for c in cams):
            raise ValueError("cameras= must be a non-empty sequence of model.Camera")
        if not all(float(c.fx) > 0 and float(c.fy) > 0 and int(c.width) > 0 and int(c.height) > 0 for c in cams):
            raise ValueError("every camera needs fx, fy > 0 and a positive image size")
        if any(c.model != "pinhole" for c in cams):
            raise ValueError("the 3-D filter's sampling rate is a pinhole camera's; fisheye cameras are not supported")
        object.__setattr__(self, "cameras", cams)
        for name in ("variance", "near", "margin"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
                raise ValueError(f"{name} must be a finite number >= 0, got {v!r}")
        k = self.recompute_every
        if isinstance(k, bool) or not isinstance(k, int) or k < 1:
            raise ValueError(f"recompute_every must be an int >= 1, got {k!r}")


def camera_table(cameras, device):
    """The cameras as gsb_filter3d_compute takes them: float32 [C, 18] on `device`, one row per camera of
    model.camera_setup(cam, 1): viewmat rows 0..2, fx, fy, cx, cy, W, H."""
    rows = []
    for cam in cameras:
        H, W, (fx, fy, cx, cy), view, _, _ = camera_setup(cam, 1)
        rows.append(torch.cat([view[:3].reshape(12).float(),
                               torch.tensor([fx, fy, cx, cy, W, H], dtype=torch.float32)]))
    return torch.stack(rows).contiguous().to(device)


def recompute_due(strategy, cfg, step, refined):
    """Whether a trainer recomputes f after step `step`: after every step whose refinement ran, and every
    cfg.recompute_every steps once refinement has stopped (step > stop_split_at for a densify.RefineConfig, step >=
    refine_stop for an mcmc.MCMCConfig), except within the last recompute_every steps before strategy.max_steps."""
    if refined:
        return True
    from .mcmc import MCMCConfig
    k = cfg.recompute_every
    stopped = step >= strategy.refine_stop if isinstance(strategy, MCMCConfig) else step > strategy.stop_split_at
    return stopped and step % k == 0 and step < strategy.max_steps - k


def compute_filter3d(means, cameras, variance=0.2, near=0.2, margin=0.15, out=None):
    """f [n] (float32, on the means' device) for means [n,3] from `cameras` (a sequence of model.Camera, or a
    camera_table).  A Gaussian no camera sees takes the largest depth of the seen ones; f is 0 everywhere when no
    Gaussian is seen.  out: an [n] float32 tensor to write into."""
    m = capi.f32(means)
    n, d = m.shape[0], m.device
    table = cameras if isinstance(cameras, torch.Tensor) else camera_table(cameras, d)
    if table.dim() != 2 or table.shape[1] != capi.FILTER3D_CAM_FLOATS or table.shape[0] < 1:
        raise ValueError(f"cameras must be a non-empty sequence of model.Camera or a [C,{capi.FILTER3D_CAM_FLOATS}] "
                         "table")
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=d)
    elif out.dtype != torch.float32 or tuple(out.shape) != (n,) or out.device != d:
        raise ValueError(f"out must be a float32 [{n}] tensor on the means' device")
    L = capi.lib()
    ws = torch.empty(L.gsb_filter3d_workspace_bytes(), dtype=torch.uint8, device=d)
    capi.check(L.gsb_filter3d_compute(n, capi.ptr(m), table.shape[0], capi.ptr(table), float(near), float(margin),
                                      float(variance), capi.ptr(ws), ws.numel(), capi.ptr(out), capi.stream()))
    return out


def bake(params, f):
    """The filter baked into the scene `params` (the reference's six tensors, or the flat layout's means / scales /
    quats / coeffs / opacities): a new dict whose "scales" are log(e^2 + f^2) / 2 and "opacities" logit(sigmoid(l)
    c3), computed in fp64 and rounded once; the other entries are the given tensors."""
    scales, logits = capi.f32(params["scales"]), capi.f32(params["opacities"])
    n = scales.shape[0]
    if f.shape != (n,) or f.dtype != torch.float32:
        raise ValueError(f"f must be a float32 [{n}] tensor")
    out = dict(params)
    out["scales"], out["opacities"] = torch.empty_like(scales), torch.empty_like(logits)
    capi.check(capi.lib().gsb_filter3d_bake(n, capi.ptr(scales), capi.ptr(logits), capi.ptr(f.contiguous()),
                                            capi.ptr(out["scales"]), capi.ptr(out["opacities"]), capi.stream()))
    return out
