"""Per-image camera pose corrections for trainer.SplatTrainer (gsplat's pose optimisation), DESIGN.md D22:

    tr = SplatTrainer(params, pose=PoseConfig(num_images=len(cameras)))
    loss = tr.step(cam, gt, step, image=i)         # B > 1: image=[i0, i1, ...]
    deltas = tr.pose_deltas()                      # copy, [num_images, 9]
    cam_i = adjusted_camera(cam, deltas[i])        # image i's camera at its learned pose

Poses from structure-from-motion are often off by a fraction of a degree or a few millimetres; without a correction
the Gaussians absorb that error as blurred, doubled edges and floaters.  Each training image i gets e_i in R^9, a
translation e[0:3] and a 6-D rotation offset e[3:9], applied in the camera's own frame (include/gsplat_b200.h,
gsb_pose_apply).  The kernels live in csrc/pose.cu and csrc/project.cu; this file holds the four buffers (parameters,
gradient, Adam m and v), the learning-rate schedule and the Adam step counter.  There is no CPU fallback."""
from dataclasses import dataclass

import torch

from . import capi


@dataclass
class PoseConfig:
    """num_images: the training images, one correction each.  The learning rate at trainer step s (1-based) is
    lr * final_lr_factor^((s - 1) / max_steps); Adam takes betas (0.9, 0.999) and eps 1e-8, and reg is its L2 weight
    decay (the gradient gets reg * e for every image on every step that trains).  The defaults are gsplat's."""
    num_images: int
    lr: float = 1e-5
    reg: float = 1e-6
    final_lr_factor: float = 0.01
    max_steps: int = 30_000

    def __post_init__(self):
        if isinstance(self.num_images, bool) or int(self.num_images) != self.num_images or self.num_images < 1:
            raise ValueError("num_images must be an integer >= 1")
        if not self.lr >= 0:
            raise ValueError("lr must be >= 0")
        if not self.reg >= 0:
            raise ValueError("reg must be >= 0")
        if not self.final_lr_factor > 0:
            raise ValueError("final_lr_factor must be > 0")
        if isinstance(self.max_steps, bool) or int(self.max_steps) != self.max_steps or self.max_steps < 1:
            raise ValueError("max_steps must be an integer >= 1")


def learning_rate(cfg, step):
    """The corrections' learning rate at trainer step `step` (1-based)."""
    return cfg.lr * cfg.final_lr_factor ** ((step - 1) / cfg.max_steps)


def rot6d(d):
    """Rd of a 6-D rotation offset d [..., 6] (float64 torch): the rows b1, b2, b3 of gsb_pose_apply."""
    base = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0], dtype=d.dtype, device=d.device)
    a = d + base
    a1, a2 = a[..., 0:3], a[..., 3:6]
    b1 = a1 / a1.norm(dim=-1, keepdim=True)
    w = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = w / w.norm(dim=-1, keepdim=True)
    b3 = torch.linalg.cross(b1, b2, dim=-1)
    return torch.stack([b1, b2, b3], -2)


def adjusted_camera(cam, delta):
    """A model.Camera equal to `cam` at the pose the correction `delta` ([9], e.g. a row of pose_deltas()) gives it:
    camToWorld = c2w [[F Rd F, F t], [0, 1]] in the user's convention (F = diag(1, -1, -1) turns it into the
    projection's, where the correction is [R|T] Delta), computed in float64 and rounded once."""
    e = torch.as_tensor(delta, dtype=torch.float64).reshape(-1).cpu()
    if e.numel() != capi.POSE_FLOATS:
        raise ValueError(f"a pose correction has {capi.POSE_FLOATS} floats")
    F = torch.diag(torch.tensor([1.0, -1.0, -1.0], dtype=torch.float64))
    D = torch.eye(4, dtype=torch.float64)
    D[:3, :3] = F @ rot6d(e[3:9]) @ F
    D[:3, 3] = F @ e[0:3]
    c2w = torch.as_tensor(cam.camToWorld, dtype=torch.float64) @ D
    return cam.replace(cam_to_world=c2w.float())


class Poses:
    """The correction buffers [num_images, 9] and their optimiser state for one trainer."""

    def __init__(self, cfg, device):
        self.cfg = cfg
        self.deltas = torch.zeros((cfg.num_images, capi.POSE_FLOATS), dtype=torch.float32, device=device)
        self.grad = torch.zeros_like(self.deltas)
        self.exp_avg = torch.zeros_like(self.deltas)
        self.exp_avg_sq = torch.zeros_like(self.deltas)
        self.adam_t = 0

    def start_step(self):
        """Writes reg * e into the gradient buffer for every image: the step's first write of it (torch Adam's L2
        weight decay on the dense gradient)."""
        torch.mul(self.deltas, float(self.cfg.reg), out=self.grad)

    def adam_step(self, step):
        """One Adam step over every correction at trainer step `step`."""
        self.adam_t += 1
        t = self.adam_t
        capi.check(capi.lib().gsb_adam_step(self.deltas.numel(), capi.ptr(self.deltas), capi.ptr(self.grad),
                                            capi.ptr(self.exp_avg), capi.ptr(self.exp_avg_sq),
                                            learning_rate(self.cfg, step), 0.9, 0.999, 1e-8, 1.0 - 0.9 ** t,
                                            1.0 - 0.999 ** t, capi.stream()))
