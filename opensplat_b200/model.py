"""Host-side mirror of the reference's `Model` (model.hpp:22-137, model.cpp:58-248,311-500,780-784) over the
gsplat_b200 operators: the caller of the hot path, with the same members, step order and hyper-parameters, so a
training loop written against the reference reads the same here:

    model.optimizers_zero_grad(); rgb = model.forward(cam, step); loss = model.main_loss(rgb, gt, w)
    loss.backward(); model.optimizers_step(); model.schedulers_step(step); model.after_train(step)

What is fused relative to the reference (all behind the C ABI, parity-tested against the same ATen sequences):
parameter activations (exp / normalise / sigmoid / view directions) in one kernel, SH colour, projection, binning +
blend, L1+SSIM loss with gradient, one Adam kernel per tensor, densification statistics and topology edits.
There is no CPU fallback."""
import math

import torch

from . import capi, ops
from .densify import Densifier, RefineConfig
from .export import SceneWriter, load_ply


def projection_matrix(z_near, z_far, fov_x, fov_y, device):
    """model.cpp:35-47 (OpenGL-style perspective matrix with +z forward)."""
    t = z_near * math.tan(0.5 * fov_y)
    b = -t
    r = z_near * math.tan(0.5 * fov_x)
    l = -r
    return torch.tensor([[2.0 * z_near / (r - l), 0.0, (r + l) / (r - l), 0.0],
                         [0.0, 2 * z_near / (t - b), (t + b) / (t - b), 0.0],
                         [0.0, 0.0, (z_far + z_near) / (z_far - z_near), -1.0 * z_far * z_near / (z_far - z_near)],
                         [0.0, 0.0, 1.0, 0.0]], dtype=torch.float32, device=device)


class Camera:
    """The fields of the reference's Camera that Model::forward reads (input_data.hpp:12-44), and its distortion
    coefficients k1, k2, k3, p1, p2, which Camera::loadImage (images.ImageSet) undistorts the image with."""

    def __init__(self, width, height, fx, fy, cx, cy, cam_to_world, k1=0.0, k2=0.0, k3=0.0, p1=0.0, p2=0.0):
        self.width, self.height = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.camToWorld = torch.as_tensor(cam_to_world, dtype=torch.float32)
        self.k1, self.k2, self.k3, self.p1, self.p2 = float(k1), float(k2), float(k3), float(p1), float(p2)


# learning rates of Model::setupOptimizers (model.cpp:58-70)
LEARNING_RATES = {"means": 0.00016, "scales": 0.005, "quats": 0.001, "featuresDc": 0.0025, "featuresRest": 0.000125,
                  "opacities": 0.05}
MEANS_LR_FINAL = 0.0000016
MEANS_LR_INIT = float(torch.tensor(LEARNING_RATES["means"], dtype=torch.float64).float())   # the float lrInit
PARAM_NAMES = ("means", "scales", "quats", "featuresDc", "featuresRest", "opacities")


def downscale_factor(step, num_downscales, resolution_schedule):
    """Model::getDownscaleFactor (model.cpp:227-229)."""
    return int(2 ** max(num_downscales - step // resolution_schedule, 0))


def means_learning_rate(step, max_steps, lr_init):
    """OptimScheduler::step for the means (optim_scheduler.cpp:4-12): log-linear decay from lr_init (the float
    learning rate the optimizer was built with) to 1.6e-6 at max_steps."""
    t = max(min(float(step) / float(max_steps), 1.0), 0.0)
    return math.exp(math.log(lr_init) * (1.0 - t) + math.log(MEANS_LR_FINAL) * t)


def camera_setup(cam, downscale):
    """The camera block of Model::forward (model.cpp:120-142) at a downscale factor: returns (height, width,
    (fx, fy, cx, cy), view [4,4], proj [4,4], cam_pos [3]), the three tensors on the host.  The caller forms the
    full projection as `proj @ view` on the device."""
    sf = float(downscale)
    fx, fy, cx, cy = cam.fx / sf, cam.fy / sf, cam.cx / sf, cam.cy / sf
    height, width = int(float(cam.height) / sf), int(float(cam.width) / sf)
    c2w = cam.camToWorld
    R = c2w[:3, :3] @ torch.diag(torch.tensor([1.0, -1.0, -1.0]))     # flip y/z to gsplat conventions
    T = c2w[:3, 3:4]
    Rinv = R.t()
    Tinv = (-Rinv) @ T
    view = torch.eye(4)
    view[:3, :3] = Rinv
    view[:3, 3:4] = Tinv
    fov_x = 2.0 * math.atan(width / (2.0 * fx))
    fov_y = 2.0 * math.atan(height / (2.0 * fy))
    proj = projection_matrix(0.001, 1000.0, fov_x, fov_y, "cpu")
    return height, width, (fx, fy, cx, cy), view, proj, T.reshape(3)


class GaussianModel:
    def __init__(self, params, cfg=None, sh_degree=None, sh_degree_interval=1000, num_downscales=0,
                 resolution_schedule=3000, background=(0.6130, 0.0101, 0.3984), device="cuda:0", generator=None,
                 group=None, antialiased=False):
        """params: dict with the reference's six tensors (means [n,3], scales [n,3] log, quats [n,4] raw,
        featuresDc [n,3], featuresRest [n,K-1,3], opacities [n,1] logits).
        antialiased: render with the anti-aliased opacity (DESIGN D19, ops.ProjectGaussiansActivatedAntialiased):
        each Gaussian's opacity is scaled by how much the projection's 0.3 px^2 blur spread it.  The parameters, the
        refinement and the saved files keep the raw opacity."""
        from .mcmc import MCMCConfig
        if getattr(cfg, "absgrad", False):
            raise ValueError("GaussianModel's statistics take v_xy from autograd; absgrad (RefineConfig(absgrad=True)) "
                             "runs in trainer.SplatTrainer")
        if isinstance(cfg, MCMCConfig):
            raise ValueError("GaussianModel refines as the reference does (RefineConfig); the MCMC strategy "
                             "(MCMCConfig) runs in trainer.SplatTrainer")
        self.device = torch.device(device)
        self.cfg = cfg or RefineConfig()
        for k in PARAM_NAMES:
            t = torch.as_tensor(params[k]).to(device=self.device, dtype=torch.float32).contiguous().clone()
            setattr(self, k, t.requires_grad_())
        k_bases = self.featuresRest.shape[1] + 1
        self.shDegree = ops.deg_from_sh(k_bases) if sh_degree is None else int(sh_degree)
        self.shDegreeInterval = int(sh_degree_interval)
        self.numDownscales, self.resolutionSchedule = int(num_downscales), int(resolution_schedule)
        self.backgroundColor = torch.tensor(background, dtype=torch.float32, device=self.device)
        self.group = group
        self.antialiased = bool(antialiased)
        self.densifier = Densifier(self.cfg, generator=generator, group=group)
        self.writer = None
        self.xys = self.radii = None
        self.lastHeight = self.lastWidth = 0
        self.setup_optimizers()

    # ---- optimizers: six Adam instances with the reference's learning rates, fused kernel per tensor ----------
    def setup_optimizers(self):
        self.lr = dict(LEARNING_RATES)
        self.lr_init_means = MEANS_LR_INIT
        self.adam_m = {k: torch.zeros_like(getattr(self, k)) for k in PARAM_NAMES}
        self.adam_v = {k: torch.zeros_like(getattr(self, k)) for k in PARAM_NAMES}
        self.adam_t = 0

    def params(self):
        return {k: getattr(self, k) for k in PARAM_NAMES}

    def optimizers_zero_grad(self):
        for k in PARAM_NAMES:
            getattr(self, k).grad = None

    def optimizers_step(self, b1=0.9, b2=0.999, eps=1e-8):
        """torch::optim::Adam::step of the six optimizers (model.cpp:236-243); a tensor without gradient is skipped
        like torch does."""
        if self.group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            from .parallel import allreduce_tensor_grads     # data-parallel over views: one flat-bucket all-reduce
            allreduce_tensor_grads([getattr(self, k) for k in PARAM_NAMES], group=self.group)
        self.adam_t += 1
        t = self.adam_t
        L = capi.lib()
        with torch.no_grad():
            for k in PARAM_NAMES:
                p = getattr(self, k)
                if p.grad is None:
                    continue
                g = p.grad.contiguous()
                capi.check(L.gsb_adam_step(p.numel(), capi.ptr(p), capi.ptr(g), capi.ptr(self.adam_m[k]),
                                           capi.ptr(self.adam_v[k]), self.lr[k], b1, b2, eps, 1.0 - b1 ** t,
                                           1.0 - b2 ** t, capi.stream()))

    def schedulers_step(self, step):
        """OptimScheduler::step for the means (optim_scheduler.cpp:4-12): log-linear decay to 1.6e-6 at maxSteps."""
        self.lr["means"] = means_learning_rate(step, self.cfg.max_steps, self.lr_init_means)

    def get_downscale_factor(self, step):
        return downscale_factor(step, self.numDownscales, self.resolutionSchedule)

    # ---- Model::forward (model.cpp:83-225) ------------------------------------------------------------------
    def forward(self, cam, step):
        dev = self.device
        height, width, (fx, fy, cx, cy), view, proj, cam_pos = camera_setup(cam, self.get_downscale_factor(step))
        self.lastHeight, self.lastWidth = height, width
        view, proj, cam_pos = view.to(dev), proj.to(dev), cam_pos.to(dev)
        tb = ops.tile_bounds(width, height)
        # model.cpp:148-150,200 inside the projection: exp(scales), quaternion normalisation, sigmoid(opacities)
        project = ops.ProjectGaussiansActivatedAntialiased if self.antialiased else ops.ProjectGaussiansActivated
        xys, depths, radii, conics, num_tiles_hit, _, opac = project.apply(
            self.means, self.scales, 1.0, self.quats, self.opacities, view, proj @ view, fx, fy, cx, cy, height,
            width, tb)
        self.xys, self.radii, self.numTilesHit = xys, radii, num_tiles_hit
        xys.retain_grad()
        if float(radii.sum()) == 0.0:
            return self.backgroundColor.repeat(height, width, 1)
        degrees_to_use = min(step // self.shDegreeInterval, self.shDegree)
        # model.cpp:176-177,186-192 in one pass: no cat of featuresDc / featuresRest, view directions formed inside,
        # + 0.5 and clamp_min fused (and their gradients written straight into the two feature tensors' grads)
        rgbs = ops.SphericalHarmonicsRgb.apply(degrees_to_use, self.means.detach(), cam_pos, self.featuresDc,
                                               self.featuresRest)
        # model.cpp:213-222: rasterize + clamp_max(rgb, 1) in the blend kernel's epilogue
        return ops.RasterizeGaussiansClamped.apply(xys, depths, radii, conics, num_tiles_hit, rgbs, opac, height,
                                                   width, self.backgroundColor)

    def main_loss(self, rgb, gt, ssim_weight):
        """Model::mainLoss (model.cpp:780-784), fused forward + gradient."""
        return ops.MainLoss.apply(rgb, gt, ssim_weight)

    # ---- Model::afterTrain (model.cpp:311-500) ---------------------------------------------------------------
    def after_train(self, step):
        if self.xys is None:
            return {"refined": False}
        # xys.grad undefined <=> this view hit no Gaussian (model.cpp:315).  Single process: nothing to do.  Under a
        # process group the densifier still has to take part in the refine step's collectives (zero statistics).
        v_xy = self.xys.grad.detach().contiguous() if self.xys.grad is not None else None
        if v_xy is None and self.densifier._world() <= 1:
            return {"refined": False}
        with torch.no_grad():
            p = {k: getattr(self, k).detach() for k in PARAM_NAMES}
            new_p, new_m, new_v, info = self.densifier.after_train(
                step, p, self.adam_m, self.adam_v, v_xy, self.radii, self.lastHeight, self.lastWidth)
            if new_p is not p:
                for k in PARAM_NAMES:
                    setattr(self, k, new_p[k].requires_grad_())
                self.adam_m, self.adam_v = new_m, new_v
        return info

    # ---- Model::save (model.cpp:496-594) -----------------------------------------------------------------------
    def save(self, filename, step=0, keep_crs=False, scale=1.0, translation=(0.0, 0.0, 0.0), wait=True):
        if self.writer is None:
            self.writer = SceneWriter(self.device)
        p = {k: getattr(self, k).detach() for k in PARAM_NAMES}
        self.writer.save(filename, p, step, keep_crs, scale, translation)
        if wait:
            self.writer.wait()

    def load_ply(self, filename, keep_crs=False, scale=1.0, translation=(0.0, 0.0, 0.0)):
        """Model::loadPly (model.cpp:614-778): replaces the parameters, re-creates the optimizers, returns the step
        recorded in the file (the reference resumes training from it, opensplat.cpp:139-147)."""
        p, step = load_ply(filename, self.device, keep_crs, scale, translation)
        for k in PARAM_NAMES:
            setattr(self, k, p[k].requires_grad_())
        self.shDegree = ops.deg_from_sh(self.featuresRest.shape[1] + 1)
        self.setup_optimizers()
        self.densifier.xys_grad_norm = self.densifier.vis_counts = self.densifier.max_2d_size = None
        return step
