"""Fisheye cameras on the H100 (DESIGN D27).

1. Kernels against the float64 restatement (tests/project_fisheye_f64.py) on random scenes out to theta_lim, on the
   axis, either side of the small-r switch, beyond theta_lim and behind the camera: forward outputs within the
   certified bound, radii and num_tiles_hit exact on certified Gaussians, the VJP against float64 autograd of the map
   (J by autograd too); the accumulating and camera-gradient forms against the plain one.
2. Geometry: small blobs rendered by SplatTrainer.render land at fx theta_d(theta) cos(phi) + cx - 0.5.
3. Trainer: one fisheye step matches the autograd composition (ops.ProjectGaussiansFisheye); mixed pinhole / fisheye
   steps; the refusals; a fisheye scene recovered from a perturbed start.
"""
import gc
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pose_f64 as pf64  # noqa: E402
import project_fisheye_f64 as pf  # noqa: E402
import test_gpu_trainer as tg  # noqa: E402
from test_gpu_mask import _compare, _frozen, _grads, _masks, _problem  # noqa: E402
from util import rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = (0.05, -0.02, 0.004, -0.0005)
GEOM = ("means", "scales", "quats", "opacities")


@pytest.fixture(autouse=True)
def _release_cached_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _fwd(cam, m, a, q, ol, aa):
    from opensplat_b200 import capi
    L, P = capi.lib(), capi.ptr
    n = m.shape[0]
    o = dict(cov3d=torch.empty(n, 6, device=DEV), xys=torch.empty(n, 2, device=DEV), depths=torch.empty(n, device=DEV),
             radii=torch.empty(n, dtype=torch.int32, device=DEV), conics=torch.empty(n, 3, device=DEV),
             num_tiles_hit=torch.empty(n, dtype=torch.int32, device=DEV), opacities=torch.empty(n, device=DEV))
    capi.check(L.gsb_project_forward_fisheye(
        n, P(m), P(a), 1.0, P(q), P(ol), P(cu(cam.V)), cam.fx, cam.fy, cam.cx, cam.cy, *cam.k, cam.theta_lim, cam.H,
        cam.W, cam.tiles_x, cam.tiles_y, cam.clip, P(o["cov3d"]), P(o["xys"]), P(o["depths"]), P(o["radii"]),
        P(o["conics"]), P(o["num_tiles_hit"]), P(o["opacities"]), int(aa), capi.stream()))
    return o


def _bwd(cam, m, a, q, ol, o, cot, aa, acc=0, prev=None, part=None):
    from opensplat_b200 import capi
    L, P = capi.lib(), capi.ptr
    n = m.shape[0]
    g = prev or dict(v_mean3d=torch.zeros(n, 3, device=DEV), v_scale=torch.zeros(n, 3, device=DEV),
                     v_quat=torch.zeros(n, 4, device=DEV), v_opacity_logits=torch.zeros(n, device=DEV))
    capi.check(L.gsb_project_backward_fisheye(
        n, P(m), P(a), 1.0, P(q), P(ol), P(cu(cam.V)), cam.fx, cam.fy, *cam.k, cam.theta_lim, cam.H, cam.W,
        P(o["radii"]), P(o["conics"]), P(cot[0]), P(cot[1]), P(cot[2]), P(cot[3]), P(g["v_mean3d"]),
        P(g["v_scale"]), P(g["v_quat"]), P(g["v_opacity_logits"]), acc, int(aa), P(part), capi.stream()))
    return g


@pytest.mark.parametrize("n", [1000, 100_000])
@pytest.mark.parametrize("aa", [0, 1])
@pytest.mark.parametrize("identity", [False, True])
def test_kernels_against_the_float64_restatement(n, aa, identity):
    cam = pf.fisheye_camera(1280, 960, 11 + n, k=K, identity=identity)
    host = pf.random_fisheye_gaussians(cam, n, 7 + n)
    m, a, q, ol = (cu(x) for x in host)
    o = _fwd(cam, m, a, q, ol, aa)
    rng = np.random.default_rng(n)
    cot = [cu(rng.standard_normal(s).astype(np.float32)) for s in ((n, 2), (n,), (n, 3), (n,))]
    g = _bwd(cam, m, a, q, ol, o, cot, aa)
    torch.cuda.synchronize()
    ref = pf.project(cam, *(torch.as_tensor(x) for x in host), aa=bool(aa),
                     v_xy=cot[0].cpu(), v_depth=cot[1].cpu(), v_conic=cot[2].cpu(), v_opacity=cot[3].cpu())
    cert, kept = ref["cert"], ref["kept"]
    print(f"n={n} kept={int(kept.sum())} cert={float(cert.double().mean()):.4f} series={int(ref['series'].sum())}")
    assert float(cert.double().mean()) > 0.98 and int(ref["series"].sum()) > 0
    for name in ("radii", "num_tiles_hit"):
        got = o[name].cpu().to(torch.int64)
        assert torch.equal(got[cert], ref[name][cert]), name
    for name in ("xys", "depths", "conics", "cov3d", "opacities"):
        got = o[name].cpu().double()
        msk = cert if got.dim() == 1 else cert[:, None].expand_as(got)
        err = (got - ref[name]).abs()[msk]
        bound = 2.0 * ref["B_" + name][msk] + 1e-30
        worst = float((err / bound).max()) if err.numel() else 0.0
        print(f"  {name}: worst err/bound {worst:.3g}")
        assert worst <= 1.0, name
    # the VJP against float64 autograd, per row relative to its largest entry.  v_mean3d carries every fisheye term (the
    # pixel centre through t and J's own derivatives) and is held on every row; v_scale and v_quat go through the
    # pinhole's covariance chain, whose fp32 conditioning on near-degenerate covariances is not bounded here, so they
    # are held on 99.8 % of the rows (a wrong convention fails on most rows)
    for name, frac in (("v_mean3d", 1.0), ("v_scale", 0.998), ("v_quat", 0.998), ("v_opacity_logits", 1.0)):
        got, want = g[name].cpu().double(), ref[name]
        rows = cert & torch.isfinite(want.reshape(n, -1)).all(1)
        d = (got - want).abs().reshape(n, -1)[rows]
        scale = want.abs().reshape(n, -1)[rows].amax(1, keepdim=True) + 1e-6
        rel = (d / scale).amax(1)
        ok = float((rel <= 1e-2).double().mean())
        print(f"  {name}: worst rel err {float(rel.max()):.3g}, rows within 1e-2: {ok:.5f}")
        assert ok >= frac, name


def test_accumulate_and_camera_gradient_forms():
    from opensplat_b200 import capi
    n = 20_000
    cam = pf.fisheye_camera(1280, 960, 3, k=K)
    host = pf.random_fisheye_gaussians(cam, n, 4)
    m, a, q, ol = (cu(x) for x in host)
    for aa in (0, 1):
        o = _fwd(cam, m, a, q, ol, aa)
        rng = np.random.default_rng(aa)
        cot = [cu(rng.standard_normal(s).astype(np.float32)) for s in ((n, 2), (n,), (n, 3), (n,))]
        plain = _bwd(cam, m, a, q, ol, o, cot, aa)
        part = torch.empty(capi.lib().gsb_project_camera_partials_floats(n), device=DEV)
        cg = _bwd(cam, m, a, q, ol, o, cot, aa, part=part)
        for k in plain:
            assert torch.equal(plain[k], cg[k]), k
        prev = {k: torch.randn_like(v) for k, v in plain.items()}
        acc = _bwd(cam, m, a, q, ol, o, cot, aa, acc=1, prev={k: v.clone() for k, v in prev.items()})
        for k in plain:
            assert torch.equal(acc[k], prev[k] + plain[k]), k
        vv, vp = torch.empty(4, 4, device=DEV), torch.empty(4, 4, device=DEV)
        L = capi.lib()
        capi.check(L.gsb_project_camera_grad_reduce(part.numel() // capi.CAMGRAD_TERMS, capi.ptr(part),
                                                    capi.ptr(vv), capi.ptr(vp), capi.stream()))
        part2 = torch.empty_like(part)
        _bwd(cam, m, a, q, ol, o, cot, aa, part=part2)
        assert torch.equal(part, part2)
        assert torch.count_nonzero(vp) == 0
        # float64 autograd of the map w.r.t. the view matrix
        ref = pf.project(cam, *(torch.as_tensor(x) for x in host), aa=bool(aa))
        kept = ref["kept"]
        V = torch.as_tensor(cam.V).double().reshape(4, 4).requires_grad_()
        ins = [torch.as_tensor(x).double() for x in host]
        uv, depth, conic, op = pf.forward_map(cam, *ins, aa=bool(aa), V=V)
        c = [x.cpu().double() for x in cot]
        keep = kept[:, None]
        loss = ((torch.where(keep, uv, 0) * c[0]).sum() + (torch.where(kept, depth, 0) * c[1]).sum()
                + (torch.where(keep, conic, 0) * c[2]).sum()
                + (torch.where(kept | (not aa), op, 0) * c[3]).sum())
        want, = torch.autograd.grad(loss, V)
        got = vv.cpu().double()
        rel = float((got[:3] - want[:3]).abs().max() / want[:3].abs().max())
        print(f"  aa={aa}: camera gradient rel err {rel:.3g}")
        assert rel <= 1e-3
        assert torch.count_nonzero(vv[3]) == 0


def _fish_camera(W, H, k, c2w=None):
    from opensplat_b200.model import Camera
    th = pf.fisheye_camera(W, H, 0, k=k).theta_lim
    tdl = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
    f = 0.5 * min(W, H) / tdl
    c2w = np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32) if c2w is None else c2w
    return Camera(W, H, f, f, 0.5 * W, 0.5 * H, c2w, k1=k[0], k2=k[1], k3=k[2], k4=k[3], model="fisheye")


def test_blob_centroids_follow_the_fisheye_map():
    from opensplat_b200.trainer import SplatTrainer
    W = H = 1024
    cam = _fish_camera(W, H, K)
    thetas = [0.0, 0.3, 0.7, 1.0, 1.3]
    phis = [0.0, 1.1, 2.5, 4.0, 5.5]
    t = []
    for th, ph in zip(thetas, phis):
        d = np.array([math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th)])
        t.append(3.0 * d)
    t = np.array(t)
    # c2w = diag(1, -1, -1) is camera_setup's identity view: a view-space point t sits at world t
    means = t
    n = len(t)
    s = np.log(np.full((n, 3), 3.0 * 0.6 / cam.fx))
    params = dict(means=means.astype(np.float32), scales=s.astype(np.float32),
                  quats=np.tile([1.0, 0, 0, 0], (n, 1)).astype(np.float32),
                  featuresDc=np.ones((n, 3), np.float32), featuresRest=np.zeros((n, 15, 3), np.float32),
                  opacities=np.full((n, 1), 0.0, np.float32))
    tr = SplatTrainer(params, device=DEV, background=(0.0, 0.0, 0.0))
    r = tr.render(cam, 1)
    alpha = r["alpha"].double().cpu().numpy()
    yy, xx = np.mgrid[0:H, 0:W]
    for th, ph in zip(thetas, phis):
        tdp = th * (1 + K[0] * th ** 2 + K[1] * th ** 4 + K[2] * th ** 6 + K[3] * th ** 8)
        u = cam.fx * tdp * math.cos(ph) + cam.cx - 0.5
        v = cam.fy * tdp * math.sin(ph) + cam.cy - 0.5
        win = (np.abs(xx - u) < 12) & (np.abs(yy - v) < 12)
        w = alpha * win
        cu_, cv_ = (w * xx).sum() / w.sum(), (w * yy).sum() / w.sum()
        print(f"theta={th}: centroid off by ({cu_ - u:.4f}, {cv_ - v:.4f}) px")
        assert abs(cu_ - u) <= 0.05 and abs(cv_ - v) <= 0.05


def _fish_cams(cams, k=K):
    return [c.replace(model="fisheye", k1=k[0], k2=k[1], k3=k[2], k4=k[3], p1=0.0, p2=0.0) for c in cams]


def _composition(tr, params, cams, gts, views, aa=False, masks=None, priors=None, step=7, grids=None, cam_grad=False):
    """Gradients of mean_b(MainLoss [of the render sliced through grids[b]] + w(step) depth_loss) through the autograd
    operators (ops.ProjectGaussiansFisheye for a fisheye view) at the trainer's view matrices and colours of its last
    step: ({name: grad}, [(viewmat, projmat or None)] per view, with .grad when cam_grad)."""
    from opensplat_b200 import ops
    from opensplat_b200.depth import depth_weight
    from opensplat_b200.model import fisheye_theta_limit
    pp = tr.pipe
    H, W = pp.H, pp.W
    dev = {k: v.to(DEV).clone().requires_grad_() for k, v in params.items() if k in GEOM}
    total, cams_out = 0.0, []
    for b, v in enumerate(views):
        c = cams[v]
        Vm = tr.viewmats[b].clone().requires_grad_(cam_grad)
        a = (dev["means"], dev["scales"], 1.0, dev["quats"], dev["opacities"], Vm)
        Pm = None
        if c.model == "fisheye":
            k = (c.k1, c.k2, c.k3, c.k4)
            xys, depths, radii, conics, nth, _, opac = ops.ProjectGaussiansFisheye.apply(
                *a, c.fx, c.fy, c.cx, c.cy, k, fisheye_theta_limit(*k), H, W, ops.tile_bounds(W, H), 0.01, aa)
        else:
            Pm = tr.projmats[b].clone().requires_grad_(cam_grad)
            proj = ops.ProjectGaussiansActivatedAntialiased if aa else ops.ProjectGaussiansActivated
            xys, depths, radii, conics, nth, _, opac = proj.apply(*a, Pm, c.fx, c.fy, c.cx, c.cy, H, W,
                                                                  ops.tile_bounds(W, H))
        prior = None if priors is None else priors[b]
        if prior is None:
            img = ops.RasterizeGaussiansClamped.apply(xys, depths, radii, conics, nth, tr.rgbs_views[b].detach(),
                                                      opac, H, W, pp.background)
        else:
            inv = torch.where(radii > 0, 1.0 / torch.where(radii > 0, depths, 1.0), 0.0)
            img, R, _ = ops.RasterizeGaussiansDepthClamped.apply(xys, depths, radii, conics, nth,
                                                                 tr.rgbs_views[b].detach(), opac, H, W, pp.background,
                                                                 inv)
        if grids is not None:
            img = ops.BilateralGridSlice.apply(grids[b], img)
        loss = ops.MainLoss.apply(img, gts[v], tr.ssim_weight, None if masks is None else masks[b])
        if prior is not None:
            ok = torch.isfinite(prior) & (prior > 0)
            loss = loss + depth_weight(tr.depth, step) * ((R - torch.where(ok, prior, 0.0)).abs() * ok).sum() / (H * W)
        total = total + loss
        cams_out.append((Vm, Pm))
    (total / len(views)).backward()
    return {k: dev[k].grad for k in GEOM}, cams_out


def _priors(H, W, V=3):
    """Inverse-depth priors with invalid pixels (0, NaN, inf, negative), as test_gpu_depth_prior's."""
    yy, xx = np.mgrid[0:H, 0:W]
    out = []
    for v in range(V):
        P = (0.25 + 0.04 * np.sin(0.05 * xx + v) * np.cos(0.04 * yy)).astype(np.float32)
        P[(xx % 7 == 0) | (yy % 9 == 0)] = 0.0
        P[0, :4] = [np.nan, np.inf, -1.0, 0.0]
        out.append(cu(P))
    return out


@pytest.mark.parametrize("mode", ["one_view", "mixed_two_views", "antialiased_mask", "appearance", "depth",
                                  "depth_mixed_two_views"])
def test_one_step_matches_the_autograd_composition(mode):
    from opensplat_b200.appearance import AppearanceConfig
    from opensplat_b200.depth import DepthConfig
    params, cams, gts, H, W = _problem()
    fish = _fish_cams(cams)
    aa, ms, ps, grids, use = False, None, None, None, fish
    if mode == "one_view":
        tr = _frozen(params)
        views = [1]
        tr.step(fish[1], gts[1], 7)
    elif mode == "mixed_two_views":
        tr = _frozen(params, 2)
        use = [cams[0], fish[1], fish[2]]
        views = [0, 1]
        tr.step([use[0], use[1]], gts[[0, 1]], 7)
    elif mode == "antialiased_mask":
        tr = _frozen(params, antialiased=True)
        views, aa, ms = [2], True, [_masks(H, W)[2]]
        tr.step(fish[2], gts[2], 7, mask=ms[0])
    elif mode == "appearance":
        tr = _frozen(params, appearance=AppearanceConfig(num_images=3))
        tr.appearance.adam_step = lambda step: None
        views = [0]
        tr.step(fish[0], gts[0], 7, image=0)
        grids = [tr.appearance_grids()[0]]
    elif mode == "depth":
        tr = _frozen(params, depth=DepthConfig(weight=2.0))
        views, ps = [1], [_priors(H, W)[1]]
        tr.step(fish[1], gts[1], 7, depth=ps[0])
    else:
        tr = _frozen(params, 2, depth=DepthConfig(weight=2.0))
        use = [fish[0], cams[1], fish[2]]
        views, ps = [0, 1], [_priors(H, W)[0], _priors(H, W)[1]]
        tr.step([use[0], use[1]], gts[[0, 1]], 7, depth=ps)
    torch.cuda.synchronize()
    got = _grads(tr)
    assert float(got["means"].abs().sum()) > 0
    want, _ = _composition(tr, params, use, gts, views, aa, ms, ps, 7, grids)
    _compare(got, want, tol=1e-3 if grids is not None else 2e-4)
    if ps is not None:
        # the depth term is a real part of it: without the priors the gradient differs
        plain, _ = _composition(tr, params, use, gts, views, aa, ms, None, 7, grids)
        assert rel_l2(got["means"].cpu().numpy(), plain["means"].reshape(-1).cpu().numpy()) > 1e-2


@pytest.mark.parametrize("mixed", [False, True])
def test_pose_correction_gradient_through_a_fisheye_view(mixed):
    """The camera gradient of a fisheye view (cam_partials -> gsb_project_camera_grad_reduce, v_projmat = 0 ->
    gsb_pose_backward) against float64 autograd of the correction through the composition's viewmat gradient; at
    B = 2 next to a pinhole view whose gradient also takes the projmat path, and with a depth prior."""
    from opensplat_b200.depth import DepthConfig
    from opensplat_b200.pose import PoseConfig
    params, cams, gts, H, W = _problem()
    fish = _fish_cams(cams)
    B = 2 if mixed else 1
    tr = _frozen(params, B, pose=PoseConfig(num_images=3, reg=0.0), depth=DepthConfig(weight=2.0))
    tr.poses.adam_step = lambda step: None
    tr.poses.deltas.copy_(torch.stack([torch.from_numpy(pf64.random_pose(i, 0.01, 0.02)) for i in range(3)]))
    e0 = tr.poses.deltas.clone()
    if mixed:
        use, views, images, ps = [fish[0], cams[1], fish[2]], [0, 1], [2, 1], [_priors(H, W)[0], None]
        tr.step([use[0], use[1]], gts[[0, 1]], 5, image=images, depth=ps)
    else:
        use, views, images, ps = fish, [1], [2], [_priors(H, W)[1]]
        tr.step(fish[1], gts[1], 5, image=2, depth=ps[0])
    torch.cuda.synchronize()
    grads, cams_out = _composition(tr, params, use, gts, views, priors=ps, step=5, cam_grad=True)
    _compare(_grads(tr), grads)
    for b, (Vm, Pm) in enumerate(cams_out):
        img = images[b]
        G_P = torch.zeros(4, 4, dtype=torch.float64) if Pm is None else Pm.grad.cpu().double()
        want = pf64.pose_grad(e0[img].cpu(), tr.base_viewmats[b].cpu().double(), tr.projs[b].cpu().double(),
                              Vm.grad.cpu().double(), G_P)      # the composition's loss already carries 1/B
        got = tr.poses.grad[img].cpu().double()
        err = float((got - want).abs().max() / want.abs().max())
        print(f"view {b} ({use[views[b]].model}): pose gradient rel err {err:.3g}")
        assert err <= 2e-4


def test_fisheye_steps_with_mcmc_and_absgrad():
    from opensplat_b200.mcmc import MCMCConfig
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem()
    fish = _fish_cams(cams)
    for cfg in (MCMCConfig(cap_max=5000), tg.refine_config(absgrad=True, warmup_length=2, refine_every=2)):
        tr = SplatTrainer(params, cfg, device=DEV)
        for s in range(1, 6):
            loss = tr.step(fish[s % 3], gts[s % 3], s)
        assert torch.isfinite(loss).all() and tr.n > 0


def test_parallel_world1_replicas_with_fisheye_views():
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1",
                        "--master-addr", "127.0.0.1", "--master-port", "29577",
                        os.path.join(ROOT, "tools", "check_parallel_fisheye.py")], capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-4000:])
    if r.returncode != 0:
        print(r.stderr[-6000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "check_ok=True" in r.stdout and "plain_trainer_bit_identical=True" in r.stdout


def test_image_set_renders_the_distortion_instead_of_resampling():
    """A fisheye camera's image and mask only take the downscale resize: no undistortion, new_k None, the whole image
    as roi, and bytes equal to those of a distortion-free pinhole camera of the same size; the returned camera keeps
    the model and k1..k4, with the intrinsics rescaled."""
    from opensplat_b200.images import ImageSet
    from opensplat_b200.model import Camera
    rng = np.random.default_rng(5)
    h, w = 301, 403
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    m = (rng.uniform(size=(h, w)) > 0.2).astype(np.uint8)
    c2w = np.eye(4, dtype=np.float32)
    fish = Camera(w, h, 150.0, 151.0, 200.5, 150.25, c2w, k1=0.05, k2=-0.02, k3=0.004, k4=-0.0005, model="fisheye")
    plain = Camera(w, h, 150.0, 151.0, 200.5, 150.25, c2w)
    for factor in (1.0, 1.5, 2.0):
        a = ImageSet([fish], [img], downscale_factor=factor, masks=[m], device=DEV)
        b = ImageSet([plain], [img], downscale_factor=factor, masks=[m], device=DEV)
        assert a.new_k == [None]
        lv = a.level(0)
        assert a.roi == [(0, 0, lv.shape[1], lv.shape[0])] == b.roi
        assert torch.equal(lv, b.level(0)) and torch.equal(a.level(0, 2), b.level(0, 2))
        assert torch.equal(a.mask(0), b.mask(0)) and torch.equal(a.mask(0, 2), b.mask(0, 2))
        c, d = a.cameras[0], b.cameras[0]
        assert (c.model, c.k1, c.k2, c.k3, c.k4, c.p1, c.p2) == ("fisheye", fish.k1, fish.k2, fish.k3, fish.k4, 0, 0)
        assert (c.width, c.height, c.fx, c.fy, c.cx, c.cy) == (d.width, d.height, d.fx, d.fy, d.cx, d.cy)
        if factor > 1:
            assert c.width < w and c.fx < fish.fx
    # the same distortion on a pinhole camera is undistorted and cropped: a different image
    dist = Camera(w, h, 150.0, 151.0, 200.5, 150.25, c2w, k1=0.05, k2=-0.02, k3=0.004)
    u = ImageSet([dist], [img], masks=[m], device=DEV)
    assert u.new_k[0] is not None and not torch.equal(u.level(0), ImageSet([fish], [img], device=DEV).level(0))


def test_refusals():
    from opensplat_b200.filter3d import Filter3DConfig
    from opensplat_b200.model import GaussianModel
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem()
    fish = _fish_cams(cams)
    with pytest.raises(ValueError):
        Filter3DConfig(cameras=[cams[0], fish[1]])
    tr = SplatTrainer(params, device=DEV, filter3d=Filter3DConfig(cameras=cams))
    with pytest.raises(ValueError):
        tr.step(fish[0], gts[0], 1)
    model = GaussianModel(params, device=DEV)
    with pytest.raises(ValueError):
        model.forward(fish[0], 1)


def _psnr(a, b):
    return float(-10 * torch.log10(((a - b) ** 2).mean()))


def test_training_recovers_a_fisheye_scene():
    from opensplat_b200.trainer import SplatTrainer
    k = (0.08, -0.03, 0.006, -0.0006)
    p, c2w, _, intr, H, W = tg.make_problem(n=6000, V=6, H=128, W=128)
    cams = [_fish_camera(W, H, k, c2w[v]) for v in range(6)]
    truth = SplatTrainer(p, device=DEV)
    gts = [truth.render(c, 1)["rgb"].clone() for c in cams]
    rng = np.random.default_rng(0)
    q = {kk: v.copy() for kk, v in p.items()}
    q["means"] = (q["means"] + rng.normal(0, 0.08, q["means"].shape)).astype(np.float32)
    q["featuresDc"] = (q["featuresDc"] + rng.normal(0, 0.8, q["featuresDc"].shape)).astype(np.float32)
    tr = SplatTrainer(q, tg.refine_config(warmup_length=10 ** 6), device=DEV)
    before = _psnr(tr.render(cams[5], 1)["rgb"], gts[5])
    for s in range(1, 301):
        v = s % 5
        tr.step(cams[v], gts[v], s)
    after = _psnr(tr.render(cams[5], 1)["rgb"], gts[5])
    print(f"held-out fisheye PSNR {before:.2f} -> {after:.2f} dB")
    assert after - before >= 6.0
