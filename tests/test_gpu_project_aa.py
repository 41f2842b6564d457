"""GPU: the anti-aliased projection (DESIGN D19) -- gsb_project_forward_activated_aa, gsb_project_backward_activated_aa
and _aa_acc, the operators ops.ProjectGaussiansActivatedAntialiased / gsb::ProjectGaussiansActivatedAntialiased, and
GaussianModel / SplatTrainer(antialiased=True).

  * forward: every output but the opacity is bit-identical to gsb_project_forward_activated's; the opacity lies within
    C B of the float64 map (tests/project_aa_f64.py) on the Gaussians it certifies, and is 0 where radii == 0;
  * backward: the writing and accumulating kernels within C B of float64 autograd per element, acc == prior + write
    bit for bit, a NULL v_opacity gives the plain kernel's gradients and a zero opacity gradient, degenerate Gaussians
    give finite values and a zero opacity;
  * the Python and C++ operators give identical bits;
  * a sub-pixel Gaussian rendered at downscale 1, 2 and 4 keeps its light (sum of alpha x downscale^2) as the float64
    model of the blend says it should, and the plain projection does not;
  * the trainer follows the model, a B = 2 step is the mean of two one-view passes, the step's launch sequence is the
    default one with the _aa entry points, and 300 steps on flat Gaussians keep every gradient and moment finite."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import project_aa_f64 as pa  # noqa: E402
import project_f64 as pf  # noqa: E402
import test_gpu_trainer as tg  # noqa: E402
import test_gpu_trainer_launches as tl  # noqa: E402
import test_gpu_trainer_views as tv  # noqa: E402
from test_gpu_project_f64 import Worst  # noqa: E402
from test_project_aa_f64_reference import _scene, degenerate_gaussians  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRADS = ("v_mean3d", "v_scale", "v_quat", "v_opacity_logits")
FWD = ("cov3d", "xys", "depths", "radii", "conics", "num_tiles_hit")


def cu(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype).contiguous()


def _forward(fn, cam, m, s, q, ol, gs):
    from opensplat_b200 import capi, ops
    n, P = m.shape[0], capi.ptr
    V, Pm = cu(cam.V.reshape(4, 4)), cu(cam.P.reshape(4, 4))
    tb = ops.tile_bounds(cam.W, cam.H)
    out = dict(cov3d=torch.empty((n, 6), device=DEV), xys=torch.empty((n, 2), device=DEV),
               depths=torch.empty((n,), device=DEV), radii=torch.empty((n,), dtype=torch.int32, device=DEV),
               conics=torch.empty((n, 3), device=DEV), num_tiles_hit=torch.empty((n,), dtype=torch.int32, device=DEV),
               opacities=torch.empty((n,), device=DEV))
    capi.check(fn(n, P(m), P(s), gs, P(q), P(ol), P(V), P(Pm), cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W, tb[0],
                  tb[1], cam.clip, *[P(out[k]) for k in FWD + ("opacities",)], capi.stream()))
    return out


def _backward(fn, cam, m, s, q, opac_or_logits, gs, out, c, vo, outs=None):
    from opensplat_b200 import capi
    n, P = m.shape[0], capi.ptr
    V, Pm = cu(cam.V.reshape(4, 4)), cu(cam.P.reshape(4, 4))
    if outs is None:
        outs = [torch.full((n, 3), float("nan"), device=DEV), torch.full((n, 3), float("nan"), device=DEV),
                torch.full((n, 4), float("nan"), device=DEV), torch.full((n,), float("nan"), device=DEV)]
    capi.check(fn(n, P(m), P(s), gs, P(q), P(opac_or_logits), P(V), P(Pm), cam.fx, cam.fy, cam.H, cam.W,
                  P(out["radii"]), P(out["conics"]), P(c["v_xy"]), P(c["v_depth"]), P(c["v_conic"]), P(vo),
                  *[P(o) for o in outs], capi.stream()))
    return outs


def _cotangents(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = dict(v_xy=torch.randn((n, 2), device=DEV, generator=g), v_depth=torch.randn((n,), device=DEV, generator=g),
             v_conic=torch.randn((n, 3), device=DEV, generator=g), v_opacity=torch.randn((n,), device=DEV, generator=g))
    z = dict(c, v_xy=torch.zeros_like(c["v_xy"]), v_depth=torch.zeros_like(c["v_depth"]))
    return [c, z]


def run_case(name, cam, m, s, q, ol, gs, seed=0, min_cert=0.99, operators=True):
    from opensplat_b200 import capi, cpp_ops, ops
    L = capi.lib()
    m, s, q, ol = cu(m), cu(s), cu(q), cu(ol)
    n = m.shape[0]
    r = pa.project_aa(cam, m, s, q, ol, gs, device=DEV)
    cert = r["cert"]
    assert float(cert.double().mean()) >= min_cert, f"{name}: certified {float(cert.double().mean()):.4f}"
    w = Worst(name)
    plain = _forward(L.gsb_project_forward_activated, cam, m, s, q, ol, gs)
    aa = _forward(L.gsb_project_forward_activated_aa, cam, m, s, q, ol, gs)
    for k in FWD:
        assert torch.equal(aa[k], plain[k]), f"{name}: {k} differs from the plain projection"
    w.check("fwd.", aa["opacities"], r, "opacities", cert)
    assert bool((aa["opacities"][aa["radii"] <= 0] == 0).all())
    g = torch.Generator(device=DEV).manual_seed(seed + 99)
    for ci, c in enumerate(_cotangents(n, seed)):
        rb = pa.project_aa(cam, m, s, q, ol, gs, device=DEV, **c)
        tag = f"bwd{ci}."
        vjp = _backward(L.gsb_project_backward_activated_aa, cam, m, s, q, ol, gs, aa, c, c["v_opacity"])
        for k, o in zip(GRADS, vjp):
            assert bool(torch.isfinite(o).all()), f"{name}: non-finite {k}"
            w.check(tag, o, rb, k, cert)
        prior = [torch.randn(o.shape, device=DEV, generator=g) * (o.abs().mean() + 1e-30)
                 * torch.exp(torch.empty(o.shape, device=DEV).uniform_(0, 14, generator=g)) for o in vjp]
        acc = _backward(L.gsb_project_backward_activated_aa_acc, cam, m, s, q, ol, gs, aa, c, c["v_opacity"],
                        [p.clone() for p in prior])
        for k, a, p, v in zip(GRADS, acc, prior, vjp):
            assert torch.equal(a, p + v), f"{name}: acc {k} is not prior + write"
        # NULL v_opacity: the plain kernel's geometry gradients, bit for bit, and a zero logit gradient
        va = _backward(L.gsb_project_backward_activated_aa, cam, m, s, q, ol, gs, aa, c, None)
        vp = _backward(L.gsb_project_backward_activated, cam, m, s, q, plain["opacities"], gs, plain, c, None)
        for k, a, b in zip(GRADS[:3], va[:3], vp[:3]):
            assert torch.equal(a, b), f"{name}: NULL v_opacity {k}"
        assert bool((va[3] == 0).all())
        if operators and n:
            _operators(cam, m, s, q, ol, gs, c, cpp_ops.ops(), ops)
    torch.cuda.synchronize()
    w.report(cert)
    return r, aa


def _operators(cam, m, s, q, ol, gs, c, co, ops):
    """ops.ProjectGaussiansActivatedAntialiased and torch.ops.opensplat_b200.project_gaussians_activated_antialiased:
    identical outputs and gradients."""
    n = m.shape[0]
    V, Pm = cu(cam.V.reshape(4, 4)), cu(cam.P.reshape(4, 4))
    tb = ops.tile_bounds(cam.W, cam.H)
    res = []
    for which in ("py", "cpp"):
        mg, sg, qg = (x.clone().requires_grad_() for x in (m, s, q))
        og = ol.clone().reshape(n, 1).requires_grad_()
        if which == "py":
            o = ops.ProjectGaussiansActivatedAntialiased.apply(mg, sg, gs, qg, og, V, Pm, cam.fx, cam.fy, cam.cx,
                                                               cam.cy, cam.H, cam.W, tb, cam.clip)
        else:
            o = co.project_gaussians_activated_antialiased(mg, sg, gs, qg, og, V, Pm, cam.fx, cam.fy, cam.cx, cam.cy,
                                                            cam.H, cam.W, cam.clip)
        xys, depths, _, conics, _, _, opac = o
        ((xys * c["v_xy"]).sum() + (depths * c["v_depth"]).sum() + (conics * c["v_conic"]).sum()
         + (opac.reshape(n) * c["v_opacity"]).sum()).backward()
        res.append([t.detach() for t in o] + [mg.grad, sg.grad, qg.grad, og.grad])
    for a, b in zip(*res):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------ cases
@pytest.mark.parametrize("scene", ["general", "small", "axis_aligned_ties", "golden_ties"])
def test_kernels_against_the_float64_reference(scene):
    cam, m, s, q, ol, gs = _scene(scene)
    run_case(scene, cam, m, s, q, ol, gs, seed=len(m))


def test_c2_size():
    """1M Gaussians at 1920x1080, as the trainer runs them."""
    cam = pf.camera_from_setup(pf.general_camera(1920, 1080, 3))
    n = 1_000_000
    m, s, q = pf.random_gaussians(cam, n, seed=4, act=True)
    ol = np.random.default_rng(5).uniform(-8, 8, n).astype(np.float32)
    run_case("C2 1M 1920x1080", cam, m, s, q, ol, 1.0, seed=5, operators=False)


def test_degenerate_gaussians():
    """det0 == 0 exactly (two zero scales), and log-scales from -30 to 4 at depths from 0.02 to 50: finite outputs and
    gradients, opacities in [0, 1]; comp = 0 gives a zero opacity."""
    from opensplat_b200 import capi
    L = capi.lib()
    cam, m, s, q, ol = degenerate_gaussians()
    rng = np.random.default_rng(3)
    k = 64
    m2 = np.concatenate([m, np.stack([rng.uniform(-1, 1, k), rng.uniform(-1, 1, k), rng.uniform(0.02, 50, k)], -1)])
    s2 = np.concatenate([s, rng.uniform(-30, 4, (k, 3))])
    q2 = np.concatenate([q, rng.standard_normal((k, 4))])
    ol2 = np.concatenate([ol, rng.uniform(-20, 20, k)])
    m2, s2, q2, ol2 = cu(m2), cu(s2), cu(q2), cu(ol2)
    out = _forward(L.gsb_project_forward_activated_aa, cam, m2, s2, q2, ol2, 1.0)
    assert bool((out["opacities"][: len(m)] == 0).all()) and bool((out["radii"][: len(m)] > 0).all())
    assert bool(torch.isfinite(out["opacities"]).all())
    assert bool(((out["opacities"] >= 0) & (out["opacities"] <= 1)).all())
    for c in _cotangents(m2.shape[0], 1):
        for o in _backward(L.gsb_project_backward_activated_aa, cam, m2, s2, q2, ol2, 1.0, out, c, c["v_opacity"]):
            assert bool(torch.isfinite(o).all())


# ------------------------------------------------------------------------------------------------------ functional
def _alpha_model(xy, conic, opac, H, W):
    """Sum over the pixels of the blend's alpha for one Gaussian (float64): pixel (x, y) at integer coordinates,
    sigma = a dx^2 / 2 + b dx dy + c dy^2 / 2, alpha = min(0.999, o exp(-sigma)), skipped below 1/255 (and T never
    reaches 1e-4 with one Gaussian)."""
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    dx, dy = xy[0] - x, xy[1] - y
    sig = 0.5 * conic[0] * dx * dx + conic[1] * dx * dy + 0.5 * conic[2] * dy * dy
    a = torch.clamp(opac * torch.exp(-sig), max=0.999)
    return float(torch.where((sig >= 0) & (a >= 1.0 / 255.0), a, 0.0).sum())


def test_subpixel_gaussian_keeps_its_light_across_resolutions():
    """One Gaussian of opacity 0.9 and 0.8 px standard deviation at full resolution (0.2 px at downscale 4), near the
    axis of a 256x256 camera, rendered at downscale 1, 2 and 4 through the projection and the depth / alpha blend.
    Its light, sum alpha x downscale^2, is the same at every downscale up to what the blend's 1/255 cut and pixel
    sampling change; the float64 model of the blend evaluated on the kernels' own xys / conics / opacities gives that
    change, and the kernels must agree with it to 1e-4.  The plain projection's light grows with the downscale."""
    from opensplat_b200 import ops
    from opensplat_b200.model import Camera, camera_setup
    Wf = Hf = 256
    f = 300.0
    cam = Camera(Wf, Hf, f, f, 0.5 * Wf, 0.5 * Hf, np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32))
    z = 3.0
    sig_world = 0.8 * z / f                                  # 0.8 px at full resolution
    means = cu([[0.013, -0.021, z]])
    scales = cu(np.log([[sig_world, sig_world, sig_world]]))
    quats = cu([[1.0, 0.0, 0.0, 0.0]])
    logit = cu([[np.log(0.9 / 0.1)]])
    light = {}
    for aa in (False, True):
        proj_op = ops.ProjectGaussiansActivatedAntialiased if aa else ops.ProjectGaussiansActivated
        for d in (1, 2, 4):
            H, W, (fx, fy, cx, cy), view, proj, _ = camera_setup(cam, d)
            view, pm = view.to(DEV), (proj @ view).to(DEV)
            xys, depths, radii, conics, nth, _, opac = proj_op.apply(means, scales, 1.0, quats, logit, view, pm, fx,
                                                                     fy, cx, cy, H, W, ops.tile_bounds(W, H))
            assert int(radii[0]) > 0
            rgb = torch.ones((1, 3), device=DEV)
            _, _, alpha = ops.RasterizeGaussiansDepth.apply(xys, depths, radii, conics, nth, rgb, opac, H, W,
                                                            torch.zeros(3, device=DEV))
            got = float(alpha.double().sum())
            model = _alpha_model(xys[0].double().cpu(), conics[0].double().cpu(), float(opac[0]), H, W)
            assert abs(got - model) <= 1e-4 * model, (aa, d, got, model)
            light[aa, d] = (got * d * d, model * d * d)
    print("\nlight (kernel, float64 model) x downscale^2: " + str(light))
    # the model's own spread (about 3 %: the 1/255 cut takes more of the fainter, smaller footprint); 2 % above it is
    # what the kernels may add
    ref = light[True, 1][1]
    spread = max(abs(light[True, d][1] / ref - 1) for d in (2, 4))
    assert spread <= 0.06, spread
    for d in (2, 4):
        assert abs(light[True, d][0] / light[True, 1][0] - 1) <= spread + 0.02
        assert light[False, d][0] / light[False, 1][0] >= 1.5          # the dilation: brighter when smaller


# ------------------------------------------------------------------------------------------------------ trainers
def test_trainer_follows_gaussian_model_through_refinements():
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV)}
    steps, seed = 34, 11
    model, lm, cm = tg.run_model(p, cams, gts_d, steps, seed, cfg=tg.refine_config(), sh_degree_interval=8,
                                 antialiased=True)
    tr, lt, ct = tg.run_trainer(p, cams, gts_d, steps, seed, cfg=tg.refine_config(), sh_degree_interval=8,
                                antialiased=True)
    assert cm[18] == len(p["means"]) and cm[19] != cm[18] and cm[29] != cm[28]
    tg._compare(model, tr, lm, lt, cm, ct, exact=True)
    # and the mode changes the training: the plain trainer's losses differ
    _, lp, _ = tg.run_trainer(p, cams, gts_d, 4, seed, cfg=tg.refine_config(), sh_degree_interval=8)
    assert np.abs(lp - lt[:4]).max() > 1e-4


def test_trainer_follows_gaussian_model_through_the_downscale_schedule():
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV), 2: torch.from_numpy(tg._half(gts)).to(DEV)}
    kw = dict(sh_degree_interval=8, num_downscales=1, resolution_schedule=6, antialiased=True)
    model, lm, cm = tg.run_model(p, cams, gts_d, 12, 3, cfg=tg.refine_config(), **kw)
    tr, lt, ct = tg.run_trainer(p, cams, gts_d, 12, 3, cfg=tg.refine_config(), **kw)
    assert tr.resolution == (W, H) and tr.pixel_reallocs == 1
    tg._compare(model, tr, lm, lt, cm, ct, exact=True)


def test_two_view_step_is_the_mean_of_two_one_view_passes():
    from opensplat_b200.trainer import SplatTrainer
    B = 2
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    views, step = [0, 1], 9
    grads, losses1, _ = tv._single_view_grads(p, cams, gt, views, step, sh_degree_interval=8, antialiased=True)
    tr = tv._no_adam(SplatTrainer(tv._params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV,
                                  ssim_weight=tv.SSIM_W, sh_degree_interval=8, views_per_step=B, antialiased=True))
    lossB = tr.step([cams[v] for v in views], gt[views], step)
    torch.cuda.synchronize()
    assert float((lossB - losses1).abs().max()) <= 1e-6
    mean = (grads[0] + grads[1]) * (1.0 / B)
    pp = tr.pipe
    geom = pp.geom_numel
    assert torch.equal(pp.grad_flat[:geom], mean[:geom])
    o, c, _ = pp.offs["coeffs"]
    assert tv._rel_l2(pp.grad_flat[o:o + c], mean[o:o + c]) <= 1e-6


AA_NAMES = {"gsb_project_forward_activated": "gsb_project_forward_activated_aa",
            "gsb_project_backward_activated": "gsb_project_backward_activated_aa",
            "gsb_project_backward_activated_acc": "gsb_project_backward_activated_aa_acc"}


@pytest.mark.parametrize("case", ["one_view", "two_views"])
def test_step_issues_the_default_sequence_with_the_aa_projection(case, monkeypatch):
    from opensplat_b200 import capi
    from opensplat_b200.trainer import SplatTrainer
    B, _, expected = tl.CASES[case]
    expected = [AA_NAMES.get(x, x) for x in expected]
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    log = []
    monkeypatch.setattr(capi, "_lib", tl._Recorder(capi.lib(), log))
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, tg.refine_config(warmup_length=10 ** 6),
                      device=DEV, views_per_step=B, antialiased=True)

    def args(views):
        return (views[0], gt[0]) if B == 1 else (views, gt[:B])
    for step in range(1, 6):
        tr.step(*args([cams[(step - 1 + b) % 3] for b in range(B)]), step)
    torch.cuda.synchronize()
    del log[:]
    tr.step(*args([cams[b] for b in range(B)]), 6)
    torch.cuda.synchronize()
    assert [x for x in log if not x.startswith("gsb_densify_stats_")] == expected, log


def test_flat_gaussians_train_300_steps_with_finite_state():
    """One log-scale of every Gaussian at -12 (flat discs, comp small when seen edge-on): 300 antialiased steps with
    refinements and an alpha reset keep every gradient and Adam moment finite."""
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem(n=3000)
    p["scales"][:, 0] = -12.0
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    tr = SplatTrainer(tv._params(p), tg.refine_config(max_steps=300, reset_alpha_every=30), device=DEV,
                      sh_degree_interval=50, antialiased=True)
    for step in range(1, 301):
        loss = tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
        pp = tr.pipe
        assert bool(torch.isfinite(pp.grad_flat).all()), step
        assert bool(torch.isfinite(pp.adam_m).all()) and bool(torch.isfinite(pp.adam_v).all()), step
        assert bool(torch.isfinite(pp.param_flat).all()) and bool(torch.isfinite(loss).all()), step
    print(f"\nflat run: {tr.n} Gaussians after 300 steps, last loss {float(loss[0]):.4f}")
