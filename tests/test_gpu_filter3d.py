"""Mip-Splatting's 3-D smoothing filter on the H100 (DESIGN D24): gsb_filter3d_compute against the fp32 restatement
bit for bit, the filtered projection against its unfiltered counterpart at f = 0 (bit for bit) and against the
float64 map at f > 0, the footprint bound, the reset and the bake, the trainer (at f = 0 it is the plain trainer bit
for bit; every option combination runs), the exported scene, and the zoom-in test the filter exists for."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter3d_f64 as ff  # noqa: E402
import project_f64 as pf  # noqa: E402
from test_filter3d_f64_reference import orbit_cameras  # noqa: E402

from opensplat_b200 import capi, ops  # noqa: E402
from opensplat_b200.filter3d import Filter3DConfig, bake, camera_table, compute_filter3d  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------------------------ the filter value
@pytest.mark.parametrize("n", [0, 1, 255, 256, 65537])
def test_filter_is_the_fp32_restatement(n):
    cams = orbit_cameras(9, centred=False, seed=n % 7)
    table = ff.camera_rows(cams)
    means = (np.random.default_rng(n).normal(size=(n, 3)) * 2.5).astype(np.float32)
    got = compute_filter3d(_cu(means), cams).cpu().numpy()
    want = ff.filter_fp32(means, table)
    assert got.dtype == np.float32 and got.shape == (n,)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if n > 1000:
        f64, cert = ff.filter_f64(means, table)
        np.testing.assert_allclose(got[cert], f64[cert], rtol=2e-6)


def test_filter_at_scale_is_deterministic():
    n, k = 1_000_000, 300
    cams = orbit_cameras(k, W=320, H=240, fx=300.0, centred=False, seed=11)
    means = (np.random.default_rng(3).normal(size=(n, 3)) * 2.0).astype(np.float32)
    table = camera_table(cams, DEV)
    m = _cu(means)
    a = compute_filter3d(m, table)
    b = compute_filter3d(m, table)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    want = ff.filter_fp32(means, table.cpu().numpy())
    assert np.array_equal(a.cpu().numpy().view(np.uint32), want.view(np.uint32))


def test_all_unseen_gives_zero():
    cams = orbit_cameras(4)
    f = compute_filter3d(_cu(np.full((300, 3), 1e4, np.float32)), cams)
    assert (f == 0).all()


# ------------------------------------------------------------------------------------------------ the projection
def _problem(n, seed, wide=False):
    g = np.random.default_rng(seed)
    cam = pf.camera_from_setup(orbit_cameras(1, W=160, H=120, fx=140.0)[0])
    means = (g.normal(size=(n, 3)) * 0.7).astype(np.float32)
    lo, hi = (-20.0, 20.0) if wide else (-6.0, -1.0)
    scales = g.uniform(lo, hi, size=(n, 3)).astype(np.float32)
    quats = g.normal(size=(n, 4)).astype(np.float32)
    logits = (g.normal(size=n) * 2).astype(np.float32)
    cot = dict(v_xy=g.normal(size=(n, 2)).astype(np.float32), v_depth=g.normal(size=n).astype(np.float32),
               v_conic=g.normal(size=(n, 3)).astype(np.float32), v_opacity=g.normal(size=n).astype(np.float32))
    return cam, means, scales, quats, logits, cot


def _forward(cam, means, scales, quats, logits, f, aa):
    n = means.shape[0]
    L = capi.lib()
    o = dict(cov3d=torch.empty((n, 6), device=DEV), xys=torch.empty((n, 2), device=DEV),
             depths=torch.empty(n, device=DEV), radii=torch.empty(n, dtype=torch.int32, device=DEV),
             conics=torch.empty((n, 3), device=DEV), nth=torch.empty(n, dtype=torch.int32, device=DEV),
             opac=torch.empty(n, device=DEV))
    V, Pm = _cu(cam.V), _cu(cam.P)
    head = (n, capi.ptr(means), capi.ptr(scales), 1.0, capi.ptr(quats), capi.ptr(logits))
    tail = (capi.ptr(V), capi.ptr(Pm), cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W, cam.tiles_x, cam.tiles_y, 0.01,
            *(capi.ptr(o[k]) for k in ("cov3d", "xys", "depths", "radii", "conics", "nth", "opac")))
    if f is None:
        fn = L.gsb_project_forward_activated_aa if aa else L.gsb_project_forward_activated
        capi.check(fn(*head, *tail, capi.stream()))
    else:
        capi.check(L.gsb_project_forward_activated_filter3d(*head, capi.ptr(f), *tail, int(aa), capi.stream()))
    return o


def _backward(cam, means, scales, quats, logits, f, fw, cot, aa, acc, cg, prev=None):
    n = means.shape[0]
    L = capi.lib()
    V, Pm = _cu(cam.V), _cu(cam.P)
    out = prev if prev is not None else dict(v_means=torch.zeros((n, 3), device=DEV),
                                             v_scales=torch.zeros((n, 3), device=DEV),
                                             v_quats=torch.zeros((n, 4), device=DEV),
                                             v_logits=torch.zeros(n, device=DEV))
    out = {k: v.clone() for k, v in out.items()}
    part = torch.zeros(max(L.gsb_project_camera_partials_floats(n), 1), device=DEV)
    c = {k: _cu(v) for k, v in cot.items()}
    opac = logits if (aa or f is not None) else fw["opac"]
    args = [n, capi.ptr(means), capi.ptr(scales), 1.0, capi.ptr(quats), capi.ptr(opac), capi.ptr(V), capi.ptr(Pm),
            cam.fx, cam.fy, cam.H, cam.W, capi.ptr(fw["radii"]), capi.ptr(fw["conics"]), capi.ptr(c["v_xy"]),
            capi.ptr(c["v_depth"]), capi.ptr(c["v_conic"]), capi.ptr(c["v_opacity"]),
            *(capi.ptr(out[k]) for k in ("v_means", "v_scales", "v_quats", "v_logits"))]
    if f is not None:
        capi.check(L.gsb_project_backward_activated_filter3d(*args[:6], capi.ptr(f), *args[6:], int(acc), int(aa),
                                                             int(cg), capi.ptr(part) if cg else None, capi.stream()))
    elif cg:
        capi.check(L.gsb_project_backward_activated_camgrad(*args, int(acc), int(aa), capi.ptr(part), capi.stream()))
    else:
        fn = {(0, 0): L.gsb_project_backward_activated, (1, 0): L.gsb_project_backward_activated_acc,
              (0, 1): L.gsb_project_backward_activated_aa, (1, 1): L.gsb_project_backward_activated_aa_acc}
        capi.check(fn[(int(acc), int(aa))](*args, capi.stream()))
    torch.cuda.synchronize()
    return out, part


def _same_bits(a, b, zero_sign=False):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    if zero_sign:
        a, b = np.where(a == 0, 0, a), np.where(b == 0, 0, b)
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.parametrize("n", [1, 257, 65537])
def test_f_zero_is_the_unfiltered_projection_bit_for_bit(n):
    cam, means, scales, quats, logits, cot = _problem(n, n, wide=True)
    m, s, q, l = _cu(means), _cu(scales), _cu(quats), _cu(logits)
    zero = torch.zeros(n, device=DEV)
    for aa in (False, True):
        a, b = _forward(cam, m, s, q, l, None, aa), _forward(cam, m, s, q, l, zero, aa)
        for k in a:
            assert _same_bits(a[k], b[k]), (aa, k)
        prev = _backward(cam, m, s, q, l, None, a, cot, aa, False, False)[0]
        for acc in (False, True):
            for cg in (False, True):
                ra, pa = _backward(cam, m, s, q, l, None, a, cot, aa, acc, cg, prev if acc else None)
                rb, pb = _backward(cam, m, s, q, l, zero, b, cot, aa, acc, cg, prev if acc else None)
                for k in ra:
                    assert _same_bits(ra[k], rb[k], zero_sign=True), (aa, acc, cg, k)
                if cg:
                    assert _same_bits(pa, pb, zero_sign=True)


@pytest.mark.parametrize("aa", [False, True])
def test_f_positive_matches_the_float64_map(aa):
    n = 4000
    cam, means, scales, quats, logits, cot = _problem(n, 7)
    f = np.random.default_rng(8).uniform(0.0, 0.03, n).astype(np.float32)
    m, s, q, l, fd = _cu(means), _cu(scales), _cu(quats), _cu(logits), _cu(f)
    fw = _forward(cam, m, s, q, l, fd, aa)
    g, _ = _backward(cam, m, s, q, l, fd, fw, cot, aa, False, False)
    kept = fw["radii"].cpu() > 0
    t = lambda a: torch.from_numpy(np.asarray(a)).to(torch.float64)
    xy, tz, conic, o = ff.filtered_map(cam, t(means), t(scales), t(quats), t(logits), t(f), aa, kept)
    k = kept.numpy()
    assert k.mean() > 0.5
    worst = 0.0
    for got, want in ((fw["xys"], xy), (fw["conics"], conic), (fw["opac"], o)):
        got, want = got.cpu().double().numpy()[k], want.detach().numpy()[k]
        tol = 1e-4 * np.abs(want) + 1e-4 * np.abs(want).max()
        worst = max(worst, float((np.abs(got - want) / tol).max()))
    vg = ff.filtered_vjp(cam, t(means), t(scales), t(quats), t(logits), t(f), *(t(cot[c]) for c in (
        "v_xy", "v_depth", "v_conic", "v_opacity")), aa=aa, kept=kept)
    for name, want in zip(("v_means", "v_scales", "v_quats", "v_logits"), vg):
        got, want = g[name].cpu().double().numpy()[k], want.numpy()[k]
        tol = 1e-3 * np.abs(want) + 1e-4 * np.abs(want).max()
        r = np.abs(got - want) / tol
        worst = max(worst, float(np.quantile(r, 0.999)))
    print(f"filtered projection, aa={aa}: worst err/tol {worst:.3g}")
    assert worst <= 1.0


def test_footprint_bound_at_the_setting_camera():
    """At the camera that sets f[i], the filtered screen covariance before the 0.3 px^2 blur satisfies
    lambda_min >= variance (min(fx, fy) / F)^2, up to fp32 error."""
    n = 20000
    cams = orbit_cameras(5, W=128, H=96, fx=100.0)
    table = ff.camera_rows(cams)
    g = np.random.default_rng(9)
    means = (g.normal(size=(n, 3)) * 1.2).astype(np.float32)
    scales = g.uniform(-14, -3, size=(n, 3)).astype(np.float32)
    quats = g.normal(size=(n, 4)).astype(np.float32)
    logits = np.zeros(n, np.float32)
    f = compute_filter3d(_cu(means), cams)
    fx_max = table[:, 12].max()
    seen_by = np.full(n, -1)
    best = np.full(n, np.inf)
    for j, c in enumerate(table):
        V = c[:12].reshape(3, 4).astype(np.float64)
        z = means @ V[:, :3].T[:, 2] + V[2, 3]
        x = means @ V[0, :3] + V[0, 3]
        y = means @ V[1, :3] + V[1, 3]
        u, v = c[12] * x / z + c[14], c[13] * y / z + c[15]
        ok = (z > 0.2) & (u >= -0.15 * c[16]) & (u <= 1.15 * c[16]) & (v >= -0.15 * c[17]) & (v <= 1.15 * c[17])
        upd = ok & (z < best)
        best[upd], seen_by[upd] = z[upd], j
    checked = 0
    for j, cam in enumerate(cams):
        sel = np.nonzero(seen_by == j)[0]
        if not len(sel):
            continue
        pc = pf.camera_from_setup(cam)
        fw = _forward(pc, _cu(means[sel]), _cu(scales[sel]), _cu(quats[sel]), _cu(logits[sel]), f[sel].contiguous(),
                      False)
        k = (fw["radii"] > 0).cpu().numpy()
        A, B, C = (fw["conics"][:, i].cpu().double().numpy()[k] for i in range(3))
        det = A * C - B * B
        cxx, cxy, cyy = C / det - 0.3, -B / det, A / det - 0.3       # the screen covariance before the blur
        tr, dt = cxx + cyy, cxx * cyy - cxy * cxy
        lam = 0.5 * tr - np.sqrt(np.maximum(0.25 * tr * tr - dt, 0))
        bound = 0.2 * (min(table[j, 12], table[j, 13]) / fx_max) ** 2
        assert (lam >= bound * (1 - 1e-3) - 1e-4).all(), (j, lam.min(), bound)
        checked += k.sum()
    assert checked > 1000


# ------------------------------------------------------------------------------------------------ reset and bake
def test_reset_and_bake_match_the_restatement():
    n = 100_000
    g = np.random.default_rng(12)
    scales = g.uniform(-8, 0, size=(n, 3)).astype(np.float32)
    logits = (g.normal(size=(n, 1)) * 3).astype(np.float32)
    f = np.where(g.uniform(size=n) < 0.3, 0, g.uniform(0, 0.05, n)).astype(np.float32)
    max_logit = float(torch.logit(torch.tensor(0.2, dtype=torch.float32)))
    L = capi.lib()
    lg, m, v = _cu(logits), torch.ones(n, device=DEV), torch.ones(n, device=DEV)
    capi.check(L.gsb_reset_opacity_filter3d(n, max_logit, 0.2, capi.ptr(_cu(scales)), capi.ptr(_cu(f)),
                                            capi.ptr(lg), capi.ptr(m), capi.ptr(v), capi.stream()))
    # the device's c3: the filtered forward's opacity at logit 100, where sigmoid is 1.f exactly
    cam = _problem(1, 0)[0]
    quats = _cu(np.tile(np.float32([1, 0, 0, 0]), (n, 1)))
    fw = _forward(cam, torch.zeros((n, 3), device=DEV), _cu(scales), quats, torch.full((n,), 100.0, device=DEV),
                  _cu(f), False)
    c3 = fw["opac"].cpu().numpy()
    want = ff.reset_f64(logits, scales, f, 0.2, max_logit, c3=c3)
    got = lg.cpu().numpy().reshape(-1)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulp.max() <= 1 and (m == 0).all() and (v == 0).all()
    one = c3 == 1
    assert one.mean() > 0.25
    assert np.array_equal(got[one], np.minimum(logits.reshape(-1)[one], np.float32(max_logit)))
    baked = bake({"scales": _cu(scales), "opacities": _cu(logits)}, _cu(f))
    a64, l64 = ff.bake_f64(scales, logits, f)
    np.testing.assert_allclose(baked["scales"].cpu().numpy(), a64, rtol=2 ** -23, atol=0)
    np.testing.assert_allclose(baked["opacities"].cpu().numpy().reshape(-1), l64, rtol=2 ** -23, atol=1e-7)


# ------------------------------------------------------------------------------------------------ the trainer
def _trainer_problem():
    from test_gpu_trainer import _cams, make_problem, refine_config
    p, c2w, gts, intr, H, W = make_problem()
    return p, _cams(c2w, H, W, intr), [_cu(g) for g in gts], refine_config()


def _run(p, cams, gts, cfg, steps=60, views=1, **kw):
    from opensplat_b200.trainer import SplatTrainer
    torch.manual_seed(0)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, cfg, device=DEV, views_per_step=views, **kw)
    for step in range(1, steps + 1):
        if views == 1:
            v = (step - 1) % len(cams)
            tr.step(cams[v], gts[v], step, **({"image": v} if "pose" in kw else {}))
        else:
            vs = [(step + b) % len(cams) for b in range(views)]
            tr.step([cams[v] for v in vs], [gts[v] for v in vs], step, **({"image": vs} if "pose" in kw else {}))
    torch.cuda.synchronize()
    return tr


@pytest.mark.parametrize("aa", [False, True])
def test_trainer_at_f_zero_is_the_plain_trainer(aa):
    """variance = 0 makes every f 0: the filtered kernels then give the plain trainer's results bit for bit, through
    refinements and an alpha reset."""
    p, cams, gts, cfg = _trainer_problem()
    a = _run(p, cams, gts, cfg, antialiased=aa)
    b = _run(p, cams, gts, cfg, antialiased=aa, filter3d=Filter3DConfig(cameras=cams, variance=0.0))
    assert (b.filter3d() == 0).all() and a.n == b.n
    pa, pb = a.params(), b.params()
    for k in pa:
        assert _same_bits(pa[k], pb[k], zero_sign=True), k


@pytest.mark.parametrize("opt", ["plain", "views2", "aa", "mcmc", "pose"])
def test_trainer_options_with_the_filter(opt):
    from opensplat_b200.mcmc import MCMCConfig
    from opensplat_b200.pose import PoseConfig
    p, cams, gts, cfg = _trainer_problem()
    kw = {"views": 2} if opt == "views2" else {}
    if opt == "aa":
        kw["antialiased"] = True
    if opt == "mcmc":
        cfg = MCMCConfig(cap_max=6000, refine_start=10, refine_stop=40, refine_every=10, max_steps=200)
    if opt == "pose":
        kw["pose"] = PoseConfig(num_images=len(cams))
    tr = _run(p, cams, gts, cfg, steps=50, filter3d=Filter3DConfig(cameras=cams), **kw)
    f = tr.filter3d()
    assert f.shape == (tr.n,) and torch.isfinite(f).all() and (f > 0).any()
    want = compute_filter3d(tr.params()["means"], cams)
    if tr.last_info.get("refined"):
        assert torch.equal(f, want)
    for v in tr.params().values():
        assert torch.isfinite(v).all()


def _composition(tr, params, cams, gts, views, f, via_operator):
    """Gradients w.r.t. the four geometry tensors of mean_b MainLoss through the autograd operators, at the trainer's
    cameras and colours of its last step.  via_operator: the operators' trailing filter3D; else torch computes the
    effective log-scales log(e^2 + f^2) / 2 and logits logit(sigmoid(l) c3) (in float64) into the unfiltered ones."""
    pp = tr.pipe
    H, W = pp.H, pp.W
    dev = {k: torch.as_tensor(params[k]).to(DEV).clone().requires_grad_() for k in ("means", "scales", "quats",
                                                                                     "opacities")}
    op = ops.ProjectGaussiansActivatedAntialiased if tr.antialiased else ops.ProjectGaussiansActivated
    if via_operator:
        scales, logits, extra = dev["scales"], dev["opacities"], (0.01, f)
    else:
        e2, f2 = torch.exp(2 * dev["scales"].double()), f.double()[:, None] ** 2
        scales = (0.5 * torch.log(e2 + f2)).float()
        p = torch.sigmoid(dev["opacities"].double()) * torch.sqrt(e2 / (e2 + f2)).prod(-1, keepdim=True)
        logits, extra = (torch.log(p) - torch.log1p(-p)).float(), ()
    total = 0.0
    for b, v in enumerate(views):
        c = cams[v]
        xys, depths, radii, conics, nth, _, opac = op.apply(dev["means"], scales, 1.0, dev["quats"], logits,
                                                            tr.viewmats[b].clone(), tr.projmats[b].clone(), c.fx,
                                                            c.fy, c.cx, c.cy, H, W, ops.tile_bounds(W, H), *extra)
        img = ops.RasterizeGaussiansClamped.apply(xys, depths, radii, conics, nth, tr.rgbs_views[b].detach(), opac, H,
                                                  W, pp.background)
        total = total + ops.MainLoss.apply(img, gts[v], tr.ssim_weight)
    (total / len(views)).backward()
    return {k: dev[k].grad.reshape(-1) for k in dev}


@pytest.mark.parametrize("mode", ["one_view", "two_views", "antialiased", "pose"])
def test_one_step_matches_the_autograd_composition(mode):
    """One step's geometry gradients (Adam frozen) against autograd of the composition, both through the operators'
    filter3D and through torch's effective parameters into the unfiltered operators."""
    import test_gpu_trainer as tg
    from opensplat_b200.pose import PoseConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gts = torch.from_numpy(gts).to(DEV)
    params = {k: torch.from_numpy(v) for k, v in p.items()}
    B = 2 if mode == "two_views" else 1
    kw = {"pose": PoseConfig(num_images=3)} if mode == "pose" else {}
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV, views_per_step=B,
                      antialiased=mode == "antialiased", filter3d=Filter3DConfig(cameras=cams, variance=0.5), **kw)
    tr._adam_step = lambda: None
    if tr.poses is not None:
        tr.poses.adam_step = lambda step: None
    views = [1] if B == 1 else [1, 2]
    f = tr.filter3d()
    assert (f > 0).all()
    if B == 1:
        tr.step(cams[1], gts[1], 7, **({"image": 1} if kw else {}))
    else:
        tr.step([cams[v] for v in views], gts[views], 7)
    torch.cuda.synchronize()
    got = {k: tr.pipe.g[k].reshape(-1).clone() for k in ("means", "scales", "quats", "opacities")}
    for via in (True, False):
        want = _composition(tr, params, cams, gts, views, f, via)
        for k in got:
            e = float((got[k] - want[k]).norm() / want[k].norm())
            print(f"  {mode} via_operator={via} {k}: rel-L2 {e:.3g}")
            assert e <= (2e-4 if via else 2e-3), (k, via)
    # the filter is a real part of it: the unfiltered composition differs
    plain = _composition(tr, params, cams, gts, views, torch.zeros_like(f), True)
    assert float((got["scales"] - plain["scales"]).norm() / plain["scales"].norm()) > 1e-2


@pytest.mark.parametrize("B", [1, 2])
def test_step_launch_sequence_with_the_filter(B, monkeypatch):
    """A steady-state step issues the plain trainer's launches with the two projections swapped for the filtered ones,
    and no recomputation."""
    import test_gpu_trainer as tg
    from test_gpu_trainer_launches import ONE_VIEW, TWO_VIEWS, _Recorder
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    log = []
    monkeypatch.setattr(capi, "_lib", _Recorder(capi.lib(), log))
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, tg.refine_config(warmup_length=10 ** 6),
                      device=DEV, views_per_step=B, filter3d=Filter3DConfig(cameras=cams))
    assert log.count("gsb_filter3d_compute") == 1               # at construction

    def args(step):
        views = [cams[(step - 1 + b) % 3] for b in range(B)]
        return (views[0], gt[0]) if B == 1 else (views, gt[:B])
    for step in range(1, 6):
        tr.step(*args(step), step)
    torch.cuda.synchronize()
    del log[:]
    tr.step(*args(6), 6)
    torch.cuda.synchronize()
    swap = {"gsb_project_forward_activated": "gsb_project_forward_activated_filter3d",
            "gsb_project_backward_activated": "gsb_project_backward_activated_filter3d",
            "gsb_project_backward_activated_acc": "gsb_project_backward_activated_filter3d"}
    expected = [swap.get(x, x) for x in (ONE_VIEW if B == 1 else TWO_VIEWS)]
    assert [x for x in log if not x.startswith("gsb_densify_stats_")] == expected, log


@pytest.mark.parametrize("strategy", ["refine", "mcmc"])
def test_recompute_launches_follow_the_schedule(strategy, monkeypatch):
    import test_gpu_trainer as tg
    from test_gpu_trainer_launches import _Recorder
    from opensplat_b200.filter3d import recompute_due
    from opensplat_b200.mcmc import MCMCConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    if strategy == "refine":
        cfg, steps = tg.refine_config(max_steps=140), 135    # refines every 10 steps from 20; split stops at 70
    else:
        cfg, steps = MCMCConfig(cap_max=6000, refine_start=10, refine_stop=40, refine_every=10, max_steps=80), 80
    f3 = Filter3DConfig(cameras=cams, recompute_every=10)
    log = []
    monkeypatch.setattr(capi, "_lib", _Recorder(capi.lib(), log))
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, cfg, device=DEV, filter3d=f3)
    torch.manual_seed(0)
    due = []
    for step in range(1, steps + 1):
        del log[:]
        tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
        calls = log.count("gsb_filter3d_compute")
        reset = bool(tr.last_info.get("alpha_reset"))
        assert calls == int(recompute_due(cfg, f3, step, tr.last_info["refined"])) + int(reset), (step, log)
        if calls:
            due.append(step)
    if strategy == "refine":
        assert due == list(range(20, 131, 10)), due
    else:
        assert due == [20, 30, 40, 50, 60], due


def test_parallel_world1_replicas_with_the_filter():
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1",
                        "--master-addr", "127.0.0.1", "--master-port", "29571",
                        os.path.join(root, "tools", "check_parallel_filter3d.py")], capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-2000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "check_ok=True" in r.stdout and "plain_trainer_bit_identical=True" in r.stdout


def test_export_bakes_the_filter(tmp_path):
    from opensplat_b200 import export
    from opensplat_b200.trainer import SplatTrainer
    p, cams, gts, cfg = _trainer_problem()
    tr = _run(p, cams, gts, cfg, steps=30, filter3d=Filter3DConfig(cameras=cams, variance=2.0))
    ref = {k: v.clone() for k, v in tr.render(cams[0], 30).items()}
    path = str(tmp_path / "scene.ply")
    tr.save(path)
    loaded, _ = export.load_ply(path, device=DEV)
    plain = SplatTrainer(loaded, cfg, device=DEV)
    got = plain.render(cams[0], 30)
    torch.cuda.synchronize()
    d = (got["rgb"] - ref["rgb"]).abs().reshape(-1)
    q, mx = torch.quantile(d[:1 << 24].float(), 0.999).item(), d.max().item()
    print(f"baked PLY render vs filtered render: 99.9% |diff| {q:.3g}, max {mx:.3g}")
    assert q < 1e-4 and mx < 5e-2
    # the .splat rows hold the baked scene too, within its quantisation
    from opensplat_b200.export import pack_splat_rows
    baked = bake(dict(tr.pipe.p), tr.filter3d())
    tr.save(str(tmp_path / "scene.splat"))
    raw = np.fromfile(str(tmp_path / "scene.splat"), dtype=np.uint8)
    assert np.array_equal(raw, pack_splat_rows(baked).view(torch.uint8).reshape(-1).cpu().numpy())
    rows = raw.reshape(-1, 32)
    scales = rows[:, 12:24].copy().view(np.float32)
    alpha = rows[:, 27].astype(np.float64) / 255.0
    want_s = np.sort(np.exp(baked["scales"].cpu().numpy()), axis=None)
    np.testing.assert_allclose(np.sort(scales, axis=None), want_s, rtol=1e-6)
    want_a = 1.0 / (1.0 + np.exp(-baked["opacities"].cpu().double().numpy().reshape(-1)))
    assert abs(np.sort(alpha) - np.sort(want_a)).max() <= 1.0 / 255 + 1e-9


# ------------------------------------------------------------------------------------------------ zoom-in
def _orbit_scene_cams(k, W, fx_per_px, radius=4.0, offset=0.0):
    from opensplat_b200.model import Camera
    cams = []
    for j in range(k):
        th = 2 * math.pi * (j + offset) / k
        eye = np.array([radius * math.cos(th), 0.6 * math.sin(3 * th), radius * math.sin(th)])
        fwd = -eye / np.linalg.norm(eye)
        right = np.cross(fwd, [0.0, 1.0, 0.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        c2w = np.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, eye
        cams.append(Camera(W, W, fx_per_px * W, fx_per_px * W, W / 2, W / 2, c2w))
    return cams


def test_filter_helps_zoom_in():
    """Students trained at 64x64 (antialiased, with and without the filter) rendered at 256x256 on held-out views
    of a synthetic teacher scene: the filtered one scores the higher PSNR."""
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.scene import make_scene
    from opensplat_b200.trainer import SplatTrainer
    sc = make_scene(20000, 64, 64, scale=0.03, sh_degree=1, opacity=(0.3, 0.9), seed=1)
    sc["means"][:, 2] = np.random.default_rng(2).uniform(-1, 1, 20000).astype(np.float32)
    teacher = {"means": sc["means"], "scales": np.log(sc["scales"]), "quats": sc["quats"],
               "featuresDc": sc["coeffs"][:, 0], "featuresRest": sc["coeffs"][:, 1:],
               "opacities": np.log(sc["opacities"] / (1 - sc["opacities"]))}
    teacher = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in teacher.items()}
    t = SplatTrainer(teacher, device=DEV, background=(0, 0, 0))
    train_lo = _orbit_scene_cams(24, 64, 1.1)
    test_hi = _orbit_scene_cams(6, 256, 1.1, offset=0.5)
    gts = [t.render(c, 1)["rgb"].clone() for c in train_lo]
    refs = [t.render(c, 1)["rgb"].clone() for c in test_hi]
    g = np.random.default_rng(4)
    n0 = 6000
    init = {"means": torch.from_numpy(g.uniform(-1, 1, (n0, 3)).astype(np.float32)),
            "scales": torch.full((n0, 3), math.log(0.03)), "quats": torch.from_numpy(g.normal(size=(n0, 4))
                                                                                      .astype(np.float32)),
            "featuresDc": torch.zeros((n0, 3)), "featuresRest": torch.zeros((n0, 3, 3)),
            "opacities": torch.full((n0, 1), -2.0)}
    steps = 3000
    cfg = RefineConfig(max_steps=steps, num_cameras=len(train_lo))
    psnr = {}
    for name, f3 in (("plain", None), ("filter", Filter3DConfig(cameras=train_lo))):
        torch.manual_seed(0)
        s = SplatTrainer(init, cfg, device=DEV, antialiased=True, background=(0, 0, 0), filter3d=f3)
        for step in range(1, steps + 1):
            v = (step - 1) % len(train_lo)
            s.step(train_lo[v], gts[v], step)
        mse = [float(((s.render(c, steps)["rgb"] - r) ** 2).mean()) for c, r in zip(test_hi, refs)]
        psnr[name] = float(np.mean([-10 * math.log10(max(e, 1e-12)) for e in mse]))
    print(f"zoom-in PSNR at 256x256 after 64x64 training: plain {psnr['plain']:.3f} dB, "
          f"filter {psnr['filter']:.3f} dB")
    assert psnr["filter"] > psnr["plain"]
