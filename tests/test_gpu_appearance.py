"""GPU: the bilateral-grid kernels (csrc/bilagrid.cu) against the float64 restatement bilagrid_f64.py within its
certified bounds, their determinism, the autograd operators, and SplatTrainer with appearance grids (DESIGN D21): one
step against the autograd composition of the existing operators, the launch sequence, B = 2 on one image, MCMC and
antialiased runs, the argument errors, evaluate / render, the steady state and a functional test on a synthetic
capture with per-image exposure and white balance."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bilagrid_f64 as ref  # noqa: E402
import test_gpu_trainer as tg  # noqa: E402  (the training problem)
from test_bilagrid_f64_reference import make_case, torch_slice  # noqa: E402
from test_gpu_trainer_launches import FORWARD, _Recorder  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _release_cached_memory():
    """Give what each test allocated back to the device: the caching allocator would otherwise keep a few hundred MB
    for the rest of the pytest process, which later tests that start CUDA subprocesses need."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def cu(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=DEV)


def _ws(H, W):
    from opensplat_b200 import capi
    return torch.empty(capi.lib().gsb_bilagrid_workspace_bytes(H, W), dtype=torch.uint8, device=DEV)


def slice_fwd(grid, rgb):
    from opensplat_b200 import capi
    H, W = rgb.shape[:2]
    out = torch.full((H, W, 3), float("nan"), device=DEV)
    capi.check(capi.lib().gsb_bilagrid_slice_forward(H, W, capi.ptr(grid), capi.ptr(rgb), capi.ptr(out),
                                                     capi.stream()))
    return out


def slice_bwd(grid, rgb, v, scale=1.0, v_grid=None, ws=None):
    from opensplat_b200 import capi
    H, W = rgb.shape[:2]
    ws = _ws(H, W) if ws is None else ws
    v_rgb = torch.full((H, W, 3), float("nan"), device=DEV)
    v_grid = torch.zeros_like(grid) if v_grid is None else v_grid
    capi.check(capi.lib().gsb_bilagrid_slice_backward(H, W, capi.ptr(grid), capi.ptr(rgb), capi.ptr(v), scale,
                                                      capi.ptr(v_rgb), capi.ptr(v_grid), capi.ptr(ws), ws.numel(),
                                                      capi.stream()))
    return v_rgb, v_grid


def worst(got, want, bound):
    """max |got - want| / bound (a ratio <= 1 is inside the bound)."""
    return float((np.abs(got.cpu().double().numpy() - want) / np.maximum(bound, 1e-300)).max())


# ---- 1. kernels against the float64 restatement -----------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (48, 64), (1080, 1920)])
def test_kernels_within_the_certified_bounds(H, W):
    grid, rgb, v = make_case(H, W, H + 3 * W)
    g, x, vv = cu(grid), cu(rgb), cu(v)
    out = slice_fwd(g, x)
    v_rgb, v_grid = slice_bwd(g, x, vv)
    torch.cuda.synchronize()
    want, ob = ref.slice_forward(grid.astype(np.float32), rgb)
    wr, rb, wg, gb = ref.slice_backward(grid.astype(np.float32), rgb, v)
    r = (worst(out, want, ob), worst(v_rgb, wr, rb), worst(v_grid, wg, gb))
    print(f"{H}x{W}: err/bound slice {r[0]:.3g}, v_rgb {r[1]:.3g}, v_grid {r[2]:.3g}")
    assert max(r) <= 1.0


@pytest.mark.parametrize("N", [1, 3])
def test_tv_within_the_certified_bounds(N):
    from opensplat_b200 import capi
    rng = np.random.default_rng(N)
    grids = (ref.identity(N) + rng.normal(0, 0.1, (N, ref.L, ref.Y, ref.X, ref.NC))).astype(np.float32)
    g = cu(grids)
    v = torch.full_like(g, float("nan"))
    val = torch.full((1,), float("nan"), device=DEV)
    capi.check(capi.lib().gsb_bilagrid_tv(N, capi.ptr(g), 2.5, capi.ptr(v), capi.ptr(val), capi.stream()))
    value, vb, grad, gb = ref.tv(grids)
    assert abs(float(val) - value) <= vb
    assert worst(v, 2.5 * grad, 2.5 * gb + 1e-45) <= 1.0
    v2 = torch.full_like(g, float("nan"))
    capi.check(capi.lib().gsb_bilagrid_tv(N, capi.ptr(g), 2.5, capi.ptr(v2), None, capi.stream()))
    assert torch.equal(v, v2)


# ---- 2. determinism and accumulation ----------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(48, 64), (1080, 1920)])
def test_backward_is_bit_deterministic_and_accumulates(H, W):
    grid, rgb, v = make_case(H, W, 7)
    g, x, vv = cu(grid), cu(rgb), cu(v)
    a_rgb, a_grid = slice_bwd(g, x, vv, 0.37)
    b_rgb, b_grid = slice_bwd(g, x, vv, 0.37)
    assert torch.equal(a_rgb, b_rgb) and torch.equal(a_grid, b_grid)
    prev = torch.randn(g.shape, device=DEV)
    _, acc = slice_bwd(g, x, vv, 0.37, v_grid=prev.clone())
    assert torch.equal(acc, prev + a_grid)
    assert bool((a_grid != 0).any())


# ---- 3. the autograd operators ------------------------------------------------------------------------------------------
def test_operators_match_torch_float64_autograd():
    from opensplat_b200 import ops
    H, W = 37, 52
    grid, rgb, v = make_case(H, W, 11)
    grid = grid.astype(np.float32)
    gs = cu(np.transpose(grid, (3, 0, 1, 2))).requires_grad_()
    x = cu(rgb).requires_grad_()
    out = ops.BilateralGridSlice.apply(gs, x)
    out.backward(cu(v))
    t_out, t_vrgb, t_vgrid = torch_slice(grid, rgb, v)
    _, ob = ref.slice_forward(grid, rgb)
    _, rb, _, gb = ref.slice_backward(grid, rgb, v)
    assert worst(out.detach(), t_out, ob) <= 1.0
    assert worst(x.grad, t_vrgb, rb) <= 1.0
    assert worst(gs.grad.permute(1, 2, 3, 0), t_vgrid, gb) <= 1.0
    rng = np.random.default_rng(2)
    grids = (ref.identity(2) + rng.normal(0, 0.1, (2, ref.L, ref.Y, ref.X, ref.NC))).astype(np.float32)
    G = cu(np.transpose(grids, (0, 4, 1, 2, 3))).requires_grad_()
    tv = ops.BilateralGridTV.apply(G)
    (3.0 * tv).backward()
    Gd = torch.tensor(np.transpose(grids, (0, 4, 1, 2, 3)), dtype=torch.float64, requires_grad=True)
    td = sum(torch.mean(torch.diff(Gd, dim=a) ** 2) for a in (4, 3, 2))
    (3.0 * td).backward()
    value, vb, _, gb = ref.tv(grids)
    assert abs(float(tv.detach()) - float(td.detach())) <= vb
    assert worst(G.grad.permute(0, 2, 3, 4, 1), np.transpose(Gd.grad.numpy(), (0, 2, 3, 4, 1)),
                 3.0 * gb + 1e-45) <= 1.0


# ---- 4. the trainer -------------------------------------------------------------------------------------------------------
def _problem(n=4000):
    p, c2w, gts, intr, H, W = tg.make_problem(n=n)
    return ({k: torch.from_numpy(v) for k, v in p.items()}, tg._cams(c2w, H, W, intr), torch.from_numpy(gts).to(DEV),
            (c2w, H, W, intr))


def _noisy_grids(tr, seed=0, sigma=0.05):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ap = tr.appearance
    ap.grids.add_(torch.randn(ap.grids.shape, device=DEV, generator=g) * sigma)
    return ap.grids.clone()


def _app(num_images=3, **kw):
    from opensplat_b200.appearance import AppearanceConfig
    return AppearanceConfig(num_images=num_images, **kw)


def test_one_step_matches_the_autograd_composition():
    from opensplat_b200 import ops
    from opensplat_b200.appearance import to_gsplat_order
    from opensplat_b200.model import GaussianModel
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    cfg = tg.refine_config(warmup_length=10 ** 6)
    tr = SplatTrainer(params, cfg, device=DEV, appearance=_app())
    g0 = _noisy_grids(tr)
    tr.step(cams[1], gts[1], 1, image=2)
    torch.cuda.synchronize()
    model = GaussianModel(params, cfg, device=DEV)
    model.optimizers_zero_grad()
    G = to_gsplat_order(g0).requires_grad_()
    rgb = model.forward(cams[1], 1)
    loss = ops.MainLoss.apply(ops.BilateralGridSlice.apply(G[2], rgb), gts[1], 0.2)
    (loss + 10.0 * ops.BilateralGridTV.apply(G)).backward()
    # the Gaussians' gradients: the same slice backward of the same loss gradient
    pg = tr.pipe.g
    for k in ("means", "scales", "quats"):
        assert torch.equal(pg[k], getattr(model, k).grad), k
    assert torch.equal(pg["opacities"].reshape(-1), model.opacities.grad.reshape(-1))
    assert torch.equal(pg["coeffs"][:, 0, :], model.featuresDc.grad)
    # the grids' gradient: tv_weight dTV then the slice's, against slice + 10 TV summed by autograd
    want = G.grad.permute(0, 2, 3, 4, 1)
    got = tr.appearance.grad
    rel = float((got - want).norm() / want.norm())
    print(f"grid gradient rel-L2 {rel:.3g}")
    assert rel <= 1e-6
    # the Gaussian Adam step equals GaussianModel's; the grid Adam step at step 1 is lr * sign(g) (m / sqrt(v))
    model.optimizers_step()
    p = tr.params()
    for k in ("means", "scales", "quats", "featuresDc", "featuresRest", "opacities"):
        assert torch.equal(p[k].reshape(-1), getattr(model, k).detach().reshape(-1)), k
    lr = ref.learning_rate(1)
    step_ = tr.appearance.grids - g0
    ulp = 2.0 ** -23 * (g0.abs() + lr)                          # the fp32 rounding of the updated grid
    big = want.abs() > 1e-4 * float(want.abs().max())
    assert bool(((step_ + lr * torch.sign(want)).abs() <= 1e-3 * lr + ulp)[big].all())
    assert bool((step_.abs() <= lr * (1 + 1e-5) + ulp).all())
    assert tr.appearance.adam_t == 1


def test_launch_sequence_adds_exactly_the_appearance_calls(monkeypatch):
    from opensplat_b200 import capi
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    log = []
    monkeypatch.setattr(capi, "_lib", _Recorder(capi.lib(), log))
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV, appearance=_app())
    for step in range(1, 6):
        tr.step(cams[(step - 1) % 3], gts[(step - 1) % 3], step, image=(step - 1) % 3)
    torch.cuda.synchronize()
    del log[:]
    tr.step(cams[0], gts[0], 6, image=0)
    torch.cuda.synchronize()
    seq = [x for x in log if not x.startswith("gsb_densify_stats_")]
    fwd = FORWARD[:-1] + ["gsb_bilagrid_slice_forward", "gsb_ssim_l1_loss", "gsb_bilagrid_slice_backward"]
    assert seq == (["gsb_sh_forward_rgb_cam", "gsb_bilagrid_tv"] + fwd
                   + ["gsb_rasterize_backward", "gsb_project_backward_activated", "gsb_sh_backward_rgb_cam",
                      "gsb_adam_step_segments", "gsb_adam_step"]), log


def test_two_views_on_one_image_add_both_halves():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    cfg = tg.refine_config(warmup_length=10 ** 6)

    def frozen(B):
        tr = SplatTrainer(params, cfg, device=DEV, views_per_step=B, appearance=_app(tv_weight=0.0))
        tr._adam_step = lambda: None
        tr.appearance.adam_step = lambda step: None
        _noisy_grids(tr)
        return tr
    one = frozen(1)
    grads = []
    for v in (0, 1):
        one.step(cams[v], gts[v], 3, image=1)
        grads.append(one.appearance.grad[1].clone())
    two = frozen(2)
    two.step([cams[0], cams[1]], gts[:2], 3, image=[1, 1])
    torch.cuda.synchronize()
    assert torch.equal(two.appearance.grad[1], (grads[0] + grads[1]) * 0.5)
    assert not bool(two.appearance.grad[0].any()) and not bool(two.appearance.grad[2].any())


@pytest.mark.parametrize("mode", ["mcmc", "antialiased", "mcmc_two_views"])
def test_mcmc_and_antialiased_runs(mode):
    from opensplat_b200.mcmc import MCMCConfig
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    B = 2 if mode == "mcmc_two_views" else 1
    cfg = (MCMCConfig(refine_start=4, refine_every=5, refine_stop=10 ** 6, cap_max=4600, max_steps=200, seed=3)
           if mode.startswith("mcmc") else tg.refine_config(warmup_length=10 ** 6))
    runs = []
    for _ in range(2):
        tr = SplatTrainer(params, cfg, device=DEV, views_per_step=B, antialiased=mode == "antialiased",
                          appearance=_app(warmup_steps=10))
        for step in range(1, 22):
            vs = [((step - 1) * B + b) % 3 for b in range(B)]
            if B == 1:
                tr.step(cams[vs[0]], gts[vs[0]], step, image=vs[0])
            else:
                tr.step([cams[v] for v in vs], gts[vs], step, image=vs)
        runs.append((tr.pipe.param_flat.clone(), tr.appearance_grids()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert bool(torch.isfinite(runs[0][1]).all()) and bool(torch.isfinite(runs[0][0]).all())
    from opensplat_b200.appearance import identity_grids, to_gsplat_order
    assert not torch.equal(runs[0][1], to_gsplat_order(identity_grids(3, DEV)))
    if mode.startswith("mcmc"):
        assert tr.n == 4600


def test_argument_errors():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem(n=500)
    cfg = tg.refine_config(warmup_length=10 ** 6)
    tr = SplatTrainer(params, cfg, device=DEV, appearance=_app())
    for bad in (None, -1, 3, 1.0, True, [0, 1]):
        with pytest.raises(ValueError):
            tr.step(cams[0], gts[0], 1, image=bad)
    tr2 = SplatTrainer(params, cfg, device=DEV, views_per_step=2, appearance=_app())
    for bad in ([0], [0, 1, 2], 0, [0, 3]):
        with pytest.raises(ValueError):
            tr2.step([cams[0], cams[1]], gts[:2], 1, image=bad)
    plain = SplatTrainer(params, cfg, device=DEV)
    with pytest.raises(ValueError):
        plain.step(cams[0], gts[0], 1, image=0)
    with pytest.raises(ValueError):
        plain.appearance_grids()
    assert tr.appearance.adam_t == 0 and tr2.appearance.adam_t == 0


def test_evaluate_and_render_are_the_plain_trainers():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    cfg = tg.refine_config(warmup_length=10 ** 6)
    tr = SplatTrainer(params, cfg, device=DEV, appearance=_app(warmup_steps=5))
    for step in range(1, 8):
        tr.step(cams[step % 3], gts[step % 3], step, image=step % 3)
    plain = SplatTrainer(tr.params(), cfg, device=DEV)
    for c in range(3):
        a = tr.evaluate(cams[c], gts[c], 8).clone()
        img_a = tr.image.clone()
        b = plain.evaluate(cams[c], gts[c], 8).clone()
        assert torch.allclose(a, b, rtol=0, atol=1e-6) and torch.equal(img_a, plain.image)
        ra, rb = tr.render(cams[c], 8), plain.render(cams[c], 8)
        for k in ("rgb", "depth", "alpha"):
            assert torch.equal(ra[k], rb[k]), k


def test_steady_state_allocates_nothing():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, _ = _problem()
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV, views_per_step=2,
                      appearance=_app())
    pairs = [gts[[v, (v + 1) % 3]].contiguous() for v in range(3)]
    for step in range(1, 4):
        tr.step([cams[step % 3], cams[(step + 1) % 3]], pairs[step % 3], step, image=[step % 3, (step + 1) % 3])
    torch.cuda.synchronize()
    before = torch.cuda.memory_stats(DEV)["allocation.all.allocated"]
    mem = torch.cuda.memory_allocated(DEV)
    for step in range(4, 10):
        tr.step([cams[step % 3], cams[(step + 1) % 3]], pairs[step % 3], step, image=[step % 3, (step + 1) % 3])
    torch.cuda.synchronize()
    assert torch.cuda.memory_stats(DEV)["allocation.all.allocated"] == before
    assert torch.cuda.memory_allocated(DEV) == mem


# ---- 5. functional: per-image exposure and white balance ------------------------------------------------------------
# Per-image (R, G, B) gains that drift smoothly along the arc of cameras, as auto-exposure and auto-white-balance
# drift over a capture: each channel's mean is 1, and the drift is what SH colour can bake into the scene.
GAINS = np.stack([np.linspace(0.82, 1.18, 8), np.linspace(1.12, 0.88, 8), np.linspace(0.86, 1.14, 8)], 1)


def _fit_score(renders, clean):
    """PSNR of the renders against the clean images after one per-channel affine map fitted over all views."""
    r = renders.reshape(-1, 3).double()
    c = clean.reshape(-1, 3).double()
    fitted = torch.empty_like(r)
    for ch in range(3):
        A = torch.stack([r[:, ch], torch.ones_like(r[:, ch])], 1)
        sol = torch.linalg.lstsq(A, c[:, ch:ch + 1]).solution
        fitted[:, ch] = (A @ sol)[:, 0]
    mse = float(((fitted - c) ** 2).mean())
    return -10.0 * np.log10(mse)


def test_appearance_grids_absorb_per_image_exposure():
    from opensplat_b200.appearance import AppearanceConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, _, intr, H, W = tg.make_problem(n=4000, V=8, H=128, W=128, seed=5)
    cams = tg._cams(c2w, H, W, intr)
    cfg = tg.refine_config(warmup_length=10 ** 6, num_cameras=8, max_steps=2000)
    teacher = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, cfg, device=DEV)
    clean = torch.stack([0.8 * teacher.render(c, 10 ** 6)["rgb"].clone() for c in cams])
    gains = torch.tensor(GAINS, dtype=torch.float32, device=DEV)
    assert abs(float(gains.mean()) - 1.0) < 0.02
    gts = (clean * gains[:, None, None, :]).contiguous()
    assert float(gts.max()) <= 1.0                           # no clipping
    rng = np.random.default_rng(9)
    start = {k: torch.from_numpy(v) for k, v in p.items()}
    start["featuresDc"] = start["featuresDc"] + torch.from_numpy(rng.normal(0, 0.3, p["featuresDc"].shape)
                                                                 .astype(np.float32))
    steps, scores = 1200, {}
    for name, app in (("plain", None), ("appearance", AppearanceConfig(num_images=8, warmup_steps=100,
                                                                         max_steps=steps))):
        # SH degree 1 from the first step: a plain run can turn the per-image gains into view-dependent colour
        tr = SplatTrainer(start, cfg, device=DEV, sh_degree_interval=1, appearance=app)
        for step in range(1, steps + 1):
            v = (step - 1) % 8
            if app is None:
                tr.step(cams[v], gts[v], step)
            else:
                tr.step(cams[v], gts[v], step, image=v)
        renders = torch.stack([tr.render(c, steps)["rgb"].clone() for c in cams])
        scores[name] = _fit_score(renders, clean)
    margin = scores["appearance"] - scores["plain"]
    print(f"PSNR after a global affine fit: plain {scores['plain']:.2f} dB, appearance {scores['appearance']:.2f} dB, "
          f"margin {margin:.2f} dB")
    # measured on an H100 80GB HBM3 (700 W): plain 30.07 dB, appearance 34.35 dB, a margin of 4.28 dB
    assert margin >= 2.0
