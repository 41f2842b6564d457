"""trainer.SplatTrainer on the H100: its three new kernels entry points against the ones they stand in for (segmented
Adam vs six per-tensor Adam calls, SH with camera view directions on the merged block vs the split variants, the
visible count of the binning stats vs radii), and the trainer against model.GaussianModel on the training problem of
test_gpu_model.py: Gaussian counts, losses, parameters and Adam moments step by step, through two refinements, an
alpha reset and the downscale schedule; plus the empty view, capacity growth, the steady state (no allocation, one
host wait per step) and the PLY writer."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util import PARAM_NAMES  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libopensplat_model_b200.so")


def make_problem(n=4000, V=3, H=96, W=128, k=4, seed=5):
    """The training problem of test_gpu_model.py."""
    rng = np.random.default_rng(seed)
    f = np.float32
    p = {
        "means": (rng.uniform(-1, 1, (n, 3)) * np.array([1.6, 1.2, 0.5])).astype(f),
        "scales": np.log(rng.uniform(0.02, 0.12, (n, 3))).astype(f),
        "quats": rng.standard_normal((n, 4)).astype(f),
        "featuresDc": rng.uniform(-1.5, 1.5, (n, 3)).astype(f),
        "featuresRest": (rng.standard_normal((n, k - 1, 3)) * 0.1).astype(f),
        "opacities": rng.uniform(-2.0, 1.0, (n, 1)).astype(f),
    }
    c2w = np.tile(np.eye(4, dtype=f), (V, 1, 1))
    for v in range(V):                       # OpenGL-style poses on a circle of radius 4, looking at the origin
        a = 0.25 * (v - (V - 1) / 2)
        c2w[v, :3, :3] = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]], dtype=f)
        c2w[v, :3, 3] = np.array([-4.0 * np.sin(a), 0.0, 4.0 * np.cos(a)], dtype=f)
    yy, xx = np.mgrid[0:H, 0:W]
    gts = np.stack([np.stack([0.5 + 0.5 * np.sin(0.07 * xx + v), 0.5 + 0.5 * np.cos(0.05 * yy - v),
                              0.5 + 0.25 * np.sin(0.03 * (xx + yy))], -1) for v in range(V)]).astype(f)
    return p, c2w, gts, (0.9 * W, 0.9 * W, W / 2.0, H / 2.0), H, W


def refine_config(**kw):
    from opensplat_b200.densify import RefineConfig
    c = dict(refine_every=10, warmup_length=15, reset_alpha_every=30, densify_grad_thresh=2e-5,
             densify_size_thresh=0.05, stop_screen_size_at=4000, split_screen_size=0.05, max_steps=200, num_cameras=3)
    c.update(kw)
    return RefineConfig(**c)


def _cams(c2w, H, W, intr):
    from opensplat_b200.model import Camera
    return [Camera(W, H, *intr, c2w[v]) for v in range(len(c2w))]


def _half(gts):
    V, H, W, _ = gts.shape
    return gts.reshape(V, H // 2, 2, W // 2, 2, 3).mean(axis=(2, 4)).astype(np.float32)


def run_model(p, cams, gts_by_factor, steps, seed, ssim_w=0.2, **kw):
    from opensplat_b200.model import GaussianModel
    model = GaussianModel({k: torch.from_numpy(v) for k, v in p.items()}, kw.pop("cfg"), device=DEV, **kw)
    torch.manual_seed(seed)
    losses, counts = [], []
    for step in range(1, steps + 1):
        v = (step - 1) % len(cams)
        model.optimizers_zero_grad()
        rgb = model.forward(cams[v], step)
        loss = model.main_loss(rgb, gts_by_factor[model.get_downscale_factor(step)][v], ssim_w)
        loss.backward()
        losses.append(float(loss.detach()))
        model.optimizers_step()
        model.schedulers_step(step)
        model.after_train(step)
        counts.append(model.means.shape[0])
    return model, np.array(losses), np.array(counts)


def run_trainer(p, cams, gts_by_factor, steps, seed, ssim_w=0.2, **kw):
    from opensplat_b200.model import downscale_factor
    from opensplat_b200.trainer import SplatTrainer
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, kw.pop("cfg"), device=DEV, ssim_weight=ssim_w,
                      **kw)
    torch.manual_seed(seed)
    losses, counts = [], []
    for step in range(1, steps + 1):
        v = (step - 1) % len(cams)
        f = downscale_factor(step, tr.num_downscales, tr.resolution_schedule)
        loss = tr.step(cams[v], gts_by_factor[f][v], step)
        losses.append(float(loss[0]))
        counts.append(tr.n)
    return tr, np.array(losses), np.array(counts)


def _compare(model, tr, losses_m, losses_t, counts_m, counts_t, exact=False):
    """Same Gaussian counts at every step and losses to 1e-6.  With `exact`, parameters and Adam moments must be
    bit-identical: at one view per step without a group the two runs execute the same kernels in the same order, and
    the segmented Adam rounds every float as the six per-tensor calls do (test_segmented_adam_is_six_per_tensor_adam_
    steps).  Otherwise (several views per step, which run other kernels by design) they are bounded loosely, 1e-3 of
    their range: Adam divides by sqrt(v), so a last-bit difference in a near-zero gradient can move a parameter by up
    to about one learning rate.  The largest differences are printed.  Returns whether parameters and moments are
    bit-identical (the loss value itself is summed with float atomics, so it varies in its last bits from run to
    run)."""
    assert np.array_equal(counts_m, counts_t), (counts_m, counts_t)
    assert np.abs(losses_m - losses_t).max() <= 1e-6, np.abs(losses_m - losses_t).max()
    same = True
    pt = tr.params()
    mt, vt = tr.adam_state()
    for k in PARAM_NAMES:
        diffs = []
        for a, b in ((getattr(model, k).detach(), pt[k]), (model.adam_m[k], mt[k]), (model.adam_v[k], vt[k])):
            assert a.shape == b.shape, k
            d = float((a - b).abs().max()) if a.numel() else 0.0
            assert d <= 1e-3 * (1.0 + float(a.abs().max())), k
            same = same and torch.equal(a, b)
            diffs.append(d)
        print(f"  {k}: max |d| param {diffs[0]:.3g}, exp_avg {diffs[1]:.3g}, exp_avg_sq {diffs[2]:.3g}")
    assert same or not exact, "parameters or moments differ from GaussianModel's"
    return same


# ---- 1. segmented Adam ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 1000, 4097])
@pytest.mark.parametrize("k", [1, 4, 16])
def test_segmented_adam_is_six_per_tensor_adam_steps(n, k):
    _segmented_vs_per_tensor(n, k)


def test_segmented_adam_is_six_per_tensor_adam_steps_at_scale():
    """300 000 Gaussians at K = 16: featuresRest has 13.5 M floats, so gsb_adam_step runs its two-float4 loop."""
    _segmented_vs_per_tensor(300_000, 16)


def _segmented_vs_per_tensor(n, k):
    """Three steps of the segmented Adam on the trainer's flat layout against six gsb_adam_step calls on the split
    tensors: bit-identical floats, padding untouched."""
    from opensplat_b200 import capi, parallel
    from opensplat_b200.model import LEARNING_RATES
    from opensplat_b200.trainer import adam_segments
    L = capi.lib()
    offs, numel = parallel.flat_layout(n, k)
    g = torch.Generator(device=DEV).manual_seed(n * 31 + k)
    pad = torch.ones(numel, dtype=torch.bool, device=DEV)
    for o, c, _ in offs.values():
        pad[o:o + c] = False
    sentinel = 12345.0
    bufs = []
    for _ in range(3):                                   # param, exp_avg, exp_avg_sq
        t = torch.randn(numel, device=DEV, generator=g)
        t[pad] = sentinel
        bufs.append(t)
    bufs[2].abs_()
    param, m, v = bufs
    lr = dict(LEARNING_RATES)
    lr["means"] = 1.3e-4                                 # a scheduled means rate, as the trainer passes it

    def split(flat):
        views = parallel.flat_views(flat, offs)
        c = views["coeffs"]
        d = {x: views[x].clone() for x in ("means", "scales", "quats", "opacities")}
        d["featuresDc"], d["featuresRest"] = c[:, 0, :].contiguous(), c[:, 1:, :].contiguous()
        return d
    ref_p, ref_m, ref_v = split(param), split(m), split(v)
    for t in range(1, 4):
        grad = torch.randn(numel, device=DEV, generator=g)
        grad[pad] = sentinel
        ref_g = split(grad)
        bc1, bc2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
        for x in PARAM_NAMES:
            capi.check(L.gsb_adam_step(ref_p[x].numel(), capi.ptr(ref_p[x]), capi.ptr(ref_g[x]), capi.ptr(ref_m[x]),
                                       capi.ptr(ref_v[x]), lr[x], 0.9, 0.999, 1e-8, bc1, bc2, capi.stream()))
        segs = adam_segments(offs, lr)
        table = (capi.AdamSegment * len(segs))(*[capi.AdamSegment(*s) for s in segs])
        capi.check(L.gsb_adam_step_segments(len(segs), C.addressof(table), capi.ptr(param), capi.ptr(grad),
                                            capi.ptr(m), capi.ptr(v), 0.9, 0.999, 1e-8, bc1, bc2, capi.stream()))
        for flat, ref in zip((param, m, v), (ref_p, ref_m, ref_v)):
            got = split(flat)
            for x in PARAM_NAMES:
                # both kernels round every float through the same adam_update, whatever its path or vector lane
                assert torch.equal(got[x], ref[x]), (t, x)
            assert bool((flat[pad] == sentinel).all())     # padding floats untouched


# ---- 2. SH colour with camera view directions on the merged block ----------------------------------------------
@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("n", [0, 1, 127, 129, 5000])
def test_sh_camera_mode_on_merged_block_is_the_split_variant(degree, n):
    from opensplat_b200 import capi, ops
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    K = ops.num_sh_bases(degree)
    g = torch.Generator(device=DEV).manual_seed(degree * 1000 + n)
    means = torch.randn((n, 3), device=DEV, generator=g) * 2.0
    cam_pos = torch.tensor([0.3, -0.7, 4.0], device=DEV)
    coeffs = torch.randn((n, K, 3), device=DEV, generator=g) * 0.5
    dc, rest = coeffs[:, 0, :].contiguous(), coeffs[:, 1:, :].contiguous()
    v_rgbs = torch.randn((n, 3), device=DEV, generator=g)
    for use in range(degree + 1):
        rgbs_split = torch.empty((n, 3), device=DEV)
        rgbs_cam = torch.empty((n, 3), device=DEV)
        capi.check(L.gsb_sh_forward_split(n, degree, use, P(means), P(cam_pos), P(dc), P(rest) if K > 1 else None,
                                          0.5, P(rgbs_split), s))
        capi.check(L.gsb_sh_forward_rgb_cam(n, degree, use, P(means), P(cam_pos), P(coeffs), 0.5, P(rgbs_cam), s))
        assert torch.equal(rgbs_cam, rgbs_split), use
        v_dc = torch.empty((n, 3), device=DEV)
        v_rest = torch.empty((n, K - 1, 3), device=DEV)
        v_coeffs = torch.full((n, K, 3), float("nan"), device=DEV)
        capi.check(L.gsb_sh_backward_split(n, degree, use, P(means), P(cam_pos), P(rgbs_split), P(v_rgbs), P(v_dc),
                                           P(v_rest) if K > 1 else None, s))
        capi.check(L.gsb_sh_backward_rgb_cam(n, degree, use, P(means), P(cam_pos), P(rgbs_cam), P(v_rgbs),
                                             P(v_coeffs), s))
        assert torch.equal(v_coeffs, torch.cat([v_dc[:, None, :], v_rest], 1)), use


# ---- 3. visible count in the binning stats ----------------------------------------------------------------------
def _bin_stats(xys, radii, conics, opac, W=256, H=192):
    from opensplat_b200 import ops
    tb = ops.tile_bounds(W, H)
    colors = torch.full((xys.shape[0], 3), 0.5, device=DEV)
    _, _, plain, _ = ops.bucket_tile_ranges(xys, radii, conics, colors, opac, tb, 1 << 20, 1024)
    _, _, stats, _ = ops.bucket_tile_ranges(xys, radii, conics, colors, opac, tb, 1 << 20, 1024, count_visible=True)
    plan = ops.BinPlan()
    plan.read_back(stats)
    plan.wait()
    stats = stats.cpu().tolist()
    assert plain.cpu().tolist() == stats[:3] + [0]      # without the request: the stats callers already read
    return stats, plan.visible


def _project(means, opac_logits, W=256, H=192):
    from opensplat_b200 import ops
    n = means.shape[0]
    g = torch.Generator(device=DEV).manual_seed(7)
    scales = torch.log(torch.rand((n, 3), device=DEV, generator=g) * 0.1 + 0.02)
    quats = torch.randn((n, 4), device=DEV, generator=g)
    view = torch.eye(4, device=DEV)
    proj = torch.tensor([[2 * 200.0 / W, 0, 0, 0], [0, 2 * 200.0 / H, 0, 0], [0, 0, 1.0, -0.01], [0, 0, 1, 0]],
                        device=DEV)
    xys, _, radii, conics, _, _, opac = ops.ProjectGaussiansActivated.apply(
        means, scales, 1.0, quats, opac_logits, view, proj @ view, 200.0, 200.0, W / 2.0, H / 2.0, H, W,
        ops.tile_bounds(W, H))
    return xys, radii, conics, opac.reshape(n)


def test_visible_count_of_the_binning_stats():
    g = torch.Generator(device=DEV).manual_seed(11)
    n = 5001
    # mixed: behind the camera, off screen, on screen
    means = torch.stack([torch.rand(n, device=DEV, generator=g) * 8 - 4, torch.rand(n, device=DEV, generator=g) * 6 - 3,
                         torch.rand(n, device=DEV, generator=g) * 9 - 3], 1)
    xys, radii, conics, opac = _project(means, torch.randn((n, 1), device=DEV, generator=g))
    vis = int((radii > 0).sum())
    assert 0 < vis < n
    stats, plan_visible = _bin_stats(xys, radii, conics, opac)
    assert stats[3] == vis and plan_visible == vis and stats[0] > 0
    # visible (radii > 0) but so faint that the cull leaves them in no tile list: centres on half-pixels, extent 0.01 px
    xs = torch.randint(0, 256, (n,), device=DEV, generator=g).float() + 0.5
    ys = torch.randint(0, 192, (n,), device=DEV, generator=g).float() + 0.5
    radii = torch.randint(0, 5, (n,), device=DEV, generator=g, dtype=torch.int32)
    conics = torch.tensor([0.5, 0.0, 0.5], device=DEV).repeat(n, 1)
    stats, plan_visible = _bin_stats(torch.stack([xs, ys], 1), radii, conics, torch.full((n,), 1e-4, device=DEV))
    vis = int((radii > 0).sum())
    assert stats[0] == 0 and stats[3] == vis > 0 and plan_visible == vis
    # every Gaussian behind the camera
    means[:, 2] = -2.0 - torch.rand(n, device=DEV, generator=g)
    xys, radii, conics, opac = _project(means, torch.randn((n, 1), device=DEV, generator=g))
    assert int((radii > 0).sum()) == 0
    stats, plan_visible = _bin_stats(xys, radii, conics, opac)
    assert stats[0] == 0 and stats[3] == 0 and plan_visible == 0
    # n = 0
    e = torch.empty((0, 2), device=DEV)
    stats, plan_visible = _bin_stats(e, torch.empty(0, dtype=torch.int32, device=DEV), torch.empty((0, 3), device=DEV),
                                     torch.empty(0, device=DEV))
    assert stats == [0, 0, 0, 0] and plan_visible == 0


# ---- 4. / 5. trajectory against GaussianModel --------------------------------------------------------------------
def test_trainer_follows_gaussian_model_through_refinements():
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV)}
    steps, seed = 34, 11
    model, lm, cm = run_model(p, cams, gts_d, steps, seed, cfg=refine_config(), sh_degree_interval=8)
    tr, lt, ct = run_trainer(p, cams, gts_d, steps, seed, cfg=refine_config(), sh_degree_interval=8)
    assert cm[18] == len(p["means"]) and cm[19] != cm[18] and cm[29] != cm[28]    # two refinements happened
    _compare(model, tr, lm, lt, cm, ct, exact=True)


def test_trainer_follows_gaussian_model_through_the_downscale_schedule():
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV), 2: torch.from_numpy(_half(gts)).to(DEV)}
    kw = dict(sh_degree_interval=8, num_downscales=1, resolution_schedule=6)
    model, lm, cm = run_model(p, cams, gts_d, 12, 3, cfg=refine_config(), **kw)
    tr, lt, ct = run_trainer(p, cams, gts_d, 12, 3, cfg=refine_config(), **kw)
    assert tr.resolution == (W, H) and tr.pixel_reallocs == 1
    _compare(model, tr, lm, lt, cm, ct, exact=True)


# ---- 6. a view that hits nothing ----------------------------------------------------------------------------------
def test_empty_view_renders_background_and_trains_nothing():
    from opensplat_b200.model import Camera
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    bg = (0.25, 0.5, 0.75)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, refine_config(), background=bg, device=DEV)
    for step in range(1, 4):
        tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
    away = c2w[0].copy()
    away[:3, :3] = away[:3, :3] @ np.diag([-1.0, 1.0, -1.0]).astype(np.float32)   # turned around: faces away
    pp, d = tr.pipe, tr.densifier
    before = [t.clone() for t in (pp.param_flat, pp.adam_m, pp.adam_v, d.xys_grad_norm, d.vis_counts, d.max_2d_size)]
    t_before = pp.adam_t
    loss = tr.step(Camera(W, H, *intr, away), gt[0], 4)
    torch.cuda.synchronize()
    assert pp.plan.visible == 0
    assert torch.equal(tr.image, torch.tensor(bg, device=DEV).expand(H, W, 3))
    assert bool(torch.isfinite(loss).all()) and float(loss[0]) > 0
    after = (pp.param_flat, pp.adam_m, pp.adam_v, d.xys_grad_norm, d.vis_counts, d.max_2d_size)
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert pp.adam_t == t_before and tr.last_info == {"refined": False}


# ---- 7. capacity growth -----------------------------------------------------------------------------------------
def test_capacity_growth_does_not_change_the_trajectory(monkeypatch):
    from opensplat_b200 import ops
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV)}
    waits = []
    orig = ops.BinPlan.wait

    def counting_wait(self):
        waits.append(1)
        return orig(self)
    monkeypatch.setattr(ops.BinPlan, "wait", counting_wait)
    small, ls, _ = run_trainer(p, cams, gts_d, 5, 1, cfg=refine_config(), m_capacity=1)
    redone = len(waits) - 5
    big, lb, _ = run_trainer(p, cams, gts_d, 5, 1, cfg=refine_config(), m_capacity=10 ** 6)
    assert redone > 0 and small.pipe.plan.m_cap < big.pipe.plan.m_cap      # the small plan overflowed and grew
    assert np.abs(ls - lb).max() <= 1e-6                 # the loss value: float atomics, last bits vary run to run
    assert torch.equal(small.pipe.param_flat, big.pipe.param_flat)
    assert torch.equal(small.pipe.adam_m, big.pipe.adam_m) and torch.equal(small.pipe.adam_v, big.pipe.adam_v)


# ---- 8. steady state ----------------------------------------------------------------------------------------------
def test_steady_state_step_allocates_nothing_and_waits_once(monkeypatch):
    from opensplat_b200 import ops
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, refine_config(warmup_length=10 ** 6),
                      device=DEV)
    for step in range(1, 6):                                           # warm-up: plan, bins, statistics, cuBLAS
        tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
    torch.cuda.synchronize()
    waits, tripped = [], []
    orig = ops.BinPlan.wait

    def wait_outside_sync_check(self):
        # The one intended host wait.  Record whether Event.synchronize alone trips the sync check, then wait.
        waits.append(1)
        try:
            return orig(self)
        except RuntimeError:
            tripped.append(1)
            torch.cuda.set_sync_debug_mode(0)
            try:
                return orig(self)
            finally:
                torch.cuda.set_sync_debug_mode("error")
    monkeypatch.setattr(ops.BinPlan, "wait", wait_outside_sync_check)
    before = torch.cuda.memory_stats()["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        for step in range(6, 16):
            tr.step(cams[(step - 1) % 3], gt[(step - 1) % 3], step)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.cuda.memory_stats()["allocation.all.allocated"] == before
    assert len(waits) == 10
    print(f"Event.synchronize trips set_sync_debug_mode('error'): {bool(tripped)}")


# ---- 9. the PLY writer --------------------------------------------------------------------------------------------
def test_trainer_save_writes_the_bytes_gaussian_model_writes(tmp_path):
    from opensplat_b200.model import GaussianModel
    from opensplat_b200.trainer import SplatTrainer
    from util import scene_edit_inputs
    p = scene_edit_inputs(1001, 16, 4)[0]
    model = GaussianModel({k: torch.from_numpy(v) for k, v in p.items()}, device=DEV)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, device=DEV)
    a, b = str(tmp_path / "model.ply"), str(tmp_path / "trainer.ply")
    model.save(a, step=77)
    tr.save(b, step=77)
    assert open(a, "rb").read() == open(b, "rb").read()


# ---- 10. against the reference's unchanged model.cpp ---------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(LIB), reason="libopensplat_model_b200.so not built (needs /root/reference at build time)")
def test_trainer_against_the_reference_model_cpp():
    from opensplat_b200 import cpp_ops
    cpp_ops.ops()
    torch.ops.load_library(LIB)
    p, c2w, gts, (fx, fy, cx, cy), H, W = make_problem()
    steps, seed, ssim_w, sh_int = 34, 11, 0.2, 8
    cfg = refine_config()
    params = [torch.from_numpy(p[x]).to(DEV) for x in PARAM_NAMES]
    out = torch.ops.opensplat_b200_model.train(
        params, torch.from_numpy(c2w), torch.from_numpy(gts), fx, fy, cx, cy, H, W, 1, steps, ssim_w, seed, sh_int,
        cfg.num_cameras, cfg.refine_every, cfg.warmup_length, cfg.reset_alpha_every, cfg.densify_grad_thresh,
        cfg.densify_size_thresh, cfg.stop_screen_size_at, cfg.split_screen_size, cfg.max_steps)
    ref_loss, ref_cnt, ref_rgb = out[0].numpy(), out[1].numpy(), out[2]
    ref_params = dict(zip(PARAM_NAMES, out[3:9]))
    cams = _cams(c2w, H, W, (fx, fy, cx, cy))
    tr, losses, counts = run_trainer(p, cams, {1: torch.from_numpy(gts).to(DEV)}, steps, seed, ssim_w, cfg=cfg,
                                     sh_degree_interval=sh_int)
    assert np.abs(losses[:20] - ref_loss[:20]).max() <= 5e-5, np.abs(losses[:20] - ref_loss[:20]).max()
    assert np.abs(counts - ref_cnt).max() <= 0.02 * ref_cnt.max(), (counts[[19, 29]], ref_cnt[[19, 29]])
    assert np.abs(losses - ref_loss).max() <= 5e-3, np.abs(losses - ref_loss).max()
    if np.array_equal(counts, ref_cnt):
        pt = tr.params()
        for k in PARAM_NAMES:
            a, b = pt[k], ref_params[k]
            assert a.shape == b.shape
            assert float((a - b).abs().max()) <= 2e-3 * (1.0 + float(b.abs().max())), k
        assert float((tr.image - ref_rgb).abs().max()) <= 2e-2
