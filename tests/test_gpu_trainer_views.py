"""GPU: trainer.SplatTrainer with several camera views per step (views_per_step=B).
 * gsb_sh_forward_rgb_cam_multiview bit-identical to B calls of gsb_sh_forward_rgb_cam;
 * gsb_project_backward_activated_acc == prev + gsb_project_backward_activated, bit for bit;
 * one B-view step's gradient buffer against the mean of B one-view backward passes from the same parameters;
 * the trajectory against model.GaussianModel run view by view (gradients scaled by 1/B, statistics per view) through
   the SH degree and downscale schedules, an alpha reset and two densifications;
 * empty views, the steady state (no allocation, one host wait per view) and, under torch.distributed.run,
   tools/check_parallel_trainer.py --views-per-rank 2."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_trainer as tg  # noqa: E402  (the training problem and _compare's bounds)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SSIM_W = 0.2


# ---- fixtures -------------------------------------------------------------------------------------------------------
def _params(p):
    return {k: torch.from_numpy(v) for k, v in p.items()}


def _away(c2w, H, W, intr):
    from opensplat_b200.model import Camera
    away = c2w[0].copy()
    away[:3, :3] = away[:3, :3] @ np.diag([-1.0, 1.0, -1.0]).astype(np.float32)   # turned around: faces away
    return Camera(W, H, *intr, away)


def _views(cams, B, step):
    """The B view indices of `step` (1-based)."""
    return [((step - 1) * B + b) % len(cams) for b in range(B)]


def _no_adam(tr):
    """Keep the parameters fixed, so that gradient buffers of several steps come from the same parameters."""
    tr._adam_step = lambda: None
    return tr


def _rel_l2(a, b):
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


# ---- 1. multi-view SH forward -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 3, 8, 9])
@pytest.mark.parametrize("n", [0, 1, 127, 129, 5000])
@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
def test_multiview_sh_forward_is_b_single_view_calls(degree, n, B):
    from opensplat_b200 import capi, ops
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    K = ops.num_sh_bases(degree)
    g = torch.Generator(device=DEV).manual_seed(degree * 1000 + n * 10 + B)
    means = torch.randn((n, 3), device=DEV, generator=g) * 2.0
    cams = torch.randn((B, 3), device=DEV, generator=g) * 3.0 + torch.tensor([0.0, 0.0, 6.0], device=DEV)
    coeffs = torch.randn((n, K, 3), device=DEV, generator=g) * 0.5
    for use in range(degree + 1):
        got = torch.full((B, n, 3), float("nan"), device=DEV)
        capi.check(L.gsb_sh_forward_rgb_cam_multiview(n, degree, use, P(means), B, P(cams), P(coeffs), 0.5, P(got), s))
        for b in range(B):
            ref = torch.full((n, 3), -1.0, device=DEV)
            capi.check(L.gsb_sh_forward_rgb_cam(n, degree, use, P(means), P(cams[b]), P(coeffs), 0.5, P(ref), s))
            assert torch.equal(got[b], ref), (use, b)


# ---- 2. accumulating projection backward ------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 4099])
def test_accumulating_projection_backward_adds_the_vjp(n):
    from opensplat_b200 import capi
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    g = torch.Generator(device=DEV).manual_seed(n)
    W, H, fx, fy = 256, 192, 200.0, 200.0

    def rnd(*shape, scale=1.0):
        return torch.randn(shape, device=DEV, generator=g) * scale

    means = torch.stack([rnd(n) * 1.5, rnd(n) * 1.0, torch.rand(n, device=DEV, generator=g) * 4 + 2], 1).contiguous()
    log_scales = torch.log(torch.rand((n, 3), device=DEV, generator=g) * 0.1 + 0.02)
    quats = rnd(n, 4)
    opac = torch.sigmoid(rnd(n))
    view = torch.eye(4, device=DEV)
    proj = torch.tensor([[2 * fx / W, 0, 0, 0], [0, 2 * fy / H, 0, 0], [0, 0, 1.0, -0.01], [0, 0, 1, 0]], device=DEV)
    projmat = proj @ view
    radii = torch.randint(-1, 4, (n,), device=DEV, generator=g, dtype=torch.int32)   # radii <= 0 included
    conics = torch.stack([torch.rand(n, device=DEV, generator=g) + 0.5, rnd(n, scale=0.1),
                          torch.rand(n, device=DEV, generator=g) + 0.5], 1).contiguous()
    v_xy, v_conic, v_opac = rnd(n, 2), rnd(n, 3), rnd(n)
    prev = [rnd(n, 3), rnd(n, 3), rnd(n, 4), rnd(n)]
    vjp = [torch.full_like(t, float("nan")) for t in prev]
    acc = [t.clone() for t in prev]

    def call(fn, outs):
        capi.check(fn(n, P(means), P(log_scales), 1.0, P(quats), P(opac), P(view), P(projmat), fx, fy, H, W, P(radii),
                      P(conics), P(v_xy), None, P(v_conic), P(v_opac), *[P(t) for t in outs], s))
    call(L.gsb_project_backward_activated, vjp)
    call(L.gsb_project_backward_activated_acc, acc)
    for a, p0, v in zip(acc, prev, vjp):
        assert bool(torch.isfinite(v).all())
        assert torch.equal(a, p0 + v)
    culled = radii <= 0
    assert bool(culled.any()) and torch.equal(acc[0][culled], prev[0][culled])   # radii <= 0: adds zero


# ---- 3. one B-view step vs B one-view backward passes -------------------------------------------------------------------
def _single_view_grads(p, cams, gts, views, step, **kw):
    """pipe.grad_flat of the one-view trainer on each view, from the same (fixed) parameters, and the losses."""
    from opensplat_b200.trainer import SplatTrainer
    tr = _no_adam(SplatTrainer(_params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV, ssim_weight=SSIM_W,
                               **kw))
    grads, losses = [], []
    for v in views:
        losses.append(tr.step(cams[v], gts[v], step).clone())
        grads.append(tr.pipe.grad_flat.clone())
    return grads, torch.stack(losses), tr.pipe


@pytest.mark.parametrize("B", [2, 4])
def test_b_view_step_is_the_mean_of_b_one_view_backward_passes(B):
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    views, step = [0, 1, 2, 1][:B], 9            # degree 1 (sh_degree_interval 8), distinct and repeated views
    grads, losses1, pp1 = _single_view_grads(p, cams, gt, views, step, sh_degree_interval=8)
    tr = _no_adam(SplatTrainer(_params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV, ssim_weight=SSIM_W,
                               sh_degree_interval=8, views_per_step=B))
    lossB = tr.step([cams[v] for v in views], gt[views], step)
    torch.cuda.synchronize()
    assert lossB.shape == (B, 3) and float((lossB - losses1).abs().max()) <= 1e-6
    mean = grads[0].clone()
    for gr in grads[1:]:
        mean = mean + gr                          # the order the accumulating projection backward sums in
    mean = mean * (1.0 / B)
    pp = tr.pipe
    geom = pp.geom_numel
    assert torch.equal(pp.grad_flat[:geom], mean[:geom])               # means, scales, quats, opacities: exact
    o, c, _ = pp.offs["coeffs"]
    rel = _rel_l2(pp.grad_flat[o:o + c], mean[o:o + c])                # the SH block: FMA re-association only
    print(f"B={B}: coefficient gradients rel-L2 {rel:.3g}, bit-identical {torch.equal(pp.grad_flat, mean)}")
    assert rel <= 1e-6


# ---- 4. trajectory against GaussianModel run view by view -----------------------------------------------------------
STEPS = 22
KW = dict(sh_degree_interval=8, num_downscales=1, resolution_schedule=10)


def _cfg():
    # refinements at steps 6 (alpha reset), 12 and 18 (densifications)
    return tg.refine_config(refine_every=6, warmup_length=5, reset_alpha_every=4)


def _model_views_step(model, pairs, step):
    """GaussianModel's B-view step: forward, loss and backward per view (the leaf gradients sum over the views),
    gradients x 1/B, one optimizer step, then each view's statistics in view order and one refine decision."""
    from opensplat_b200.model import PARAM_NAMES
    model.optimizers_zero_grad()
    losses, stats = [], []
    for cam, gt in pairs:
        loss = model.main_loss(model.forward(cam, step), gt, SSIM_W)
        if loss.requires_grad:
            loss.backward()
        losses.append(float(loss.detach()))
        gxy = model.xys.grad
        stats.append((gxy.detach().clone() if gxy is not None else None, model.radii.clone()))
    with torch.no_grad():
        for k in PARAM_NAMES:
            if getattr(model, k).grad is not None:
                getattr(model, k).grad.mul_(1.0 / len(pairs))
    trains = any(v is not None for v, _ in stats)
    if trains:
        model.optimizers_step()
    model.schedulers_step(step)
    if trains:
        d = model.densifier
        for v_xy, radii in stats:
            d.accumulate_view(step, v_xy, radii, model.lastHeight, model.lastWidth)
        with torch.no_grad():
            prm = {k: getattr(model, k).detach() for k in PARAM_NAMES}
            new_p, new_m, new_v, _ = d.finish_step(step, prm, model.adam_m, model.adam_v, model.lastHeight,
                                                   model.lastWidth)
            if new_p is not prm:
                for k in PARAM_NAMES:
                    setattr(model, k, new_p[k].requires_grad_())
                model.adam_m, model.adam_v = new_m, new_v
    return losses


@pytest.mark.parametrize("B", [2, 4])
def test_b_view_trainer_follows_gaussian_model_view_by_view(B):
    from opensplat_b200.model import GaussianModel, downscale_factor
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gts_d = {1: torch.from_numpy(gts).to(DEV), 2: torch.from_numpy(tg._half(gts)).to(DEV)}

    def pairs(step):
        f = downscale_factor(step, KW["num_downscales"], KW["resolution_schedule"])
        return [(cams[v], gts_d[f][v]) for v in _views(cams, B, step)]
    model = GaussianModel(_params(p), _cfg(), device=DEV, **KW)
    torch.manual_seed(3)
    lm, cm = [], []
    for step in range(1, STEPS + 1):
        lm.extend(_model_views_step(model, pairs(step), step))
        cm.append(model.means.shape[0])
    tr = SplatTrainer(_params(p), _cfg(), device=DEV, ssim_weight=SSIM_W, views_per_step=B, **KW)
    torch.manual_seed(3)
    lt, ct, refined = [], [], []
    for step in range(1, STEPS + 1):
        pr = pairs(step)
        loss = tr.step([c for c, _ in pr], torch.stack([g for _, g in pr]), step)
        lt.extend(loss[:, 0].tolist())
        ct.append(tr.n)
        refined.append(tr.last_info.get("refined", False))
    cm, ct = np.array(cm), np.array(ct)
    assert ct[11] != ct[10] and ct[17] != ct[16] and refined[5]            # two densifications, the alpha reset
    assert tr.resolution == (W, H) and tr.pixel_reallocs == 1              # the downscale schedule
    exact = tg._compare(model, tr, np.array(lm), np.array(lt), cm, ct)
    print(f"B={B} trainer vs GaussianModel view by view over {STEPS} steps: bit-identical = {exact}")


# ---- 5. empty views ---------------------------------------------------------------------------------------------------
def test_one_empty_view_trains_on_the_others_with_divisor_b():
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    grads, _, _ = _single_view_grads(p, cams, gt, [1], 9, sh_degree_interval=8)
    tr = _no_adam(SplatTrainer(_params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV, ssim_weight=SSIM_W,
                               sh_degree_interval=8, views_per_step=2))
    tr.step([_away(c2w, H, W, intr), cams[1]], gt[[0, 1]], 9)
    torch.cuda.synchronize()
    pp = tr.pipe
    half = grads[0] * 0.5                         # the divisor stays B = 2
    assert torch.equal(pp.grad_flat[:pp.geom_numel], half[:pp.geom_numel])
    o, c, _ = pp.offs["coeffs"]
    assert _rel_l2(pp.grad_flat[o:o + c], half[o:o + c]) <= 1e-6
    # the statistics: only the visible view's (the empty one adds nothing in one process)
    ref = SplatTrainer(_params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV, sh_degree_interval=8)
    ref.step(cams[1], gt[1], 9)
    for a in ("xys_grad_norm", "vis_counts", "max_2d_size"):
        assert torch.equal(getattr(tr.densifier, a), getattr(ref.densifier, a)), a


def test_all_views_empty_trains_nothing():
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    tr = SplatTrainer(_params(p), tg.refine_config(), device=DEV, views_per_step=3)
    for step in range(1, 4):
        tr.step(cams, gt, step)
    pp, d = tr.pipe, tr.densifier
    before = [t.clone() for t in (pp.param_flat, pp.adam_m, pp.adam_v, d.xys_grad_norm, d.vis_counts, d.max_2d_size)]
    t_before = pp.adam_t
    away = _away(c2w, H, W, intr)
    loss = tr.step([away] * 3, gt, 4)
    torch.cuda.synchronize()
    assert pp.plan.visible == 0 and bool(torch.isfinite(loss).all()) and loss.shape == (3, 3)
    after = (pp.param_flat, pp.adam_m, pp.adam_v, d.xys_grad_norm, d.vis_counts, d.max_2d_size)
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert pp.adam_t == t_before and tr.last_info == {"refined": False}


# ---- 6. steady state --------------------------------------------------------------------------------------------------
def test_steady_state_allocates_nothing_and_waits_once_per_view(monkeypatch):
    from opensplat_b200 import ops
    from opensplat_b200.trainer import SplatTrainer
    B = 3
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    tr = SplatTrainer(_params(p), tg.refine_config(warmup_length=10 ** 6), device=DEV, views_per_step=B)

    def step_at(step):
        v = _views(cams, B, step)
        tr.step([cams[i] for i in v], [gt[i] for i in v], step)
    for step in range(1, 6):                                           # warm-up: plan, bins, statistics, cuBLAS
        step_at(step)
    torch.cuda.synchronize()
    waits = []
    orig = ops.BinPlan.wait

    def wait_outside_sync_check(self):
        waits.append(1)                                                # the intended host wait of each view
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
            step_at(step)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.cuda.memory_stats()["allocation.all.allocated"] == before
    assert len(waits) == 10 * B


# ---- 7. under a process group -----------------------------------------------------------------------------------------
def _run(nproc, port, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tools", "check_parallel_trainer.py"), "--views-per-rank", "2"],
                       capture_output=True, text=True, timeout=900, env=e)
    print(r.stdout[-4000:])
    if r.returncode != 0:
        print(r.stderr[-6000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "check_ok=True" in r.stdout and "views_per_rank=2" in r.stdout
    return r.stdout


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_two_views_per_rank_world1_follows_gaussian_model(overlap):
    out = _run(1, 29561 if overlap == "1" else 29563, {"GSB_EXCHANGE_OVERLAP": overlap})
    assert f"overlap={overlap == '1'}" in out and "steady_allocs=0 steady_waits=20" in out
    assert "plain_trainer_bit_identical=True" in out


def test_two_views_per_rank_2gpu_follows_gaussian_model():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run(2, 29565)
    out = _run(2, 29567, {"GSB_EXCHANGE_MULTICAST": "0"})
    assert "multicast=False" in out
