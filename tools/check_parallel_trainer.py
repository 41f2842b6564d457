"""torchrun --nproc-per-node N tools/check_parallel_trainer.py : the data-parallel trainer.SplatTrainer on N GPUs.

Every rank trains its own view sequence (rank r, step s -> view (s - 1 + r) % V) of the training problem of
tests/test_gpu_trainer.py twice, with SplatTrainer(..., group=WORLD) (the fused NVLink exchange) and with
GaussianModel(..., group=WORLD) (autograd + one NCCL all-reduce of the six gradient tensors), through the SH degree
schedule, the downscale schedule, an alpha reset and two densifications; with two or more ranks, rank 1's camera is
turned around (its view hits nothing) on a densification step.  It checks:
  * the same Gaussian count as GaussianModel at every step, losses to 1e-6, parameters and Adam moments within the
    bounds of test_gpu_trainer._compare (the SH gradient is expanded from the exchanged colour gradients instead of
    reduced, a fp32 re-association; the largest differences are printed);
  * replicas bit-identical (parameters and moments) after every step;
  * the steady state: between refinements a step allocates no device memory and waits on the host once.
GSB_EXCHANGE_MULTICAST=0 forces the peer-pointer all-reduce, GSB_EXCHANGE_OVERLAP=0 the single-launch exchange.

--views-per-rank B (default 1): every rank trains B views per step (SplatTrainer(views_per_step=B); rank r's view b
of step s is view ((s - 1) B G + r B + b) % V).  The GaussianModel reference then runs a forward, loss and backward
per view, keeps each view's xys.grad and radii, scales the leaf gradients by 1/B before optimizers_step (which
averages over the ranks) and accumulates the statistics view by view (Densifier.accumulate_view, finish_step).  On
the densification step the last view of rank 1 (of rank 0 at world size 1) is turned around.  The steady state then
expects B host waits per step.
--mcmc: the MCMC strategy instead (SplatTrainer(cfg=mcmc.MCMCConfig), DESIGN D20; GaussianModel has no counterpart):
relocations and growth from a set with faint Gaussians, replicas bit-identical (parameters and moments) after every
step, and at world size 1 the run bit-identical to the same run without a group.
Rank 0 prints one line ending in `check_ok=True|False`; the exit code is 0 iff every check held on every rank."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--views-per-rank", type=int, default=1)
ap.add_argument("--mcmc", action="store_true")
ARGS = ap.parse_args()
B = ARGS.views_per_rank
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
DEV = torch.device("cuda", local)

import test_gpu_trainer as tg  # noqa: E402  (the training problem and its refinement schedule)
from opensplat_b200 import ops, parallel  # noqa: E402
from opensplat_b200.model import Camera, GaussianModel, PARAM_NAMES, downscale_factor  # noqa: E402
from opensplat_b200.trainer import SplatTrainer  # noqa: E402

STEPS, SEED, SSIM_W = 22, 7, 0.2
# SH degree 0 -> 1 at step 8; half resolution until step 10; refinements at steps 6 (alpha reset), 12 and 18
# (densifications)
KW = dict(sh_degree_interval=8, num_downscales=1, resolution_schedule=10)
EMPTY_STEP = 18                     # rank 1 (world >= 2): its view hits nothing on this densification step


def cfg(**kw):
    return tg.refine_config(**{**dict(refine_every=6, warmup_length=5, reset_alpha_every=4), **kw})


p, c2w, gts, intr, H, W = tg.make_problem()
cams = tg._cams(c2w, H, W, intr)
V = len(cams)
gts_d = {1: torch.from_numpy(gts).to(DEV), 2: torch.from_numpy(tg._half(gts)).to(DEV)}
away = c2w[0].copy()
away[:3, :3] = away[:3, :3] @ np.diag([-1.0, 1.0, -1.0]).astype(np.float32)   # turned around: faces away
away_cam = Camera(W, H, *intr, away)


def view(step):
    v = (step - 1 + rank) % V
    cam = away_cam if (world >= 2 and rank == 1 and step == EMPTY_STEP) else cams[v]
    return cam, gts_d[downscale_factor(step, KW["num_downscales"], KW["resolution_schedule"])][v]


def views(step):
    """B > 1: this rank's B (camera, image) pairs of `step`."""
    f = downscale_factor(step, KW["num_downscales"], KW["resolution_schedule"])
    out = []
    for b in range(B):
        v = ((step - 1) * B * world + rank * B + b) % V
        empty = step == EMPTY_STEP and b == B - 1 and rank == min(1, world - 1)
        out.append((away_cam if empty else cams[v], gts_d[f][v]))
    return out


def params():
    return {k: torch.from_numpy(v) for k, v in p.items()}


def run_trainer(group, check_sync):
    tr = SplatTrainer(params(), cfg(), device=DEV, ssim_weight=SSIM_W, group=group, views_per_step=B, **KW)
    torch.manual_seed(SEED)
    losses, counts, in_sync, empty_visible = [], [], True, None
    for step in range(1, STEPS + 1):
        if B == 1:
            cam, gt = view(step)
            loss = tr.step(cam, gt, step)
            losses.append(float(loss[0]))
        else:
            vs = views(step)
            loss = tr.step([c for c, _ in vs], [g for _, g in vs], step)
            losses.extend(float(x) for x in loss[:, 0].tolist())
        counts.append(tr.n)
        if step == EMPTY_STEP:
            empty_visible = tr.pipe.plan.visible
        if check_sync:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m, pp.adam_v))
    return tr, np.array(losses), np.array(counts), in_sync, empty_visible


def run_model():
    if B > 1:
        return run_model_views()
    model = GaussianModel(params(), cfg(), device=DEV, group=dist.group.WORLD, **KW)
    torch.manual_seed(SEED)
    losses, counts = [], []
    for step in range(1, STEPS + 1):
        cam, gt = view(step)
        model.optimizers_zero_grad()
        loss = model.main_loss(model.forward(cam, step), gt, SSIM_W)
        if loss.requires_grad:
            loss.backward()
        losses.append(float(loss.detach()))
        model.optimizers_step()
        model.schedulers_step(step)
        model.after_train(step)
        counts.append(model.means.shape[0])
    return model, np.array(losses), np.array(counts)


def model_views_step(model, pairs, step):
    """One B-view step of GaussianModel: per view a forward, loss and backward (the leaf gradients sum over the
    views), the gradients times 1/B, optimizers_step (the mean over the ranks), then the per-view statistics and one
    refine decision.  Returns the B losses."""
    model.optimizers_zero_grad()
    losses, stats = [], []
    for cam, gt in pairs:
        loss = model.main_loss(model.forward(cam, step), gt, SSIM_W)
        if loss.requires_grad:
            loss.backward()
        losses.append(float(loss.detach()))
        g = model.xys.grad
        stats.append((g.detach().clone() if g is not None else None, model.radii.clone()))
    with torch.no_grad():
        for k in PARAM_NAMES:
            if getattr(model, k).grad is not None:
                getattr(model, k).grad.mul_(1.0 / len(pairs))
    d = model.densifier
    trains = any(v is not None for v, _ in stats) or d._world() > 1
    if trains:   # a step whose views all hit nothing trains nothing (one process)
        model.optimizers_step()
    model.schedulers_step(step)
    if trains:
        for v_xy, radii in stats:
            d.accumulate_view(step, v_xy, radii, model.lastHeight, model.lastWidth)
        with torch.no_grad():
            p = {k: getattr(model, k).detach() for k in PARAM_NAMES}
            new_p, new_m, new_v, _ = d.finish_step(step, p, model.adam_m, model.adam_v, model.lastHeight,
                                                   model.lastWidth)
            if new_p is not p:
                for k in PARAM_NAMES:
                    setattr(model, k, new_p[k].requires_grad_())
                model.adam_m, model.adam_v = new_m, new_v
    return losses


def run_model_views():
    model = GaussianModel(params(), cfg(), device=DEV, group=dist.group.WORLD, **KW)
    torch.manual_seed(SEED)
    losses, counts = [], []
    for step in range(1, STEPS + 1):
        losses.extend(model_views_step(model, views(step), step))
        counts.append(model.means.shape[0])
    return model, np.array(losses), np.array(counts)


def compare(model, tr, lm, lt, cm, ct):
    """test_gpu_trainer._compare's bounds, reported instead of asserted: (ok, max loss difference, bit-identical)."""
    ok = bool(np.array_equal(cm, ct))
    dloss = float(np.abs(lm - lt).max()) if ok else float("inf")
    ok = ok and dloss <= 1e-6
    exact = True
    pt = tr.params()
    mt, vt = tr.adam_state()
    for k in PARAM_NAMES:
        diffs = []
        for a, b in ((getattr(model, k).detach(), pt[k]), (model.adam_m[k], mt[k]), (model.adam_v[k], vt[k])):
            if a.shape != b.shape:
                ok, d = False, float("inf")
            else:
                d = float((a - b).abs().max()) if a.numel() else 0.0
                ok = ok and d <= 1e-3 * (1.0 + float(a.abs().max()))
                exact = exact and torch.equal(a, b)
            diffs.append(d)
        print(f"  rank {rank} {k}: max |d| param {diffs[0]:.3g}, exp_avg {diffs[1]:.3g}, exp_avg_sq {diffs[2]:.3g}")
    return ok, dloss, exact


def steady_state():
    """10 steps between refinements under set_sync_debug_mode('error'): (allocations, BinPlan.wait calls)."""
    tr = SplatTrainer(params(), cfg(warmup_length=10 ** 6), device=DEV, group=dist.group.WORLD, views_per_step=B,
                      **KW)

    def step_at(step):                               # full resolution, no turned-around camera
        if B == 1:
            v = (step - 1 + rank) % V
            tr.step(cams[v], gts_d[1][v], step)
        else:
            vs = [((step - 1) * B * world + rank * B + b) % V for b in range(B)]
            tr.step([cams[v] for v in vs], [gts_d[1][v] for v in vs], step)
    for step in range(11, 16):                       # warm-up: plan, bins, statistics, cuBLAS
        step_at(step)
    torch.cuda.synchronize()
    waits, orig = [], ops.BinPlan.wait

    def wait_outside_sync_check(self):
        waits.append(1)
        torch.cuda.set_sync_debug_mode(0)            # the one intended host wait
        try:
            return orig(self)
        finally:
            torch.cuda.set_sync_debug_mode("error")
    ops.BinPlan.wait = wait_outside_sync_check
    before = torch.cuda.memory_stats(DEV)["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        for step in range(16, 26):
            step_at(step)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        ops.BinPlan.wait = orig
    torch.cuda.synchronize()
    return torch.cuda.memory_stats(DEV)["allocation.all.allocated"] - before, len(waits)


def run_mcmc(group):
    """The MCMC trainer on this rank's views: (trainer, counts, relocated, replicas in sync after every step)."""
    from opensplat_b200.mcmc import MCMCConfig
    pm = params()
    pm["opacities"][:300] = -8.0                     # faint: relocated at the first refinement
    n0 = pm["means"].shape[0]
    cfg = MCMCConfig(refine_start=4, refine_every=6, cap_max=int(1.12 * n0), max_steps=200, seed=SEED)
    tr = SplatTrainer(pm, cfg, device=DEV, ssim_weight=SSIM_W, group=group, views_per_step=B, **KW)
    counts, relocated, in_sync = [], 0, True
    for step in range(1, STEPS + 1):
        if B == 1:
            tr.step(*view(step), step)
        else:
            vs = views(step)
            tr.step([c for c, _ in vs], [g for _, g in vs], step)
        counts.append(tr.n)
        relocated += tr.last_info.get("relocated", 0)
        if group is not None:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m, pp.adam_v))
    return tr, np.array(counts), relocated, in_sync


def check_mcmc():
    tr, ct, relocated, in_sync = run_mcmc(dist.group.WORLD)
    plain_exact = None
    if world == 1:
        tp, cp, _, _ = run_mcmc(None)
        plain_exact = bool(np.array_equal(cp, ct) and all(torch.equal(a, b) for a, b in (
            (tp.pipe.param_flat, tr.pipe.param_flat), (tp.pipe.adam_m, tr.pipe.adam_m),
            (tp.pipe.adam_v, tr.pipe.adam_v))))
    refined = bool(ct[-1] > ct[0] and relocated >= 300)
    flags = torch.tensor([int(in_sync), int(refined), int(plain_exact is not False)], device=DEV)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    good = bool(flags.all())
    if rank == 0:
        print(f"parallel mcmc check world={world}: counts {ct[0]}->{ct[-1]} relocated={relocated} "
              f"replicas_in_sync={bool(flags[0])} refined={bool(flags[1])} plain_trainer_bit_identical={plain_exact} "
              + (f"views_per_rank={B} " if B > 1 else "") + f"check_ok={good}")
    return good


dist.init_process_group("nccl", device_id=DEV)
if ARGS.mcmc:
    ok_mcmc = check_mcmc()
    dist.destroy_process_group()
    sys.exit(0 if ok_mcmc else 1)
tr, lt, ct, in_sync, empty_visible = run_trainer(dist.group.WORLD, check_sync=True)
model, lm, cm = run_model()
ok, dloss, exact = compare(model, tr, lm, lt, cm, ct)
refined = bool(cm[11] != cm[10] and cm[17] != cm[16])      # both densifications changed the Gaussian set
empty_ok = (world < 2 or rank != 1 or empty_visible == 0) if B == 1 else (rank != min(1, world - 1) or
                                                                        empty_visible == 0)
mc, overlap = bool(tr.exchange.multicast_ptr), tr.exchange.overlap
plain_exact = None
if world == 1:                                   # the same run without the exchange (group=None)
    tp, lp, cp, _, _ = run_trainer(None, check_sync=False)
    plain_exact = bool(np.array_equal(cp, ct) and torch.equal(tp.pipe.param_flat, tr.pipe.param_flat)
                       and torch.equal(tp.pipe.adam_m, tr.pipe.adam_m) and torch.equal(tp.pipe.adam_v, tr.pipe.adam_v))
    del tp
del tr, model
allocs, waits = steady_state()
steady_ok = allocs == 0 and waits == 10 * B
flags = torch.tensor([int(ok), int(in_sync), int(refined), int(empty_ok), int(steady_ok)], device=DEV)
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
dl = torch.tensor([dloss], dtype=torch.float64, device=DEV)
dist.all_reduce(dl, op=dist.ReduceOp.MAX)
good = bool(flags.all())
if rank == 0:
    print(f"parallel trainer check world={world} multicast={mc} overlap={overlap}: counts {ct[0]}->{ct[-1]} "
          f"max|dloss|={float(dl[0]):.3g} matches_gaussian_model={bool(flags[0])} bit_identical={exact} "
          f"plain_trainer_bit_identical={plain_exact} replicas_in_sync={bool(flags[1])} refined={bool(flags[2])} "
          f"empty_view_ok={bool(flags[3])} steady_allocs={allocs} steady_waits={waits} "
          + (f"views_per_rank={B} " if B > 1 else "") + f"check_ok={good}")
dist.destroy_process_group()
sys.exit(0 if good else 1)
