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
Rank 0 prints one line ending in `check_ok=True|False`; the exit code is 0 iff every check held on every rank."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

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


def params():
    return {k: torch.from_numpy(v) for k, v in p.items()}


def run_trainer(group, check_sync):
    tr = SplatTrainer(params(), cfg(), device=DEV, ssim_weight=SSIM_W, group=group, **KW)
    torch.manual_seed(SEED)
    losses, counts, in_sync, empty_visible = [], [], True, None
    for step in range(1, STEPS + 1):
        cam, gt = view(step)
        loss = tr.step(cam, gt, step)
        losses.append(float(loss[0]))
        counts.append(tr.n)
        if step == EMPTY_STEP:
            empty_visible = tr.pipe.plan.visible
        if check_sync:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m, pp.adam_v))
    return tr, np.array(losses), np.array(counts), in_sync, empty_visible


def run_model():
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
    tr = SplatTrainer(params(), cfg(warmup_length=10 ** 6), device=DEV, group=dist.group.WORLD, **KW)

    def step_at(step):                               # full resolution, no turned-around camera
        v = (step - 1 + rank) % V
        tr.step(cams[v], gts_d[1][v], step)
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


dist.init_process_group("nccl", device_id=DEV)
tr, lt, ct, in_sync, empty_visible = run_trainer(dist.group.WORLD, check_sync=True)
model, lm, cm = run_model()
ok, dloss, exact = compare(model, tr, lm, lt, cm, ct)
refined = bool(cm[11] != cm[10] and cm[17] != cm[16])      # both densifications changed the Gaussian set
empty_ok = world < 2 or rank != 1 or empty_visible == 0
mc, overlap = bool(tr.exchange.multicast_ptr), tr.exchange.overlap
plain_exact = None
if world == 1:                                   # the same run without the exchange (group=None)
    tp, lp, cp, _, _ = run_trainer(None, check_sync=False)
    plain_exact = bool(np.array_equal(cp, ct) and torch.equal(tp.pipe.param_flat, tr.pipe.param_flat)
                       and torch.equal(tp.pipe.adam_m, tr.pipe.adam_m) and torch.equal(tp.pipe.adam_v, tr.pipe.adam_v))
    del tp
del tr, model
allocs, waits = steady_state()
steady_ok = allocs == 0 and waits == 10
flags = torch.tensor([int(ok), int(in_sync), int(refined), int(empty_ok), int(steady_ok)], device=DEV)
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
dl = torch.tensor([dloss], dtype=torch.float64, device=DEV)
dist.all_reduce(dl, op=dist.ReduceOp.MAX)
good = bool(flags.all())
if rank == 0:
    print(f"parallel trainer check world={world} multicast={mc} overlap={overlap}: counts {ct[0]}->{ct[-1]} "
          f"max|dloss|={float(dl[0]):.3g} matches_gaussian_model={bool(flags[0])} bit_identical={exact} "
          f"plain_trainer_bit_identical={plain_exact} replicas_in_sync={bool(flags[1])} refined={bool(flags[2])} "
          f"empty_view_ok={bool(flags[3])} steady_allocs={allocs} steady_waits={waits} check_ok={good}")
dist.destroy_process_group()
sys.exit(0 if good else 1)
