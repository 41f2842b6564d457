"""torchrun --nproc-per-node N tools/check_parallel_fisheye.py : the data-parallel trainer.SplatTrainer over fisheye
and pinhole views (DESIGN D27).

Every rank trains its own view sequence (rank r, step s -> view (s - 1 + r) % V) of the training problem of
tests/test_gpu_trainer.py, whose cameras alternate between the pinhole and an OpenCV fisheye camera of the same pose
and intrinsics, with SplatTrainer(..., group=WORLD), through two densifications.  It checks that the replicas stay
bit-identical (parameters and Adam moments) after every step, that the losses are finite, and at world size 1 that
the run is bit-identical to the same run without a group (parameters and moments; the returned losses are sums through
per-tile float atomics, whose order varies from run to run, and are compared to 1e-5 relative).  Rank 0 prints one
line ending in `check_ok=True|False`; the exit code is 0 iff every check held on every rank."""
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
from opensplat_b200 import parallel  # noqa: E402
from opensplat_b200.trainer import SplatTrainer  # noqa: E402

STEPS = 22
p, c2w, gts, intr, H, W = tg.make_problem()
cams = tg._cams(c2w, H, W, intr)
V = len(cams)
gts_d = torch.from_numpy(gts).to(DEV)
K = (0.05, -0.02, 0.004, -0.0005)
cams = [c.replace(model="fisheye", k1=K[0], k2=K[1], k3=K[2], k4=K[3]) if v % 2 == 0 else c
        for v, c in enumerate(cams)]


def run(group):
    torch.manual_seed(3)    # the refinement's splits draw from the default generator
    tr = SplatTrainer({k: torch.from_numpy(x) for k, x in p.items()},
                      tg.refine_config(refine_every=6, warmup_length=5, reset_alpha_every=4), device=DEV,
                      group=group)
    in_sync, losses = True, []
    for step in range(1, STEPS + 1):
        v = (step - 1 + rank) % V
        loss = tr.step(cams[v], gts_d[v], step)
        losses.append(float(loss[0]))
        if group is not None:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m,
                                                                                   pp.adam_v))
    return tr, np.array(losses), in_sync


dist.init_process_group("nccl", device_id=DEV)
tr, losses, in_sync = run(dist.group.WORLD)
counts = tr.n
finite = bool(np.isfinite(losses).all() and (losses > 0).all())
plain_exact = None
if world == 1:
    tp, lp, _ = run(None)
    plain_exact = bool(np.allclose(lp, losses, rtol=1e-5, atol=0) and torch.equal(tp.pipe.param_flat, tr.pipe.param_flat)
                       and torch.equal(tp.pipe.adam_m, tr.pipe.adam_m) and torch.equal(tp.pipe.adam_v, tr.pipe.adam_v))
flags = torch.tensor([int(in_sync), int(finite), int(plain_exact is not False)], device=DEV)
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
good = bool(flags.all())
if rank == 0:
    print(f"parallel fisheye check world={world}: n={counts} loss {losses[0]:.4g}->{losses[-1]:.4g} "
          f"replicas_in_sync={bool(flags[0])} losses_finite={bool(flags[1])} plain_trainer_bit_identical={plain_exact} "
          f"check_ok={good}")
dist.destroy_process_group()
sys.exit(0 if good else 1)
