"""torchrun --nproc-per-node N tools/check_parallel_absgrad.py : the data-parallel trainer.SplatTrainer with AbsGS's
absolute screen-space gradients in the densification statistics (DESIGN D25).

Every rank trains its own view sequence (rank r, step s -> view (s - 1 + r) % V) of the training problem of
tests/test_gpu_trainer.py with SplatTrainer(..., group=WORLD, cfg=RefineConfig(absgrad=True)) through densifications
and an alpha reset.  It checks that the replicas stay bit-identical (parameters and Adam moments) after every step,
and at world size 1 that the run is bit-identical to the same run without a group.  Rank 0 prints one line ending in
`check_ok=True|False`; the exit code is 0 iff every check held on every rank."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
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


def run(group):
    torch.manual_seed(3)    # the refinement's splits draw from the default generator
    tr = SplatTrainer({k: torch.from_numpy(x) for k, x in p.items()},
                      tg.refine_config(refine_every=6, warmup_length=5, reset_alpha_every=4, densify_grad_thresh=8e-5,
                                       absgrad=True), device=DEV, group=group)
    in_sync, refined = True, 0
    for step in range(1, STEPS + 1):
        v = (step - 1 + rank) % V
        tr.step(cams[v], gts_d[v], step)
        refined += int(tr.last_info.get("added", 0) > 0)
        if group is not None:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m,
                                                                                   pp.adam_v))
    return tr, refined, in_sync


dist.init_process_group("nccl", device_id=DEV)
tr, refined, in_sync = run(dist.group.WORLD)
plain_exact = None
if world == 1:
    tp, _, _ = run(None)
    plain_exact = bool(tp.n == tr.n and torch.equal(tp.pipe.param_flat, tr.pipe.param_flat)
                       and torch.equal(tp.pipe.adam_m, tr.pipe.adam_m) and torch.equal(tp.pipe.adam_v, tr.pipe.adam_v))
flags = torch.tensor([int(in_sync), int(refined > 0), int(plain_exact is not False)], device=DEV)
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
good = bool(flags.all())
if rank == 0:
    print(f"parallel absgrad check world={world}: n={tr.n} densifications={refined} replicas_in_sync={bool(flags[0])} "
          f"plain_trainer_bit_identical={plain_exact} check_ok={good}")
dist.destroy_process_group()
sys.exit(0 if good else 1)
