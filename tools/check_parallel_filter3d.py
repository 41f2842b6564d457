"""torchrun --nproc-per-node N tools/check_parallel_filter3d.py : the data-parallel trainer.SplatTrainer with
Mip-Splatting's 3-D smoothing filter (DESIGN D24).

Every rank trains its own view sequence (rank r, step s -> view (s - 1 + r) % V) of the training problem of
tests/test_gpu_trainer.py with SplatTrainer(..., group=WORLD, filter3d=Filter3DConfig(cameras)), through
densifications and an alpha reset.  Every rank is given the same cameras and computes the same filter, so it checks
that the replicas stay bit-identical (parameters, Adam moments and the filter) after every step, and at world size 1
that the run is bit-identical to the same run without a group.  Rank 0 prints one line ending in
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
from opensplat_b200.filter3d import Filter3DConfig  # noqa: E402
from opensplat_b200.trainer import SplatTrainer  # noqa: E402

STEPS = 22
p, c2w, gts, intr, H, W = tg.make_problem()
cams = tg._cams(c2w, H, W, intr)
V = len(cams)
gts_d = torch.from_numpy(gts).to(DEV)


def run(group):
    torch.manual_seed(3)    # the refinement's splits draw from the default generator
    tr = SplatTrainer({k: torch.from_numpy(x) for k, x in p.items()},
                      tg.refine_config(refine_every=6, warmup_length=5, reset_alpha_every=4), device=DEV,
                      group=group, filter3d=Filter3DConfig(cameras=cams))
    in_sync, resets = True, 0
    for step in range(1, STEPS + 1):
        v = (step - 1 + rank) % V
        tr.step(cams[v], gts_d[v], step)
        resets += int(bool(tr.last_info.get("alpha_reset")))
        if group is not None:
            pp = tr.pipe
            in_sync = in_sync and all(parallel.replicas_in_sync(t, world) for t in (pp.param_flat, pp.adam_m,
                                                                                   pp.adam_v, tr.f3d))
    return tr, resets, in_sync


dist.init_process_group("nccl", device_id=DEV)
tr, resets, in_sync = run(dist.group.WORLD)
plain_exact = None
if world == 1:
    tp, _, _ = run(None)
    plain_exact = bool(torch.equal(tp.pipe.param_flat, tr.pipe.param_flat) and torch.equal(tp.pipe.adam_m, tr.pipe.adam_m)
                       and torch.equal(tp.pipe.adam_v, tr.pipe.adam_v) and torch.equal(tp.f3d, tr.f3d))
flags = torch.tensor([int(in_sync), int(resets > 0), int(plain_exact is not False)], device=DEV)
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
good = bool(flags.all())
if rank == 0:
    print(f"parallel filter3d check world={world}: n={tr.n} alpha_resets={resets} replicas_in_sync={bool(flags[0])} "
          f"plain_trainer_bit_identical={plain_exact} check_ok={good}")
dist.destroy_process_group()
sys.exit(0 if good else 1)
