"""Training-step rate of the data-parallel trainer.SplatTrainer (fused NVLink exchange) against the data-parallel
model.GaussianModel (autograd, six Adam launches, one NCCL all-reduce of the six gradient tensors), one view per
rank, config C2 (1M Gaussians, 1920x1080, SH degree 3, the scene and camera of tools/bench_model_train.py; every rank
renders that camera against its own target image):

    python -m torch.distributed.run --nproc-per-node N tools/bench_trainer_parallel.py [--steps 30] [--warmup 5]

Per rank, CUDA events around `--steps` steps after `--warmup` steps, RefineConfig(warmup_length=10**6)
(densification statistics every step, no refinement in the timed loop); the reported step time is the maximum over
the ranks.  At world size 1 the plain SplatTrainer (no process group, created before it is initialised) is timed too,
on the same camera, so that the cost of the exchange machinery at one rank is visible.  Rank 0 prints one JSON line,
with the GPU's name and power limit."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--H", type=int, default=1080)
    a = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    from bench_model_train import model_scene
    from bench_trainer import gpu_info, timed
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.model import Camera, GaussianModel
    from opensplat_b200.trainer import SplatTrainer
    W, H = a.W, a.H
    p, c2w, (fx, fy, cx, cy) = model_scene(a.n, W, H)
    cam = Camera(W, H, fx, fy, cx, cy, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(rank)).to(dev)
    ssim_w, first = 0.2, 3001
    steady = RefineConfig(warmup_length=10 ** 6)
    out = {"workload": f"trainer_parallel_{a.n}_{W}x{H}_sh3", "gpu": gpu_info(), "world": world, "steps": a.steps,
           "warmup": a.warmup}

    def params():
        return {k: torch.from_numpy(v) for k, v in p.items()}

    def rate(ms):
        return {"iters_per_s": 1e3 / ms, "ms_per_iter": ms}

    def time_trainer(tr):
        for s in range(a.warmup):
            tr.step(cam, gt, first + s)
        return timed(lambda i: tr.step(cam, gt, first + a.warmup + i), a.steps)

    if world == 1:                  # before the process group exists: the single-process trainer
        tr = SplatTrainer(params(), steady, device=dev, ssim_weight=ssim_w)
        out["splat_trainer_plain"] = rate(time_trainer(tr))
        del tr
        torch.cuda.empty_cache()

    dist.init_process_group("nccl", device_id=dev)

    def max_over_ranks(ms):
        t = torch.tensor([ms], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])

    tr = SplatTrainer(params(), steady, device=dev, ssim_weight=ssim_w, group=dist.group.WORLD)
    out["splat_trainer_data_parallel"] = rate(max_over_ranks(time_trainer(tr)))
    out["multicast"], out["overlap"] = bool(tr.exchange.multicast_ptr), tr.exchange.overlap
    del tr
    torch.cuda.empty_cache()

    model = GaussianModel(params(), steady, device=dev, group=dist.group.WORLD)

    def model_step(step):
        model.optimizers_zero_grad()
        loss = model.main_loss(model.forward(cam, step), gt, ssim_w)
        loss.backward()
        model.optimizers_step()
        model.schedulers_step(step)
        model.after_train(step)
    for s in range(a.warmup):
        model_step(first + s)
    out["gaussian_model_data_parallel"] = rate(max_over_ranks(timed(lambda i: model_step(first + a.warmup + i),
                                                                    a.steps)))
    out["speedup_data_parallel"] = (out["splat_trainer_data_parallel"]["iters_per_s"] /
                                    out["gaussian_model_data_parallel"]["iters_per_s"])
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
