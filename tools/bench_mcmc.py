"""Cost of the MCMC strategy (DESIGN D20) on one GPU, in one process:

  - the two per-step kernels (gsb_mcmc_regularize, gsb_mcmc_add_noise) at 1M (C2) and 5M (C5) Gaussians: CUDA events
    around `--launches` launches of each after a warm-up, with the bytes each moves and the rate that gives;
  - one refinement at 1M -> 1.05M (10 % of the Gaussians dead: relocation, then 5 % growth), MCMCRefiner.finish_step
    timed from the host up to a device synchronise (its one read-back included), the median over `--refines` fresh
    copies;
  - a C2 training step (1M Gaussians, 1920x1080, SH degree 3, the scene and camera of tools/bench_model_train.py) of
    SplatTrainer with the default strategy (RefineConfig, no refinement in the timed window) and with MCMCConfig (no
    refinement in the window either: regularisers and noise every step), alternating rounds of `--steps` steps.

Prints one JSON line, with the GPU's name and power limit read in the same run.

    python tools/bench_mcmc.py [--steps 30] [--rounds 5] [--launches 200] [--refines 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_trainer import gpu_info, timed  # noqa: E402
from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.mcmc import MCMCConfig, MCMCRefiner  # noqa: E402
from opensplat_b200.pipeline import SplatPipeline  # noqa: E402

DEV = "cuda:0"


def random_pipe(n, dead_frac=0.1, seed=0):
    """A SplatPipeline holding n random Gaussians (SH degree 3) with Adam moments; dead_frac of them faint."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    pp = SplatPipeline(n, 16, 16, sh_degree=3, device=DEV)
    pp.param_flat.normal_(generator=g)
    pp.p["scales"].uniform_(-6, -3, generator=g)
    pp.p["opacities"].uniform_(-3, 3, generator=g)
    pp.p["opacities"][torch.rand(n, 1, device=DEV, generator=g) < dead_frac] = -8.0
    pp.adam_m = torch.randn(pp.numel, device=DEV, generator=g) * 1e-3
    pp.adam_v = torch.rand(pp.numel, device=DEV, generator=g) * 1e-6
    return pp


def kernel_costs(n, launches):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    pp = random_pipe(n)
    p, g = pp.p, pp.g
    pp.grad_flat.zero_()

    def reg(i):
        capi.check(L.gsb_mcmc_regularize(n, P(p["opacities"]), P(p["scales"]), 1e-8, 1e-8, P(g["opacities"]),
                                         P(g["scales"]), s))

    def noise(i):
        capi.check(L.gsb_mcmc_add_noise(n, P(p["opacities"]), P(p["scales"]), P(p["quats"]), 0, 0, i + 1, 1e-9,
                                        P(p["means"]), s))
    out = {}
    # bytes: regularize reads logit + 3 log-scales and reads/writes their 4 gradients (48 B); noise reads logit,
    # 3 log-scales, 4 quaternion floats and reads/writes 3 means (56 B)
    for name, fn, nbytes in (("regularize", reg, 48), ("noise", noise, 56)):
        for i in range(20):
            fn(i)
        ms = timed(fn, launches)
        out[name] = {"us": 1e3 * ms, "bytes_per_gaussian": nbytes, "GBps": nbytes * n / (ms * 1e-3) / 1e9}
    out["per_step_us"] = out["regularize"]["us"] + out["noise"]["us"]
    del pp
    torch.cuda.empty_cache()
    return out


def refine_cost(n, repeats):
    cfg = MCMCConfig(refine_start=0, refine_every=1, cap_max=10 * n, noise_lr=0.0)
    times, info = [], None
    for r in range(repeats + 1):
        pp = random_pipe(n, seed=r)
        refiner = MCMCRefiner(cfg)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = refiner.finish_step(1000, pp, 1e-4)
        torch.cuda.synchronize()
        if r:                      # the first one loads the module and warms the allocator
            times.append(1e3 * (time.perf_counter() - t0))
        info = res[3]
        del pp, res
        torch.cuda.empty_cache()
    return {"ms_median": float(np.median(times)), "ms": times, "n_before": n, "n_after": info["n"],
            "relocated": info["relocated"], "added": info["added"]}


def trainer_steps(a):
    from bench_model_train import model_scene
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.model import Camera
    from opensplat_b200.trainer import SplatTrainer
    W, H = 1920, 1080
    p, c2w, (fx, fy, cx, cy) = model_scene(1_000_000, W, H)
    cam = Camera(W, H, fx, fy, cx, cy, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    first = 3001
    cfgs = {"default": RefineConfig(warmup_length=10 ** 6), "mcmc": MCMCConfig(refine_start=10 ** 6)}
    trainers = {}
    for k, cfg in cfgs.items():
        tr = SplatTrainer({k2: torch.from_numpy(v) for k2, v in p.items()}, cfg, device=DEV, ssim_weight=0.2)
        for s in range(a.warmup):
            tr.step(cam, gt, first + s)
        trainers[k] = tr
    ms = {k: [] for k in cfgs}
    step = first + a.warmup
    for _ in range(a.rounds):
        for k, tr in trainers.items():
            ms[k].append(timed(lambda i: tr.step(cam, gt, step + i), a.steps))
        step += a.steps
    out = {k: {"ms_per_step": float(np.median(v)), "ms_rounds": v} for k, v in ms.items()}
    out["overhead_pct"] = 100.0 * (out["mcmc"]["ms_per_step"] / out["default"]["ms_per_step"] - 1.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--refines", type=int, default=5)
    a = ap.parse_args()
    out = {"gpu": gpu_info()}
    out["kernels"] = {"C2_1M": kernel_costs(1_000_000, a.launches), "C5_5M": kernel_costs(5_000_000, a.launches)}
    out["refine_1M"] = refine_cost(1_000_000, a.refines)
    out["trainer_C2"] = trainer_steps(a)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
