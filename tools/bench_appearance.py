"""Cost of the per-image appearance grids (DESIGN D21) on one GPU, in one process:

  - the slice forward and backward (gsb_bilagrid_slice_forward / _backward) at 1920x1080: CUDA events around
    `--launches` launches of each after a warm-up, against their byte floors (forward: rgb in, out back, 24 B per
    pixel; backward: rgb and v_out in, v_rgb back, 36 B per pixel; the 96 KB grid is noise at this size);
  - the per-step grid work at N = 100, 300 and 1000 images: gsb_bilagrid_tv (writes the gradient) plus the grid Adam
    step (gsb_adam_step over all N grids; 16 B read + 12 B written per float), against those 40 B per float;
  - a C2 training step (1M Gaussians, 1920x1080, SH degree 3, the scene and camera of tools/bench_model_train.py) of
    SplatTrainer without and with AppearanceConfig(num_images=300), alternating rounds of `--steps` steps.

Prints one JSON line, with the GPU's name and power limit read in the same run.

    python tools/bench_appearance.py [--steps 30] [--rounds 5] [--launches 200]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_trainer import gpu_info, timed  # noqa: E402
from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.appearance import AppearanceConfig, identity_grids  # noqa: E402

DEV = "cuda:0"


def slice_costs(launches, W=1920, H=1080):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    g = torch.Generator(device=DEV).manual_seed(0)
    grid = identity_grids(1, DEV)[0] + torch.randn(identity_grids(1, DEV)[0].shape, device=DEV, generator=g) * 0.05
    rgb = torch.rand((H, W, 3), device=DEV, generator=g)
    v = torch.randn((H, W, 3), device=DEV, generator=g)
    out, v_rgb, v_grid = torch.empty_like(rgb), torch.empty_like(rgb), torch.zeros_like(grid)
    ws = torch.empty(L.gsb_bilagrid_workspace_bytes(H, W), dtype=torch.uint8, device=DEV)

    def fwd(i):
        capi.check(L.gsb_bilagrid_slice_forward(H, W, P(grid), P(rgb), P(out), s))

    def bwd(i):
        capi.check(L.gsb_bilagrid_slice_backward(H, W, P(grid), P(rgb), P(v), 1.0, P(v_rgb), P(v_grid), P(ws),
                                                 ws.numel(), s))
    res = {}
    for name, fn, nbytes in (("forward", fwd, 24), ("backward", bwd, 36)):
        for i in range(20):
            fn(i)
        ms = timed(fn, launches)
        floor_us = nbytes * H * W / 3.35e12 * 1e6
        res[name] = {"us": 1e3 * ms, "bytes_per_pixel_floor": nbytes, "floor_us_at_3.35TBps": floor_us,
                     "GBps_at_floor_bytes": nbytes * H * W / (ms * 1e-3) / 1e9}
    res["workspace_bytes"] = ws.numel()
    return res


def grid_step_costs(n, launches):
    from opensplat_b200.appearance import Appearance
    ap = Appearance(AppearanceConfig(num_images=n), torch.device(DEV))

    def step(i):
        ap.tv()
        ap.adam_step(i + 1)
    for i in range(10):
        step(i)
    ms = timed(step, launches)
    floats = ap.grids.numel()
    return {"us": 1e3 * ms, "floats": floats, "floor_us_at_3.35TBps": 40 * floats / 3.35e12 * 1e6}


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
    apps = {"off": None, "on_300": AppearanceConfig(num_images=300)}
    trainers = {}
    for k, app in apps.items():
        tr = SplatTrainer({k2: torch.from_numpy(v) for k2, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2, appearance=app)
        kw = {} if app is None else {"image": 7}
        for s in range(a.warmup):
            tr.step(cam, gt, first + s, **kw)
        trainers[k] = (tr, kw)
    ms = {k: [] for k in apps}
    step = first + a.warmup
    for _ in range(a.rounds):
        for k, (tr, kw) in trainers.items():
            ms[k].append(timed(lambda i: tr.step(cam, gt, step + i, **kw), a.steps))
        step += a.steps
    out = {k: {"ms_per_step": float(np.median(v)), "ms_rounds": v} for k, v in ms.items()}
    out["overhead_ms"] = out["on_300"]["ms_per_step"] - out["off"]["ms_per_step"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    out = {"gpu": gpu_info()}
    out["slice_1080p"] = slice_costs(a.launches)
    out["tv_plus_adam"] = {str(n): grid_step_costs(n, a.launches) for n in (100, 300, 1000)}
    out["trainer_C2"] = trainer_steps(a)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
