"""Training-step rate of trainer.SplatTrainer against model.GaussianModel's loop (opensplat.cpp:151-170) on one GPU,
config C2 (1M Gaussians, 1920x1080, SH degree 3, the scene and camera of tools/bench_model_train.py), in one process:

  - iterations per second of each, CUDA events around `--steps` steps after `--warmup` steps, with
    RefineConfig(warmup_length=10**6): densification statistics every step, no refinement in the timed loop;
  - one refinement of each at 1M Gaussians (a step that splits, duplicates and culls), timed as the whole step that
    contains it, next to the steady step time.

Prints one JSON line, with the GPU's name and power limit.

    python tools/bench_trainer.py [--n 1000000] [--steps 30] [--warmup 5]

With --views-per-step 1,2,4,8 it times SplatTrainer(views_per_step=B) instead, for every B of the list, in the same
process and in alternating rounds (--rounds, each round times every B once, so B = 1 and B = 4 alternate): ms per
step, views per second and the trainer's peak device memory, medians over the rounds.  The B views of a step are
the scene's camera turned about the scene centre by small angles (0.02 rad apart, around the vertical axis), so that
every view sees a similar footprint and a step's cost stays comparable across B."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def timed(fn, steps):
    """ms per call of fn(i) over `steps` calls, CUDA events around the whole loop."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def turned_views(c2w, centre, count, step_rad=0.02):
    """`count` camera poses: c2w turned about the vertical axis through `centre` by 0, +a, -a, +2a, ... radians."""
    import numpy as np
    out = []
    for b in range(count):
        ang = step_rad * ((b + 1) // 2) * (1 if b % 2 else -1)
        rot = np.eye(4, dtype=np.float32)
        rot[:3, :3] = [[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]
        shift, back = np.eye(4, dtype=np.float32), np.eye(4, dtype=np.float32)
        shift[:3, 3], back[:3, 3] = -centre, centre
        out.append((back @ rot @ shift @ c2w).astype(np.float32))
    return out


def bench_views(a, dev, out):
    """--views-per-step: SplatTrainer at each B, alternating rounds in one process."""
    import numpy as np
    from bench_model_train import model_scene
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.model import Camera
    from opensplat_b200.trainer import SplatTrainer
    W, H = a.W, a.H
    bs = [int(x) for x in a.views_per_step.split(",")]
    p, c2w, (fx, fy, cx, cy) = model_scene(a.n, W, H)
    poses = turned_views(c2w[0], p["means"].astype(np.float64).mean(0).astype(np.float32), max(bs))
    cams = [Camera(W, H, fx, fy, cx, cy, c) for c in poses]
    gts = torch.rand((max(bs), H, W, 3), generator=torch.Generator().manual_seed(0)).to(dev)
    first, trainers, peak = 3001, {}, {}
    for B in bs:   # build and warm up every trainer first; the peak is each trainer's own
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=dev, ssim_weight=0.2, views_per_step=B)
        for s in range(a.warmup):
            tr.step(cams[:B] if B > 1 else cams[0], gts[:B] if B > 1 else gts[0], first + s)
        torch.cuda.synchronize()
        peak[B] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        trainers[B] = tr
    ms = {B: [] for B in bs}
    step = first + a.warmup
    for _ in range(a.rounds):
        for B in bs:
            tr = trainers[B]
            c, g = (cams[:B], gts[:B]) if B > 1 else (cams[0], gts[0])
            ms[B].append(timed(lambda i: tr.step(c, g, step + i), a.steps))
        step += a.steps
    res = {}
    for B in bs:
        m = float(np.median(ms[B]))
        res[str(B)] = {"ms_per_step": m, "views_per_s": 1e3 * B / m, "steps_per_s": 1e3 / m,
                       "peak_mem_mb": peak[B], "ms_per_step_rounds": ms[B]}
    out["views_per_step"] = res
    out["workload"] = f"trainer_views_{a.n}_{W}x{H}_sh3"
    out["rounds"] = a.rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--H", type=int, default=1080)
    ap.add_argument("--views-per-step", default=None, help="comma-separated B values, e.g. 1,2,4,8")
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    dev = "cuda:0"
    if a.views_per_step:
        out = {"gpu": gpu_info(), "steps": a.steps, "warmup": a.warmup}
        bench_views(a, dev, out)
        print(json.dumps(out))
        return
    from bench_model_train import model_scene
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.model import Camera, GaussianModel
    from opensplat_b200.trainer import SplatTrainer
    W, H = a.W, a.H
    p, c2w, (fx, fy, cx, cy) = model_scene(a.n, W, H)
    cam = Camera(W, H, fx, fy, cx, cy, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(dev)
    ssim_w, first = 0.2, 3001
    out = {"workload": f"trainer_{a.n}_{W}x{H}_sh3", "gpu": gpu_info(), "steps": a.steps, "warmup": a.warmup}
    steady = RefineConfig(warmup_length=10 ** 6)
    # a refinement at step 200 (200 % refine_every == 0, past warmup, inside the densify window) after statistics
    # from steps 190..199; the gradient threshold is low enough that many Gaussians split, low opacities are culled
    refine = RefineConfig(refine_every=100, warmup_length=0, densify_grad_thresh=2e-6)

    def params():
        return {k: torch.from_numpy(v) for k, v in p.items()}

    def model_step(model, step):
        model.optimizers_zero_grad()
        loss = model.main_loss(model.forward(cam, step), gt, ssim_w)
        loss.backward()
        model.optimizers_step()
        model.schedulers_step(step)
        return model.after_train(step)

    # ---- GaussianModel ----
    model = GaussianModel(params(), steady, device=dev)
    for s in range(a.warmup):
        model_step(model, first + s)
    ms = timed(lambda i: model_step(model, first + a.warmup + i), a.steps)
    out["gaussian_model"] = {"iters_per_s": 1e3 / ms, "ms_per_iter": ms}
    del model
    model = GaussianModel(params(), refine, device=dev)
    for s in range(190, 200):
        model_step(model, s)
    n0 = model.means.shape[0]
    ms_r = timed(lambda i: model_step(model, 200), 1)
    info = model.densifier.last_info
    out["gaussian_model"]["refine"] = {"step_ms": ms_r, "n_before": n0, "n_after": int(model.means.shape[0]),
                                       "n_splits": info.get("n_splits"), "culled": info.get("culled")}
    del model
    torch.cuda.empty_cache()

    # ---- SplatTrainer ----
    tr = SplatTrainer(params(), steady, device=dev, ssim_weight=ssim_w)
    for s in range(a.warmup):
        tr.step(cam, gt, first + s)
    ms_t = timed(lambda i: tr.step(cam, gt, first + a.warmup + i), a.steps)
    out["splat_trainer"] = {"iters_per_s": 1e3 / ms_t, "ms_per_iter": ms_t}
    del tr
    tr = SplatTrainer(params(), refine, device=dev, ssim_weight=ssim_w)
    for s in range(190, 200):
        tr.step(cam, gt, s)
    n0 = tr.n
    losses = []
    ms_r = timed(lambda i: losses.append(tr.step(cam, gt, 200)), 1)
    info = tr.last_info
    out["splat_trainer"]["refine"] = {"step_ms": ms_r, "n_before": n0, "n_after": tr.n,
                                      "n_splits": info.get("n_splits"), "culled": info.get("culled")}
    out["speedup_iters_per_s"] = out["splat_trainer"]["iters_per_s"] / out["gaussian_model"]["iters_per_s"]
    out["final_loss_trainer"] = float(losses[-1][0])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
