"""Cost of the pose corrections (DESIGN D22): times the activated projection backward without and with the camera
gradient (gsb_project_backward_activated against gsb_project_backward_activated_camgrad), alternating the arms within
one run, at C2 (1M Gaussians, 1920x1080) and C5 (5M, 2560x1440); the reduce (gsb_project_camera_grad_reduce) of
those sizes' partial rows; then the C2 SplatTrainer step without and with PoseConfig(num_images=300), alternating
rounds.  Prints the medians with the card's name and power limit.
usage: python tools/bench_pose.py [--reps N] [--steps K] [--rounds R] [--no-trainer]"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_depth import card  # noqa: E402
from bench_model_train import model_scene  # noqa: E402
from bench_trainer import timed  # noqa: E402
from opensplat_b200 import capi, ops  # noqa: E402
from opensplat_b200.model import Camera, camera_setup  # noqa: E402

DEV = "cuda:0"
SIZES = {"C2": (1_000_000, 1920, 1080), "C5": (5_000_000, 2560, 1440)}


def _events(fn, reps, times, key):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    capi.check(fn())
    e1.record()
    times[key].append((e0, e1))


def bench_kernels(name, reps):
    n, W, H = SIZES[name]
    p, c2w, intr = model_scene(n, W, H)
    H_, W_, (fx, fy, cx, cy), view, proj, _ = camera_setup(Camera(W, H, *intr, c2w[0]), 1)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in p.items()}
    view, pm = view.to(DEV).contiguous(), (proj @ view).to(DEV).contiguous()
    tb = ops.tile_bounds(W_, H_)
    i32 = torch.int32
    out = [torch.empty((n, 6), device=DEV), torch.empty((n, 2), device=DEV), torch.empty(n, device=DEV),
           torch.empty(n, dtype=i32, device=DEV), torch.empty((n, 3), device=DEV), torch.empty(n, dtype=i32, device=DEV),
           torch.empty(n, device=DEV)]
    g = torch.Generator(device=DEV).manual_seed(0)
    v_xy, v_conic, v_opac = (torch.randn(s, device=DEV, generator=g) for s in ((n, 2), (n, 3), (n,)))
    grads = [torch.empty((n, 3), device=DEV), torch.empty((n, 3), device=DEV), torch.empty((n, 4), device=DEV),
             torch.empty(n, device=DEV)]
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    ol = t["opacities"].reshape(n)
    part = torch.empty(L.gsb_project_camera_partials_floats(n), device=DEV)
    nblocks = part.numel() // capi.CAMGRAD_TERMS
    cg = torch.empty((2, 4, 4), device=DEV)
    capi.check(L.gsb_project_forward_activated(n, P(t["means"]), P(t["scales"]), 1.0, P(t["quats"]), P(ol), P(view),
                                               P(pm), fx, fy, cx, cy, H_, W_, tb[0], tb[1], 0.01,
                                               *[P(o) for o in out], s))
    args = lambda: (n, P(t["means"]), P(t["scales"]), 1.0, P(t["quats"]), P(out[6]), P(view), P(pm), fx, fy, H_, W_,
                    P(out[3]), P(out[4]), P(v_xy), None, P(v_conic), P(v_opac), *[P(x) for x in grads])
    arms = {"bwd_plain": lambda: L.gsb_project_backward_activated(*args(), s),
            "bwd_camgrad": lambda: L.gsb_project_backward_activated_camgrad(*args(), 0, 0, P(part), s),
            "reduce": lambda: L.gsb_project_camera_grad_reduce(nblocks, P(part), P(cg[0]), P(cg[1]), s)}
    times = {k: [] for k in arms}
    for _ in range(3):
        for f in arms.values():
            capi.check(f())
    torch.cuda.synchronize()
    for r in range(reps):
        for k, f in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):
            _events(f, reps, times, k)
    torch.cuda.synchronize()
    med = {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in times.items()}
    visible = int((out[3] > 0).sum())
    print(f"{name}: n={n} {W_}x{H_} visible={visible} blocks={nblocks} reps={reps}  "
          + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items())
          + f"  camgrad {100 * (med['bwd_camgrad'] / med['bwd_plain'] - 1):+.1f}%", flush=True)


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.pose import PoseConfig
    from opensplat_b200.trainer import SplatTrainer
    n, W, H = SIZES["C2"]
    p, c2w, intr = model_scene(n, W, H)
    cam = Camera(W, H, *intr, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    first, trainers = 3001, {}
    for on in (False, True):
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2, pose=PoseConfig(num_images=300) if on else None)
        kw = {"image": 7} if on else {}
        for i in range(warmup):
            tr.step(cam, gt, first + i, **kw)
        trainers[on] = (tr, kw)
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    step = first + warmup
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            tr, kw = trainers[on]
            ms[on].append(timed(lambda i: tr.step(cam, gt, step + i, **kw), steps))
        step += steps
    for on in (False, True):
        m = float(np.median(ms[on]))
        print(f"C2 SplatTrainer pose={'PoseConfig(num_images=300)' if on else None}: {m:.3f} ms/step "
              f"({1e3 / m:.1f} steps/s), rounds " + " ".join(f"{x:.3f}" for x in ms[on]), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--no-trainer", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pose: no CUDA device")
    print("card:", card(), flush=True)
    for name in SIZES:
        bench_kernels(name, a.reps)
        torch.cuda.empty_cache()
    if not a.no_trainer:
        bench_trainer(a.steps, a.rounds)
