"""Cost of Mip-Splatting's 3-D smoothing filter (DESIGN D24): gsb_filter3d_compute at 1M and 5M Gaussians x 100 and
300 cameras; the activated projection forward and backward without and with the filter
(gsb_project_forward_activated / gsb_project_backward_activated against the _filter3d entry points), alternating the
arms within one run, at C2 (1M Gaussians, 1920x1080) and C5 (5M, 2560x1440); then the C2 SplatTrainer step without
and with Filter3DConfig, alternating rounds.  Prints the medians with the card's name and power limit.
usage: python tools/bench_filter3d.py [--reps N] [--steps K] [--rounds R] [--no-trainer]"""
import argparse
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_depth import card  # noqa: E402
from bench_model_train import model_scene  # noqa: E402
from bench_pose import SIZES, _events  # noqa: E402
from bench_trainer import timed  # noqa: E402
from opensplat_b200 import capi, ops  # noqa: E402
from opensplat_b200.filter3d import camera_table, compute_filter3d  # noqa: E402
from opensplat_b200.model import Camera, camera_setup  # noqa: E402

DEV = "cuda:0"


def orbit(k, W, H, intr, radius):
    """k cameras on a circle around the scene's centre, looking at it, with the given intrinsics."""
    cams = []
    for j in range(k):
        th = 2 * math.pi * j / k
        eye = np.array([radius * math.sin(th), 0.3 * math.sin(5 * th), -radius * math.cos(th)])
        fwd = -eye / np.linalg.norm(eye)
        right = np.cross(fwd, [0.0, 1.0, 0.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        c2w = np.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, eye
        cams.append(Camera(W, H, *intr, c2w))
    return cams


def bench_compute(reps):
    for n in (1_000_000, 5_000_000):
        p, _, intr = model_scene(n, 1920, 1080)
        means = torch.from_numpy(np.ascontiguousarray(p["means"])).to(DEV)
        for k in (100, 300):
            table = camera_table(orbit(k, 1920, 1080, intr, 8.0), DEV)
            out = torch.empty(n, device=DEV)
            for _ in range(3):
                compute_filter3d(means, table, out=out)
            torch.cuda.synchronize()
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                compute_filter3d(means, table, out=out)
                e1.record()
                ts.append((e0, e1))
            torch.cuda.synchronize()
            ms = float(np.median([a.elapsed_time(b) for a, b in ts]))
            pairs = n * k
            print(f"gsb_filter3d_compute n={n} cameras={k}: {ms:.4f} ms  ({pairs / ms / 1e6:.2f} G pairs/s, "
                  f"seen {(out > 0).float().mean().item():.3f})", flush=True)


def bench_projection(name, reps):
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
    f3 = compute_filter3d(t["means"], orbit(100, W, H, intr, 8.0))
    head = lambda: (n, P(t["means"]), P(t["scales"]), 1.0, P(t["quats"]), P(ol))
    tail = lambda: (P(view), P(pm), fx, fy, cx, cy, H_, W_, tb[0], tb[1], 0.01, *[P(o) for o in out])
    capi.check(L.gsb_project_forward_activated(*head(), *tail(), s))
    bwd = lambda opac: (P(view), P(pm), fx, fy, H_, W_, P(out[3]), P(out[4]), P(v_xy), None, P(v_conic), P(v_opac),
                        *[P(x) for x in grads])
    bh = lambda opac: (n, P(t["means"]), P(t["scales"]), 1.0, P(t["quats"]), P(opac))
    arms = {"fwd_plain": lambda: L.gsb_project_forward_activated(*head(), *tail(), s),
            "fwd_filter3d": lambda: L.gsb_project_forward_activated_filter3d(*head(), P(f3), *tail(), 0, s),
            "bwd_plain": lambda: L.gsb_project_backward_activated(*bh(out[6]), *bwd(out[6]), s),
            "bwd_filter3d": lambda: L.gsb_project_backward_activated_filter3d(*bh(ol), P(f3), *bwd(ol), 0, 0, 0, None,
                                                                              s)}
    times = {k: [] for k in arms}
    for _ in range(3):
        for fn in arms.values():
            capi.check(fn())
    torch.cuda.synchronize()
    for r in range(reps):
        for k, fn in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):
            _events(fn, reps, times, k)
    torch.cuda.synchronize()
    med = {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in times.items()}
    print(f"{name}: n={n} {W_}x{H_} visible={int((out[3] > 0).sum())} reps={reps}  "
          + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items())
          + f"  fwd {100 * (med['fwd_filter3d'] / med['fwd_plain'] - 1):+.1f}%"
          + f"  bwd {100 * (med['bwd_filter3d'] / med['bwd_plain'] - 1):+.1f}%", flush=True)


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.filter3d import Filter3DConfig
    from opensplat_b200.trainer import SplatTrainer
    n, W, H = SIZES["C2"]
    p, c2w, intr = model_scene(n, W, H)
    cam = Camera(W, H, *intr, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    first, trainers = 3001, {}
    for on in (False, True):
        f3 = Filter3DConfig(cameras=orbit(100, W, H, intr, 8.0)) if on else None
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2, filter3d=f3)
        for i in range(warmup):
            tr.step(cam, gt, first + i)
        trainers[on] = tr
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    step = first + warmup
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            tr = trainers[on]
            ms[on].append(timed(lambda i: tr.step(cam, gt, step + i), steps))
        step += steps
    for on in (False, True):
        m = float(np.median(ms[on]))
        print(f"C2 SplatTrainer filter3d={'Filter3DConfig(100 cameras)' if on else None}: {m:.3f} ms/step "
              f"({1e3 / m:.1f} steps/s), rounds " + " ".join(f"{x:.3f}" for x in ms[on]), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--no-trainer", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_filter3d: no CUDA device")
    print("card:", card(), flush=True)
    bench_compute(a.reps)
    torch.cuda.empty_cache()
    for name in SIZES:
        bench_projection(name, a.reps)
        torch.cuda.empty_cache()
    if not a.no_trainer:
        bench_trainer(a.steps, a.rounds)
