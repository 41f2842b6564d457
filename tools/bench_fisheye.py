"""Cost of fisheye cameras (DESIGN D27): the projection forward and backward (plain, anti-aliased, with the camera
gradient), pinhole (gsb_project_*_activated[_aa|_camgrad]) against fisheye (gsb_project_*_fisheye), at C2 (1M
Gaussians) and C5 (5M), 1920x1080, alternating within one run, each timed over launches queued behind a device-side
sleep; and the C2 SplatTrainer step with a pinhole against a fisheye camera, medians of alternated rounds, as CUDA
events.  Prints the medians with the card's name and power limit.
usage: python tools/bench_fisheye.py [--reps N] [--steps K] [--rounds R]"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_depth import card  # noqa: E402
from bench_mask import _time_arms  # noqa: E402
from bench_model_train import model_scene  # noqa: E402
from bench_trainer import timed  # noqa: E402
from opensplat_b200 import capi, ops  # noqa: E402
from opensplat_b200.model import Camera, camera_setup, fisheye_theta_limit  # noqa: E402

DEV = "cuda:0"
W, H = 1920, 1080
K = (0.05, -0.02, 0.004, -0.0005)


def bench_projection(n, reps):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    p, c2w, intr = model_scene(n, W, H)
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in p.items()}
    _, _, (fx, fy, cx, cy), view, proj, _ = camera_setup(Camera(W, H, *intr, c2w[0]), 1)
    vm, pm = view.to(DEV).contiguous(), (proj @ view).to(DEV).contiguous()
    th = fisheye_theta_limit(*K)
    tb = ops.tile_bounds(W, H)
    f32, i32 = torch.float32, torch.int32
    out = [torch.empty(n, 6, device=DEV), torch.empty(n, 2, device=DEV), torch.empty(n, device=DEV),
           torch.empty(n, dtype=i32, device=DEV), torch.empty(n, 3, device=DEV), torch.empty(n, dtype=i32, device=DEV),
           torch.empty(n, device=DEV)]
    o = [P(x) for x in out]
    head = (n, P(g["means"]), P(g["scales"]), 1.0, P(g["quats"]), P(g["opacities"]))
    grads = [torch.zeros(n, 3, device=DEV), torch.zeros(n, 3, device=DEV), torch.zeros(n, 4, device=DEV),
             torch.zeros(n, device=DEV)]
    cot = [torch.randn(n, 2, device=DEV), torch.randn(n, device=DEV), torch.randn(n, 3, device=DEV),
           torch.randn(n, device=DEV)]
    part = torch.empty(L.gsb_project_camera_partials_floats(n), dtype=f32, device=DEV)
    for aa in (0, 1):
        pin_f = L.gsb_project_forward_activated_aa if aa else L.gsb_project_forward_activated
        arms = {"pinhole": lambda: pin_f(*head, P(vm), P(pm), fx, fy, cx, cy, H, W, tb[0], tb[1], 0.01, *o, s),
                "fisheye": lambda: L.gsb_project_forward_fisheye(*head, P(vm), fx, fy, cx, cy, *K, th, H, W, tb[0],
                                                                 tb[1], 0.01, *o, aa, s)}
        med = _time_arms(arms, reps)
        print(f"n={n} forward{' AA' if aa else ''}: pinhole {med['pinhole']:.4f} ms, fisheye {med['fisheye']:.4f} "
              f"ms ({100 * (med['fisheye'] / med['pinhole'] - 1):+.1f}%)", flush=True)
    # backward: the radii and conics of the last fisheye forward serve both arms (the same per-Gaussian work)
    bt = (P(out[3]), P(out[4]), P(cot[0]), P(cot[1]), P(cot[2]), P(cot[3])) + tuple(P(x) for x in grads)
    for mode in ("plain", "AA", "camgrad"):
        aa = int(mode == "AA")
        pt = P(part) if mode == "camgrad" else None
        if mode == "camgrad":
            pin = lambda: L.gsb_project_backward_activated_camgrad(*head, P(vm), P(pm), fx, fy, H, W, *bt, 0, 0, pt, s)
        else:
            pf = L.gsb_project_backward_activated_aa if aa else L.gsb_project_backward_activated
            pin = lambda: pf(*head, P(vm), P(pm), fx, fy, H, W, *bt, s)
        arms = {"pinhole": pin,
                "fisheye": lambda: L.gsb_project_backward_fisheye(*head, P(vm), fx, fy, *K, th, H, W, *bt, 0, aa, pt,
                                                                  s)}
        med = _time_arms(arms, reps)
        print(f"n={n} backward {mode}: pinhole {med['pinhole']:.4f} ms, fisheye {med['fisheye']:.4f} ms "
              f"({100 * (med['fisheye'] / med['pinhole'] - 1):+.1f}%)", flush=True)


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, intr = model_scene(1_000_000, W, H)
    cams = {"pinhole": Camera(W, H, *intr, c2w[0]),
            "fisheye": Camera(W, H, *intr, c2w[0], k1=K[0], k2=K[1], k3=K[2], k4=K[3], model="fisheye")}
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    first, trainers = 3001, {}
    for name, cam in cams.items():
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2)
        for i in range(warmup):
            tr.step(cam, gt, first + i)
        trainers[name] = tr
    torch.cuda.synchronize()
    ms = {k: [] for k in cams}
    step = first + warmup
    for r in range(rounds):
        for name in (list(cams) if r % 2 == 0 else list(cams)[::-1]):
            tr, cam = trainers[name], cams[name]
            ms[name].append(timed(lambda i: tr.step(cam, gt, step + i), steps))
        step += steps
    med = {k: float(np.median(v)) for k, v in ms.items()}
    for k in cams:
        print(f"C2 SplatTrainer {k}: {med[k]:.3f} ms/step, rounds " + " ".join(f"{x:.3f}" for x in ms[k]), flush=True)
    print(f"C2 fisheye: {100 * (med['fisheye'] / med['pinhole'] - 1):+.1f}%", flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fisheye: no CUDA device")
    print("card:", card(), flush=True)
    for n in (1_000_000, 5_000_000):
        bench_projection(n, a.reps)
    bench_trainer(a.steps, a.rounds)
