"""Cost of the inverse-depth priors (DESIGN D23) on the C2 workload (1M Gaussians, 1920x1080, SH degree 3): the C2
SplatTrainer step without and with DepthConfig() and a prior on every view, alternating rounds, as CUDA events; then
the new kernels alone (gsb_inverse_depths, gsb_inverse_depths_backward, gsb_inverse_depth_l1 and the 2x level of
gsb_depth_downscale_mean), alternating within one run, each timed over launches queued behind a device-side sleep.
Prints the medians with the card's name and power limit.
usage: python tools/bench_depth_prior.py [--reps N] [--steps K] [--rounds R]"""
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
from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.model import Camera  # noqa: E402

DEV = "cuda:0"
N, W, H = 1_000_000, 1920, 1080


def _prior(seed=0):
    g = torch.Generator().manual_seed(seed)
    P = 0.15 + 0.2 * torch.rand((H, W), generator=g)
    P[torch.rand((H, W), generator=g) < 0.2] = 0.0            # a fifth of the pixels without data
    return P.to(DEV).contiguous()


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.depth import DepthConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, intr = model_scene(N, W, H)
    cam = Camera(W, H, *intr, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    prior = _prior()
    first, trainers = 3001, {}
    for on in (False, True):
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2, depth=DepthConfig() if on else None)
        kw = {"depth": prior} if on else {}
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
    med = {on: float(np.median(ms[on])) for on in (False, True)}
    for on in (False, True):
        print(f"C2 SplatTrainer depth={'DepthConfig() + prior' if on else None}: {med[on]:.3f} ms/step "
              f"({1e3 / med[on]:.1f} steps/s), rounds " + " ".join(f"{x:.3f}" for x in ms[on]), flush=True)
    print(f"C2 depth prior: {med[True] - med[False]:+.3f} ms/step ({100 * (med[True] / med[False] - 1):+.1f}%)",
          flush=True)
    tr = trainers[True][0]
    n = tr.n
    return tr.pipe.depths[:n].clone(), tr.pipe.radii[:n].clone(), prior, tr.depth_render.clone()


def bench_kernels(depths, radii, prior, rendered, reps):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    n = depths.shape[0]
    inv, v_inv, v_z = torch.empty(n, device=DEV), torch.randn(n, device=DEV), torch.empty(n, device=DEV)
    v_r = torch.empty((H, W), device=DEV)
    loss = torch.empty(1, device=DEV)
    ws = torch.empty(L.gsb_inverse_depth_l1_workspace_bytes(H, W), dtype=torch.uint8, device=DEV)
    half = torch.empty((H // 2, W // 2), device=DEV)
    arms = {
        "inverse_depths": lambda: L.gsb_inverse_depths(n, P(depths), P(radii), P(inv), s),
        "inverse_depths_backward": lambda: L.gsb_inverse_depths_backward(n, P(depths), P(radii), P(v_inv), P(v_z), s),
        "inverse_depth_l1": lambda: L.gsb_inverse_depth_l1(H, W, P(rendered), P(prior), 1.0 / (H * W), P(v_r),
                                                           P(loss), ws.data_ptr(), ws.numel(), s),
        "downscale_mean_x2": lambda: L.gsb_depth_downscale_mean(H, W, 2, P(prior), P(half), s),
    }
    for _ in range(3):
        for f in arms.values():
            capi.check(f())
    torch.cuda.synchronize()
    # Each sample is `per` back-to-back launches between two events, enqueued behind a device-side sleep so that the
    # host's launch cost (tens of microseconds through ctypes) does not leave the GPU idle inside the timed window.
    times, per = {k: [] for k in arms}, 20
    for r in range(reps):
        for k, f in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(2_000_000)
            e0.record()
            for _ in range(per):
                capi.check(f())
            e1.record()
            times[k].append((e0, e1))
        torch.cuda.synchronize()
    med = {k: float(np.median([a.elapsed_time(b) / per for a, b in v])) for k, v in times.items()}
    print(f"C2 kernels: n={n} {W}x{H} samples={reps}x{per}  " + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items()),
          flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_depth_prior: no CUDA device")
    print("card:", card(), flush=True)
    bench_kernels(*bench_trainer(a.steps, a.rounds), a.reps)
