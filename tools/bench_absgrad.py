"""Cost of AbsGS's absolute screen-space gradient (DESIGN D25): the backward blend launch without and with it
(gsb_rasterize_backward against gsb_rasterize_backward_absgrad, and the DEPTH pair gsb_rasterize_backward_depth
against gsb_rasterize_backward_absgrad with depth) on the same binned frame, alternating the arms within one run, at
C2 (1M Gaussians, 1920x1080), C3 (3M, 3840x2160) and C5 (5M, 2560x1440); then the C2 SplatTrainer step without and
with RefineConfig(absgrad=True) on the same fixed scene (no refinement runs: absgrad changes the Gaussian count, so
only a fixed scene compares like with like), alternating rounds.  Prints the medians with the card's name and power
limit.
usage: python tools/bench_absgrad.py [workload ...] [--reps N] [--steps K] [--rounds R] [--no-trainer]"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS  # noqa: E402
from bench_depth import card  # noqa: E402
from bench_model_train import model_scene  # noqa: E402
from bench_pose import SIZES  # noqa: E402
from bench_trainer import timed  # noqa: E402
from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.model import Camera  # noqa: E402
from opensplat_b200.pipeline import SplatPipeline  # noqa: E402
from opensplat_b200.scene import make_scene  # noqa: E402

DEV = "cuda:0"


def bench_blend(wl, reps):
    n, W, H, scale, opac = WORKLOADS[wl]
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=opac, seed=0)
    pp = SplatPipeline(n, W, H, device=DEV)
    pp.load_scene(sc)
    pp.target.copy_(torch.from_numpy(np.random.default_rng(1).uniform(0, 1, (H, W, 3)).astype(np.float32)))
    pp.forward_backward()
    pp.forward_backward()
    f32 = torch.float32
    od, oa = torch.empty((H, W), dtype=f32, device=DEV), torch.empty((H, W), dtype=f32, device=DEV)
    vd = torch.randn((H, W), dtype=f32, device=DEV)
    v_depths = torch.empty(n, dtype=f32, device=DEV)
    v_xy_abs = torch.empty((n, 2), dtype=f32, device=DEV)
    pp._bin_blend(pp.p["opacities"], 0, out_depth=od, out_alpha=oa)     # a depth frame: the plain frame's bits
    L, P, s = pp.L, capi.ptr, capi.stream()
    capi.check(L.gsb_mse_loss_grad(H * W * 3, P(pp.out_img), P(pp.target), P(pp.v_img), P(pp.loss),
                                   1.0 / (H * W * 3), s))
    tb, m = pp.tb, pp.m_raster
    bwd = (H, W, tb[0], tb[1], pp.n, m, P(pp.tile_bins), P(pp.tile_order), P(pp.conics), P(pp.p["opacities"]),
           P(pp.records), P(pp.cum), P(pp.background), P(pp.final_Ts), P(pp.final_idx), P(pp.v_img), None,
           P(pp.grad_rows), P(pp.v_xy), P(pp.v_conic), P(pp.v_rgbs), P(pp.g["opacities"]), 0)
    dep = (P(pp.record_depths), P(vd), P(v_depths))
    arms = {
        "bwd_plain": lambda: L.gsb_rasterize_backward(*bwd, s),
        "bwd_absgrad": lambda: L.gsb_rasterize_backward_absgrad(*bwd, None, None, None, P(v_xy_abs), s),
        "bwd_depth": lambda: L.gsb_rasterize_backward_depth(*bwd, *dep, s),
        "bwd_depth_absgrad": lambda: L.gsb_rasterize_backward_absgrad(*bwd, *dep, P(v_xy_abs), s),
    }
    times = {k: [] for k in arms}
    for _ in range(3):
        for f in arms.values():
            capi.check(f())
    torch.cuda.synchronize()
    for r in range(reps):
        for k, f in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):   # alternate the order
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            capi.check(f())
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    med = {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in times.items()}
    print(f"{wl}: n={n} {W}x{H} M={pp.m} reps={reps}  " + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items())
          + f"  absgrad {100 * (med['bwd_absgrad'] / med['bwd_plain'] - 1):+.1f}%"
          + f"  depth+absgrad {100 * (med['bwd_depth_absgrad'] / med['bwd_depth'] - 1):+.1f}%", flush=True)


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.trainer import SplatTrainer
    n, W, H = SIZES["C2"]
    p, c2w, intr = model_scene(n, W, H)
    cam = Camera(W, H, *intr, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    first, trainers = 3001, {}
    for on in (False, True):
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()},
                          RefineConfig(warmup_length=10 ** 6, absgrad=on), device=DEV, ssim_weight=0.2)
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
    med = {on: float(np.median(ms[on])) for on in ms}
    for on in (False, True):
        print(f"C2 SplatTrainer absgrad={on}: {med[on]:.3f} ms/step ({1e3 / med[on]:.1f} steps/s), rounds "
              + " ".join(f"{x:.3f}" for x in ms[on]), flush=True)
    print(f"C2 step absgrad {100 * (med[True] / med[False] - 1):+.2f}%", flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["c2_1M_1080p_sh3", "c3_3M_4k_sh3", "c5_5M_1440p_dense"])
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--no-trainer", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_absgrad: no CUDA device")
    print("card:", card(), flush=True)
    for wl in a.workloads:
        bench_blend(wl, a.reps)
        torch.cuda.empty_cache()
    if not a.no_trainer:
        bench_trainer(a.steps, a.rounds)
