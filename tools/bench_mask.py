"""Cost of the per-image loss masks (DESIGN D26): gsb_ssim_l1_loss_masked against gsb_ssim_l1_loss at 1920x1080 and
3840x2160, alternating within one run, each timed over launches queued behind a device-side sleep; the mask ingest
(gsb_resize_area_mask_u8 at loadImage factor 1.5 and getImage factor 2, gsb_undistort_mask_u8) of a 1920x1080 mask;
and the C2 SplatTrainer step (1M Gaussians, 1920x1080, SH degree 3) without and with a mask, alternating rounds, as
CUDA events.  Prints the medians with the card's name and power limit.
usage: python tools/bench_mask.py [--reps N] [--steps K] [--rounds R]"""
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


def _mask(h, w, seed=0):
    """A fifth of the pixels ignored: one rectangle and scattered pixels."""
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand((h, w), generator=g) >= 0.1).to(torch.uint8)
    m[h // 4:h // 2, w // 3:w // 2] = 0
    return m.to(DEV).contiguous()


def _time_arms(arms, reps, per=20):
    for _ in range(3):
        for f in arms.values():
            capi.check(f())
    torch.cuda.synchronize()
    # `per` back-to-back launches between two events, behind a device-side sleep so the host's launch cost does not
    # leave the GPU idle inside the timed window; the arms alternate their order every round
    times = {k: [] for k in arms}
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
    return {k: float(np.median([a.elapsed_time(b) / per for a, b in v])) for k, v in times.items()}


def bench_loss(reps):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    for w, h in ((1920, 1080), (3840, 2160)):
        g = torch.Generator(device=DEV).manual_seed(1)
        r = torch.rand((h, w, 3), device=DEV, generator=g)
        gt = torch.rand((h, w, 3), device=DEV, generator=g)
        m = _mask(h, w)
        v = torch.empty_like(r)
        out = torch.empty(3, device=DEV)
        ws = torch.empty(L.gsb_ssim_workspace_bytes(h, w) + 256, dtype=torch.uint8, device=DEV)
        off = (-ws.data_ptr()) % 256
        wp, wn = ws.data_ptr() + off, ws.numel() - off
        arms = {"unmasked": lambda: L.gsb_ssim_l1_loss(h, w, P(r), P(gt), 0.2, P(v), P(out), wp, wn, s),
                "masked": lambda: L.gsb_ssim_l1_loss_masked(h, w, P(r), P(gt), P(m), 0.2, P(v), P(out), wp, wn, s)}
        med = _time_arms(arms, reps)
        print(f"loss {w}x{h}: unmasked {med['unmasked']:.4f} ms, masked {med['masked']:.4f} ms "
              f"({100 * (med['masked'] / med['unmasked'] - 1):+.1f}%)", flush=True)


def bench_ingest(reps):
    from opensplat_b200.images import get_optimal_new_camera_matrix
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    m = _mask(H, W)
    dh, dw = 720, 1280                                     # loadImage at factor 1.5: round(1080 / 1.5), round(1920 / 1.5)
    lo = torch.empty((dh, dw), dtype=torch.uint8, device=DEV)
    half = torch.empty((H // 2, W // 2), dtype=torch.uint8, device=DEV)
    K, dist = (1500.0, 1500.0, 960.0, 540.0), (-0.1, 0.02, 0.0, 0.0, 0.0)
    newK, roi = get_optimal_new_camera_matrix(K, dist, (W, H))
    und = torch.empty((roi[3], roi[2]), dtype=torch.uint8, device=DEV)
    f15 = float(np.float32(1.0) / np.float32(1.5))
    arms = {"resize_x1.5": lambda: L.gsb_resize_area_mask_u8(H, W, P(m), dh, dw, P(lo), f15, s),
            "level_x2": lambda: L.gsb_resize_area_mask_u8(H, W, P(m), H // 2, W // 2, P(half), 0.0, s),
            "undistort": lambda: L.gsb_undistort_mask_u8(H, W, P(m), *K, *dist, *newK, *roi, P(und), s)}
    med = _time_arms(arms, reps)
    print(f"mask ingest {W}x{H}: " + "  ".join(f"{k}={v:.4f} ms" for k, v in med.items()), flush=True)


def bench_trainer(steps, rounds, warmup=5):
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.trainer import SplatTrainer
    p, c2w, intr = model_scene(N, W, H)
    cam = Camera(W, H, *intr, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(DEV)
    mask = _mask(H, W)
    first, trainers = 3001, {}
    for on in (False, True):
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6),
                          device=DEV, ssim_weight=0.2)
        kw = {"mask": mask} if on else {}
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
        print(f"C2 SplatTrainer mask={'yes' if on else None}: {med[on]:.3f} ms/step ({1e3 / med[on]:.1f} steps/s), "
              f"rounds " + " ".join(f"{x:.3f}" for x in ms[on]), flush=True)
    print(f"C2 mask: {med[True] - med[False]:+.3f} ms/step ({100 * (med[True] / med[False] - 1):+.1f}%)", flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=6)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mask: no CUDA device")
    print("card:", card(), flush=True)
    bench_loss(a.reps)
    bench_ingest(a.reps)
    bench_trainer(a.steps, a.rounds)
