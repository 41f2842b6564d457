"""Times the training-image kernels (csrc/image.cu) at 1080p and 4K on one GPU and prints one JSON line:

  - ingest per image: what images.ImageSet does for a distorted camera once the decoded u8 image is on the device --
    gsb_undistort_u8 (undistort + ROI crop) and the two getImage levels of the reference's default --num-downscales 2
    (gsb_resize_area_u8 at factors 2 and 4);
  - the per-step gt() launch (gsb_u8_to_f32_views of one full-resolution view), next to one SplatTrainer step of
    config C2 (1M Gaussians, 1920x1080, SH degree 3, the scene of tools/bench_model_train.py).

Each kernel figure is given twice.  `*_ms`: CUDA events around `--reps` back-to-back calls on the same buffers, so the
inputs sit in the 50 MB L2 (a 1080p u8 level is 6 MB).  `*_cold_ms`: the median of single calls timed with CUDA
events, each after a 256 MB write that evicts L2.  Both leave out the host: `ingest_host_ms` is the wall time of
ImageSet([camera], [host u8 image]) plus the two levels, to a device synchronise -- the host-to-device upload of the
decoded image and the host fp64 get_optimal_new_camera_matrix included.  The card's name and power limit are read in
the same run.

    python tools/bench_images.py [--reps 50] [--n 1000000]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def timed_cold(fn, reps, flush):
    """Median ms of single fn() calls, CUDA events around each, L2 evicted before each by writing `flush`."""
    ms = []
    for _ in range(reps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(0)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def ingest_host_ms(cam, host_img, reps, dev):
    """Median wall ms of ImageSet construction from a host image plus its levels at 2 and 4, to a synchronise."""
    import time
    from opensplat_b200.images import ImageSet
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s = ImageSet([cam], [host_img], device=dev)
        s.level(0, 2)
        s.level(0, 4)
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0))
        del s
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--n", type=int, default=1_000_000)
    a = ap.parse_args()
    from bench_trainer import gpu_info, timed
    from opensplat_b200 import capi
    from opensplat_b200.images import ImageSet, get_optimal_new_camera_matrix
    from opensplat_b200.model import Camera
    dev = "cuda:0"
    L, P = capi.lib(), capi.ptr
    out = {"gpu": gpu_info(), "reps": a.reps, "sizes": {}}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for label, (W, H) in (("1080p", (1920, 1080)), ("4K", (3840, 2160))):
        host_img = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
        img = host_img.to(dev)
        K = (0.8 * W, 0.8 * W, W / 2 + 0.3, H / 2 - 0.2)
        dist = (-0.1, 0.02, 0.0005, -0.0004, 0.0)
        new_k, (rx, ry, rw, rh) = get_optimal_new_camera_matrix(K, dist, (W, H))
        und = torch.empty((rh, rw, 3), dtype=torch.uint8, device=dev)
        l2 = torch.empty((rh // 2, rw // 2, 3), dtype=torch.uint8, device=dev)
        l4 = torch.empty((rh // 4, rw // 4, 3), dtype=torch.uint8, device=dev)

        def ingest(_):
            s = capi.stream()
            capi.check(L.gsb_undistort_u8(H, W, P(img), *K, *dist, *new_k, rx, ry, rw, rh, P(und), s))
            capi.check(L.gsb_resize_area_u8(rh, rw, P(und), rh // 2, rw // 2, P(l2), 0.0, s))
            capi.check(L.gsb_resize_area_u8(rh, rw, P(und), rh // 4, rw // 4, P(l4), 0.0, s))

        def undistort_only(_):
            capi.check(L.gsb_undistort_u8(H, W, P(img), *K, *dist, *new_k, rx, ry, rw, rh, P(und), capi.stream()))

        cam = Camera(W, H, *K, np.eye(4, dtype=np.float32), k1=dist[0], k2=dist[1], p1=dist[2], p2=dist[3])
        s = ImageSet([cam], [img], device=dev)
        for f in (1, 2, 4):
            s.level(0, f)
        for _ in range(3):
            ingest(0)
            s.gt(0, 1)
        out["sizes"][label] = {
            "image": [W, H], "roi": [rx, ry, rw, rh],
            "ingest_ms": timed(ingest, a.reps),
            "ingest_cold_ms": timed_cold(ingest, a.reps, flush),
            "undistort_crop_ms": timed(undistort_only, a.reps),
            "undistort_crop_cold_ms": timed_cold(undistort_only, a.reps, flush),
            "gt_ms": timed(lambda _: s.gt(0, 1), a.reps),
            "gt_cold_ms": timed_cold(lambda _: s.gt(0, 1), a.reps, flush),
            "ingest_host_ms": ingest_host_ms(cam, host_img, 10, dev),
        }
        del s, und, l2, l4, img, host_img
        torch.cuda.empty_cache()
    # one C2 step next to the gt launch
    from bench_model_train import model_scene
    from opensplat_b200.densify import RefineConfig
    from opensplat_b200.trainer import SplatTrainer
    W, H = 1920, 1080
    p, c2w, (fx, fy, cx, cy) = model_scene(a.n, W, H)
    cam = Camera(W, H, fx, fy, cx, cy, c2w[0])
    gt = torch.rand((H, W, 3), generator=torch.Generator().manual_seed(0)).to(dev)
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, RefineConfig(warmup_length=10 ** 6), device=dev)
    first = 3001
    for i in range(5):
        tr.step(cam, gt, first + i)
    out["c2_step_ms"] = timed(lambda i: tr.step(cam, gt, first + 5 + i), 30)
    out["gt_share_of_c2_step_1080p"] = out["sizes"]["1080p"]["gt_ms"] / out["c2_step_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
