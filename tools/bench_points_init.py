"""Times the point-cloud initialisation: gsb_knn_mean_dist (csrc/knn.cu) and the whole points.params_from_points, on a
uniform cloud and an SfM-like clustered cloud (1 % far outliers, duplicate groups of 2..5000 points, a planar patch),
against a CPU stand-in for the reference's single-threaded nanoflann search: scipy cKDTree(workers=1) build + 4-NN
query (skipped when scipy is missing).  Each workload's k-NN is checked bit for bit against a device brute force on
sampled queries (outliers and duplicate-group members included).

    python tools/bench_points_init.py [--sizes 1000000,5000000] [--reps 7] [--no-cpu]

Prints the GPU's name and power limit, one line per workload, and a JSON line with all results."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import points_init as pi  # noqa: E402
from opensplat_b200 import capi, points  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def time_kernel(xyz_dev, reps):
    """Median ms of gsb_knn_mean_dist over `reps` calls (CUDA events per call, after 2 warm-up calls)."""
    L, n = capi.lib(), xyz_dev.shape[0]
    ws = torch.empty(L.gsb_knn_workspace_bytes(n), dtype=torch.uint8, device=xyz_dev.device)
    out = torch.empty(n, dtype=torch.float32, device=xyz_dev.device)
    call = lambda: capi.check(L.gsb_knn_mean_dist(n, capi.ptr(xyz_dev), capi.ptr(out), capi.ptr(ws), ws.numel(),
                                                  capi.stream()))
    for _ in range(2):
        call()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), out, ws.numel()


def time_params(xyz, rgb, reps):
    """Median s of params_from_points from host arrays (host clock around a device synchronise)."""
    points.params_from_points(xyz, rgb)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        points.params_from_points(xyz, rgb)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def time_cpu_standin(xyz):
    try:
        from scipy.spatial import cKDTree
    except ImportError:
        return None
    t0 = time.perf_counter()
    tree = cKDTree(xyz)
    tree.query(xyz, k=4, workers=1)
    return time.perf_counter() - t0


def check_sampled(xyz_dev, got, cloud, samples=8192):
    """Bit-exactness on `samples` queries: half random, half from the outliers and duplicate-group members."""
    rng = np.random.default_rng(0)
    special = np.concatenate([cloud["outliers"], cloud["duplicates"]])
    k = min(len(special), samples // 2)
    q = np.unique(np.concatenate([rng.choice(special, k, replace=False) if k else special[:0],
                                  rng.choice(len(cloud["xyz"]), samples - k, replace=False)]))
    want = pi.knn_mean_dist_brute_torch(xyz_dev, q)
    return int((got.cpu().numpy()[q].view(np.int32) != want.view(np.int32)).sum()), len(q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,5000000")
    ap.add_argument("--kinds", default="uniform,clustered")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--no-cpu", action="store_true", help="skip the scipy cKDTree stand-in")
    a = ap.parse_args()
    info = gpu_info()
    print("gpu:", info or torch.cuda.get_device_name(0), flush=True)
    rows = []
    for n in (int(s) for s in a.sizes.split(",")):
        for kind in a.kinds.split(","):
            cloud = pi.make_cloud(kind, n, seed=1)
            xyz = cloud["xyz"]
            rgb = np.random.default_rng(2).integers(0, 256, xyz.shape, dtype=np.uint8)
            xyz_dev = torch.from_numpy(xyz).cuda()
            kernel_ms, md, ws_bytes = time_kernel(xyz_dev, a.reps)
            bad, checked = check_sampled(xyz_dev, md, cloud)
            params_s = time_params(xyz, rgb, max(3, a.reps // 2))
            cpu_s = None if a.no_cpu else time_cpu_standin(xyz)
            row = dict(kind=kind, n=n, knn_ms=round(kernel_ms, 3), params_from_points_ms=round(1e3 * params_s, 2),
                       workspace_mb=round(ws_bytes / 2 ** 20, 1), sampled_queries=checked, mismatches=bad,
                       cpu_ckdtree_s=None if cpu_s is None else round(cpu_s, 2))
            rows.append(row)
            print(row, flush=True)
            del xyz_dev, md
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": info, "results": rows}))
    if any(r["mismatches"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
