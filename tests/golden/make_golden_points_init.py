"""Writes tests/golden/points_init.npz: the reference's Model constructor (model.hpp:23-57) on six small clouds, at SH
degrees 1 and 3.

The parameter tensors come from the UNMODIFIED reference constructor on the CPU (oracle/_ref/libopensplat_ref_points.so,
built by oracle/build_points_ref.py where the reference checkout exists).  Its PointsTensor::scales() is nanoflann,
which cannot be built offline, so the driver is handed the nearest-neighbour mean distances; they come from the numpy
brute force of oracle/points_init.py, and this script refuses to write the file unless scipy's cKDTree restatement
agrees with it bit for bit.

Per case <c>: <c>/xyz [n,3] fp32, <c>/rgb [n,3] u8, <c>/mean_dist [n], and per degree <d>: <c>/d<d>/{scales, quats,
featuresDc, featuresRest_shape, opacities} (means are xyz; featuresRest is all zeros, its shape is stored)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import build_points_ref, points_init  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "points_init.npz")
DEGREES = (1, 3)


def cases():
    rng = np.random.default_rng(2024)
    f = np.float32
    t = rng.uniform(-2, 2, 600).astype(f)
    line = np.column_stack([0.5 + t, -1.0 + 2 * t, 0.25 - 3 * t]).astype(f)
    line = np.concatenate([line, line[:40]])                      # collinear, with duplicates
    plane = np.column_stack([rng.uniform(-1, 1, 1500), rng.uniform(-1, 1, 1500), np.full(1500, 0.75)]).astype(f)
    return {
        "uniform": points_init.make_cloud("uniform", 5000, seed=11)["xyz"],
        "clustered": points_init.make_cloud("clustered", 5000, seed=12, max_dup=50)["xyz"],
        "collinear": line,
        "planar": plane,
        "four": np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3]], f),
        "identical": np.tile(np.array([[0.3, -1.2, 2.5]], f), (64, 1)),
    }


def main():
    lib = build_points_ref.build()
    if lib is None:
        raise SystemExit("needs the reference checkout to build oracle/_ref/libopensplat_ref_points.so")
    torch.ops.load_library(lib)
    ref = torch.ops.opensplat_ref_points
    rng = np.random.default_rng(7)
    out = {}
    for name, xyz in cases().items():
        xyz = np.ascontiguousarray(xyz, np.float32)
        rgb = rng.integers(0, 256, xyz.shape, dtype=np.uint8)
        md = points_init.knn_mean_dist_brute(xyz)
        kd = points_init.knn_mean_dist_kdtree(xyz)
        assert np.array_equal(md.view(np.int32), kd.view(np.int32)), f"{name}: the two k-NN restatements disagree"
        out[f"{name}/xyz"], out[f"{name}/rgb"], out[f"{name}/mean_dist"] = xyz, rgb, md
        for d in DEGREES:
            r = ref.init_model(torch.from_numpy(xyz), torch.from_numpy(rgb), d, torch.from_numpy(md))
            names = ("means", "scales", "quats", "featuresDc", "featuresRest", "opacities")
            r = dict(zip(names, (t.numpy() for t in r)))
            assert np.array_equal(r["means"], xyz) and not r["featuresRest"].any()
            for k in ("scales", "quats", "featuresDc", "opacities"):
                out[f"{name}/d{d}/{k}"] = r[k]
            out[f"{name}/d{d}/featuresRest_shape"] = np.array(r["featuresRest"].shape, np.int64)
        print(f"{name}: n={len(xyz)} mean_dist in [{md.min():.3g}, {md.max():.3g}]")
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
