"""Restatement of the reference's Model constructor (model.hpp:23-57) -- TEST INFRASTRUCTURE ONLY.

    init_model(xyz, rgb, sh_degree) -> {means, scales, quats, featuresDc, featuresRest, opacities} (CPU torch tensors)

The nearest-neighbour step, PointsTensor::scales (kdtree_tensor.cpp:4-22, a nanoflann k-d tree), is restated twice,
independently, because the reference's tree cannot be built offline:
  - knn_mean_dist_brute: numpy brute force over all pairs, every fp32 operation a separate ufunc (nothing contracted);
  - knn_mean_dist_kdtree: scipy cKDTree's 16 nearest candidates in float64, re-evaluated in fp32 with the
    reference's operation order.
Both compute d(i,j) = ((dx*dx) + (dy*dy)) + dz*dz with dx = x_i - x_j in fp32, take the four smallest values (i itself
included) and return ((sqrt(d1) + sqrt(d2)) + sqrt(d3)) / 3 in fp32.  The rest of the constructor is torch on the
CPU, as the reference runs it; tests/native/points_driver.cpp pins it against the reference's own constructor."""
import math

import numpy as np
import torch

SH_C0 = 0.28209479177387814


def _dist_fp32(q, p):
    """d for query rows q [c,3] against points p [m,3] (all queries) or [c,m,3] (per query), fp32, separate
    roundings."""
    dx, dy, dz = (np.subtract(q[:, None, a], p[..., a], dtype=np.float32) for a in range(3))
    s = np.add(np.multiply(dx, dx, dtype=np.float32), np.multiply(dy, dy, dtype=np.float32), dtype=np.float32)
    return np.add(s, np.multiply(dz, dz, dtype=np.float32), dtype=np.float32)


def _mean_of_sorted(d4):
    """((sqrt(d1) + sqrt(d2)) + sqrt(d3)) / 3 in fp32 from the sorted four smallest values [c,4]."""
    r = np.sqrt(d4.astype(np.float32))
    s = np.add(np.add(r[:, 1], r[:, 2], dtype=np.float32), r[:, 3], dtype=np.float32)
    return np.divide(s, np.float32(3.0), dtype=np.float32)


def _check(xyz):
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    if xyz.ndim != 2 or xyz.shape[1] != 3 or xyz.shape[0] < 4:
        raise ValueError("xyz must be [n,3] with n >= 4")
    return xyz


def knn_mean_dist_brute(xyz, chunk_elems=1 << 23):
    """Brute force over all pairs: [n] fp32."""
    xyz = _check(xyz)
    n = xyz.shape[0]
    c = max(1, min(n, chunk_elems // n))
    out = np.empty(n, np.float32)
    for a in range(0, n, c):
        d = _dist_fp32(xyz[a:a + c], xyz)
        d4 = np.sort(np.partition(d, 3, axis=1)[:, :4], axis=1)
        out[a:a + c] = _mean_of_sorted(d4)
    return out


def knn_mean_dist_kdtree(xyz, k=16):
    """scipy cKDTree's k nearest candidates (float64), re-evaluated in fp32: [n] fp32."""
    from scipy.spatial import cKDTree
    xyz = _check(xyz)
    k = min(k, xyz.shape[0])
    _, idx = cKDTree(xyz.astype(np.float64)).query(xyz.astype(np.float64), k=k)
    d = _dist_fp32(xyz, xyz[idx])
    d4 = np.sort(d, axis=1)[:, :4]
    return _mean_of_sorted(d4)


def knn_mean_dist_brute_torch(xyz_dev, queries, chunk=None):
    """mean_dist of the rows `queries` (indices) of a CUDA fp32 [n,3] tensor by brute force on the device, for clouds
    too large for numpy: one torch op per rounding (each op is its own kernel, so nothing is contracted), the four
    smallest by topk(4, largest=False), then sqrt / sum / division in numpy fp32.  [len(queries)] fp32."""
    n = xyz_dev.shape[0]
    chunk = chunk or max(1, min(256, (1 << 27) // n))
    px, py, pz = xyz_dev[:, 0], xyz_dev[:, 1], xyz_dev[:, 2]
    out = []
    for a in range(0, len(queries), chunk):
        q = xyz_dev[torch.as_tensor(np.asarray(queries[a:a + chunk]), device=xyz_dev.device)]
        dx = q[:, 0:1] - px[None]
        dy = q[:, 1:2] - py[None]
        dz = q[:, 2:3] - pz[None]
        d = (dx * dx + dy * dy) + dz * dz
        del dx, dy, dz
        v = torch.topk(d, 4, dim=1, largest=False).values
        out.append(torch.sort(v, dim=1).values.cpu().numpy())
    return _mean_of_sorted(np.concatenate(out))


def random_quats(n):
    """randomQuatTensor(n) (model.cpp:23-33) after torch::manual_seed(42)."""
    g = torch.Generator().manual_seed(42)
    u, v, w = (torch.rand(n, generator=g) for _ in range(3))
    return torch.stack([torch.sqrt(1 - u) * torch.sin(2 * math.pi * v), torch.sqrt(1 - u) * torch.cos(2 * math.pi * v),
                        torch.sqrt(u) * torch.sin(2 * math.pi * w), torch.sqrt(u) * torch.cos(2 * math.pi * w)], -1)


def init_model(xyz, rgb, sh_degree, mean_dist=None):
    """The six tensors of Model's constructor on the CPU; mean_dist [n] defaults to the brute force."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    n = xyz.shape[0]
    if mean_dist is None:
        mean_dist = knn_mean_dist_brute(xyz)
    k = (sh_degree + 1) ** 2
    means = torch.from_numpy(xyz.copy())
    scales = torch.from_numpy(np.ascontiguousarray(mean_dist, dtype=np.float32)).reshape(n, 1).repeat(1, 3).log()
    shs = torch.zeros((n, k, 3), dtype=torch.float32)
    shs[:, 0, :3] = ((torch.from_numpy(rgb).to(torch.float64) / 255.0 - 0.5) / SH_C0).to(torch.float32)
    return {"means": means, "scales": scales, "quats": random_quats(n), "featuresDc": shs[:, 0, :].clone(),
            "featuresRest": shs[:, 1:, :].clone(),
            "opacities": torch.logit(float(np.float32(0.1)) * torch.ones(n, 1))}


def make_cloud(kind, n, seed=0, max_dup=5000):
    """Test clouds: {"xyz" [n,3] fp32, "outliers" (indices), "duplicates" (indices)}.
    uniform: the unit cube.  clustered: SfM-like -- Gaussian clusters of size ~0.01 in [-1,1]^3, 1 % far outliers
    spread over 1e4x the cluster size, duplicate groups of 2..max_dup identical points, a planar patch (z constant)."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return {"xyz": rng.uniform(-1, 1, (n, 3)).astype(np.float32), "outliers": np.zeros(0, np.int64),
                "duplicates": np.zeros(0, np.int64)}
    assert kind == "clustered", kind
    n_out = max(1, n // 100)
    n_plane = n // 20
    sizes, left = [], n // 50
    s = 2
    while left >= 2:                       # group sizes 2, 5, 20, ... up to max_dup, then repeated
        g = min(s, left, max_dup)
        sizes.append(g)
        left -= g
        s = 2 if s >= max_dup else min(max_dup, s * 4 + (1 if s == 2 else 0))
    n_dup = sum(sizes)
    n_cl = n - n_out - n_plane - n_dup
    centres = rng.uniform(-1, 1, (max(8, n // 2000), 3))
    cl = centres[rng.integers(0, len(centres), n_cl)] + rng.normal(0, 0.01, (n_cl, 3))
    out = rng.uniform(-50, 50, (n_out, 3))
    plane = np.column_stack([rng.uniform(0.2, 0.4, n_plane), rng.uniform(-0.3, -0.1, n_plane),
                             np.full(n_plane, 0.25)])
    dup = np.concatenate([np.repeat(cl[rng.integers(0, n_cl)][None] if i % 2 else rng.uniform(-1, 1, (1, 3)), g, 0)
                          for i, g in enumerate(sizes)]) if sizes else np.zeros((0, 3))
    xyz = np.concatenate([cl, out, plane, dup]).astype(np.float32)
    kind_of = np.concatenate([np.zeros(n_cl), np.ones(n_out), np.full(n_plane, 2), np.full(n_dup, 3)])
    perm = rng.permutation(n)
    xyz, kind_of = xyz[perm], kind_of[perm]
    return {"xyz": np.ascontiguousarray(xyz), "outliers": np.nonzero(kind_of == 1)[0],
            "duplicates": np.nonzero(kind_of == 3)[0]}
