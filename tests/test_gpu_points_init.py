"""Point-cloud initialisation on the H100: points.knn_mean_dist (csrc/knn.cu) and points.params_from_points against
the reference constructor's golden vectors, the k-NN against a device brute force on a 1M-point SfM-like cloud,
determinism and permutation equivariance, the edge cases, and SplatTrainer trained from a point cloud."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import points_init as pi  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(ROOT, "tests", "golden", "points_init.npz")
CASES = ["uniform", "clustered", "collinear", "planar", "four", "identical"]


def _bits(t):
    a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a).view(np.uint8)


def _bits_equal(a, b):
    a = a.detach().cpu() if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))
    b = b.detach().cpu() if isinstance(b, torch.Tensor) else torch.from_numpy(np.asarray(b))
    return tuple(a.shape) == tuple(b.shape) and a.dtype == b.dtype and np.array_equal(_bits(a), _bits(b))


def _ulp_distance(a, b):
    """|a - b| in units in the last place of fp32 (both finite, same sign)."""
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("degree", [1, 3])
def test_golden_constructor(case, degree):
    from opensplat_b200 import points
    g = np.load(GOLDEN)
    xyz, rgb = g[f"{case}/xyz"], g[f"{case}/rgb"]
    md = points.knn_mean_dist(torch.from_numpy(xyz).to(DEV))
    assert md.is_cuda and _bits_equal(md, torch.from_numpy(g[f"{case}/mean_dist"]))
    p = points.params_from_points(xyz, rgb, sh_degree=degree, device=DEV)
    assert all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in p.values())
    assert _bits_equal(p["means"], torch.from_numpy(xyz))
    for k in ("quats", "featuresDc", "opacities"):
        assert _bits_equal(p[k], torch.from_numpy(g[f"{case}/d{degree}/{k}"])), k
    assert tuple(p["featuresRest"].shape) == tuple(g[f"{case}/d{degree}/featuresRest_shape"])
    assert not bool(p["featuresRest"].any())
    s, want = p["scales"].cpu().numpy(), g[f"{case}/d{degree}/scales"]
    assert s.shape == want.shape
    inf = np.isneginf(want)
    assert np.array_equal(np.isneginf(s), inf)
    assert np.isfinite(s[~inf]).all()
    assert _ulp_distance(s[~inf], want[~inf]).max(initial=0) <= 2


@pytest.fixture(scope="module")
def big_cloud():
    return pi.make_cloud("clustered", 1_000_000, seed=3)


def test_million_point_cloud_matches_device_brute_force(big_cloud):
    from opensplat_b200 import points
    xyz = torch.from_numpy(big_cloud["xyz"]).to(DEV)
    md = points.knn_mean_dist(xyz)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(md).all()) and bool((md >= 0).all())
    rng = np.random.default_rng(0)
    q = np.unique(np.concatenate([rng.choice(len(xyz), 8192, replace=False), big_cloud["outliers"],
                                  big_cloud["duplicates"]]))
    want = pi.knn_mean_dist_brute_torch(xyz, q)
    got = md.cpu().numpy()[q]
    bad = np.nonzero(got.view(np.int32) != want.view(np.int32))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(q)} queries differ, e.g. {q[bad[:5]]}: {got[bad[:5]]} vs {want[bad[:5]]}"


def test_deterministic_and_permutation_equivariant(big_cloud):
    from opensplat_b200 import points
    xyz = torch.from_numpy(big_cloud["xyz"]).to(DEV)
    a = points.knn_mean_dist(xyz)
    b = points.knn_mean_dist(xyz)
    assert _bits_equal(a, b)
    perm = torch.randperm(len(xyz), generator=torch.Generator().manual_seed(1)).to(DEV)
    c = points.knn_mean_dist(xyz[perm].contiguous())
    assert _bits_equal(c, a[perm])


def test_edge_cases():
    from opensplat_b200 import points
    p = points.params_from_points(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8), sh_degree=3, device=DEV)
    assert {k: tuple(v.shape) for k, v in p.items()} == {
        "means": (0, 3), "scales": (0, 3), "quats": (0, 4), "featuresDc": (0, 3), "featuresRest": (0, 15, 3),
        "opacities": (0, 1)}
    assert all(v.is_cuda for v in p.values())
    assert points.knn_mean_dist(torch.zeros((0, 3), device=DEV)).shape == (0,)
    four = np.array([[0, 0, 0], [3, 0, 0], [0, 4, 0], [0, 0, 12]], np.float32)
    assert _bits_equal(points.knn_mean_dist(four), torch.from_numpy(pi.knn_mean_dist_brute(four)))
    same = np.tile(np.array([[1.5, -2.0, 0.25]], np.float32), (1000, 1))
    p = points.params_from_points(same, np.full((1000, 3), 128, np.uint8), sh_degree=0, device=DEV)
    assert not bool(points.knn_mean_dist(same).any())
    assert bool(torch.isneginf(p["scales"]).all()) and p["featuresRest"].shape == (1000, 0, 3)


def test_trainer_from_point_cloud():
    """SplatTrainer(params_from_points(...)) on test_gpu_trainer's synthetic problem: 10 steps, finite losses."""
    from opensplat_b200.points import params_from_points
    from opensplat_b200.trainer import SplatTrainer
    from test_gpu_trainer import _cams, make_problem, refine_config
    p, c2w, gts, intr, H, W = make_problem()
    rgb = np.random.default_rng(0).integers(0, 256, (len(p["means"]), 3), dtype=np.uint8)
    params = params_from_points(p["means"], rgb, sh_degree=1, device=DEV)
    tr = SplatTrainer(params, refine_config(), device=DEV)
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    losses = []
    for step in range(1, 11):
        losses.append(tr.step(cams[(step - 1) % len(cams)], gt[(step - 1) % len(cams)], step)[0].item())
    assert np.isfinite(losses).all(), losses
