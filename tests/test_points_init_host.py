"""Point-cloud initialisation, CPU side: the two k-NN restatements of oracle/points_init.py against each other and
the golden vectors, the restatement of Model's constructor against the reference's own constructor
(tests/native/points_driver.cpp), the argument checks of points.params_from_points / knn_mean_dist and of the C ABI
entry point.  No GPU."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import points_init as pi  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "points_init.npz")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libopensplat_ref_points.so")
CASES = ["uniform", "clustered", "collinear", "planar", "four", "identical"]
DEGREES = (1, 3)
NAMES = ("means", "scales", "quats", "featuresDc", "featuresRest", "opacities")


def _golden():
    return np.load(GOLDEN)


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("case", CASES)
def test_knn_restatements_agree_with_each_other_and_the_golden(case):
    pytest.importorskip("scipy")
    g = _golden()
    xyz = g[f"{case}/xyz"]
    brute = pi.knn_mean_dist_brute(xyz)
    kd = pi.knn_mean_dist_kdtree(xyz)
    assert _bits_equal(brute, kd)
    assert _bits_equal(brute, g[f"{case}/mean_dist"])


def test_knn_restatement_edge_values():
    g = _golden()
    assert not g["identical/mean_dist"].any()                   # all points identical: mean 0
    four = g["four/xyz"]                                        # 4 points: every point's neighbours are the other 3
    d = [np.sort([np.float32(((np.float32(p[0] - q[0]) ** 2 + np.float32(p[1] - q[1]) ** 2)
                              + np.float32(p[2] - q[2]) ** 2)) for q in four]) for p in four]
    want = [np.float32((np.sqrt(x[1]) + np.sqrt(x[2]) + np.sqrt(x[3])) / np.float32(3)) for x in d]
    assert np.allclose(g["four/mean_dist"], want, rtol=1e-6)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("degree", DEGREES)
def test_oracle_constructor_matches_golden(case, degree):
    g = _golden()
    xyz, rgb = g[f"{case}/xyz"], g[f"{case}/rgb"]
    o = {k: v.numpy() for k, v in pi.init_model(xyz, rgb, degree).items()}
    assert _bits_equal(o["means"], xyz)
    for k in ("scales", "quats", "featuresDc", "opacities"):
        assert _bits_equal(o[k], g[f"{case}/d{degree}/{k}"]), k
    assert tuple(o["featuresRest"].shape) == tuple(g[f"{case}/d{degree}/featuresRest_shape"])
    assert not o["featuresRest"].any()
    if case == "identical":
        assert np.isneginf(o["scales"]).all()                     # the reference's log(0)


@pytest.mark.skipif(not os.path.exists(REF_LIB),
                    reason="libopensplat_ref_points.so not built (needs the reference checkout at build time)")
@pytest.mark.parametrize("degree", [0, 1, 3, 4])
def test_oracle_constructor_matches_reference_constructor(degree):
    """oracle.points_init.init_model against the UNMODIFIED Model constructor (through points_driver.cpp) on a fresh
    cloud (not the golden one), all six tensors bit for bit."""
    torch.ops.load_library(REF_LIB)
    c = pi.make_cloud("clustered", 3000, seed=40 + degree, max_dup=40)
    xyz = c["xyz"]
    rgb = np.random.default_rng(degree).integers(0, 256, xyz.shape, dtype=np.uint8)
    md = pi.knn_mean_dist_brute(xyz)
    ref = torch.ops.opensplat_ref_points.init_model(torch.from_numpy(xyz), torch.from_numpy(rgb), degree,
                                                    torch.from_numpy(md))
    o = pi.init_model(xyz, rgb, degree, md)
    for name, r in zip(NAMES, ref):
        assert _bits_equal(o[name].numpy(), r.numpy()), name


def test_product_host_helpers_match_oracle():
    """The CPU halves of points.params_from_points (quaternions, colours, opacity) against the restatement, and the
    quaternion stream against torch.manual_seed(42)'s global one; the caller's global RNG is left untouched."""
    from opensplat_b200 import points
    g = _golden()
    rgb = g["clustered/rgb"]
    o = pi.init_model(g["clustered/xyz"], rgb, 3, g["clustered/mean_dist"])
    state = torch.get_rng_state()
    q = points.random_quats(len(rgb))
    assert torch.equal(torch.get_rng_state(), state)
    assert _bits_equal(q.numpy(), o["quats"].numpy())
    with torch.random.fork_rng():
        torch.manual_seed(42)
        u, v, w = torch.rand(len(rgb)), torch.rand(len(rgb)), torch.rand(len(rgb))
    g2 = torch.Generator().manual_seed(42)
    assert all(torch.equal(a, torch.rand(len(rgb), generator=g2)) for a in (u, v, w))
    assert _bits_equal(points.rgb_to_features_dc(torch.from_numpy(rgb)).numpy(), o["featuresDc"].numpy())
    assert np.float32(points.opacity_logit()) == o["opacities"].numpy()[0, 0]


def _bad_inputs():
    f, u8 = np.float32, np.uint8
    ok3 = np.zeros((8, 3), f)
    rgb8 = np.zeros((8, 3), u8)
    nan = ok3.copy()
    nan[3, 1] = np.nan
    inf = ok3.copy()
    inf[5, 2] = -np.inf
    return {
        "xyz_float64": (ok3.astype(np.float64), rgb8, 3),
        "xyz_shape": (np.zeros((8, 4), f), rgb8, 3),
        "xyz_1d": (np.zeros(24, f), rgb8, 3),
        "rgb_dtype": (ok3, rgb8.astype(np.int32), 3),
        "rgb_shape": (ok3, np.zeros((8, 4), u8), 3),
        "rgb_count": (ok3, np.zeros((7, 3), u8), 3),
        "one_point": (np.zeros((1, 3), f), np.zeros((1, 3), u8), 3),
        "three_points": (np.zeros((3, 3), f), np.zeros((3, 3), u8), 3),
        "nan": (nan, rgb8, 3),
        "inf": (inf, rgb8, 3),
        "degree_negative": (ok3, rgb8, -1),
        "degree_5": (ok3, rgb8, 5),
        "degree_float": (ok3, rgb8, 2.0),
        "xyz_list": ([[0.0, 0.0, 0.0]] * 8, rgb8, 3),
    }


@pytest.mark.parametrize("case", sorted(_bad_inputs()))
def test_params_from_points_rejects_bad_input_before_the_device(case, monkeypatch):
    from opensplat_b200 import capi, points
    xyz, rgb, deg = _bad_inputs()[case]

    def no_device(*a, **k):
        raise AssertionError("the library was reached before the arguments were checked")
    monkeypatch.setattr(capi, "lib", no_device)
    with pytest.raises(ValueError):
        points.params_from_points(xyz, rgb, sh_degree=deg, device="cpu")


@pytest.mark.parametrize("case", ["xyz_float64", "xyz_shape", "one_point", "three_points", "nan", "inf"])
def test_knn_mean_dist_rejects_bad_input(case):
    from opensplat_b200 import points
    xyz = _bad_inputs()[case][0]
    with pytest.raises(ValueError):
        points.knn_mean_dist(xyz, device="cpu")


def test_params_from_points_empty_cloud():
    from opensplat_b200 import points
    p = points.params_from_points(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8), sh_degree=2, device="cpu")
    shapes = {k: tuple(v.shape) for k, v in p.items()}
    assert shapes == {"means": (0, 3), "scales": (0, 3), "quats": (0, 4), "featuresDc": (0, 3),
                      "featuresRest": (0, 8, 3), "opacities": (0, 1)}
    assert all(v.dtype == torch.float32 for v in p.values())


def test_capi_knn_argument_checks():
    """The C entry point's host-side checks (no kernel runs): n = 0 is a no-op, 1 <= n < 4 and n < 0 are rejected, an
    unaligned or short workspace is rejected, and the workspace size grows with n."""
    from opensplat_b200 import capi
    L = capi.lib()
    assert L.gsb_knn_workspace_bytes(0) == 0
    sizes = [L.gsb_knn_workspace_bytes(n) for n in (4, 33, 1000, 1 << 20)]
    assert sizes == sorted(sizes) and sizes[0] > 0
    assert L.gsb_knn_mean_dist(0, None, None, None, 0, None) == 0
    for n in (-1, 1, 2, 3):
        assert L.gsb_knn_mean_dist(n, C.c_void_p(256), C.c_void_p(256), C.c_void_p(256), 1 << 30, None) == -1
    assert L.gsb_knn_mean_dist(4, C.c_void_p(256), C.c_void_p(256), C.c_void_p(260), 1 << 30, None) == -1
    assert L.gsb_knn_mean_dist(4, C.c_void_p(256), C.c_void_p(256), C.c_void_p(256), 16, None) == -2
