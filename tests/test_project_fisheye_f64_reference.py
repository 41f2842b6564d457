"""CPU checks of the fisheye projection's float64 restatement (tests/project_fisheye_f64.py, DESIGN D27): the kernel's
operation tree equals the exact map, the map is OpenCV's fisheye model, it meets the pinhole on the axis, the theta
limit is the first stationary point of theta_d, and the check tells known-wrong conventions apart."""
import math

import numpy as np
import pytest
import torch

import project_fisheye_f64 as pf
from opensplat_b200.model import fisheye_theta_limit

F8 = torch.float64
KS = [(0.0, 0.0, 0.0, 0.0), (0.05, -0.02, 0.004, -0.0005), (-0.3, 0.1, -0.02, 0.002), (0.2, 0.05, 0.01, 0.001)]


def _scene(k, n=3000, seed=0, identity=False):
    cam = pf.fisheye_camera(640, 480, seed, k=k, identity=identity)
    return cam, [torch.as_tensor(x).to(F8) for x in pf.random_fisheye_gaussians(cam, n, seed + 1)]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("identity", [False, True])
def test_tree_values_equal_the_exact_map(k, identity):
    cam, (m, a, q, ol) = _scene(k, identity=identity)
    out = pf.project(cam, m, a, q, ol, aa=True)
    uv, depth, conic, op = pf.forward_map(cam, m, a, q, ol, aa=True)
    kept = out["kept"]
    assert int(kept.sum()) > 500 and int(out["series"].sum()) > 50
    for name, ref in (("xys", uv), ("conics", conic), ("opacities", op)):
        got, B = out[name][kept], out["B_" + name][kept]
        err = (got - ref[kept]).abs()
        # the tree's float64 evaluation differs from the map by float64 rounding and the series remainder in B
        assert bool((err <= 1e-9 * (got.abs() + 1) + B).all()), name


def test_map_is_opencv_fisheye_projectPoints():
    rng = np.random.default_rng(3)
    k = (0.03, -0.01, 0.002, -0.0003)
    fx, fy, cx, cy = 300.0, 310.0, 320.5, 240.25
    X = rng.uniform(-1, 1, (500, 3))
    X[:, 2] = rng.uniform(0.05, 2, 500)
    # cv::fisheye::projectPoints (undistorted point a = x / z, b = y / z), alpha = 0
    a, b = X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    r = np.sqrt(a * a + b * b)
    th = np.arctan(r)
    thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
    sc = thd / r
    want = np.stack([fx * a * sc + cx, fy * b * sc + cy], -1) - 0.5
    got = pf.pixel_map(torch.as_tensor(X), k, fx, fy, cx, cy).numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)


@pytest.mark.parametrize("k", KS)
def test_on_the_axis_J_is_the_pinhole_J(k):
    fx, fy = 400.0, 410.0
    for tz in (0.3, 1.0, 7.0):
        t = torch.tensor([[0.0, 0.0, tz]], dtype=F8, requires_grad=True)
        uv = pf.pixel_map(t, k, fx, fy, 0.0, 0.0)
        J = torch.stack([torch.autograd.grad(uv[0, i], t, retain_graph=True)[0][0] for i in range(2)])
        want = torch.tensor([[fx / tz, 0, 0], [0, fy / tz, 0]], dtype=F8)
        assert torch.isfinite(J).all()
        torch.testing.assert_close(J, want, rtol=1e-14, atol=1e-14)


def test_small_r_branch_is_continuous():
    k = KS[2]
    tz = 1.3
    for rho in (1e-5, 0.099999, 0.1, 0.100001, 0.3):
        t = torch.tensor([[rho * tz * 0.6, rho * tz * 0.8, tz]], dtype=F8)
        ref = torch.tensor([[rho * tz * 0.6, rho * tz * 0.8, tz]], dtype=torch.float64)
        got = pf.pixel_map(t, k, 500.0, 500.0, 0.0, 0.0)
        th = math.atan(rho)
        thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
        want = 500.0 * thd / (rho * tz) * ref[0, :2] - 0.5
        torch.testing.assert_close(got[0], want, rtol=1e-13, atol=1e-12)
        # the fp32 tree: both branches agree with the exact map within the bound there
        Rt = [pf.R(t[:, i]) for i in range(3)]
        f = pf._fisheye_terms(tuple(pf.f32(x) for x in k), *Rt)
        assert bool(((f["g"].v - (thd / (rho * tz))).abs() <= f["g"].b + 1e-15).all())


@pytest.mark.parametrize("k,expect", [((0.0, 0.0, 0.0, 0.0), None), ((0.1, 0.01, 0.0, 0.0), None),
                                      ((-0.3, 0.0, 0.0, 0.0), "root"), ((0.05, -0.2, 0.0, 0.0), "root"),
                                      ((0.0, 0.0, 0.0, -0.05), "root")])
def test_theta_limit(k, expect):
    lim = fisheye_theta_limit(*k)
    assert lim == float(np.float32(lim))
    if expect is None:
        assert lim == float(np.float32(0.5 * math.pi))
        return
    c = [9 * k[3], 7 * k[2], 5 * k[1], 3 * k[0], 1.0]
    x = [r.real for r in np.roots(np.trim_zeros(c, "f")) if abs(r.imag) < 1e-12 and 0 < r.real < (0.5 * math.pi) ** 2]
    want = math.sqrt(min(x))
    assert lim == float(np.float32(want))
    def d(th):
        return 1 + 3 * k[0] * th ** 2 + 5 * k[1] * th ** 4 + 7 * k[2] * th ** 6 + 9 * k[3] * th ** 8
    assert d(0.999 * want) > 0 and abs(d(want)) < 1e-9


@pytest.mark.parametrize("a,b", [(0.7, 0.0), (1.0, 0.3), (1.3, 1.0), (2.0, 0.3), (0.5, 0.0)])
def test_theta_limit_at_a_double_root(a, b):
    """d theta_d / d theta = (1 - x / a)^2 (1 + b x), x = theta^2, touches 0 at theta = sqrt(a) without crossing:
    theta_d stops growing there, so that is the limit (np.roots returns most of these as a conjugate pair)."""
    import numpy as np
    c = np.polymul(np.polymul([-1.0 / a, 1.0], [-1.0 / a, 1.0]), [b, 1.0])      # [7 k3, 5 k2, 3 k1, 1]
    c = np.concatenate([np.zeros(4 - len(c)), c])             # polymul drops a leading 0 (b = 0)
    k3, k2, k1 = c[0] / 7.0, c[1] / 5.0, c[2] / 3.0
    lim = fisheye_theta_limit(k1, k2, k3, 0.0)
    assert abs(lim - math.sqrt(a)) <= 1e-6 * math.sqrt(a)


def test_theta_limit_refuses_non_finite():
    with pytest.raises(ValueError):
        fisheye_theta_limit(float("nan"), 0, 0, 0)


@pytest.mark.parametrize("alt", ["no_half", "theta", "eps"])
def test_check_rejects_wrong_conventions(alt):
    k = KS[2]
    cam, (m, a, q, ol) = _scene(k, n=2000, identity=True)
    out = pf.project(cam, m, a, q, ol)
    uv, _, conic, _ = pf.forward_map(cam, m, a, q, ol, alt=alt)
    kept = out["kept"]
    err = (out["xys"][kept] - uv[kept]).abs() - 4 * out["B_xys"][kept]
    err_c = (out["conics"][kept] - conic[kept]).abs() - 4 * out["B_conics"][kept]
    assert bool((err > 0).any() or (err_c > 0).any())
