"""Pins tests/project_aa_f64.py, the float64 reference of the anti-aliased projection (DESIGN D19), on the CPU:
  * its bound's evaluation (the kernels' operation tree on value-plus-bound numbers) has the values of torch autograd
    of an independently written map, sigmoid(l) sqrt(clamp_min(det S0 / det(S0 + 0.3 I), 0)) chained onto the
    projection, to float64 precision: forward opacity and the VJP w.r.t. means, log-scales, raw quaternions, logits;
  * the check rejects known wrong conventions, each on Gaussians where it differs by more than the bound;
  * a constructed det0 == 0 exactly gives comp = 0, a zero opacity and no gradient from the comp term."""
import numpy as np
import pytest
import torch

import project_aa_f64 as pa
import project_f64 as pf
from opensplat_b200.model import Camera
from util import load_golden

C_BOUND = 2.0
GRADS = ("v_mean3d", "v_scale", "v_quat", "v_opacity_logits")


def _axis_cam(W=128, H=96):
    """camera_setup's y / z flip makes this camToWorld the identity view: t = mean exactly in fp32."""
    return pf.camera_from_setup(Camera(W, H, 100.0, 80.0, 0.5 * W + 7.0, 0.5 * H - 5.0,
                                       np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32)))


def _scene(name):
    """(cam, means, log-scales, quats, logits, glob_scale)."""
    if name == "general":
        cam = pf.camera_from_setup(pf.general_camera(320, 200, 0))
        m, s, q = pf.random_gaussians(cam, 4000, 1, act=True)
        gs = 1.3
    elif name == "small":      # sub-pixel footprints: comp far below 1
        cam = pf.camera_from_setup(pf.general_camera(320, 200, 4))
        m, s, q = pf.random_gaussians(cam, 3000, 5, px_std=(0.01, 0.5), act=True)
        gs = 1.0
    elif name == "axis_aligned_ties":
        cam = _axis_cam()
        mt, st, qt = pf.tie_gaussians(cam, 5)
        mg, sg, qg = pf.random_gaussians(cam, 300, 6, act=True)
        m, s, q = np.concatenate([mt, mg]), np.concatenate([np.log(st), sg]), np.concatenate([qt, qg])
        gs = 1.0
    else:                      # the golden fov-clamp ties' inputs, scales taken as exp(log-scale)
        g = load_golden("projection_ties")
        fx, fy, cx, cy = [float(v) for v in g["intrins"]]
        H, W = [int(v) for v in g["hw"]]
        cam = pf.Cam(g["viewmat"], g["projmat"], fx, fy, cx, cy, H, W, float(g["clip_thresh"]))
        m, s, q, gs = g["means"], np.log(g["scales"]).astype(np.float32), g["quats"], float(g["glob_scale"])
    ol = np.random.default_rng(len(m)).uniform(-6, 6, len(m)).astype(np.float32)
    return cam, m, s.astype(np.float32), q, ol, gs


def _cot(n, seed):
    rng = np.random.default_rng(seed)
    return dict(v_xy=rng.standard_normal((n, 2)).astype(np.float32), v_depth=rng.standard_normal(n).astype(np.float32),
                v_conic=rng.standard_normal((n, 3)).astype(np.float32),
                v_opacity=rng.standard_normal(n).astype(np.float32))


@pytest.mark.parametrize("scene", ["general", "small", "axis_aligned_ties", "golden_ties"])
def test_bound_evaluation_is_the_autograd_value(scene):
    cam, m, s, q, ol, gs = _scene(scene)
    n = len(m)
    r = pa.project_aa(cam, m, s, q, ol, gs, **_cot(n, 3))
    k, pos = r["kept"], r["comp_pos"]
    assert float(k.double().mean()) > 0.5 and bool((pos == k).all())
    assert float(r["comp"][k].min()) > 0 and float(r["comp"][k].max()) < 1
    if scene.endswith("ties"):
        assert int((k & (r["tie_x"] | r["tie_y"])).sum()) >= 16
    # forward: the tree's opacity against the map's
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    comp, _ = pa.comp_map(cam, t(m), t(s), t(q), gs)
    want = torch.where(k, torch.sigmoid(t(ol)) * comp, 0.0)
    d = (r["opacities"] - want).abs()
    assert bool((d <= 1e-6 * r["B_opacities"] + 1e-300).all()), float((d / r["B_opacities"]).nan_to_num().max())
    for nm in GRADS:
        d = (r["re_" + nm] - r[nm]).abs()
        assert bool((d <= 1e-6 * r["B_" + nm] + 1e-300).all()), (nm, float((d / r["B_" + nm]).nan_to_num().max()))
        assert float(r[nm].abs().max()) > 0
    # the comp term is what moves the geometry gradients away from the plain projection's
    p = pf.project(cam, m, s, q, gs, act=True, opacity_logits=ol, **_cot(n, 3))
    assert float((r["v_scale"] - p["v_scale"]).abs().max()) > 0


def _rejected(r, ra, sel):
    """Per Gaussian: some output or gradient of the alternative lies outside C_BOUND B of the reference."""
    bad = torch.zeros_like(sel)
    for nm in ("opacities",) + GRADS:
        key = nm if nm == "opacities" else "re_" + nm
        err = (ra[key] - r[nm]).abs()
        over = err > C_BOUND * r["B_" + nm]
        bad |= over if over.dim() == 1 else over.any(-1)
    return bad & sel


@pytest.mark.parametrize("alt", pa.ALTS)
def test_check_rejects_known_wrong_conventions(alt):
    """Each alternative, evaluated on the kernels' tree, must fall outside C_BOUND B on many certified Gaussians: the
    per-entry off-diagonal cotangent doubled, gsplat's comp + 1e-6 in the backward's denominator (visible where comp
    is small: the sub-pixel scene), the compensation left out of v_logit, and det / det0 in place of det0 / det."""
    cam, m, s, q, ol, gs = _scene("small" if alt == "comp_eps" else "general")
    n = len(m)
    c = _cot(n, 7)
    r = pa.project_aa(cam, m, s, q, ol, gs, **c)
    ra = pa.project_aa(cam, m, s, q, ol, gs, alt=alt, **c)
    sel = r["kept"] & r["cert"] & r["comp_pos"]
    frac = float(_rejected(r, ra, sel).double().sum() / sel.double().sum())
    print(f"\n{alt}: rejected on {frac:.3f} of {int(sel.sum())}")
    assert frac >= (0.03 if alt == "comp_eps" else 0.5), frac     # comp_eps: measured 0.053


def degenerate_gaussians():
    """Gaussians with det0 == 0 exactly at the identity-view camera: identity quaternion and two zero scales (log-scale
    -inf) leave one axis, x or y, so S0 has a zero row; the blur keeps det > 0 and the Gaussian visible."""
    cam = _axis_cam()
    rng = np.random.default_rng(11)
    n = 12
    m = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n), rng.uniform(1.0, 4.0, n)], -1)
    s = np.full((n, 3), -np.inf)
    s[: n // 2, 0] = np.log(rng.uniform(0.01, 0.2, n // 2))
    s[n // 2:, 1] = np.log(rng.uniform(0.01, 0.2, n - n // 2))
    q = np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (n, 1)) * rng.uniform(0.5, 2.0, (n, 1))
    ol = rng.uniform(-3, 3, n)
    return cam, m.astype(np.float32), s.astype(np.float32), q.astype(np.float32), ol.astype(np.float32)


def test_det0_zero_contributes_nothing():
    cam, m, s, q, ol = degenerate_gaussians()
    n = len(m)
    c = _cot(n, 9)
    r = pa.project_aa(cam, m, s, q, ol, 1.0, **c)
    p = pf.project(cam, m, s, q, 1.0, act=True, opacity_logits=ol, **c)
    k = r["kept"]
    assert bool(k.all()) and bool(r["cert"].all()) and not bool(r["comp_pos"].any())
    assert bool((r["comp"] == 0).all()) and bool((r["B_comp"] == 0).all())
    assert bool((r["opacities"] == 0).all()) and bool((r["v_opacity_logits"] == 0).all())
    assert bool((r["re_v_opacity_logits"] == 0).all())
    for nm in ("v_mean3d", "v_scale", "v_quat"):
        assert torch.equal(r["re_" + nm], p["re_" + nm]), nm      # the plain tree, bit for bit
        assert bool(torch.isfinite(r[nm]).all())
        d = (r[nm] - p[nm]).abs()
        assert bool((d <= 1e-6 * r["B_" + nm] + 1e-300).all()), nm
