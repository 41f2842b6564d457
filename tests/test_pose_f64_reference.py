"""CPU: pins the float64 restatement of the camera gradient and the pose chain (tests/pose_f64.py, DESIGN D22) --
the tree against autograd and central differences of the float64 projection map, the identity correction, the
product's own camera helpers, and the wrong conventions it must reject."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pose_f64 as ref  # noqa: E402
import project_f64 as pf  # noqa: E402

F8 = torch.float64


def scene(seed=3, n=300, W=96, H=64):
    """A general camera, Gaussians in its view (the kept, certified ones) and cotangents."""
    mcam = pf.general_camera(W, H, seed)
    cam = pf.camera_from_setup(mcam)
    m, s, q = pf.random_gaussians(cam, n, seed, frac_near=0.0, act=True)
    rng = np.random.default_rng(seed + 1)
    ol = rng.normal(0, 1.5, n).astype(np.float32)
    out = pf.project(cam, m, s, q, act=True, opacity_logits=ol)
    keep = (out["radii"] > 0) & out["cert"]
    m, s, q, ol = m[keep.numpy()], s[keep.numpy()], q[keep.numpy()], ol[keep.numpy()]
    k = m.shape[0]
    vx = rng.normal(0, 1, (k, 2)).astype(np.float32)
    vc = rng.normal(0, 1, (k, 3)).astype(np.float32)
    vo = rng.normal(0, 1, k).astype(np.float32)
    return mcam, cam, m, s, q, ol, vx, vc, vo


def _loss(cam, m, s, q, ol, vx, vc, vo, aa, V, P):
    """The float64 loss of the projection at viewmat V and projmat P (float64 [4,4])."""
    import project_aa_f64 as paa
    c = copy.copy(cam)
    c.V, c.P = V.reshape(16), P.reshape(16)
    t = [torch.as_tensor(x, dtype=F8) for x in (m, s, q, ol, vx, vc, vo)]
    xy, _, conic, _, _ = pf.forward_map(c, t[0], t[1], t[2], 1.0, True)
    L = (xy * t[4]).sum() + (conic * t[5]).sum()
    if aa:
        comp, _ = paa.comp_map(c, t[0], t[1], t[2])
        L = L + (torch.sigmoid(t[3]) * comp * t[6]).sum()
    return L


@pytest.mark.parametrize("aa", [False, True])
def test_restatement_equals_autograd_and_central_differences(aa):
    _, cam, m, s, q, ol, vx, vc, vo = scene()
    assert m.shape[0] > 100
    GV, GP = ref.camgrad_autograd(cam, m, s, q, ol, vx, vc, vo, aa)
    TV, TP, BV, BP = ref.camgrad_tree(cam, m, s, q, ol, vx, vc, vo, aa)
    # the tree's values are the exact map's
    assert torch.allclose(TV, GV, rtol=1e-9, atol=1e-9 * float(GV.abs().max()))
    assert torch.allclose(TP, GP, rtol=1e-9, atol=1e-9 * float(GP.abs().max()))
    assert not bool(GV[3].any()) and not bool(GP[2].any())
    assert bool((BV[:3] > 0).all()) and bool(torch.isfinite(BV).all()) and not bool(BV[3].any())
    # central differences of the float64 map
    V0 = torch.tensor(cam.V, dtype=F8).reshape(4, 4)
    P0 = torch.tensor(cam.P, dtype=F8).reshape(4, 4)
    for which, G in (("V", GV), ("P", GP)):
        fd = torch.zeros(4, 4, dtype=F8)
        for r in range(4):
            for c in range(4):
                base = V0 if which == "V" else P0
                h = 1e-6 * max(1.0, abs(float(base[r, c])))
                d = torch.zeros(4, 4, dtype=F8)
                d[r, c] = h
                args = [(V0 + d, P0), (V0 - d, P0)] if which == "V" else [(V0, P0 + d), (V0, P0 - d)]
                fd[r, c] = (_loss(cam, m, s, q, ol, vx, vc, vo, aa, *args[0]) -
                            _loss(cam, m, s, q, ol, vx, vc, vo, aa, *args[1])) / (2 * h)
        err = float((fd - G).abs().max() / G.abs().max())
        print(f"{which}: central differences rel err {err:.3g}")
        assert err < 1e-5


def test_tree_rejects_a_dropped_JvT_term():
    """Without the J^T vT columns the tree no longer equals autograd of the map."""
    _, cam, m, s, q, ol, vx, vc, vo = scene()
    GV, _ = ref.camgrad_autograd(cam, m, s, q, ol, vx, vc)
    TV, _, _, _ = ref.camgrad_tree(cam, m, s, q, ol, vx, vc, alt="no_JvT")
    err = float((TV - GV)[:3, :3].abs().max() / GV.abs().max())
    print(f"dropped J^T vT: rel err {err:.3g}")
    assert err > 1e-2


def test_identity_correction_is_exact():
    e = torch.zeros(9, dtype=F8)
    assert torch.equal(ref.rot6d(e[3:]), torch.eye(3, dtype=F8))
    from opensplat_b200 import pose
    assert torch.equal(pose.rot6d(torch.zeros(6, dtype=F8)), torch.eye(3, dtype=F8))
    mcam = pf.general_camera(64, 48, 7)
    adj = pose.adjusted_camera(mcam, torch.zeros(9))
    assert torch.equal(adj.camToWorld, mcam.camToWorld)


def test_rot6d_rows_and_the_product_helper():
    th = 0.3
    d = torch.tensor([math.cos(th) - 1, math.sin(th), 0.0, -math.sin(th), math.cos(th) - 1, 0.0], dtype=F8)
    want = torch.tensor([[math.cos(th), math.sin(th), 0], [-math.sin(th), math.cos(th), 0], [0, 0, 1]], dtype=F8)
    assert torch.allclose(ref.rot6d(d), want, atol=1e-15)
    assert not torch.allclose(ref.rot6d(d, "columns"), want, atol=1e-3)
    from opensplat_b200 import pose
    d2 = torch.tensor(ref.random_pose(4)[3:], dtype=F8)
    assert torch.allclose(pose.rot6d(d2), ref.rot6d(d2), atol=1e-15)


def _setup(cam):
    from opensplat_b200.model import camera_setup
    _, _, _, view, proj, centre = camera_setup(cam, 1.0)
    return view.double(), proj.double(), centre.double()


def test_pose_apply_matches_the_adjusted_camera_and_rejects_wrong_frames():
    from opensplat_b200 import pose
    mcam = pf.general_camera(64, 48, 11)
    view, proj, centre = _setup(mcam)
    e = torch.tensor(ref.random_pose(2, rot=0.05, trans=0.2), dtype=F8)
    v_adj, _, c_adj = _setup(pose.adjusted_camera(mcam, e.float()))
    vp, c = ref.pose_apply(e, view, centre)
    assert float((vp - v_adj).abs().max()) < 1e-5 and float((c - c_adj).abs().max()) < 1e-5
    for alt in ("left", "columns", "centre_unmoved"):
        va, ca = ref.pose_apply(e, view, centre, alt)
        assert float((va - v_adj).abs().max()) > 1e-3 or float((ca - c_adj).abs().max()) > 1e-3, alt


@pytest.mark.parametrize("alt", [None, "no_fold", "left", "columns"])
def test_pose_gradient_is_the_composition_derivative(alt):
    """pose_grad from the camera gradient equals central differences in e of the float64 projection loss at the
    corrected camera; each wrong convention does not."""
    mcam, cam, m, s, q, ol, vx, vc, vo = scene(seed=5, n=200)
    view, proj, _ = _setup(mcam)
    e = torch.tensor(ref.random_pose(8), dtype=F8)
    vp, _ = ref.pose_apply(e, view, torch.zeros(3, dtype=F8))
    c = copy.copy(cam)
    c.V, c.P = vp.reshape(16).numpy(), (proj @ vp).reshape(16).numpy()
    GV, GP = ref.camgrad_autograd(c, m, s, q, ol, vx, vc)
    g = ref.pose_grad(e, view, proj, GV, GP, alt)
    fd = torch.zeros(9, dtype=F8)
    for k in range(9):
        h = 1e-6
        vals = []
        for sg in (1, -1):
            ee = e.clone()
            ee[k] += sg * h
            v2, _ = ref.pose_apply(ee, view, torch.zeros(3, dtype=F8))
            vals.append(_loss(cam, m, s, q, ol, vx, vc, vo, False, v2, proj @ v2))
        fd[k] = (vals[0] - vals[1]) / (2 * h)
    err = float((g - fd).abs().max() / fd.abs().max())
    print(f"{alt}: rel err {err:.3g}")
    if alt is None:
        assert err < 1e-5
    else:
        assert err > 1e-2
