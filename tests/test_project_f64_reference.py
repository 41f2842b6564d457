"""Pins tests/project_f64.py, the float64 projection reference the GPU projection tests are held to (CPU only):
  * its bound's evaluation (the kernel's operation tree on value-plus-bound numbers) has the autograd values of its
    forward map to float64 precision, so the bound is taken along the right computation;
  * the fp32 oracle (oracle/gsplat_oracle.c, the kernels' tree in the same order) lies within C_BOUND B of it on every
    certified Gaussian, per element, with no aggregate norm and no flip allowance;
  * the reference's own numbers (tests/golden/projection_*.npz: its CPU back end and torch autograd) lie within
    C_GOLD B of it, per element;
  * the check rejects each known wrong gradient convention on most of the Gaussians that convention changes."""
import numpy as np
import pytest
import torch

import project_f64 as pf
from oracle import oracle as orc
from opensplat_b200.model import Camera
from util import load_golden

U = pf.U
# fp32 vs the float64 map: B is a first-order bound of the fp32 evaluation of the kernels' tree.  The factor 2 covers
# the second-order terms it drops, and the u |exact| it charges per operation where the fp32 result is |computed|.
C_BOUND = 2.0
# The reference's CPU back end evaluates the same map in fp32 in ITS order: 3-term matmul dot products (in any order,
# possibly fused), pow(x, 2) = x * x, divisions by det where the kernel multiplies by 1/det, and autograd's tree for the
# backward rather than the hand-written VJP.  These regroup the same products and sums.  A k-term sum in another
# order has partial sums no larger than the sum of the magnitudes of its terms, so its rounding is at most (k - 1) = 2
# times what B charges for it in the kernels' order (the matmuls' 3-term sums), hence 2 x C_BOUND.  B is not a proof
# for autograd's backward tree, which is not the one B follows; the measured worst ratio on the golden vectors is
# about 0.13 of this tolerance.
C_GOLD = 4.0
GRADS = ("v_mean3d", "v_scale", "v_quat")


def _general(n=4000, seed=0, act=False, glob_scale=1.3, W=320, H=200):
    cam = pf.camera_from_setup(pf.general_camera(W, H, seed))
    m, s, q = pf.random_gaussians(cam, n, seed + 1, act=act)
    return cam, m, s, q, glob_scale


def _axis_aligned(seed=5, n=300):
    """The identity-view camera with exact ties among ordinary Gaussians."""
    W, H = 128, 96
    cam = pf.camera_from_setup(Camera(W, H, 100.0, 80.0, 0.5 * W + 7.0, 0.5 * H - 5.0,
                                      np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32)))
    mt, st, qt = pf.tie_gaussians(cam, seed)
    mg, sg, qg = pf.random_gaussians(cam, n, seed + 1)
    return cam, np.concatenate([mt, mg]), np.concatenate([st, sg]), np.concatenate([qt, qg]), 1.0


def _cot(n, seed, act=False):
    rng = np.random.default_rng(seed)
    c = dict(v_xy=rng.standard_normal((n, 2)).astype(np.float32), v_depth=rng.standard_normal(n).astype(np.float32),
             v_conic=rng.standard_normal((n, 3)).astype(np.float32))
    if act:
        c["v_opacity"] = rng.standard_normal(n).astype(np.float32)
    return c


def cotangent_sets(n, seed):
    """Random (v_xy, v_depth, v_conic), and v_conic alone.  The fov clamp and the quaternion enter only through the
    conic, whose gradients are small against those of the pixel centre: with v_xy present, the bound of v_mean3d is
    set by the pixel-centre path and hides a wrong clamp gradient.  The conic-only set exposes it."""
    c = _cot(n, seed)
    z = dict(c, v_xy=np.zeros_like(c["v_xy"]), v_depth=np.zeros_like(c["v_depth"]))
    return c, z


def _within(got, r, name, mask, C):
    got = torch.as_tensor(np.asarray(got, np.float64))
    err = (got - r[name]).abs()
    bound = C * r["B_" + name]
    m = mask if err.dim() == 1 else mask[:, None].expand_as(err)
    ratio = float((err[m] / bound[m].clamp_min(1e-300)).max()) if bool(m.any()) else 0.0
    return bool((err[m] <= bound[m]).all()), ratio


@pytest.mark.parametrize("scene", ["general", "activated", "axis_aligned_ties"])
def test_bound_evaluation_is_the_autograd_value(scene):
    if scene == "axis_aligned_ties":
        cam, m, s, q, gs = _axis_aligned()
    else:
        cam, m, s, q, gs = _general(act=scene == "activated")
    act = scene == "activated"
    n = m.shape[0]
    ol = np.random.default_rng(9).uniform(-30, 30, n).astype(np.float32) if act else None
    r = pf.project(cam, m, s, q, gs, act=act, opacity_logits=ol, **_cot(n, 3, act))
    k = r["kept"]
    assert float(k.double().mean()) > 0.5 and bool((k & r["clamp_x"]).any()) and bool((k & r["clamp_y"]).any())
    if scene == "axis_aligned_ties":
        assert int((k & r["tie_x"]).sum()) >= 8 and int((k & r["tie_y"]).sum()) >= 8
    for nm in GRADS + (("v_opacity_logits",) if act else ()):
        d = (r["re_" + nm] - r[nm]).abs()
        assert bool((d <= 1e-6 * r["B_" + nm] + 1e-300).all()), (nm, float((d / r["B_" + nm]).nan_to_num().max()))
        assert float(r[nm].abs().max()) > 0


@pytest.mark.parametrize("scene", ["general", "axis_aligned_ties", "near_and_wide"])
def test_certified_gaussians_match_oracle(scene):
    if scene == "axis_aligned_ties":
        cam, m, s, q, gs = _axis_aligned()
    elif scene == "near_and_wide":
        cam, m, s, q, gs = _general(n=3000, seed=7, glob_scale=0.7, W=17, H=33)
    else:
        cam, m, s, q, gs = _general()
    n = m.shape[0]
    c = _cot(n, 4)
    r = pf.project(cam, m, s, q, gs, **c)
    cert = r["cert"]
    assert float(cert.double().mean()) >= 0.99, float(cert.double().mean())
    o = orc.project_forward(m, s, gs, q, *cam.args())
    cn = cert.numpy()
    for nm in ("radii", "num_tiles_hit"):
        assert np.array_equal(o[nm][cn], r[nm].numpy()[cn]), nm
    worst = {}
    for nm in ("xys", "depths", "conics", "cov3d"):
        ok, worst[nm] = _within(o[nm], r, nm, cert, C_BOUND)
        assert ok, (nm, worst[nm])
    g = orc.project_backward(m, s, gs, q, *cam.args(), o["radii"], o["conics"], c["v_xy"], c["v_depth"], c["v_conic"])
    for nm in GRADS:
        ok, worst[nm] = _within(g[nm], r, nm, cert, C_BOUND)
        assert ok, (nm, worst[nm])
    if scene == "axis_aligned_ties":
        ties = (r["tie_x"] | r["tie_y"]) & r["kept"]
        assert bool((ties <= cert).all()) and int(ties.sum()) >= 16
    print(f"\n{scene}: certified {float(cert.double().mean()):.4f}; worst err/bound "
          + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


def _golden_inputs(name):
    g = load_golden(name)
    fx, fy, cx, cy = [float(v) for v in g["intrins"]]
    H, W = [int(v) for v in g["hw"]]
    cam = pf.Cam(g["viewmat"], g["projmat"], fx, fy, cx, cy, H, W, float(g["clip_thresh"]))
    return g, cam, float(g["glob_scale"])


@pytest.mark.parametrize("name", ["projection_general", "projection_ties"])
def test_matches_reference_golden(name):
    """The reference's CPU back end differs from the CUDA semantics in two known ways: its xys ignore cx / cy (offset
    by exactly cx - W/2, cy - H/2), and it forms rw = 1/max(w, 1e-6) instead of 1/(w + 1e-6) (D3).  The float64 map
    is evaluated its way ("cpu") for the comparison, on the Gaussians the CUDA semantics keep and certify."""
    g, cam, gs = _golden_inputs(name)
    rc = pf.project(cam, g["means"], g["scales"], g["quats"], gs, v_xy=g["v_xy"], v_conic=g["v_conic"], d3="cpu")
    rk = pf.project(cam, g["means"], g["scales"], g["quats"], gs)
    sel = rk["kept"] & rk["cert"] & rc["cert"]
    assert float(sel.double().sum() / rk["kept"].double().sum()) >= 0.99
    if name == "projection_ties":
        ties = (rk["tie_x"] | rk["tie_y"]) & rk["kept"]
        assert int(ties.sum()) >= 16 and bool((ties <= sel).all())
    else:
        assert int((sel & rk["clamp_x"]).sum()) > 50 and int((sel & rk["clamp_y"]).sum()) > 50
        assert int((sel & (rk["depths"] <= 0.2)).sum()) > 20
    sn = sel.numpy()
    assert np.array_equal(g["ref_radii"][sn], rk["radii"].numpy()[sn])
    worst = {}
    for nm, key in (("xys", "ref_xys"), ("conics", "ref_conics")):
        ok, worst[nm] = _within(g[key], rc, nm, sel, C_GOLD)
        assert ok, (nm, worst[nm])
    for nm, key in (("v_mean3d", "ref_v_means"), ("v_scale", "ref_v_scales"), ("v_quat", "ref_v_quats")):
        ok, worst[nm] = _within(g[key], rc, nm, sel, C_GOLD)
        assert ok, (nm, worst[nm])
    print(f"\n{name}: compared {int(sel.sum())}; worst err/bound " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("name", ["projection_general", "projection_ties"])
def test_oracle_matches_reference_golden(name):
    """The fp32 oracle against the reference's own vectors, per element, with the D3 and cx / cy differences taken
    out through the float64 map: oracle - map(cuda) + map(cpu) must lie within the two bounds of the reference."""
    g, cam, gs = _golden_inputs(name)
    o = orc.project_forward(g["means"], g["scales"], gs, g["quats"], *cam.args())
    rk = pf.project(cam, g["means"], g["scales"], g["quats"], gs, v_xy=g["v_xy"], v_conic=g["v_conic"])
    rc = pf.project(cam, g["means"], g["scales"], g["quats"], gs, v_xy=g["v_xy"], v_conic=g["v_conic"], d3="cpu")
    sel = rk["kept"] & rk["cert"] & rc["cert"]
    assert np.array_equal(o["radii"][sel.numpy()], g["ref_radii"][sel.numpy()])
    b = orc.project_backward(g["means"], g["scales"], gs, g["quats"], *cam.args(), o["radii"], o["conics"], g["v_xy"],
                             None, g["v_conic"])
    for nm, key in (("v_mean3d", "ref_v_means"), ("v_scale", "ref_v_scales"), ("v_quat", "ref_v_quats")):
        shifted = torch.as_tensor(b[nm], dtype=torch.float64) - rk[nm] + rc[nm]
        err = (shifted - torch.as_tensor(g[key], dtype=torch.float64)).abs()[sel]
        bound = (C_BOUND * rk["B_" + nm] + C_GOLD * rc["B_" + nm])[sel]
        assert bool((err <= bound).all()), (nm, float((err / bound).max()))


ALTS = ["no_d8", "no_d11", "no_d12", "d13_factor2", "JVt", "no_glob_scale", "full_clamp"]


@pytest.mark.parametrize("alt", ALTS)
def test_check_rejects_known_wrong_conventions(alt):
    """Each alternative, built in float64, must fail |g - reference| <= C_BOUND B on most of the certified Gaussians
    whose gradient it changes: the bound is tight enough to tell the conventions apart.  The alternatives: D8's clamp
    sub-gradient dropped (the reference's CUDA VJP), D11's normalisation Jacobian dropped, D12's perspective-divide term
    dropped, D13's factor 2 on v_conic[1], T = J V^T, glob_scale missing from v_scale, and the clamped branch at a
    tie (this kernel before D16).  Measured: D8 about 0.66 (its change is small where the clamp barely acts), D11
    0.76, D12 0.90, the others 0.97 and above; required: 0.6."""
    if alt == "full_clamp":
        cam, m, s, q, gs = _axis_aligned()
    else:
        cam, m, s, q, gs = _general(n=3000, seed=2)
    n = m.shape[0]
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    changed = torch.zeros(n, dtype=torch.bool)
    rejected = torch.zeros(n, dtype=torch.bool)
    for c in cotangent_sets(n, 6):
        r = pf.project(cam, m, s, q, gs, **c)
        args = (cam, t(m), t(s), t(q), t(c["v_xy"]), t(c["v_depth"]))
        vc = t(c["v_conic"])
        if alt == "d13_factor2":
            g = pf.vjp(*args, vc * torch.tensor([1.0, 2.0, 1.0], dtype=torch.float64), gs)
        else:
            g = pf.vjp(*args, vc, gs, alt=None if alt == "no_glob_scale" else alt)
        g = list(g[:3])
        if alt == "no_glob_scale":
            g[1] = g[1] / gs
        sel = r["kept"] & r["cert"]
        for nm, ga in zip(GRADS, g):
            d = torch.where(sel[:, None], (ga - r[nm]).abs(), 0)
            changed |= (d > 1e-12 * (r[nm].abs() + r["B_" + nm] / U)).any(-1)
            rejected |= (d > C_BOUND * r["B_" + nm]).any(-1)
    n_changed = int(changed.sum())
    frac = float((rejected & changed).sum()) / max(n_changed, 1)
    print(f"\n{alt}: changes {n_changed} certified Gaussians, rejected on {frac:.4f} of them")
    assert n_changed >= (16 if alt == "full_clamp" else 100)
    assert frac >= 0.6, frac
