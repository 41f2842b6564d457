"""Pins tests/sh_f64.py and tests/loss_f64.py, the float64 references the GPU SH and loss tests are held to (CPU only):
  * each bound's evaluation (the kernel's operation tree on value-plus-bound numbers) has the values of float64
    autograd of a plain formula to float64 precision, so the bound is taken along the right computation;
  * the oracle (oracle/gsplat_oracle.c's SH, oracle.main_loss) lies within C_BOUND B of it, per element;
  * the reference's own numbers (tests/golden: its CPU SH and its SSIM + l1_loss under libtorch autograd) lie within
    C_GOLD B, per element; loss_ties_48x80 holds exact ties, saturated 0 / 1 areas and flat blocks;
  * the check rejects each known wrong convention on most of the elements that convention changes."""
import numpy as np
import pytest
import torch

import loss_f64 as lf
import sh_f64 as sf
from oracle import oracle as orc
from util import load_golden

F8 = torch.float64
# first-order bound: the factor 2 covers the second-order terms and the u |exact| charged where fp32 rounds u |computed|
C_BOUND = 2.0
# The reference's CPU back end and libtorch evaluate the same maps in their own order (SSIM: a 121-tap 2-D conv2d
# instead of two 11-tap passes; SH: its own expression order), so its rounding is not the one B follows.  Measured
# worst ratios are printed; the tolerance is 4 B.
C_GOLD = 4.0


def _ratio(got, want, bound, mask=None):
    got = torch.as_tensor(np.asarray(got, np.float64)) if not torch.is_tensor(got) else got.double()
    err = (got - want).abs()
    if mask is not None:
        err, bound = err[mask], bound[mask]
    ok = bool((err <= bound).all())
    return ok, float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _sh_inputs(n, degree, seed):
    rng = np.random.default_rng(seed)
    K = sf.num_bases(degree)
    co = rng.standard_normal((n, K, 3)).astype(np.float32)
    means = rng.uniform(-2, 2, (n, 3)).astype(np.float32)
    vd = rng.standard_normal((n, 3)).astype(np.float32)
    cp = np.array([0.3, -4.0, 1.5], np.float32)
    v = rng.standard_normal((n, 3)).astype(np.float32)
    return co, means, vd, cp, v


@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("mode", ["viewdirs", "cam_rgb"])
def test_sh_bound_evaluation_is_the_autograd_value(degree, mode):
    for use in range(degree + 1):
        co, means, vd, cp, v = _sh_inputs(500, degree, 10 * degree + use)
        kw = dict(viewdirs=vd) if mode == "viewdirs" else dict(means=means, cam_pos=cp, bias=0.5)
        r = sf.sh(degree, use, co, v_colors=v, **kw)
        d = (r["re_v_coeffs"] - r["v_coeffs"]).abs()
        assert bool((d <= 1e-6 * r["B_v_coeffs"] + 1e-300).all())
        assert float(r["v_coeffs"].abs().max()) > 0
        # forward values against the plain colour formula
        vdir = torch.as_tensor(vd, dtype=F8) if mode == "viewdirs" else (torch.as_tensor(means, dtype=F8)
                                                                         - torch.as_tensor(cp, dtype=F8))
        nb = sf.num_bases(use)
        col = sf._plain_colour(nb, vdir, torch.as_tensor(co, dtype=F8))
        if mode == "cam_rgb":
            col = (col + 0.5).clamp_min(0)
        assert bool(((r["colors"] - col).abs() <= 1e-6 * r["B_colors"] + 1e-12 * col.abs()).all())
        if mode == "cam_rgb":
            assert float(r["cert"].double().mean()) >= 0.99 and (nb > 1 or bool(r["cert"].all()))


def test_sh_multiview_bound_evaluation_is_the_autograd_value():
    n, degree, views = 400, 3, 5
    co, means, _, _, _ = _sh_inputs(n, degree, 3)
    rng = np.random.default_rng(4)
    cams = rng.uniform(-3, 3, (views, 3)).astype(np.float32) + np.array([0, 0, -6], np.float32)
    v = rng.standard_normal((views, n, 3)).astype(np.float32)
    v[1] = 0
    r = sf.sh_multiview(degree, 2, co, means, cams, v, 1.0 / views)
    d = (r["re_v_coeffs"] - r["v_coeffs"]).abs()
    assert bool((d <= 1e-6 * r["B_v_coeffs"] + 1e-300).all()) and float(r["v_coeffs"].abs().max()) > 0
    assert bool((r["v_coeffs"][:, 9:] == 0).all())


@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
def test_sh_oracle_within_bound(degree):
    co, _, vd, _, v = _sh_inputs(3000, degree, 100 + degree)
    K = sf.num_bases(degree)
    worst = []
    for use in range(degree + 1):
        r = sf.sh(degree, use, co, viewdirs=vd, v_colors=v)
        ok, q = _ratio(orc.sh_forward(use, vd, co), r["colors"], C_BOUND * r["B_colors"])
        assert ok, (use, q)
        ok2, q2 = _ratio(orc.sh_backward(use, K, vd, v), r["v_coeffs"], C_BOUND * r["B_v_coeffs"])
        assert ok2, (use, q2)
        worst += [q, q2]
    print(f"\nSH degree {degree} oracle: worst err/bound {max(worst):.3f}")


@pytest.mark.parametrize("name", ["sh_deg3", "sh_deg4"])
def test_sh_golden_within_bound(name):
    g = load_golden(name)
    deg = int(g["degree"])
    worst = []
    for use in range(deg + 1):
        r = sf.sh(deg, use, g["coeffs"], viewdirs=g["viewdirs"], v_colors=g["wgt"])
        ok, q = _ratio(g[f"ref_colors_d{use}"], r["colors"], C_GOLD * r["B_colors"])
        assert ok, (use, q)
        ok2, q2 = _ratio(g[f"ref_v_coeffs_d{use}"], r["v_coeffs"], C_GOLD * r["B_v_coeffs"])
        assert ok2, (use, q2)
        worst += [q / C_GOLD, q2 / C_GOLD]
    print(f"\n{name}: worst err/B {max(worst):.3f}")


def test_sh_tie_is_exact_and_passes_the_gradient():
    """featuresDc = -1.7724538f at degrees_to_use 0: fl(C0 c) = -0.5, so the fp32 colour + 0.5 is exactly 0 and the
    clamp passes the gradient (D17), though the float64 product lies below -0.5."""
    assert np.float32(sf.C0) * np.float32(sf.TIE_DC) == np.float32(-0.5)
    assert float(sf.C0) * float(sf.TIE_DC) < -0.5
    n = 64
    co, means, _, cp, v = _sh_inputs(n, 2, 7)
    co[:, 0, 1] = sf.TIE_DC
    r = sf.sh(2, 0, co, means=means, cam_pos=cp, bias=0.5, v_colors=v)
    assert bool(r["tie"][:, 1].all()) and bool(r["cert"].all()) and bool(r["mask"][:, 1].all())
    assert bool((r["v_coeffs"][:, 0, 1] == sf.C0 * torch.as_tensor(v[:, 1], dtype=F8)).all())
    blocked = sf.sh(2, 0, co, means=means, cam_pos=cp, bias=0.5, v_colors=v, alt="tie_blocked")
    assert bool((blocked["v_coeffs"][:, 0, 1] == 0).all())
    err = (blocked["v_coeffs"] - r["v_coeffs"]).abs()[:, 0, 1]
    assert bool((err > C_BOUND * r["B_v_coeffs"][:, 0, 1]).all())       # rejected at every tie


# ------------------------------------------------------------------------------------------------ loss
def _loss_images(kind, H, W, seed):
    if kind == "ties":
        return lf.tie_images(H, W, seed)
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0, 1, (H, W, 3)).astype(np.float32)
    rend = np.clip(gt + 0.15 * rng.standard_normal((H, W, 3)).astype(np.float32), 0, 1).astype(np.float32)
    return rend, gt


def _plain_grad(rend, gt, w, alt=None):
    r = torch.as_tensor(rend, dtype=F8).requires_grad_()
    total, l1, ssim = lf.plain_loss(r, torch.as_tensor(gt, dtype=F8), w, alt=alt)
    (g,) = torch.autograd.grad(total, [r])
    return g, float(total.detach()), float(l1.detach()), float(ssim.detach())


@pytest.mark.parametrize("kind,H,W", [("random", 37, 29), ("ties", 48, 80), ("random", 1, 37), ("ties", 17, 16)])
@pytest.mark.parametrize("w", [0.0, 0.2, 1.0])
def test_loss_bound_evaluation_is_the_autograd_value(kind, H, W, w):
    rend, gt = _loss_images(kind, H, W, H * W)
    r = lf.loss(rend, gt, w, band=7)              # several bands, so the band halo is exercised
    g, total, l1, ssim = _plain_grad(rend, gt, w)
    d = (r["v_rendered"] - g).abs()
    assert bool((d <= 1e-6 * r["B_v_rendered"] + 1e-300).all()), float((d / r["B_v_rendered"]).nan_to_num().max())
    for k, val in (("loss", total), ("l1", l1), ("ssim", ssim)):
        assert abs(r[k] - val) <= 1e-6 * r["B_" + k], (k, r[k], val)
    one = lf.loss(rend, gt, w)                    # one band
    assert torch.equal(one["v_rendered"], r["v_rendered"]) and torch.equal(one["B_v_rendered"], r["B_v_rendered"])


@pytest.mark.parametrize("kind,H,W", [("random", 45, 70), ("ties", 48, 80), ("ties", 33, 31)])
@pytest.mark.parametrize("w", [0.0, 0.2, 1.0])
def test_loss_oracle_within_bound(kind, H, W, w):
    rend, gt = _loss_images(kind, H, W, 3 + H)
    r = lf.loss(rend, gt, w)
    o = orc.main_loss(rend, gt, w)
    ok, q = _ratio(o["v_rendered"], r["v_rendered"], C_BOUND * r["B_v_rendered"])
    assert ok, q
    for k in ("loss", "l1", "ssim"):
        assert abs(o[k] - r[k]) <= C_BOUND * r["B_" + k], k
    print(f"\nloss {kind} {H}x{W} w={w} oracle: worst err/bound {q:.3f}")


@pytest.mark.parametrize("name", ["loss_45x70", "loss_ties_48x80"])
def test_loss_golden_within_bound(name):
    g = load_golden(name)
    w = float(g["ssim_weight"])
    r = lf.loss(g["rendered"], g["gt"], w)
    ok, q = _ratio(g["ref_v_rendered"], r["v_rendered"], C_GOLD * r["B_v_rendered"])
    assert ok, q
    assert abs(float(g["ref_loss"]) - r["loss"]) <= C_GOLD * r["B_loss"]
    if name == "loss_ties_48x80":
        same = torch.as_tensor(g["rendered"] == g["gt"])
        assert float(same.double().mean()) > 0.3
    print(f"\n{name}: worst err/B {q / C_GOLD:.3f}")


LOSS_ALTS = ["sgn0_plus", "untransposed", "centred", "edge_pad", "swap_c"]


@pytest.mark.parametrize("alt", LOSS_ALTS)
def test_loss_check_rejects_known_wrong_conventions(alt):
    """Each alternative must fail |v - reference| <= C_BOUND B on most of the elements whose gradient it changes:
    sgn(0) = +1, the untransposed window in the backward, a centred window, edge-clamped padding, C1 and C2 swapped.
    The tie content is used, so sgn(0) and the flat blocks are present."""
    rend, gt = lf.tie_images(48, 80, 11)
    r = lf.loss(rend, gt, 0.2)
    a = lf.loss(rend, gt, 0.2, alt=alt)
    d = (a["v_rendered"] - r["v_rendered"]).abs()
    changed = d > 1e-12 * (r["v_rendered"].abs() + r["B_v_rendered"] / lf.U)
    frac = float((changed & (d > C_BOUND * r["B_v_rendered"])).sum()) / max(int(changed.sum()), 1)
    print(f"\n{alt}: changes {int(changed.sum())} elements, rejected on {frac:.4f} of them")
    assert int(changed.sum()) >= 100 and frac >= 0.6, frac
