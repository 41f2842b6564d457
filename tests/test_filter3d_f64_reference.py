"""CPU: the restatement of the 3-D smoothing filter (tests/filter3d_f64.py, DESIGN D24) against an independent
float64 transcription of Mip-Splatting's formulas, torch autograd and central differences, and the wrong conventions
it must reject."""
import math

import numpy as np
import pytest
import torch

import filter3d_f64 as ff
import project_f64 as pf
from opensplat_b200.model import Camera


def orbit_cameras(k, W=64, H=48, fx=60.0, radius=4.0, centred=True, seed=0):
    g = np.random.default_rng(seed)
    cams = []
    for j in range(k):
        th = 2 * math.pi * j / k
        eye = np.array([radius * math.cos(th), 0.5 * (j % 3 - 1), radius * math.sin(th)])
        fwd = -eye / np.linalg.norm(eye)
        right = np.cross(fwd, [0.0, 1.0, 0.0])
        right /= np.linalg.norm(right)
        up = np.cross(right, fwd)
        c2w = np.eye(4)
        # camera_setup flips y / z (the reference's convention): camera axes right, up, -forward
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, eye
        f = fx * (1.0 + 0.3 * (j % 2))
        cx, cy = (W / 2, H / 2) if centred else (W / 2 + g.uniform(-8, 8), H / 2 + g.uniform(-6, 6))
        cams.append(Camera(W, H, f, f * 1.05, cx, cy, c2w))
    return cams


def mip_cams(table):
    """(R, T, fx, fy, W, H) of Mip-Splatting's cameras from a camera table: xyz @ R + T = V[:3,:3] xyz + V[:3,3]."""
    out = []
    for c in table.astype(np.float64):
        V = c[:12].reshape(3, 4)
        out.append((V[:, :3].T, V[:, 3], c[12], c[13], c[16], c[17]))
    return out


def gaussians(n, seed, spread=2.5):
    g = np.random.default_rng(seed)
    return (g.normal(size=(n, 3)) * spread).astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1])
def test_matches_mip_splatting_at_centred_cameras(seed):
    table = ff.camera_rows(orbit_cameras(7, seed=seed))
    means = gaussians(3000, seed)
    # S is float32(sqrt(float32(0.2))) here, sqrt(0.2) there
    ref = ff.mip_splatting_filter(means, mip_cams(table)) * (float(np.float32(math.sqrt(np.float32(0.2)))) /
                                                              math.sqrt(0.2))
    f64, cert = ff.filter_f64(means, table)
    f32 = ff.filter_fp32(means, table)
    assert cert.mean() > 0.99
    np.testing.assert_allclose(f64[cert], ref[cert], rtol=1e-12)
    np.testing.assert_allclose(f32[cert], ref[cert], rtol=1e-5)


def test_off_centre_cameras_use_their_principal_point():
    cams = orbit_cameras(5, centred=False, seed=3)
    table = ff.camera_rows(cams)
    means = gaussians(4000, 4)
    f64, cert = ff.filter_f64(means, table)
    f32 = ff.filter_fp32(means, table)
    np.testing.assert_allclose(f32[cert], f64[cert], rtol=1e-5)
    # Mip-Splatting's W/2 convention decides some Gaussians differently here
    centred = ff.mip_splatting_filter(means, mip_cams(table))
    assert (np.abs(centred - f64) > 1e-6 * np.abs(f64)).any()


def test_unseen_and_all_unseen():
    table = ff.camera_rows(orbit_cameras(4))
    means = np.concatenate([gaussians(200, 5, 0.5), np.full((3, 3), 1e4, np.float32)])
    f = ff.filter_fp32(means, table)
    seen = f[:200]
    assert (f[200:] == seen.max()).all() and (f[200:] > 0).all()
    assert (ff.filter_fp32(np.full((5, 3), 1e4, np.float32), table) == 0).all()


@pytest.mark.parametrize("alt", ["euclid", "min_focal", "no_margin", "unseen_zero"])
def test_rejects_wrong_filter_conventions(alt):
    table = ff.camera_rows(orbit_cameras(6))
    means = np.concatenate([gaussians(3000, 6), np.full((2, 3), 1e4, np.float32)])
    ref = ff.mip_splatting_filter(means, mip_cams(table))
    bad = ff.filter_fp32(means, table, alt=alt)
    assert np.abs(bad - ref).max() > 1e-3 * np.abs(ref).max(), alt


# ------------------------------------------------------------------------------------------------ projection VJP
def _cam():
    return pf.camera_from_setup(orbit_cameras(1, W=96, H=80)[0])


def _inputs(n, seed):
    g = np.random.default_rng(seed)
    means = torch.tensor(g.normal(size=(n, 3)) * 0.6, dtype=torch.float64)
    scales = torch.tensor(g.uniform(-5, -1, size=(n, 3)), dtype=torch.float64)
    quats = torch.tensor(g.normal(size=(n, 4)), dtype=torch.float64)
    logits = torch.tensor(g.normal(size=n), dtype=torch.float64)
    f = torch.tensor(g.uniform(0.001, 0.05, size=n), dtype=torch.float64)
    cot = [torch.tensor(g.normal(size=s), dtype=torch.float64) for s in ((n, 2), (n,), (n, 3), (n,))]
    return means, scales, quats, logits, f, cot


@pytest.mark.parametrize("aa", [False, True])
def test_closed_forms_match_autograd(aa):
    """The kernel's v_scale / v_logit closed forms equal autograd of the filtered map, given the sigma cotangent."""
    cam = _cam()
    means, scales, quats, logits, f, (vxy, vz, vc, vo) = _inputs(40, 1)
    kept = None
    s = scales.clone().requires_grad_()
    l = logits.clone().requires_grad_()
    a_eff, c3, o = ff.effective(s, l, f)
    sig = torch.exp(a_eff)
    sig_leaf = sig.detach().clone().requires_grad_()
    import project_aa_f64 as paa
    xy, tz, conic, _, _ = pf.forward_map(cam, means, torch.log(sig_leaf), quats, 1.0, True)
    comp = paa.comp_map(cam, means, torch.log(sig_leaf), quats)[0] if aa else None
    out = (xy * vxy).sum() + (conic * vc).sum() + (tz * vz).sum()
    if aa:
        out = out + (o.detach() * comp * vo).sum()
    (v_sigma,) = torch.autograd.grad(out, [sig_leaf])
    g_s, g_l = ff.filtered_vjp(cam, means, scales, quats, logits, f, vxy, vz, vc, vo, aa=aa, kept=kept)[1::2]
    v_a, v_l = ff.vjp_terms(scales, logits, f, v_sigma.numpy(), vo.numpy(),
                            comp=comp.detach().numpy() if aa else None)
    np.testing.assert_allclose(v_a, g_s.numpy(), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(v_l, g_l.numpy(), rtol=1e-9, atol=1e-12)


def test_vjp_matches_central_differences():
    cam = _cam()
    means, scales, quats, logits, f, (vxy, vz, vc, vo) = _inputs(6, 2)
    g = ff.filtered_vjp(cam, means, scales, quats, logits, f, vxy, vz, vc, vo, aa=True)

    def loss(m, s, q, l):
        xy, tz, conic, o = ff.filtered_map(cam, m, s, q, l, f, aa=True)
        return float((xy * vxy).sum() + (conic * vc).sum() + (tz * vz).sum() + (o * vo).sum())
    base = [means, scales, quats, logits]
    h = 1e-6
    for k in range(4):
        flat = base[k].reshape(-1)
        for idx in range(0, flat.numel(), 3):
            up = [b.clone() for b in base]
            dn = [b.clone() for b in base]
            up[k].reshape(-1)[idx] += h
            dn[k].reshape(-1)[idx] -= h
            fd = (loss(*up) - loss(*dn)) / (2 * h)
            assert abs(fd - float(g[k].reshape(-1)[idx])) <= 1e-5 * (1 + abs(fd)), (k, idx)


@pytest.mark.parametrize("alt", ["scale_add", "logscale_add", "no_sqrt", "sqrt_twice"])
def test_rejects_wrong_effective_gaussian(alt):
    scales = torch.tensor([[-3.0, -2.0, -4.0]], dtype=torch.float64)
    logits = torch.tensor([0.3], dtype=torch.float64)
    f = torch.tensor([0.03], dtype=torch.float64)
    a, c3, o = ff.effective(scales, logits, f)
    a2, c32, o2 = ff.effective(scales, logits, f, alt)
    # the definitions: sigma^2 = e^2 + f^2, c3 = sqrt(det(diag e^2) / det(diag e^2 + f^2))
    e2 = torch.exp(2 * scales)
    assert torch.allclose(torch.exp(2 * a), e2 + f[:, None] ** 2, rtol=1e-14)
    assert torch.allclose(c3, torch.sqrt(e2.prod(-1) / (e2 + f[:, None] ** 2).prod(-1)), rtol=1e-14)
    assert not (torch.allclose(a, a2, rtol=1e-6) and torch.allclose(c3, c32, rtol=1e-6))


def test_f_zero_is_the_identity():
    scales = np.linspace(-20, 20, 41).repeat(3).reshape(-1, 3).astype(np.float32)
    assert (ff.c3_fp32(scales, np.zeros(len(scales), np.float32)) == 1).all()


def test_one_minus_r_squared_cancels():
    """At log-scale -12 (e ~ 6.1e-6) with a filter a few thousand times smaller, the opacity's share of the scale
    gradient, (f / sigma)^2 ~ 1e-8, is exact to a few ulp in the kernel's form, while 1 - r^2 loses every digit."""
    a = np.float32(-12.0)
    e = np.exp(a, dtype=np.float32)
    for f in (np.float32(1e-9), np.float32(3e-10)):
        sig = np.sqrt(e * e + f * f, dtype=np.float32)
        r = e / sig
        good = (f / sig) * (f / sig)
        bad = np.float32(1) - r * r
        exact = 1.0 / (1.0 + (float(e) / float(f)) ** 2)
        assert abs(float(good) - exact) <= 8 * ff.EPS32 * exact
        assert abs(float(bad) - exact) >= 0.5 * exact           # no correct digit left
    # the float64 closed forms agree with each other where nothing cancels
    scales = np.array([[-12.0, -3.0, 0.5]])
    v1, _ = ff.vjp_terms(scales, np.array([0.2]), np.array([1e-5]), np.ones((1, 3)), np.array([1.0]))
    v2, _ = ff.vjp_terms(scales, np.array([0.2]), np.array([1e-5]), np.ones((1, 3)), np.array([1.0]), cancel=True)
    np.testing.assert_allclose(v1, v2, rtol=1e-6)


# ------------------------------------------------------------------------------------------------ reset and bake
def test_reset_matches_definition():
    g = np.random.default_rng(7)
    n = 2000
    scales = g.uniform(-6, 0, size=(n, 3)).astype(np.float32)
    logits = g.normal(size=n).astype(np.float32) * 3
    f = np.where(g.uniform(size=n) < 0.3, 0, g.uniform(0, 0.05, size=n)).astype(np.float32)
    max_logit = float(torch.logit(torch.tensor(0.2, dtype=torch.float32)))
    out = ff.reset_f64(logits, scales, f, 0.2, max_logit)
    c3 = ff.c3_fp32(scales, f).astype(np.float64)
    # effective opacity after the reset never exceeds r (beyond one fp32 rounding of the logit)
    o_eff = c3 / (1 + np.exp(-out.astype(np.float64)))
    assert (o_eff <= 0.2 * (1 + 1e-6)).all()
    # untouched where already below; equal to the plain reset where c3 == 1
    below = c3 / (1 + np.exp(-logits.astype(np.float64))) < 0.2 * (1 - 1e-6)
    assert (out[below] == logits[below]).all()
    one = c3 == 1
    assert one.any() and (out[one] == np.minimum(logits[one], np.float32(max_logit))).all()


def test_bake_matches_definition():
    g = np.random.default_rng(8)
    n = 500
    scales = g.uniform(-8, 1, size=(n, 3))
    logits = g.normal(size=n) * 4
    f = g.uniform(0, 0.1, size=n)
    a, l = ff.bake_f64(scales, logits, f)
    # the baked Gaussian has the filtered covariance and the effective opacity
    np.testing.assert_allclose(np.exp(2 * a), np.exp(2 * scales) + f[:, None] ** 2, rtol=1e-12)
    c3 = np.sqrt(np.exp(2 * scales) / (np.exp(2 * scales) + f[:, None] ** 2)).prod(-1)
    np.testing.assert_allclose(1 / (1 + np.exp(-l)), c3 / (1 + np.exp(-logits)), rtol=1e-10)
