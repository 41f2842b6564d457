"""Pins tests/fused_f64.py, the float64 reference the GPU tests of csrc/fused.cu are held to (CPU only):
  * each bound's evaluation (the kernel's operation tree on value-plus-bound numbers) has the value of the plain
    formula or of float64 autograd to float64 precision, so the bound is taken along the right computation;
  * the reference's own numbers lie within C_GOLD B per element: torch.optim.Adam (CPU float32, foreach=False) one
    step at a time over several steps with the state fed forward, float32 torch autograd of exp, normalize and sigmoid,
    and oracle/scene_edit.densify_stats, whose counts and maxima must match exactly;
  * the check rejects each known wrong convention on most of the elements that convention changes."""
import math

import numpy as np
import pytest
import torch

import fused_f64 as ff
from oracle import scene_edit

F8 = torch.float64
# first-order bound: the factor 2 covers the second-order terms and the u |exact| charged where fp32 rounds u |computed|
C_BOUND = 2.0
# torch.optim.Adam and torch's float32 autograd evaluate the same maps in their own order (Adam: exp_avg by lerp, the
# step as (step_size m) / den), so their rounding is not the one B follows; the tolerance is 4 B.
C_GOLD = 4.0


def _ratio(got, want, bound, mask=None):
    got = got.double() if torch.is_tensor(got) else torch.as_tensor(np.asarray(got, np.float64))
    err = (got - want).abs()
    if mask is not None:
        err, bound = err[mask], bound[mask]
    ok = bool((err <= bound).all())
    return ok, float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _rejects(alt_v, ref_v, bound, what):
    """The alternative fails |alt - reference| <= C_BOUND B on >= 60 % of the elements it changes (>= 100 of them)."""
    d = (alt_v - ref_v).abs()
    changed = d > 1e-12 * (ref_v.abs() + bound / ff.U)
    frac = float((changed & (d > C_BOUND * bound)).sum()) / max(int(changed.sum()), 1)
    print(f"\n{what}: changes {int(changed.sum())} elements, rejected on {frac:.4f} of them")
    assert int(changed.sum()) >= 100 and frac >= 0.6, frac


# ------------------------------------------------------------------------------------------------ Adam
def adam_state(n, seed, gmin=-30.0, gmax=2.0):
    """fp32 (p, g, m, v): |g| log-uniform in [10^gmin, 10^gmax] with random signs and 5 % exact zeros; a state
    as after some steps (m ~ 0.1 |g|-ish, v ~ 1e-3 g^2-ish, each log-spread)."""
    rng = np.random.default_rng(seed)
    mag = 10.0 ** rng.uniform(gmin, gmax, n)
    g = np.where(rng.uniform(size=n) < 0.05, 0.0, mag * rng.choice([-1.0, 1.0], n))
    p = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1, n)
    m = 0.1 * g * 10.0 ** rng.uniform(-1, 1, n)
    v = 1e-3 * g * g * 10.0 ** rng.uniform(-1, 1, n)
    return [np.asarray(x, np.float32) for x in (p, g, m, v)]


@pytest.mark.parametrize("t", [1, 2, 10, 1000, 30000])
def test_adam_bound_evaluation_is_the_plain_value(t):
    p, g, m, v = (torch.as_tensor(x, dtype=F8) for x in adam_state(20000, t))
    r = ff.adam(p, g, m, v, 1.6e-4, t)
    pp, mp, vp = ff.adam_plain(p, g, m, v, 1.6e-4, t)
    assert not bool(r["ovf"].any()) and bool(r["cert"].all())
    assert bool(((r["re_p"] - pp).abs() <= 1e-6 * r["B_p"]).all())
    assert bool(((r["p"] - pp).abs() <= 1e-6 * r["B_p"]).all())
    assert torch.equal(r["m"], mp) and torch.equal(r["v"], vp)
    assert bool((r["B_p"] > 0).all())


def test_adam_overflow_is_a_certified_decision():
    """|g| past sqrt(FLT_MAX / (1 - b2)) ~ 5.8e20 from v = 0: v' = inf and p unchanged; a state already at inf stays
    there.  A gradient at the threshold itself is not certified."""
    thr = math.sqrt(ff.OVF / ff.f32(1 - 0.999))
    g = np.array([1e19, 1.8e19, 1e20, 5.7e20, 5.9e20, 1e21, 1e30, 1.0, thr], np.float32)
    n = g.size
    p = np.full(n, 0.25, np.float32)
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    v[7] = np.inf
    r = ff.adam(p, g, m, v, 1e-2, 3)
    assert r["ovf"].tolist() == [False, False, False, False, True, True, True, True, float(g[8]) ** 2 * ff.f32(
        1 - 0.999) >= ff.OVF]
    assert r["cert"][:8].all() and not bool(r["cert"][8])
    assert bool((r["p"][r["ovf"]] == 0.25).all()) and bool(torch.isinf(r["v"][r["ovf"]]).all())


def test_adam_torch_within_bound():
    """torch.optim.Adam on the CPU (float32, foreach=False), six steps with the state fed forward; each step
    restated from the fp32 state before it.  Gradients from 1e-30 to 1e19 with exact zeros, a large gradient followed
    by tiny ones, and overflowing ones (v = inf from then on, p frozen)."""
    n = 40000
    rng = np.random.default_rng(3)
    p0 = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1, n)).astype(np.float32)
    pt = torch.tensor(p0).requires_grad_()
    opt = torch.optim.Adam([pt], lr=1.6e-4, foreach=False)
    worst = 0.0
    for t in range(1, 7):
        mag = 10.0 ** rng.uniform(-30, 19, n)
        g = mag * rng.choice([-1.0, 1.0], n)
        g[rng.uniform(size=n) < 0.05] = 0.0
        g[:2000] = 1e3 if t == 1 else 1e-30 * t         # a large gradient, then tiny ones: v ~ 0 relative to m
        g[2000:2100] = 1e21 if t == 2 else 1.0           # overflow at step 2
        g = g.astype(np.float32)
        if t == 1:
            before = [p0, np.zeros(n, np.float32), np.zeros(n, np.float32)]
        else:
            st = opt.state[pt]
            before = [pt.detach().numpy().copy(), st["exp_avg"].numpy().copy(), st["exp_avg_sq"].numpy().copy()]
        r = ff.adam(before[0], g, before[1], before[2], 1.6e-4, t)
        pt.grad = torch.tensor(g)
        opt.step()
        st = opt.state[pt]
        assert bool(r["cert"].all())
        for key, got in (("p", pt.detach()), ("m", st["exp_avg"]), ("v", st["exp_avg_sq"])):
            exact = r["ovf"] if key != "m" else torch.zeros_like(r["ovf"])
            assert torch.equal(got.double()[exact], r[key][exact]), (t, key)
            ok, q = _ratio(got, r[key], C_GOLD * r["B_" + key], ~exact)
            assert ok, (t, key, q)
            worst = max(worst, q)
        assert t < 2 or bool(torch.isinf(st["exp_avg_sq"][2000:2100]).all())
    print(f"\ntorch.optim.Adam: worst err/B {worst * C_GOLD:.3f}")


@pytest.mark.parametrize("alt,t", [("eps_in_sqrt", 5), ("bc2_unsqrt", 5), ("no_bc", 5), ("no_bc", 1000)])
def test_adam_check_rejects_known_wrong_conventions(alt, t):
    p, g, m, v = adam_state(20000, 100 + t, gmin=-14, gmax=1)
    r = ff.adam(p, g, m, v, 1e-2, t)
    a = ff.adam(p, g, m, v, 1e-2, t, alt=alt)
    _rejects(a["p"], r["p"], r["B_p"], f"Adam {alt} t={t}")


def test_segment_rates():
    segs, n = ff.synthetic_segments(1)
    lr, inside = ff.segment_rates(n, segs)
    for o, c, row, head, lh, lrest in segs:
        for e in range(0, c, max(1, c // 97)):
            assert float(lr[o + e]) == (lh if e % row < head else lrest)
    assert int(inside.sum()) == sum(s[1] for s in segs) and not bool(inside[:4].any())


@pytest.mark.parametrize("alt", ["head_whole_row", "buffer_rows", "per_float4"])
def test_segmented_rate_check_rejects_known_wrong_conventions(alt):
    segs, n = ff.synthetic_segments(2)
    p, g, m, v = adam_state(n, 7, gmin=-2, gmax=1)
    lr, inside = ff.segment_rates(n, segs)
    bad = ff.segment_rates_alt(n, segs, alt)
    r = ff.adam(p, g, m, v, torch.where(inside, lr, 0.0), 4)
    a = ff.adam(p, g, m, v, torch.where(inside, bad, 0.0), 4)
    _rejects(a["p"][inside], r["p"][inside], r["B_p"][inside], f"segment rates {alt}")


# ------------------------------------------------------------------------------------------------ activations
def act_inputs(n, seed):
    """Log-scales in [-30, 88]; raw quaternions with norms 1e-15 .. 1e15, a quarter axis-aligned; logits in +-[0, 100]
    with exact zeros; means 1e-6 .. 1e6 from the camera."""
    rng = np.random.default_rng(seed)
    ls = rng.uniform(-30, 88, (n, 3))
    q = rng.standard_normal((n, 4))
    ax = rng.uniform(size=n) < 0.25
    q[ax] = 0.0
    q[ax, rng.integers(0, 4, int(ax.sum()))] = rng.choice([-1.0, 1.0], int(ax.sum()))
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * 10.0 ** rng.uniform(-15, 15, (n, 1))
    x = rng.uniform(-100, 100, n)
    x[rng.uniform(size=n) < 0.03] = 0.0
    cam = np.array([0.3, -2.7, 4.1], np.float32)
    d = rng.standard_normal((n, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 10.0 ** rng.uniform(-6, 6, (n, 1))
    means = cam.astype(np.float64) + d
    vs, vq, vo = rng.standard_normal((n, 3)), rng.standard_normal((n, 4)), rng.standard_normal(n)
    return [np.asarray(a, np.float32) for a in (means, ls, q, x, cam, vs, vq, vo)]


def test_activation_bound_evaluation_is_the_autograd_value():
    means, ls, q, x, cam, vs, vq, vo = act_inputs(20000, 1)
    r = ff.activate(means, ls, q, x, cam, vs, vq, vo)
    pl = r["plain"]
    for k in ("scales", "quats", "opacities", "viewdirs"):
        want = pl[k].reshape(r[k].shape)
        fin = torch.isfinite(r[k]) & (r[k] != 0) if k in ("scales", "opacities") else torch.ones_like(r[k], dtype=bool)
        assert bool(((r[k] - want).abs()[fin] <= 1e-6 * r["B_" + k][fin]).all()), k
    for k in ("v_log_scales", "v_raw_quats", "v_logits"):
        fin = torch.isfinite(r[k]) & (r[k] != 0)
        assert bool(((r["re_" + k] - r[k]).abs()[fin] <= 1e-6 * r["B_" + k][fin]).all()), k
        assert int(fin.sum()) > 1000


def test_activation_decisions():
    """exp overflow at log-scale ln(FLT_MAX) = 88.7228: +inf above, finite below; sigmoid saturation at logit
    -88.7228: exactly 0 with a VJP of exactly 0 below.  The fp32 neighbours of the threshold bracket it, and only
    those within 4 u of it may be uncertified."""
    s0 = np.float32(math.log(ff.FLT_MAX))
    near = np.array([np.nextafter(s0, -np.inf, dtype=np.float32), s0, np.nextafter(s0, np.inf, dtype=np.float32)])
    ls = np.array([80.0, 88.0, 88.7, 88.8, 89.0, 100.0, *near], np.float32)
    n = ls.size
    ls3 = np.repeat(ls[:, None], 3, 1)
    x = -ls
    means, q = np.ones((n, 3), np.float32), np.ones((n, 4), np.float32)
    r = ff.activate(means, ls3, q, x, np.zeros(3, np.float32), np.ones((n, 3), np.float32), np.ones((n, 4)),
                    np.ones(n, np.float32))
    assert r["s_ovf"][:, 0].tolist()[:6] == [False, False, False, True, True, True]
    assert r["o_zero"].tolist()[:6] == [False, False, False, True, True, True]
    assert bool(r["cert_s"][:6].all()) and bool(r["cert_o"][:6].all())
    assert bool(torch.isinf(r["scales"][3:6]).all()) and bool((r["opacities"][3:6] == 0).all())
    assert bool((r["v_logits"][3:6] == 0).all())
    assert int((~r["cert_s"][:, 0]).sum()) <= 2


def test_activation_torch_float32_within_bound():
    means, ls, q, x, cam, vs, vq, vo = act_inputs(20000, 2)
    ls = np.minimum(ls, 88.0)
    r = ff.activate(means, ls, q, x, cam, vs, vq, vo)
    assert bool(r["cert_vls"].all()) and int((~torch.isfinite(r["v_log_scales"])).sum()) > 0
    t = [torch.tensor(a).requires_grad_() for a in (ls, q, x)]
    sc, qn, op, vd = ff.act_map(torch.tensor(means), *t, torch.tensor(cam))
    ((sc * torch.tensor(vs)).sum() + (qn * torch.tensor(vq)).sum() + (op * torch.tensor(vo)).sum()).backward()
    worst = []
    for name, got in (("scales", sc), ("quats", qn), ("opacities", op), ("viewdirs", vd),
                      ("v_log_scales", t[0].grad), ("v_raw_quats", t[1].grad), ("v_logits", t[2].grad)):
        exact = ~torch.isfinite(r[name])                  # v * exp(s) overflowing to +-inf: the same in float32 torch
        assert torch.equal(got.detach().double()[exact], r[name][exact]), name
        ok, qr = _ratio(got.detach(), r[name], C_GOLD * r["B_" + name], ~exact)
        assert ok, (name, qr)
        worst.append(qr)
    print(f"\nfloat32 torch activations: worst err/B {max(worst) * C_GOLD:.3f}")


@pytest.mark.parametrize("alt,key", [("sig_oo", "v_logits"), ("sig_o1po", "v_logits"), ("q_no_proj", "v_raw_quats")])
def test_activation_check_rejects_known_wrong_conventions(alt, key):
    means, ls, q, x, cam, vs, vq, vo = act_inputs(20000, 3)
    x = (np.random.default_rng(4).standard_normal(x.size) * 3).astype(np.float32)   # where sigmoid is not saturated
    r = ff.activate(means, ls, q, x, cam, vs, vq, vo)
    a = ff.activate(means, ls, q, x, cam, vs, vq, vo, alt=alt)
    _rejects(a[key], r[key], r["B_" + key], f"activation {alt}")


# ------------------------------------------------------------------------------------------------ densification
def stats_inputs(n, seed, H=300, W=480):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 2)) * 10.0 ** rng.uniform(-15, 15, (n, 1))
    v[rng.uniform(size=n) < 0.03] = 0.0
    r = rng.integers(-1, 3000, n).astype(np.int32)
    r[rng.uniform(size=n) < 0.2] = 0
    return v.astype(np.float32), r


@pytest.mark.parametrize("H,W", [(300, 480), (481, 299)])
def test_densify_stats_reference_and_oracle(H, W):
    n = 20000
    v1, r1 = stats_inputs(n, 1)
    v2, r2 = stats_inputs(n, 2)
    st = ff.densify_stats(v1, r1, H, W)
    assert bool(((st["xys_grad_norm"] - st["plain"]).abs() <= 1e-6 * st["B_xys_grad_norm"]).all())
    o = scene_edit.densify_stats(None, v1, r1, H, W)
    ok, q1 = _ratio(o[0], st["xys_grad_norm"], C_GOLD * st["B_xys_grad_norm"])
    assert ok, q1
    assert torch.equal(o[1].double(), st["vis_counts"]) and torch.equal(o[2].double(), st["max_2d_size"])
    state32 = [x.float() for x in (o[0], o[1], o[2])]
    up = ff.densify_stats(v2, r2, H, W, state=state32)
    assert bool(((up["xys_grad_norm"] - up["plain"]).abs() <= 1e-6 * up["B_xys_grad_norm"] + 1e-300).all())
    o2 = scene_edit.densify_stats(state32, v2, r2, H, W)
    ok, q2 = _ratio(o2[0], up["xys_grad_norm"], C_GOLD * up["B_xys_grad_norm"] + (up["B_xys_grad_norm"] == 0) * 0)
    assert ok, q2
    assert torch.equal(o2[1].double(), up["vis_counts"]) and torch.equal(o2[2].double(), up["max_2d_size"])
    print(f"\ndensify stats {H}x{W}: worst err/B {max(q1, q2):.3f}")


def test_densify_stats_check_rejects_known_wrong_conventions():
    n, H, W = 20000, 300, 480
    v, r = stats_inputs(n, 5)
    good = ff.densify_stats(v, r, H, W)
    bad = ff.densify_stats(v, r, H, W, alt="min_hw")
    vis = torch.as_tensor(r > 0)
    assert bool((bad["max_2d_size"] != good["max_2d_size"])[vis].float().mean() > 0.99)
    state = [torch.full((n,), 7.0, dtype=torch.float32)] * 3
    bad = ff.densify_stats(v, r, H, W, state=state, alt="init_visible")
    assert bool((bad["vis_counts"] != good["vis_counts"])[~vis].all())
    assert bool(((bad["xys_grad_norm"] - good["xys_grad_norm"]).abs() > C_BOUND * good["B_xys_grad_norm"])[~vis]
                .float().mean() > 0.95)


# ------------------------------------------------------------------------------------------------ MSE
def test_mse_reference():
    rng = np.random.default_rng(0)
    n = 12345
    a = rng.uniform(0, 1, n).astype(np.float32)
    b = rng.uniform(0, 1, n).astype(np.float32)
    b[:100] = a[:100]
    inv = 1.0 / n
    r = ff.mse(a, b, inv, 132)
    d = a - b
    want = (np.float32(2) * np.float32(inv)) * d
    assert np.array_equal(r["v_img"].numpy(), want) and bool((r["v_img"][:100] == 0).all())
    exact = float(np.mean((a.astype(np.float64) - b) ** 2))
    assert abs(r["loss"] - exact) <= 1e-6 * r["B_loss"] + abs(ff.f32(inv) * n - 1) * exact
    ref32 = torch.nn.functional.mse_loss(torch.tensor(a), torch.tensor(b))
    assert abs(float(ref32) - r["loss"]) <= C_GOLD * r["B_loss"]
    bad = ff.mse(a, b, inv, 132, alt="no_two")
    assert bool((bad["v_img"] != r["v_img"])[100:].all())
