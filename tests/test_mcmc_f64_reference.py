"""CPU: pins the float64 MCMC restatement (tests/mcmc_f64.py) that the GPU tests compare the kernels against --
Philox against the Random123 known-answer vectors, the relocation ratio o/D against a 50-digit evaluation of the
double-sum definition, the update's identities, the sampling rule and the regulariser gradient against autograd."""
import math
import os
import sys
from decimal import Decimal, localcontext

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mcmc_f64 as ref  # noqa: E402


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = tuple(int(w) for w in ref.philox(*ctr, *key))
    assert got == want, [hex(g) for g in got]


def test_uniforms_and_normals_are_exact_functions_of_the_words():
    w = ref.draws(4096, seed=0x123456789abcdef, step=7, tag=1)
    u = ref.uniform(w[:, 0], w[:, 1])
    assert (u >= 0).all() and (u < 1).all()
    # the 53-bit integer behind u is exact: u * 2^53 is an integer < 2^53
    assert np.array_equal(u * 2.0 ** 53, np.floor(u * 2.0 ** 53))
    assert ref.uniform(np.array([MAX := 0xffffffff], np.uint64), np.array([MAX], np.uint64))[0] == 1 - 2.0 ** -53
    z = ref.normals(w)
    assert np.isfinite(z).all() and abs(z.mean()) < 0.05 and abs(z.std() - 1) < 0.05
    # u1 = 1 (a >> 8 = 2^24 - 1) gives a zero radius; the smallest u1 = 2^-24 the largest one
    zc, _ = ref.box_muller(np.array([0xffffffff], np.uint64), np.array([0], np.uint64))
    assert zc[0] == 0
    zc, _ = ref.box_muller(np.array([0], np.uint64), np.array([0], np.uint64))
    assert zc[0] == pytest.approx(math.sqrt(48 * math.log(2)))


def _o_over_D_decimal(o, r):
    """o / D with D = sum_{i=1..r} sum_{k=0..i-1} C(i-1,k) (-1)^k / sqrt(k+1) alpha^(k+1), alpha = 1 - (1-o)^(1/r),
    at 50 significant digits."""
    with localcontext() as ctx:
        ctx.prec = 50
        od = Decimal(float(o))
        alpha = 1 - (1 - od) ** (Decimal(1) / Decimal(r))
        sq = [Decimal(k + 1).sqrt() for k in range(r)]
        pw = [alpha ** (k + 1) for k in range(r)]
        D = Decimal(0)
        for i in range(1, r + 1):
            for k in range(i):
                t = Decimal(math.comb(i - 1, k)) / sq[k] * pw[k]
                D += -t if k & 1 else t
        return od / D


OS = np.concatenate([np.geomspace(1e-3, 0.5, 6), 1 - np.geomspace(0.3, 1e-7, 6)])


@pytest.mark.parametrize("r", range(1, 52))
def test_ratio_against_a_50_digit_evaluation(r):
    alpha = -np.expm1(np.log1p(-OS) / r)
    got = OS / ref.relocation_D(alpha, r)
    want = np.array([float(_o_over_D_decimal(o, r)) for o in OS])
    rel = np.abs(got - want) / np.abs(want)
    assert rel.max() <= 1e-11, (r, rel.max())


def test_update_identities():
    o = np.float32(np.concatenate([np.geomspace(1e-3, 0.5, 50), 1 - np.geomspace(0.5, 1e-6, 50)]))
    s = np.float32(np.random.default_rng(0).uniform(-6, 0, (100, 3)))
    # r = 1: the Gaussian is unchanged (the new logit is logit(o) up to its fp32 rounding)
    lg, sc = ref.ratio_update(o, s, np.ones(100, int), 1e-9)
    assert np.array_equal(sc, s)
    o_new = 1 / (1 + np.exp(-lg.astype(np.float64)))
    assert np.allclose(o_new, o.astype(np.float64), rtol=2e-6, atol=0)
    # 1 - (1 - alpha)^r = o: r copies of the new opacity composite to the old one
    for r in (2, 3, 7, 51):
        alpha = -np.expm1(np.log1p(-o.astype(np.float64)) / r)
        assert np.allclose(-np.expm1(r * np.log1p(-alpha)), o.astype(np.float64), rtol=1e-13, atol=0)
    # the clamp: the logit never reaches the fp32 sigmoid's 1 and never falls below logit(min_opacity)
    lg, _ = ref.ratio_update(np.float32([1.0, 1e-4]), np.zeros((2, 3), np.float32), np.array([2, 51]), 0.005)
    assert np.isfinite(lg).all() and lg[1] == np.float32(math.log(0.005 / 0.995))


def test_sampling_rule_never_draws_a_zero_weight():
    rng = np.random.default_rng(3)
    o = rng.uniform(0, 1, 5000).astype(np.float32)
    o[rng.uniform(size=5000) < 0.3] = 0.001
    cdf = np.cumsum(ref.weights(o, 0.005))
    s, u = ref.draw_samples(cdf, 20000, 11, 600, ref.RELOCATE_TAG)
    assert (o[s] > 0.005).all() and (s < 5000).all()
    # the drawn frequencies follow the weights
    f = np.bincount(s, minlength=5000) / 20000.0
    w = ref.weights(o, 0.005) / cdf[-1]
    assert abs(f[w > 0].sum() - 1) < 1e-12 and np.corrcoef(f, w)[0, 1] > 0.5
    # ties at a boundary go to the first index above: u T == c_i draws i + 1
    assert ref.sample(np.array([1.0, 2.0, 3.0]), np.array([1 / 3])) == 1


def test_regulariser_gradient_against_autograd():
    rng = np.random.default_rng(1)
    n = 777
    logit = torch.tensor(rng.uniform(-6, 6, n), dtype=torch.float64, requires_grad=True)
    s = torch.tensor(rng.uniform(-7, 0, (n, 3)), dtype=torch.float64, requires_grad=True)
    loss = 0.01 * torch.sigmoid(logit).abs().mean() + 0.03 * torch.exp(s).abs().mean()
    loss.backward()
    go, gs = ref.regularizer_grad(torch.sigmoid(logit).detach().numpy(), s.detach().numpy(), 0.01, 0.03)
    assert np.allclose(go, logit.grad.numpy(), rtol=1e-14, atol=0)
    assert np.allclose(gs, s.grad.numpy(), rtol=1e-14, atol=0)


def test_relocation_and_growth_of_a_set():
    rng = np.random.default_rng(2)
    n, K = 300, 4
    p = {"means": rng.standard_normal((n, 3)).astype(np.float32),
         "scales": rng.uniform(-5, -1, (n, 3)).astype(np.float32),
         "quats": rng.standard_normal((n, 4)).astype(np.float32),
         "opacities": rng.uniform(-8, 3, (n, 1)).astype(np.float32),
         "coeffs": rng.standard_normal((n, K, 3)).astype(np.float32)}
    m = {k: rng.standard_normal(t.shape).astype(np.float32) for k, t in p.items()}
    v = {k: rng.uniform(0, 1, t.shape).astype(np.float32) for k, t in p.items()}
    o = (1 / (1 + np.exp(-p["opacities"][:, 0].astype(np.float64)))).astype(np.float32)
    m0 = {k: t.copy() for k, t in m.items()}
    out = ref.relocate(p, m, v, o, 600, 5, 0.005)
    dead = out["dead"]
    assert out["n_dead"] == (o <= 0.005).sum() > 0
    for k in p:
        assert np.array_equal(p[k][dead], p[k][out["samples"]])
        assert np.array_equal(m[k][dead], m0[k][dead])            # the dead rows' moments are kept (gsplat)
        assert not m[k][out["samples"]].any()                     # the drawn rows' moments are zeroed
    o2 = (1 / (1 + np.exp(-p["opacities"][:, 0].astype(np.float64)))).astype(np.float32)
    assert (o2 > 0.005 * 0.999).all()
    new_p, new_m, new_v, info = ref.grow(p, m, v, o2, 600, 5, 0.005, 10 ** 6)
    assert info["added"] == int(1.05 * n) - n and new_p["means"].shape[0] == int(1.05 * n)
    assert not new_m["means"][n:].any() and np.array_equal(new_p["coeffs"][n:], p["coeffs"][info["samples"]])
