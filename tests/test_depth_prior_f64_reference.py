"""CPU: pins tests/depth_prior_f64.py (the restatement of csrc/depth.cu, DESIGN D23) against torch autograd of the
definitions -- the loss (|R - P| * mask).sum() / (H W) with its gradient, the chain through where(radii > 0, 1 / z, 0),
the mean-pool levels of a prior -- with ties R == P, invalid priors (0, negative, NaN, +-inf) and radii == 0; and
DepthConfig's validation and weight schedule."""
import math

import numpy as np
import pytest
import torch

import depth_prior_f64 as ref

F8 = torch.float64
BAD = [0.0, -1.0, float("nan"), float("inf"), float("-inf")]


def _maps(H, W, seed):
    """R and P with every kind of pixel: ordinary ones, ties R == P and each invalid prior."""
    rng = np.random.default_rng(seed)
    R = rng.uniform(0.0, 2.0, (H, W)).astype(np.float32)
    P = rng.uniform(0.01, 2.0, (H, W)).astype(np.float32)
    k = rng.integers(0, 8, (H, W))
    P = np.where(k == 0, R, P)                                   # ties
    for j, b in enumerate(BAD):
        P = np.where(k == j + 1, np.float32(b), P)
    return R, P.astype(np.float32)


def _autograd_loss(R, P, weight):
    r = torch.from_numpy(R).to(F8).requires_grad_()
    p = torch.from_numpy(P).to(F8)
    mask = torch.isfinite(p) & (p > 0)
    loss = ((r - torch.where(mask, p, 0.0)).abs() * mask).sum() / (R.shape[0] * R.shape[1])
    (weight * loss).backward()
    return float(loss.detach()), r.grad.numpy()


@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (64, 48)])
def test_loss_and_gradient_match_autograd(H, W):
    R, P = _maps(H, W, H * W)
    if H * W == 1:
        P[0, 0] = R[0, 0]
    want, grad = _autograd_loss(R, P, 0.37)
    loss, bound = ref.l1_loss_f64(R, P)
    # the fp32 terms |fp32(R - P)| differ from the exact |R - P| by at most u32 each
    assert abs(loss - want) <= bound + ref.U32 * want + 1e-300
    assert np.array_equal(ref.l1_grad_f64(R, P, 0.37), grad)
    g32 = np.float32(0.37 / (H * W))
    assert np.array_equal(ref.l1_grad_f32(R, P, g32).astype(np.float64), grad / (0.37 / (H * W)) * float(g32))
    # ties and invalid pixels take no gradient; every invalid kind is present on the larger maps
    dead = ~ref.valid(P) | (R == P)
    assert not ref.l1_grad_f32(R, P, g32)[dead].any()
    if H * W > 100:
        for b in BAD:
            assert (P == np.float32(b)).any() or (math.isnan(b) and np.isnan(P).any())


def test_all_invalid_gives_zero():
    R = np.ones((4, 6), np.float32)
    P = np.zeros((4, 6), np.float32)
    assert ref.l1_loss_f64(R, P)[0] == 0.0 and not ref.l1_grad_f32(R, P, 1.0).any()


def test_chain_matches_autograd():
    rng = np.random.default_rng(3)
    n = 4000
    z = np.exp(rng.uniform(np.log(0.01), np.log(1e4), n)).astype(np.float32)
    radii = rng.integers(0, 3, n).astype(np.int32)               # a third with radii == 0
    v = rng.normal(0, 1, n).astype(np.float32)
    zt = torch.from_numpy(z).to(F8).requires_grad_()
    inv = torch.where(torch.from_numpy(radii) > 0, 1.0 / zt, 0.0)
    (inv * torch.from_numpy(v).to(F8)).sum().backward()
    assert np.array_equal(ref.inverse_depths_f64(z, radii), inv.detach().numpy())
    assert np.allclose(ref.inverse_depths_backward_f64(z, radii, v), zt.grad.numpy(), rtol=1e-15, atol=0)
    # the fp32 chain: 1/z and -(v inv) inv, each rounding within u32 of float64
    i32 = ref.inverse_depths_f32(z, radii).astype(np.float64)
    i64 = ref.inverse_depths_f64(z, radii)
    assert np.all(np.abs(i32 - i64) <= ref.U32 * np.abs(i64))
    b32 = ref.inverse_depths_backward_f32(z, radii, v).astype(np.float64)
    b64 = zt.grad.numpy()
    assert np.all(np.abs(b32 - b64) <= 5 * ref.U32 * np.abs(b64) + 1e-300)
    assert not b32[radii == 0].any() and not i32[radii == 0].any()


@pytest.mark.parametrize("h,w,f", [(8, 8, 2), (17, 23, 4), (33, 31, 8), (5, 9, 1)])
def test_downscale_mean_matches_masked_average_pool(h, w, f):
    rng = np.random.default_rng(h * w + f)
    src = rng.uniform(0.1, 3.0, (h, w)).astype(np.float32)
    k = rng.integers(0, 6, (h, w))
    for j, b in enumerate(BAD):
        src = np.where(k == j + 1, np.float32(b), src)
    if h // f >= 2:
        src[:f, :f] = 0.0                                        # a block with no valid sample
    s = torch.from_numpy(src).to(F8)
    ok = torch.isfinite(s) & (s > 0)
    num = torch.nn.functional.avg_pool2d(torch.where(ok, s, 0.0)[None, None], f)[0, 0]
    den = torch.nn.functional.avg_pool2d(ok.to(F8)[None, None], f)[0, 0]
    want = torch.where(den > 0, num / den.clamp_min(1e-300), 0.0).numpy()
    got64, count = ref.downscale_mean_f64(src, f)
    assert got64.shape == (h // f, w // f)
    assert np.allclose(got64, want, rtol=1e-14, atol=0)
    got32 = ref.downscale_mean_f32(src, f).astype(np.float64)
    # f*f - 1 fp32 additions of positive terms and one division
    assert np.all(np.abs(got32 - want) <= (f * f + 1) * ref.U32 * want)
    if h // f >= 2:
        assert got32[0, 0] == 0.0 and count[0, 0] == 0


def test_depth_config_validation_and_weight_schedule():
    from opensplat_b200.depth import DepthConfig, depth_weight
    c = DepthConfig()
    assert (c.weight, c.final_weight_factor, c.max_steps) == (1.0, 0.01, 30_000)
    assert depth_weight(c, 1) == 1.0
    assert math.isclose(depth_weight(c, 15_001), 0.1, rel_tol=1e-12)
    assert math.isclose(depth_weight(c, 30_001), 0.01, rel_tol=1e-12)
    assert depth_weight(c, 90_000) == depth_weight(c, 30_001)       # held at the final value
    c2 = DepthConfig(weight=0.5, final_weight_factor=0.2, max_steps=10)
    for s in range(1, 30):
        assert depth_weight(c2, s) == 0.5 * 0.2 ** (min(s - 1, 10) / 10)
    assert DepthConfig(weight=0.0).weight == 0.0
    for kw in ({"weight": -1.0}, {"weight": float("nan")}, {"final_weight_factor": 0.0},
               {"final_weight_factor": -0.5}, {"max_steps": 0}, {"max_steps": 1.5}, {"max_steps": True}):
        with pytest.raises(ValueError):
            DepthConfig(**kw)
