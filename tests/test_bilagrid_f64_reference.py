"""CPU: pins the float64 restatement of the bilateral-grid kernels (bilagrid_f64.py) against torch float64 autograd
of F.grid_sample(align_corners=True, padding_mode="border") plus the affine map, and its TV against the definition,
at z = 0, z = 1, an interior cell boundary, pure black and white pixels, 1x1 and non-square images.  It also shows
the comparison rejects four wrong conventions: the align_corners=False pixel mapping, a v_rgb without the luma path,
column-major coefficients and a TV normalised per grid."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bilagrid_f64 as ref  # noqa: E402

f32 = np.float32


def tie_grey(k):
    """A near-grey pixel (fp32) whose luma gives gz = k exactly, 0 < z < 1 (its blue channel stepped by ulps)."""
    c = f32(k / 7.0)
    px = np.array([[[c, c, c]]], f32)
    for _ in range(4096):
        g = ref.gz32(ref.luma32(px))[0, 0]
        if g == k:
            return px[0, 0].copy()
        px[0, 0, 2] = np.nextafter(px[0, 0, 2], f32(2) if g < k else f32(-1), dtype=f32)
    raise AssertionError(k)


def make_case(H, W, seed):
    rng = np.random.default_rng(seed)
    rgb = rng.uniform(0, 1, (H, W, 3)).astype(f32)
    flat = rgb.reshape(-1, 3)
    special = [np.zeros(3, f32), np.ones(3, f32), np.array([0, 0.5, 1], f32), np.array([1, 0, 0], f32)]
    special += [tie_grey(k) for k in (1, 3, 6)]
    for i, v in enumerate(special[:flat.shape[0]]):
        flat[(i * 7) % flat.shape[0]] = v
    grid = ref.identity() + rng.normal(0, 0.1, (ref.L, ref.Y, ref.X, ref.NC))
    v = rng.normal(0, 1, (H, W, 3)).astype(f32)
    return grid, rgb, v


def torch_slice(grid, rgb, v, align_corners=True, column_major=False):
    """out, v_rgb, v_grid [L,Y,X,12] by torch f64 autograd through F.grid_sample."""
    H, W = rgb.shape[:2]
    s = ref.locate(rgb)
    G = torch.tensor(np.transpose(grid, (3, 0, 1, 2))[None], dtype=torch.float64, requires_grad=True)
    x = torch.tensor(rgb, dtype=torch.float64, requires_grad=True)
    lw = torch.tensor([float(c) for c in ref.LUMA32], dtype=torch.float64)
    zlin = (x * lw).sum(-1)
    z32 = torch.tensor(s["z"].astype(np.float64))
    inside = (z32 > 0) & (z32 < 1)
    # the fp32 gz the kernels compute, carried with the luma's derivative
    zval = torch.where(inside, torch.tensor(s["gz"]) / (ref.L - 1), z32)
    zt = zval + (zlin - zlin.detach())
    xn = torch.tensor(s["gx"] / (ref.X - 1) * 2 - 1)
    yn = torch.tensor(s["gy"] / (ref.Y - 1) * 2 - 1)
    coords = torch.stack([xn, yn, 2 * zt - 1], -1).view(1, 1, H, W, 3)
    coef = F.grid_sample(G, coords, mode="bilinear", align_corners=align_corners, padding_mode="border")
    coef = coef[0, :, 0].permute(1, 2, 0)
    A = coef.reshape(H, W, 4, 3).transpose(-1, -2) if column_major else coef.reshape(H, W, 3, 4)
    out = (A[..., :3] * x[..., None, :]).sum(-1) + A[..., 3]
    (out * torch.tensor(v, dtype=torch.float64)).sum().backward()
    return (out.detach().numpy(), x.grad.numpy(), np.transpose(G.grad[0].numpy(), (1, 2, 3, 0)))


def close(a, b, tol=1e-11):
    return float(np.abs(a - b).max()) <= tol * max(1.0, float(np.abs(b).max()))


CASES = [(1, 1), (5, 7), (7, 5), (13, 40), (48, 64)]


@pytest.mark.parametrize("H,W", CASES)
def test_slice_and_gradients_match_grid_sample_autograd(H, W):
    grid, rgb, v = make_case(H, W, H * 100 + W)
    out, ob = ref.slice_forward(grid, rgb)
    v_rgb, rb, v_grid, gb = ref.slice_backward(grid, rgb, v)
    t_out, t_vrgb, t_vgrid = torch_slice(grid, rgb, v)
    assert close(out, t_out) and close(v_rgb, t_vrgb) and close(v_grid, t_vgrid)
    assert (ob > 0).all() and (rb >= 0).all() and (gb >= 0).all()


def test_tie_rules():
    """z <= 0 and z >= 1 (black, white) carry no luma derivative; at an interior integer gz = k it is the forward
    difference of cells k and k + 1."""
    grid = ref.identity()
    grid[..., 3] = np.arange(ref.L)[:, None, None] ** 2 * 0.01           # b_r = 0.01 l^2: dout_r/dgz per cell
    cells = [np.zeros(3, f32), np.ones(3, f32)] + [tie_grey(k) for k in (1, 3, 6)]
    rgb = np.stack(cells)[None].astype(f32)
    v = np.zeros_like(rgb)
    v[..., 0] = 1.0
    v_rgb, _, _, _ = ref.slice_backward(grid, rgb, v)
    _, t_vrgb, _ = torch_slice(grid, rgb, v)
    assert close(v_rgb, t_vrgb)
    lw = np.array([float(c) for c in ref.LUMA32])
    for i, k in enumerate([None, None, 1, 3, 6]):
        dz = 0.0 if k is None else 7 * 0.01 * ((k + 1) ** 2 - k ** 2)
        assert np.allclose(v_rgb[0, i], np.array([1.0, 0, 0]) + lw * dz, rtol=1e-12, atol=1e-12), i


def test_tv_matches_its_definition():
    rng = np.random.default_rng(3)
    grids = ref.identity(3) + rng.normal(0, 0.1, (3, ref.L, ref.Y, ref.X, ref.NC))
    gs = np.transpose(grids, (0, 4, 1, 2, 3))
    value, vb, grad, gb = ref.tv(grids)
    want = ref.tv_definition(gs)
    assert abs(value - want) <= 1e-6 * want                 # the restatement squares the fp32 differences
    G = torch.tensor(gs, requires_grad=True)
    tv = sum(torch.mean(torch.diff(G, dim=a) ** 2) for a in (4, 3, 2))
    tv.backward()
    assert abs(float(tv) - want) <= 1e-13 * want
    assert close(grad, np.transpose(G.grad.numpy(), (0, 2, 3, 4, 1)), 1e-13)
    assert vb > 0 and (gb >= 0).all()


# ---- the comparison rejects wrong conventions ---------------------------------------------------------------------
def _excess(got, want, bound):
    return float((np.abs(got - want) / np.maximum(bound, 1e-300)).max())


def test_rejects_align_corners_false():
    grid, rgb, v = make_case(13, 40, 1)
    out, ob = ref.slice_forward(grid, rgb)
    t_out, _, _ = torch_slice(grid, rgb, v, align_corners=False)
    assert _excess(t_out, out, ob) > 100


def test_rejects_v_rgb_without_the_luma_path():
    grid, rgb, v = make_case(13, 40, 2)
    v_rgb, rb, _, _ = ref.slice_backward(grid, rgb, v)
    s = ref.locate(rgb)
    A, _ = ref._interp(np.asarray(grid, np.float64), s)
    no_luma = np.einsum("hwcj,hwc->hwj", A[..., :3], v.astype(np.float64))
    assert _excess(no_luma, v_rgb, rb) > 100


def test_rejects_column_major_coefficients():
    grid, rgb, v = make_case(13, 40, 4)
    out, ob = ref.slice_forward(grid, rgb)
    t_out, _, _ = torch_slice(grid, rgb, v, column_major=True)
    assert _excess(t_out, out, ob) > 100


def test_rejects_tv_normalised_per_grid():
    rng = np.random.default_rng(5)
    grids = ref.identity(4) + rng.normal(0, 0.1, (4, ref.L, ref.Y, ref.X, ref.NC))
    gs = np.transpose(grids, (0, 4, 1, 2, 3))
    value, vb, _, _ = ref.tv(grids)
    per_grid = sum(ref.tv_definition(gs[i:i + 1]) for i in range(4))
    assert abs(per_grid - value) > 100 * vb


def test_learning_rate_schedule():
    assert ref.learning_rate(1) == pytest.approx(2e-3 * 0.01, rel=1e-15)
    assert ref.learning_rate(1001) == pytest.approx(2e-3 * 0.01 ** (1000 / 30000), rel=1e-15)
    assert ref.learning_rate(30000) == pytest.approx(2e-3 * 0.01 ** (29999 / 30000), rel=1e-15)
