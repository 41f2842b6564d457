"""A float64 restatement of the bilateral-grid kernels (csrc/bilagrid.cu, DESIGN D21) with an fp32 error bound for
each output, derived from the kernels' operation order.

Inputs are what the kernels see: grids channels-last [L,Y,X,12] (or [N,L,Y,X,12]) and fp32 images.  The pixel
coordinates gx, gy, the luma z and gz = clamp(z, 0, 1)(L - 1) are computed in numpy float32, operation by operation as
the kernels round them (no contraction), so both sides choose the same cell; from there everything is float64.

Bounds (u = 2^-24), each an upper bound on |kernel - reference|:
 * slice: coef_k is 8 fmas over weights w = (wz wy) wx (three roundings each), out_c three more fmas: |err| <=
   32 u sum_j |A|_cj |x_j| with x = (r, g, b, 1) and |A| the coefficients interpolated from |G| (about 2.3x the first-
   order count).
 * v_rgb: the same, over |A|^T |v| plus the luma path 7 |lw_j| sum_c |v_c| (|dA|_c |x|), |dA| interpolated from
   |G_z0| + |G_z0+1|.
 * v_grid: each float is a sequential fp32 sum of at most CHUNK pixel terms per (cell, chunk) slot, then of at most
   4 * chunks slots, then scale times it added: |err| <= (CHUNK + 4 chunks + 8) u sum |terms| (the terms' own four
   roundings included), times 1.01.
 * TV gradient: at most six fmas of fp32 differences, inv_a rounded to fp32, times the weight: 12 u sum |terms|.
 * TV value: fp32 differences squared and summed in fp64, rounded once: 4 u TV."""
import math

import numpy as np

X, Y, L, NC = 16, 16, 8, 12
U = 2.0 ** -24
CHUNK = 4 * L * 4 * NC         # bilagrid.cu: CHUNK = 4 * BT, BT = L * 4 * 12
LUMA32 = (np.float32(0.299), np.float32(0.587), np.float32(0.114))
f32 = np.float32


def chunks(H, W):
    """bilagrid.cu chunks_for: (cell, chunk) slots per spatial cell."""
    nx, ny = min(W, W // (X - 1) + 2), min(H, H // (Y - 1) + 2)
    return -(-(nx * ny) // CHUNK)


def identity(n=None):
    g = np.zeros((L, Y, X, NC))
    g[..., 0] = g[..., 5] = g[..., 10] = 1.0
    return g if n is None else np.repeat(g[None], n, 0)


def axis32(n, cells):
    """fp32 g = ((p + 0.5) / n)(cells - 1) for p < n."""
    p = np.arange(n, dtype=f32)
    return ((p + f32(0.5)) / f32(n) * f32(cells - 1)).astype(f32)


def luma32(rgb):
    rgb = np.asarray(rgb, dtype=f32)
    return ((LUMA32[0] * rgb[..., 0] + LUMA32[1] * rgb[..., 1]) + LUMA32[2] * rgb[..., 2]).astype(f32)


def gz32(z):
    return (np.clip(z, f32(0), f32(1)).astype(f32) * f32(L - 1)).astype(f32)


def locate(rgb):
    """Per pixel of an fp32 [H,W,3] image: integer cells (x0, y0, z0), fractions (fx, fy, fz) in f64, the fp32 luma z
    and fp32 coordinates (gx, gy, gz), all [H,W]."""
    H, W = rgb.shape[:2]
    gx = np.broadcast_to(axis32(W, X)[None, :], (H, W)).astype(np.float64)
    gy = np.broadcast_to(axis32(H, Y)[:, None], (H, W)).astype(np.float64)
    z = luma32(rgb)
    gz = gz32(z).astype(np.float64)
    x0 = np.minimum(np.floor(gx).astype(int), X - 2)
    y0 = np.minimum(np.floor(gy).astype(int), Y - 2)
    z0 = np.minimum(np.floor(gz).astype(int), L - 2)
    return dict(x0=x0, y0=y0, z0=z0, fx=gx - x0, fy=gy - y0, fz=gz - z0, z=z, gx=gx, gy=gy, gz=gz)


def _corners(s):
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                w = ((s["fz"] if dz else 1 - s["fz"]) * (s["fy"] if dy else 1 - s["fy"])
                     * (s["fx"] if dx else 1 - s["fx"]))
                yield dz, dy, dx, w


def _interp(grid, s):
    coef, coef_abs = 0.0, 0.0
    for dz, dy, dx, w in _corners(s):
        g = grid[s["z0"] + dz, s["y0"] + dy, s["x0"] + dx]           # [H,W,12]
        coef = coef + w[..., None] * g
        coef_abs = coef_abs + w[..., None] * np.abs(g)
    return coef.reshape(coef.shape[:2] + (3, 4)), coef_abs.reshape(coef.shape[:2] + (3, 4))


def _dz(grid, s):
    d, d_abs = 0.0, 0.0
    for dy in (0, 1):
        for dx in (0, 1):
            w = (s["fy"] if dy else 1 - s["fy"]) * (s["fx"] if dx else 1 - s["fx"])
            g0 = grid[s["z0"], s["y0"] + dy, s["x0"] + dx]
            g1 = grid[s["z0"] + 1, s["y0"] + dy, s["x0"] + dx]
            d = d + w[..., None] * (g1 - g0)
            d_abs = d_abs + w[..., None] * (np.abs(g1) + np.abs(g0))
    return d.reshape(d.shape[:2] + (3, 4)), d_abs.reshape(d.shape[:2] + (3, 4))


def _x1(rgb):
    return np.concatenate([np.asarray(rgb, np.float64), np.ones(rgb.shape[:2] + (1,))], -1)


def slice_forward(grid, rgb):
    """(out [H,W,3], bound [H,W,3]) for one grid [L,Y,X,12] and an fp32 image [H,W,3]."""
    s = locate(rgb)
    A, A_abs = _interp(np.asarray(grid, np.float64), s)
    x = _x1(rgb)
    out = np.einsum("hwcj,hwj->hwc", A, x)
    bound = 32 * U * np.einsum("hwcj,hwj->hwc", A_abs, np.abs(x))
    return out, bound


def slice_backward(grid, rgb, v_out):
    """(v_rgb [H,W,3], v_rgb bound, v_grid [L,Y,X,12], v_grid bound) of out = slice(grid, rgb) for the cotangent
    v_out (fp32 [H,W,3]), at scale 1."""
    grid = np.asarray(grid, np.float64)
    H, W = rgb.shape[:2]
    s = locate(rgb)
    A, A_abs = _interp(grid, s)
    dA, dA_abs = _dz(grid, s)
    x, v = _x1(rgb), np.asarray(v_out, np.float64)
    inside = (s["z"] > 0) & (s["z"] < 1)
    dz = np.where(inside, (L - 1) * np.einsum("hwc,hwcj,hwj->hw", v, dA, x), 0.0)
    dz_abs = np.where(inside, (L - 1) * np.einsum("hwc,hwcj,hwj->hw", np.abs(v), dA_abs, np.abs(x)), 0.0)
    lw = np.array([float(c) for c in LUMA32])
    v_rgb = np.einsum("hwcj,hwc->hwj", A[..., :3], v) + lw * dz[..., None]
    b_rgb = 32 * U * (np.einsum("hwcj,hwc->hwj", A_abs[..., :3], np.abs(v)) + lw * dz_abs[..., None])
    v_grid = np.zeros((L, Y, X, NC))
    t_abs = np.zeros((L, Y, X, NC))
    vx = (v[..., :, None] * x[..., None, :]).reshape(H, W, NC)          # v_c x_j at 4c + j
    for dz_, dy, dx, w in _corners(s):
        idx = (s["z0"] + dz_, s["y0"] + dy, s["x0"] + dx)
        t = w[..., None] * vx
        np.add.at(v_grid, idx, t)
        np.add.at(t_abs, idx, np.abs(t))
    b_grid = 1.01 * (CHUNK + 4 * chunks(H, W) + 8) * U * t_abs
    return v_rgb, b_rgb, v_grid, b_grid


def _diffs(grids):
    """The fp32 neighbour differences along x, y and l of channels-last grids [N,L,Y,X,12], as f64."""
    g = np.asarray(grids, f32)
    return [(np.diff(g, axis=a).astype(f32)).astype(np.float64) for a in (3, 2, 1)]


def tv(grids):
    """(TV value, its bound, dTV/dG [N,L,Y,X,12], gradient bound) at weight 1."""
    g = np.asarray(grids, np.float64)
    n = g.shape[0]
    value, grad, g_abs = 0.0, np.zeros_like(g), np.zeros_like(g)
    d32 = _diffs(grids)
    for a, axis in enumerate((3, 2, 1)):
        d = np.diff(g, axis=axis)
        cnt = d.size
        value += float((d32[a] ** 2).sum()) / cnt
        t = 2.0 * d / cnt
        sl_lo = [slice(None)] * 5
        sl_hi = [slice(None)] * 5
        sl_lo[axis], sl_hi[axis] = slice(0, -1), slice(1, None)
        grad[tuple(sl_hi)] += t          # (G - G_prev) on the later element
        grad[tuple(sl_lo)] -= t          # -(G_next - G) on the earlier one
        g_abs[tuple(sl_hi)] += np.abs(t)
        g_abs[tuple(sl_lo)] += np.abs(t)
    assert n >= 1
    return value, 4 * U * value + 1e-45, grad, 12 * U * g_abs


def tv_definition(grids_gs):
    """TV of grids in gsplat order [N,12,L,Y,X], written from its definition (f64)."""
    g = np.asarray(grids_gs, np.float64)
    return sum(float(np.mean(np.diff(g, axis=a) ** 2)) for a in (4, 3, 2))


def learning_rate(step, lr=2e-3, final=0.01, w0=0.01, warmup=1000, max_steps=30000):
    s = step - 1
    return lr * final ** (s / max_steps) * (w0 + (1 - w0) * min(s, warmup) / warmup)


def lr_bound(step, **kw):
    """The fp32 learning-rate argument is one rounding of the f64 value the host computes."""
    return U * abs(learning_rate(step, **kw)) + math.ulp(learning_rate(step, **kw))
