"""Restatement of the inverse-depth prior kernels (csrc/depth.cu, DESIGN D23) in numpy fp32 (what the kernels compute,
rounding by rounding) and in float64 (what they approximate), taking the kernels' fp32 decisions as given: which
pixels are valid, the sign of R - P, which Gaussians have radii > 0.

A prior sample p is valid iff it is finite and > 0."""
import numpy as np

F4 = np.float32
U32 = 2.0 ** -24
U64 = 2.0 ** -53


def valid(p):
    p = np.asarray(p)
    return np.isfinite(p) & (p > 0)


# ---- fp32, rounding by rounding ---------------------------------------------------------------------------------------
def inverse_depths_f32(depths, radii):
    z = np.asarray(depths, F4)
    with np.errstate(divide="ignore", over="ignore"):
        return np.where(np.asarray(radii) > 0, F4(1.0) / z, F4(0.0)).astype(F4)


def inverse_depths_backward_f32(depths, radii, v_inv):
    inv = inverse_depths_f32(depths, radii)
    with np.errstate(over="ignore", invalid="ignore"):
        g = -((np.asarray(v_inv, F4) * inv) * inv)
    return np.where(np.asarray(radii) > 0, g, F4(0.0)).astype(F4)


def l1_grad_f32(rendered, prior, g):
    """v_rendered = g sgn(R - P) on valid pixels (sgn(0) = 0), 0 elsewhere."""
    r, p, g = np.asarray(rendered, F4), np.asarray(prior, F4), F4(g)
    with np.errstate(invalid="ignore"):
        s = np.where(r > p, g, np.where(r < p, -g, F4(0.0)))
    return np.where(valid(p), s, F4(0.0)).astype(F4)


def l1_terms_f32(rendered, prior):
    """|fp32(R - P)| on valid pixels, 0 elsewhere: the terms the kernel sums."""
    r, p = np.asarray(rendered, F4), np.asarray(prior, F4)
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.abs(r - p)
    return np.where(valid(p), d, F4(0.0)).astype(F4)


def downscale_mean_f32(src, factor):
    """dst [h/f, w/f]: the mean of the valid samples of each f x f block, summed in fp32 in row-major order and divided
    by their count; 0 when the block has none."""
    src = np.asarray(src, F4)
    f = int(factor)
    dh, dw = src.shape[0] // f, src.shape[1] // f
    s = np.zeros((dh, dw), F4)
    c = np.zeros((dh, dw), np.int64)
    for j in range(f):
        for i in range(f):
            p = src[j:dh * f:f, i:dw * f:f]
            ok = valid(p)
            with np.errstate(over="ignore"):
                s = np.where(ok, s + np.where(ok, p, F4(0.0)), s).astype(F4)
            c += ok
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(c > 0, s / np.maximum(c, 1).astype(F4), F4(0.0))
    return out.astype(F4)


# ---- float64 ----------------------------------------------------------------------------------------------------------
def l1_loss_f64(rendered, prior):
    """(sum over the valid pixels of |R - P|) / (H W) in float64, from the fp32 terms, and the bound on the kernel's
    loss: the fp64 sum of N terms (N u64 of the sum) plus the one rounding to fp32 (u32 of the value)."""
    t = l1_terms_f32(rendered, prior).astype(np.float64)
    count = t.size
    loss = float(t.sum()) / count
    bound = U32 * abs(loss) + 2 * count * U64 * abs(loss) + 1e-45
    return loss, bound


def l1_grad_f64(rendered, prior, weight):
    """The gradient of weight * loss w.r.t. R in float64: weight / (H W) sgn(R - P) on valid pixels."""
    r, p = np.asarray(rendered, F4), np.asarray(prior, F4)
    with np.errstate(invalid="ignore"):
        s = np.where(r > p, 1.0, np.where(r < p, -1.0, 0.0))
    return np.where(valid(p), s * (weight / r.size), 0.0)


def inverse_depths_f64(depths, radii):
    z = np.asarray(depths, np.float64)
    with np.errstate(divide="ignore"):
        return np.where(np.asarray(radii) > 0, 1.0 / z, 0.0)


def inverse_depths_backward_f64(depths, radii, v_inv):
    """d/dz of sum v_inv * (1/z) = -v_inv / z^2 where radii > 0, 0 elsewhere."""
    z = np.asarray(depths, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(np.asarray(radii) > 0, -np.asarray(v_inv, np.float64) / (z * z), 0.0)


def downscale_mean_f64(src, factor):
    src = np.asarray(src, F4)
    f = int(factor)
    dh, dw = src.shape[0] // f, src.shape[1] // f
    blk = src[:dh * f, :dw * f].reshape(dh, f, dw, f).transpose(0, 2, 1, 3).reshape(dh, dw, f * f)
    ok = valid(blk)
    s = np.where(ok, blk, 0).astype(np.float64).sum(-1)
    c = ok.sum(-1)
    return np.where(c > 0, s / np.maximum(c, 1), 0.0), c
