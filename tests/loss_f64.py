"""Float64 restatement of the fused training loss gsb_ssim_l1_loss (csrc/ssim.cu) with a per-element error bound.

The loss is Model::mainLoss (model.cpp:780-784): (1 - w) L1 + w (1 - SSIM), with the reference's SSIM (ssim.cpp): the
window exp(-floor((i - 11) / 2)^2 / 4.5), i = 0..10, normalised -- a one-sided staircase whose heaviest taps sit at +4
and +5 px -- zero padding of 5, C1 = 0.01^2, C2 = 0.03^2, the mean over [H,W,3].  `loss` follows the kernels' tree:
  * the forward's separable evaluation: a horizontal 11-tap fmaf chain over x = gt, y = rendered, x x, y y and x y
    (each square or product rounded first), then the vertical chain over the five filtered rows;
  * the SSIM map and the three partial maps dS/dmu_y, dS/de22, dS/de12 exactly as ssim.cu:105-115 writes them;
  * the backward's transposed window w[10 - k], horizontal then vertical, over the three maps (zero outside the image);
  * v = ssim_scale (dmu + 2 y de22 + x de12) + l1_scale sgn(y - x), with ssim_scale = -w / count and l1_scale =
    (1 - w) / count formed in fp32 as the host does.
The values are those of the exact map, so they equal float64 autograd of the plain formula (conv2d, ssim.cpp's
expression, torch's abs whose gradient at 0 is 0) to float64 precision; `plain_loss` is that formula.

The bound.  The kernel's window is normalised in double and narrowed (ssim.cu), the reference's in fp32; they differ by
1 ulp on some taps, so each weight is charged 2u relative.  C1 and C2 are the reference's fp32 constants, charged the
distance to the kernel's `0.01f * 0.01f`.  Every other fp32 operation adds u |result| (project_f64.R), and an fmaf adds
it once.  The maps carry their bounds into the backward.  ssim.cu is built with --fmad=true; the bound of a separately
rounded multiply-add is at least that of the fused one, so it holds either way.

The certificate.  The only decision is sgn(y - x), and it is exact in fp32: fl(y - x) has the sign of y - x and is 0
only when y == x.  Every element is certified.

The scalars {total, L1, SSIM} are fp32 sums: per thread over 3 channels, a 256-thread shuffle tree (5 + 3 levels), then
one float atomic per 16 x 16 tile in any order.  A sum through a tree of depth d has error <= d u sum |terms|; the
atomics add depth n_tiles.  Their bounds add that to the sum of the per-element bounds, then the finalize step's
roundings.

The image is processed in row bands, so 2160 x 3840 fits on any device.
"""
import numpy as np
import torch

from project_f64 import F8, U, R, f32

TILE = 16
RAD = 5


def window(alt=None):
    """The reference's window in float64; alt "centred": the symmetric Gaussian exp(-(i - 5)^2 / 4.5)."""
    i = np.arange(11, dtype=np.float64)
    d = (i - 5.0) if alt == "centred" else np.floor((i - 11.0) / 2.0)
    g = np.exp(-d * d / 4.5)
    return g / g.sum()


def _rfma(w, a, acc):
    """fmaf(w, a, acc) on R with one rounding; w a float64 weight R over a scalar, acc None for 0."""
    v = w.v * a.v + (acc.v if acc is not None else 0.0)
    b = w.v.abs() * a.b + a.v.abs() * w.b + (acc.b if acc is not None else 0.0)
    return R(v, b + U * v.abs())


def _shift(a, k, n, dim):
    return R(a.v.narrow(dim, k, n), a.b.narrow(dim, k, n))


def _filter(a, w, dim):
    """sum_k w[k] a[p - 5 + k] along dim (a zero padded by 5 on both sides there), as the kernels' fmaf chain."""
    n = a.v.shape[dim] - 2 * RAD
    acc = None
    for k in range(11):
        acc = _rfma(w[k], _shift(a, k, n, dim), acc)
    return acc


def _pad_band(img, y0, y1, H):
    """Rows y0 - 5 .. y1 + 5 of img [H,W,3] (float64), zero outside the image, and 5 zero columns on each side."""
    lo, hi = max(y0 - RAD, 0), min(y1 + RAD, H)
    band = torch.nn.functional.pad(img[lo:hi].permute(2, 0, 1), (RAD, RAD, lo - (y0 - RAD), (y1 + RAD) - hi))
    return band.permute(1, 2, 0)


def _pad_band_r(m, y0, y1, H, pad):
    return R(pad(m.v, y0, y1, H), pad(m.b, y0, y1, H))


def _consts():
    c1r, c2r = f32(0.01 * 0.01), f32(0.03 * 0.03)
    c1k, c2k = f32(f32(0.01) * f32(0.01)), f32(f32(0.03) * f32(0.03))
    return (c1r, abs(c1k - c1r)), (c2r, abs(c2k - c2r))


def _rc(v, b, like):
    return R(torch.tensor(v, dtype=F8, device=like.device), torch.tensor(b, dtype=F8, device=like.device))


def loss(rendered, gt, ssim_weight, device=None, band=None, alt=None):
    """The float64 reference of gsb_ssim_l1_loss for rendered, gt [H,W,3] (fp32 values).  Returns float64 on `device`:
    v_rendered [H,W,3] and B_v_rendered; loss, l1, ssim (Python floats) with B_loss, B_l1, B_ssim; the maps d_mu,
    d_e22, d_e12 (with B_ bounds).  alt: a known wrong convention, for the sensitivity checks -- "sgn0_plus" (sgn(0) =
    +1), "untransposed" (w[k] in the backward), "centred" (a symmetric window), "edge_pad" (edge-clamped padding
    instead of zero padding), "swap_c" (C1 and C2 swapped)."""
    dev = device if device is not None else (rendered.device if torch.is_tensor(rendered) else "cpu")
    y = torch.as_tensor(np.asarray(rendered) if not torch.is_tensor(rendered) else rendered).to(dev, F8)
    x = torch.as_tensor(np.asarray(gt) if not torch.is_tensor(gt) else gt).to(dev, F8)
    H, W, _ = y.shape
    if band is None:
        band = max(1, min(H, (1 << 21) // (3 * (W + 2 * RAD))))
    w64 = window("centred" if alt == "centred" else None)
    wf = [_rc(float(v), 2 * U * float(v), y) for v in w64]
    wt = wf[::-1] if alt != "untransposed" else wf
    (c1, c1b), (c2, c2b) = _consts()
    if alt == "swap_c":
        (c1, c1b), (c2, c2b) = (c2, c2b), (c1, c1b)
    C1, C2 = _rc(c1, c1b, y), _rc(c2, c2b, y)
    ws = f32(ssim_weight)
    pad = _pad_band if alt != "edge_pad" else _edge_band
    maps = {k: R(torch.zeros_like(y), torch.zeros_like(y)) for k in ("d_mu", "d_e22", "d_e12")}
    s_sum, s_bnd, s_abs = 0.0, 0.0, 0.0
    l1_sum = 0.0
    for y0 in range(0, H, band):
        y1 = min(H, y0 + band)
        xb, yb = R(pad(x, y0, y1, H)), R(pad(y, y0, y1, H))
        prods = [xb, yb, xb * xb, yb * yb, xb * yb]
        hz = [_filter(p, wf, 1) for p in prods]
        mx, my, exx, eyy, exy = [_filter(h, wf, 0) for h in hz]
        sxx, syy, sxy = exx - mx * mx, eyy - my * my, exy - mx * my
        A1, A2 = 2.0 * mx * my + C1, 2.0 * sxy + C2
        B1, B2 = mx * mx + my * my + C1, sxx + syy + C2
        inv = 1.0 / (B1 * B2)
        S = A1 * A2 * inv
        d_e12 = 2.0 * A1 * inv
        d_e22 = -S / B2
        d_mu = 2.0 * mx * (A2 - A1) * inv - 2.0 * my * S / B1 + 2.0 * my * S / B2
        for k, m in (("d_mu", d_mu), ("d_e22", d_e22), ("d_e12", d_e12)):
            maps[k].v[y0:y1], maps[k].b[y0:y1] = m.v, m.b
        s_sum += float(S.v.sum())
        s_bnd += float(S.b.sum())
        s_abs += float(S.v.abs().sum())
        l1_sum += float((y[y0:y1] - x[y0:y1]).abs().sum())
    count_exact = float(H * W * 3)
    count32 = f32(f32(f32(H) * f32(W)) * 3.0)
    tiles = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    depth = 3 + 5 + 3 + tiles
    cnt = _rc(count_exact, abs(count32 - count_exact), y)
    inv_count = 1.0 / cnt
    ssim = _rc(s_sum, s_bnd + depth * U * s_abs, y) * inv_count
    l1 = _rc(l1_sum, (1 + depth) * U * l1_sum, y) * inv_count      # fabsf(y - x): one rounding each, then the sum
    wr = _rc(ws, 0.0, y)
    total = (1.0 - wr) * l1 + wr * (1.0 - ssim)
    # backward: host scales, then the transposed filter of the three maps
    ssim_scale = -wr / cnt
    l1_scale = (1.0 - wr) / cnt
    v = R(torch.zeros_like(y), torch.zeros_like(y))
    for y0 in range(0, H, band):
        y1 = min(H, y0 + band)
        acc = [_filter(_filter(_pad_band_r(maps[k], y0, y1, H, pad), wt, 1), wt, 0) for k in ("d_mu", "d_e22", "d_e12")]
        xv, yv = R(x[y0:y1]), R(y[y0:y1])
        dssim = acc[0] + 2.0 * yv * acc[1] + xv * acc[2]
        dd = y[y0:y1] - x[y0:y1]
        sgn = torch.sign(dd) if alt != "sgn0_plus" else torch.where(dd >= 0, 1.0, -1.0).to(F8)
        vb = ssim_scale * dssim + l1_scale * R(sgn)
        v.v[y0:y1], v.b[y0:y1] = vb.v, vb.b
    out = dict(v_rendered=v.v, B_v_rendered=v.b, loss=float(total.v), B_loss=float(total.b), l1=float(l1.v),
               B_l1=float(l1.b), ssim=float(ssim.v), B_ssim=float(ssim.b))
    for k, m in maps.items():
        out[k], out["B_" + k] = m.v, m.b
    return out


def _edge_band(img, y0, y1, H):
    """alt "edge_pad": the band padded by repeating the edge pixels."""
    idx = torch.arange(y0 - RAD, y1 + RAD, device=img.device).clamp(0, H - 1)
    b = img[idx].permute(2, 0, 1)
    return torch.nn.functional.pad(b[None], (RAD, RAD, 0, 0), mode="replicate")[0].permute(1, 2, 0)


def plain_loss(rendered, gt, ssim_weight, alt=None):
    """The reference's formula in float64 torch (differentiable in `rendered`): conv2d with the 2-D window, zero
    padding 5, ssim.cpp's expression, torch's l1_loss (mean |y - x|, gradient sgn(y - x) with sgn(0) = 0)."""
    w1 = torch.as_tensor(window("centred" if alt == "centred" else None), dtype=F8, device=rendered.device)
    win = (w1[:, None] * w1[None, :]).expand(3, 1, 11, 11).contiguous()
    y = rendered.permute(2, 0, 1)[None]
    x = gt.permute(2, 0, 1)[None]
    conv = lambda a: torch.nn.functional.conv2d(a, win, padding=RAD, groups=3)
    mu1, mu2 = conv(x), conv(y)
    s11, s22, s12 = conv(x * x) - mu1 * mu1, conv(y * y) - mu2 * mu2, conv(x * y) - mu1 * mu2
    (c1, _), (c2, _) = _consts()
    S = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s11 + s22 + c2))
    w = f32(ssim_weight)
    l1 = (y - x).abs().mean()
    ssim = S.mean()
    return (1 - w) * l1 + w * (1 - ssim), l1, ssim


# ------------------------------------------------------------------------------------------------ images
def tie_images(H, W, seed):
    """Training-like content for the loss: u8/255 ground truth with a saturated 0 block, a saturated 1 block and a
    constant mid-grey block, each wider than the window where the image allows; the rendered image equals the ground
    truth on about 30 % of the pixels (sgn(0) = 0 decides their L1 gradient), is clamped to [0, 1] elsewhere (exact 0
    and 1 where it saturates), equals the ground truth on the black block and is a different constant on the white
    and grey blocks (flat regions).  Returns (rendered, gt) fp32 [H,W,3]."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    bh, bw = max(1, H // 3), max(1, W // 4)
    g[:bh, :bw] = 0
    g[:bh, bw:2 * bw] = 255
    g[bh:2 * bh, :bw] = 128
    gt = g.astype(np.float32) / np.float32(255)
    r = np.clip(gt + np.float32(0.25) * rng.standard_normal((H, W, 3)).astype(np.float32), 0, 1).astype(np.float32)
    same = rng.uniform(size=(H, W)) < 0.3
    r[same] = gt[same]
    r[:bh, :bw] = 0
    r[:bh, bw:2 * bw] = np.float32(0.75)
    r[bh:2 * bh, :bw] = np.float32(0.3)
    return r, gt
