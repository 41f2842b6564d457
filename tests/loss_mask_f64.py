"""Float64 restatement of the masked training loss gsb_ssim_l1_loss_masked (csrc/ssim.cu, DESIGN D26) with a
per-element error bound, built on loss_f64's restatement of the unmasked kernels.

A mask m [H,W] (nonzero = used) selects both images: x~ = m ? gt : 0, y~ = m ? rendered : 0.  The kernels' tree is
loss_f64's on x~ and y~, with three changes:
  * the forward's sums keep only used pixels (S and |y - x|), and the three partial maps are m ? d : 0;
  * N = sum m is an integer; the count is fl(fl(N) * 3) and the finalize kernel forms 1/count, -w/count and
    (1 - w)/count on the device with IEEE division -- the roundings the host forms for the unmasked loss;
  * v_rendered is m ? (ssim_scale dssim + l1_scale sgn) : 0.
N = 0 gives {total 0, L1 0, SSIM 1} and v = 0.  The bound follows the same kernel tree, so it is loss_f64's bound with
the ignored terms removed; every element stays certified (the only decision is sgn, exact in fp32).

`plain_loss` is the plain formula of D26 in float64 torch (differentiable in `rendered`).
"""
import numpy as np
import torch

from loss_f64 import RAD, TILE, _consts, _filter, _pad_band, _pad_band_r, _rc, window
from project_f64 import F8, U, R, f32


def _t(a, dev):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev)


def loss(rendered, gt, mask, ssim_weight, device=None, band=None):
    """The float64 reference of gsb_ssim_l1_loss_masked for rendered, gt [H,W,3] (fp32 values, any content on ignored
    pixels) and mask [H,W] (nonzero = used).  Returns what loss_f64.loss returns, plus n (the used-pixel count)."""
    dev = device if device is not None else (rendered.device if torch.is_tensor(rendered) else "cpu")
    m = _t(mask, dev) != 0
    m3 = m[..., None]
    y = torch.where(m3, _t(rendered, dev).to(F8), 0.0)
    x = torch.where(m3, _t(gt, dev).to(F8), 0.0)
    H, W, _ = y.shape
    n = int(m.sum())
    zeros = torch.zeros_like(y)
    if n == 0:
        out = dict(v_rendered=zeros, B_v_rendered=zeros.clone(), loss=0.0, B_loss=0.0, l1=0.0, B_l1=0.0, ssim=1.0,
                   B_ssim=0.0, n=0)
        for k in ("d_mu", "d_e22", "d_e12"):
            out[k], out["B_" + k] = zeros.clone(), zeros.clone()
        return out
    if band is None:
        band = max(1, min(H, (1 << 21) // (3 * (W + 2 * RAD))))
    wf = [_rc(float(v), 2 * U * float(v), y) for v in window()]
    wt = wf[::-1]
    (c1, c1b), (c2, c2b) = _consts()
    C1, C2 = _rc(c1, c1b, y), _rc(c2, c2b, y)
    ws = f32(ssim_weight)
    maps = {k: R(torch.zeros_like(y), torch.zeros_like(y)) for k in ("d_mu", "d_e22", "d_e12")}
    s_sum, s_bnd, s_abs, l1_sum = 0.0, 0.0, 0.0, 0.0
    for y0 in range(0, H, band):
        y1 = min(H, y0 + band)
        mb = m3[y0:y1]
        xb, yb = R(_pad_band(x, y0, y1, H)), R(_pad_band(y, y0, y1, H))
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
        for k, d in (("d_mu", d_mu), ("d_e22", d_e22), ("d_e12", d_e12)):
            maps[k].v[y0:y1] = torch.where(mb, d.v, 0.0)
            maps[k].b[y0:y1] = torch.where(mb, d.b, 0.0)
        Sv, Sb = torch.where(mb, S.v, 0.0), torch.where(mb, S.b, 0.0)
        s_sum += float(Sv.sum())
        s_bnd += float(Sb.sum())
        s_abs += float(Sv.abs().sum())
        l1_sum += float((y[y0:y1] - x[y0:y1]).abs().sum())     # 0 on ignored pixels: both are 0 there
    count_exact = float(3 * n)
    count32 = f32(f32(n) * f32(3.0))
    tiles = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    depth = 3 + 5 + 3 + tiles
    cnt = _rc(count_exact, abs(count32 - count_exact), y)
    inv_count = 1.0 / cnt
    ssim = _rc(s_sum, s_bnd + depth * U * s_abs, y) * inv_count
    l1 = _rc(l1_sum, (1 + depth) * U * l1_sum, y) * inv_count
    wr = _rc(ws, 0.0, y)
    total = (1.0 - wr) * l1 + wr * (1.0 - ssim)
    ssim_scale = -wr / cnt
    l1_scale = (1.0 - wr) / cnt
    v = R(torch.zeros_like(y), torch.zeros_like(y))
    for y0 in range(0, H, band):
        y1 = min(H, y0 + band)
        acc = [_filter(_filter(_pad_band_r(maps[k], y0, y1, H, _pad_band), wt, 1), wt, 0)
               for k in ("d_mu", "d_e22", "d_e12")]
        xv, yv = R(x[y0:y1]), R(y[y0:y1])
        dssim = acc[0] + 2.0 * yv * acc[1] + xv * acc[2]
        sgn = torch.sign(y[y0:y1] - x[y0:y1])
        vb = ssim_scale * dssim + l1_scale * R(sgn)
        mb = m3[y0:y1]
        v.v[y0:y1] = torch.where(mb, vb.v, 0.0)
        v.b[y0:y1] = torch.where(mb, vb.b, 0.0)
    out = dict(v_rendered=v.v, B_v_rendered=v.b, loss=float(total.v), B_loss=float(total.b), l1=float(l1.v),
               B_l1=float(l1.b), ssim=float(ssim.v), B_ssim=float(ssim.b), n=n)
    for k, mp in maps.items():
        out[k], out["B_" + k] = mp.v, mp.b
    return out


def plain_loss(rendered, gt, mask, ssim_weight):
    """D26's formula in float64 torch, differentiable in `rendered`: x~ = m ? gt : 0, y~ = m ? rendered : 0 (selected),
    S the reference's SSIM map of x~ and y~ (conv2d, zero padding 5), L1 = sum m |y - x| / 3N, SSIM = sum m S / 3N,
    total = (1 - w) L1 + w (1 - SSIM); N = 0 gives (0, 0, 1)."""
    m = (mask != 0)
    n = int(m.sum())
    w = f32(ssim_weight)
    if n == 0:
        z = (rendered * 0.0).nan_to_num().sum() * 0.0
        return z, z.detach(), z.detach() + 1.0
    m3 = m[..., None]
    yt = torch.where(m3, rendered, torch.zeros((), dtype=rendered.dtype, device=rendered.device))
    xt = torch.where(m3, gt, torch.zeros((), dtype=gt.dtype, device=gt.device))
    w1 = torch.as_tensor(window(), dtype=F8, device=rendered.device)
    win = (w1[:, None] * w1[None, :]).expand(3, 1, 11, 11).contiguous()
    yy = yt.permute(2, 0, 1)[None]
    xx = xt.permute(2, 0, 1)[None]
    conv = lambda a: torch.nn.functional.conv2d(a, win, padding=RAD, groups=3)
    mu1, mu2 = conv(xx), conv(yy)
    s11, s22, s12 = conv(xx * xx) - mu1 * mu1, conv(yy * yy) - mu2 * mu2, conv(xx * yy) - mu1 * mu2
    (c1, _), (c2, _) = _consts()
    S = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s11 + s22 + c2))
    mm = m.to(F8)[None, None]
    l1 = ((yt - xt).abs()).sum() / (3 * n)
    ssim = (S * mm).sum() / (3 * n)
    return (1 - w) * l1 + w * (1 - ssim), l1, ssim


# ------------------------------------------------------------------------------------------------ masks
def make_mask(H, W, kind, seed):
    """Seeded u8 [H,W] test masks (1 = used): "random" (~30 % ignored, i.i.d.), "blobs" (a few ignored discs and
    rectangles, with isolated single ignored pixels), "single" (one used pixel), "zero" (nothing used), "ones"."""
    rng = np.random.default_rng(seed)
    if kind == "ones":
        return np.ones((H, W), np.uint8)
    if kind == "zero":
        return np.zeros((H, W), np.uint8)
    if kind == "single":
        m = np.zeros((H, W), np.uint8)
        m[rng.integers(H), rng.integers(W)] = 1
        return m
    if kind == "random":
        return (rng.uniform(size=(H, W)) >= 0.3).astype(np.uint8)
    assert kind == "blobs", kind
    m = np.ones((H, W), np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    for _ in range(4):
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        r = rng.uniform(0.05, 0.2) * max(H, W)
        m[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 0
    y0, x0 = rng.integers(0, H), rng.integers(0, W)
    m[y0:y0 + max(1, H // 5), x0:x0 + max(1, W // 4)] = 0
    k = max(1, H * W // 200)
    m[rng.integers(0, H, k), rng.integers(0, W, k)] = 0
    return m
