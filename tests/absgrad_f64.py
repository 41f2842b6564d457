"""Float64 reference of AbsGS's absolute screen-space gradient (DESIGN D25), built on tests/blend_f64.py without
changing it.

Per blended pair the gradient of the Gaussian's 2-D mean is g = -w (a dx + b dy, b dx + c dy), w = alpha_unclamped *
v_alpha as in blend_f64's backward (with the depth map's cotangent, d = rgb . v_out + z v_depth, when depths are
given); v_xy is the sum of g over the pairs and v_xy_abs the sum of |g|, component by component.

The pair decisions are recomputed here with blend_f64's formulas, and the certificates (pix_cert, gauss_cert), the
clamp mask and n_tiles come from blend_f64.blend itself (depth_f64.blend_depth with depths), so a Gaussian certified
there has exactly these pairs in any correct fp32 implementation.

Error scale, per term: |w| (e_w |a dx + b dy| + GAMMA (|a dx| + |b dy|)), where e_w is the relative error bound of w
that blend_f64 carries for its v_xy terms (the alpha errors amplified through T, amp_b u, on the magnitude wm of w)
and the second part bounds the rounding of the inner product, which may cancel.  |.| is 1-Lipschitz, so the bound of
the sum is the sum of the terms' bounds.  A_v_xy_abs = sum wm |a dx + b dy| is the magnitude the summation order
acts on.  Both are returned in units of u, as blend_f64's A / B: the tests hold the kernel to
|delta| <= C u (B + (8 + n_tiles) A)."""
import torch

import blend_f64 as bf
import depth_f64 as df


def absgrad(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background, img_h, img_w, v_output,
            v_output_alpha=None, clamp=False, depths=None, v_output_depth=None, budget=1 << 24):
    """blend_f64.blend's result (depth_f64.blend_depth's when depths are given) plus v_xy_abs [N,2] with A_v_xy_abs /
    B_v_xy_abs, and v_xy_pairs [N,2]: v_xy summed pair by pair from the same w (equal to the result's v_xy up to the
    order of the sum)."""
    dev = xys.device
    f8 = torch.float64
    H, W = int(img_h), int(img_w)
    U, TILE = bf.U, bf.TILE
    if depths is None:
        r = bf.blend(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background, H, W,
                     v_output=v_output, v_output_alpha=v_output_alpha, clamp=clamp, budget=budget)
    else:
        r = df.blend_depth(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, depths, background, H, W,
                           v_output=v_output, v_output_depth=v_output_depth, v_output_alpha=v_output_alpha,
                           clamp=clamp, budget=budget)
    tx_n = (W + TILE - 1) // TILE
    gs = gaussian_ids_sorted.to(dev).long()
    bins = tile_bins.to(dev).long().reshape(-1, 2)
    xy = xys.to(dev, f8).reshape(-1, 2)
    con = conics.to(dev, f8).reshape(-1, 3)
    col = colors.to(dev, f8).reshape(-1, 3)
    op = opacities.to(dev, f8).reshape(-1)
    zz = depths.to(dev, f8).reshape(-1) if depths is not None else None
    bg = torch.as_tensor(background).to(dev, f8).reshape(3)
    N = xy.shape[0]
    vout_img = v_output.to(dev, f8).reshape(H, W, 3)
    voa_img = v_output_alpha.to(dev, f8).reshape(H, W) if v_output_alpha is not None else None
    vd_img = None
    if depths is not None:
        vd_img = (v_output_depth.to(dev, f8).reshape(H, W) if v_output_depth is not None
                  else torch.zeros(H, W, dtype=f8, device=dev))
    sat = r["sat"]
    out = {k: torch.zeros(N, 2, dtype=f8, device=dev) for k in ("v_xy_abs", "A_v_xy_abs", "B_v_xy_abs",
                                                                 "v_xy_pairs")}
    lens = (bins[:, 1] - bins[:, 0]).clamp_min(0)
    lx = torch.arange(256, device=dev) % TILE
    ly = torch.arange(256, device=dev) // TILE
    zero = torch.zeros((), dtype=f8, device=dev)
    one = torch.ones((), dtype=f8, device=dev)
    for tiles, L in bf._batches(lens, budget):
        if L == 0:
            continue
        nt = tiles.shape[0]
        s = bins[tiles, 0]
        ln = lens[tiles]
        kk = torch.arange(L, device=dev)
        pad = kk[None, :] < ln[:, None]
        gid = gs[(s[:, None] + kk[None, :]).clamp(max=max(gs.shape[0] - 1, 0))]
        gid = torch.where(pad, gid, torch.zeros_like(gid))
        X = (tiles % tx_n)[:, None] * TILE + lx[None, :]
        Y = (tiles // tx_n)[:, None] * TILE + ly[None, :]
        inimg = (X < W) & (Y < H)
        Xc, Yc = X.clamp(max=W - 1), Y.clamp(max=H - 1)
        dx = xy[gid, 0][:, None, :] - X[:, :, None].to(f8)
        dy = xy[gid, 1][:, None, :] - Y[:, :, None].to(f8)
        a, b, c = (con[gid, i][:, None, :] for i in range(3))
        o = op[gid][:, None, :]
        # ---- blend_f64's pair decisions and alpha error bound
        ta, tb_, tc = 0.5 * a * dx * dx, b * dx * dy, 0.5 * c * dy * dy
        sigma = ta + tb_ + tc
        dsig = bf.GAMMA * (ta.abs() + tb_.abs() + tc.abs())
        au = o * torch.exp(-sigma)
        alpha = au.clamp(max=0.999)
        pad3 = pad[:, None, :]
        valid = pad3 & (sigma >= 0) & (alpha >= bf.ALPHA_MIN)
        eps = dsig + bf.KAPPA * U * (1.0 + torch.log(o.clamp_min(1e-30)).abs() + sigma.clamp_min(0))
        P = torch.cumprod(torch.where(valid, 1.0 - alpha, one), -1)
        blended = valid & (P > bf.T_EPS)
        fb = torch.where(blended, 1.0 - alpha, one)
        Tf = torch.cumprod(fb, -1)[..., -1]
        ue = eps / U
        amp_f = torch.where(blended, ue * alpha / (1.0 - alpha) + 2.0, zero)
        nb = blended.sum(-1)
        amp_b = amp_f.sum(-1, keepdim=True) + ue + 2.0 * nb[..., None].to(f8)
        # ---- blend_f64's backward, with the depth channel in d
        vo = vout_img[Yc, Xc] * inimg[..., None]
        vo = torch.where(sat[Yc, Xc], zero, vo)
        voa = voa_img[Yc, Xc] * inimg if voa_img is not None else torch.zeros_like(Tf)
        a2 = au.clamp(max=0.99)
        ra = torch.where(blended, 1.0 / (1.0 - a2), one)
        rev = torch.flip(torch.cumprod(torch.flip(ra, [-1]), -1), [-1])
        Tk = Tf[..., None] * rev
        fac2 = torch.where(blended, a2 * Tk, zero)
        cg = col[gid][:, None, :, :]
        d = (cg * vo[:, :, None, :]).sum(-1)
        dabs = (cg.abs() * vo[:, :, None, :].abs()).sum(-1)
        if zz is not None:
            vD = vd_img[Yc, Xc] * inimg
            zg = zz[gid][:, None, :]
            d = d + zg * vD[..., None]
            dabs = dabs + zg.abs() * vD.abs()[..., None]
        q0 = Tf * ((bg * vo).sum(-1) - voa)
        q0abs = Tf * ((bg * vo).abs().sum(-1) + voa.abs())
        behind = torch.flip(torch.cumsum(torch.flip(d * fac2, [-1]), -1), [-1]) - d * fac2
        behind_abs = torch.flip(torch.cumsum(torch.flip(dabs * fac2, [-1]), -1), [-1]) - dabs * fac2
        v_alpha = d * Tk - ra * (q0[..., None] + behind)
        m_alpha = dabs * Tk + ra * (q0abs[..., None] + behind_abs)
        w = torch.where(blended, au * v_alpha, zero)
        wm = torch.where(blended, au * m_alpha, zero)
        ix, iy = a * dx + b * dy, b * dx + c * dy
        sx, sy = (a * dx).abs() + (b * dy).abs(), (b * dx).abs() + (c * dy).abs()
        g = torch.stack([-w * ix, -w * iy], -1)
        mag = torch.stack([wm * ix.abs(), wm * iy.abs()], -1)
        err = torch.stack([wm * (amp_b * ix.abs() + (bf.GAMMA / U) * sx),
                           wm * (amp_b * iy.abs() + (bf.GAMMA / U) * sy)], -1)
        sel = pad.reshape(-1)
        gi = gid.reshape(-1)[sel]
        for name, val in (("v_xy_abs", g.abs()), ("A_v_xy_abs", mag), ("B_v_xy_abs", err), ("v_xy_pairs", g)):
            out[name].index_add_(0, gi, val.sum(1).reshape(nt * L, 2)[sel])
    r.update(out)
    return r
