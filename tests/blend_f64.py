"""Float64 restatement of the blend kernels' per-pixel semantics, with a certificate of its threshold decisions.

The forward is the front-to-back compositing of raster_fwd.cu: integer pixel coordinates,
sigma = 1/2 (a dx^2 + c dy^2) + b dx dy, skip the pair if sigma < 0, alpha = min(0.999, o exp(-sigma)), skip it if
alpha < 1/255, stop BEFORE blending once T (1 - alpha) <= 1e-4, out = sum c alpha T + T_final bg, final_idx = sorted
index of the last blended pair (0 if none).  The backward is that of raster_bwd.cu: alpha clamped at 0.99, T rebuilt
from T_final by dividing by (1 - alpha) back to front, v_conic with the factor 1/2 on every entry, plus the
v_output_alpha term.  With clamp=True the image is clamp_max(out, 1) and the cut channels get no gradient (the
GSB_RASTER_CLAMP_MAX_ONE instantiations).

The kernels and the fp32 oracle evaluate every threshold in fp32, so a pair whose exact alpha lies within rounding of
1/255, or a pixel whose T (1 - alpha) lies within rounding of 1e-4, may legitimately go either way.  The certificate
marks the decisions that cannot: sigma carries the error bound GAMMA (|a dx^2 / 2| + |b dx dy| + |c dy^2 / 2|), alpha the
relative bound eps = dsigma + KAPPA u (1 + |ln o| + sigma) (log2 of the opacity, the fma into the exponent and ex2 /
expf); a pair is decided when sigma and alpha lie clear of 0 and 1/255 by those bounds, the termination when T (1 - alpha)
lies clear of 1e-4 by the accumulated bound of the product, the clamp when out lies clear of 1.  Every pixel whose pairs
and termination (and clamp) are all decided is `certified`: any correct fp32 implementation takes exactly the decisions
of this reference there.  A Gaussian is certified when none of its pairs that may blend (sigma and alpha not certainly
below 0 and 1/255, and not certainly behind the pixel's termination) lies at an uncertified pixel: everywhere else in
its tiles it contributes exactly nothing whichever way that pixel's decisions go, so every pixel its gradient sums over
is certified.

Alongside the results it returns, per output element, the magnitude A = sum |term| over the element's contributions,
and the error scale B = sum |term| x (the term's amplification of the relative alpha and rounding errors through T, in
units of u = 2^-24).  The tests hold the kernels to |delta| <= C u (k A + B).

Works on any device; tiles are processed in batches of similar list length so that the padded [tiles, 256, L] pair
tensors stay within `budget` elements.
"""
import torch

U = 2.0 ** -24          # unit roundoff of fp32
GAMMA = 8 * U           # relative error of each sigma term: dx rounding, two products, the fmas
KAPPA = 8.0             # alpha: log2(opacity) (1 ulp of |lo|), the fma into the exponent, ex2.approx (2 ulp) / expf
TILE = 16
ALPHA_MIN = 1.0 / 255.0
T_EPS = 1e-4


def _batches(lens, budget):
    """Tile ids grouped by list length (longest first) so that n_tiles * 256 * L_max <= budget per group."""
    order = torch.argsort(lens, descending=True)
    ls = lens[order].tolist()
    i, out = 0, []
    while i < len(ls):
        L = max(ls[i], 1)
        nt = max(1, budget // (256 * L))
        j = i
        while j < len(ls) and j - i < nt and ls[j] > 0:
            j += 1
        if j == i:          # the rest are empty tiles
            out.append((order[i:], 0))
            break
        out.append((order[i:j], ls[i]))
        i = j
    return out


def blend(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background, img_h, img_w,
          v_output=None, v_output_alpha=None, clamp=False, clamp_margin=8.0, budget=1 << 24):
    """Forward (and, if v_output is given, backward) of the blend on the sorted lists.  Returns a dict:
    out_img [H,W,3], final_Ts [H,W], final_idx [H,W] (int64), n_blend [H,W], A_out / B_out [H,W,3], A_T / B_T [H,W],
    pix_cert [H,W] (bool), gauss_cert [N] (bool), sat [H,W,3] (bool, clamp only) and, with v_output, v_xy [N,2],
    v_conic [N,3], v_colors [N,3], v_opacity [N,1] with their A_* / B_* and the per-Gaussian tile count n_tiles [N].
    All floating outputs are float64 on the device of `xys`."""
    dev = xys.device
    f8 = torch.float64
    H, W = int(img_h), int(img_w)
    tx_n = (W + TILE - 1) // TILE
    gs = gaussian_ids_sorted.to(dev).long()
    bins = tile_bins.to(dev).long().reshape(-1, 2)
    xy = xys.to(dev, f8).reshape(-1, 2)
    con = conics.to(dev, f8).reshape(-1, 3)
    col = colors.to(dev, f8).reshape(-1, 3)
    op = opacities.to(dev, f8).reshape(-1)
    bg = torch.as_tensor(background).to(dev, f8).reshape(3)
    N = xy.shape[0]
    bwd = v_output is not None
    if bwd:
        vout_img = v_output.to(dev, f8).reshape(H, W, 3)
        voa_img = v_output_alpha.to(dev, f8).reshape(H, W) if v_output_alpha is not None else None

    out = torch.zeros(H, W, 3, dtype=f8, device=dev)
    fT = torch.ones(H, W, dtype=f8, device=dev)
    fI = torch.zeros(H, W, dtype=torch.int64, device=dev)
    nbl = torch.zeros(H, W, dtype=torch.int64, device=dev)
    A_out = torch.zeros(H, W, 3, dtype=f8, device=dev)
    B_out = torch.zeros(H, W, 3, dtype=f8, device=dev)
    A_T = torch.ones(H, W, dtype=f8, device=dev)
    B_T = torch.zeros(H, W, dtype=f8, device=dev)
    cert = torch.ones(H, W, dtype=torch.bool, device=dev)
    sat = torch.zeros(H, W, 3, dtype=torch.bool, device=dev)
    bad = torch.zeros(N, dtype=f8, device=dev)      # > 0: the Gaussian may blend at an undecided pixel
    res = {}
    if bwd:
        names = ("v_xy", "v_conic", "v_colors", "v_opacity")
        widths = (2, 3, 3, 1)
        for nm, w in zip(names, widths):
            for p in ("", "A_", "B_"):
                res[p + nm] = torch.zeros(N, w, dtype=f8, device=dev)
    out[:] = bg
    A_out[:] = bg.abs()

    lens = (bins[:, 1] - bins[:, 0]).clamp_min(0)
    lx = torch.arange(256, device=dev) % TILE
    ly = torch.arange(256, device=dev) // TILE
    for tiles, L in _batches(lens, budget):
        if L == 0:
            continue
        nt = tiles.shape[0]
        s = bins[tiles, 0]
        ln = lens[tiles]
        kk = torch.arange(L, device=dev)
        pad = kk[None, :] < ln[:, None]                                        # [nt, L]
        gid = gs[(s[:, None] + kk[None, :]).clamp(max=max(gs.shape[0] - 1, 0))]
        gid = torch.where(pad, gid, torch.zeros_like(gid))
        X = (tiles % tx_n)[:, None] * TILE + lx[None, :]                       # [nt, 256]
        Y = (tiles // tx_n)[:, None] * TILE + ly[None, :]
        inimg = (X < W) & (Y < H)
        Xc, Yc = X.clamp(max=W - 1), Y.clamp(max=H - 1)
        dx = xy[gid, 0][:, None, :] - X[:, :, None].to(f8)                     # [nt, 256, L]
        dy = xy[gid, 1][:, None, :] - Y[:, :, None].to(f8)
        a, b, c = (con[gid, i][:, None, :] for i in range(3))
        o = op[gid][:, None, :]
        ta, tb_, tc = 0.5 * a * dx * dx, b * dx * dy, 0.5 * c * dy * dy
        sigma = ta + tb_ + tc
        dsig = GAMMA * (ta.abs() + tb_.abs() + tc.abs())
        del ta, tb_, tc
        au = o * torch.exp(-sigma)
        alpha = au.clamp(max=0.999)
        pad3 = pad[:, None, :]
        valid = pad3 & (sigma >= 0) & (alpha >= ALPHA_MIN)
        lno = torch.log(o.clamp_min(1e-30)).abs()
        eps = dsig + KAPPA * U * (1.0 + lno + sigma.clamp_min(0))              # relative bound of alpha
        pair_dec = ((sigma - dsig >= 0) | (sigma + dsig < 0)) & (
            (sigma + dsig < 0) | (au * (1 - eps) >= ALPHA_MIN) | (au * (1 + eps) < ALPHA_MIN))
        possible = ~((sigma + dsig < 0) | (au * (1 + eps) < ALPHA_MIN))       # the pair may blend
        del lno, dsig
        one = torch.ones((), dtype=f8, device=dev)
        fac = torch.where(valid, 1.0 - alpha, one)
        P = torch.cumprod(fac, -1)
        Pprev = torch.cat([torch.ones_like(P[..., :1]), P[..., :-1]], -1)
        blended = valid & (P > T_EPS)
        reach = pad3 & (Pprev > T_EPS)                 # pairs the blend still looks at (up to the stopping one)
        # relative bound of T(1-alpha): alpha's error through (1 - alpha), 2 roundings per factor
        zero_ = torch.zeros((), dtype=f8, device=dev)
        rel_f = torch.where(valid, eps * alpha / (1.0 - alpha) + 2 * U, zero_)
        E = torch.cumsum(rel_f, -1)
        term_dec = ~(valid & reach) | ((P - T_EPS).abs() > E * P)
        pix_ok = torch.all(~reach | (pair_dec & term_dec), -1)                # [nt, 256]
        # pairs the blend may still look at whichever way the pixel's decisions go: T before them can be larger by
        # the errors of the decided factors and by a factor 1 / (1 - alpha) per undecided pair
        a_hi = (au * (1 + eps)).clamp(max=0.999)
        grow = torch.cumsum(rel_f + torch.where(pad3 & ~pair_dec, a_hi / (1.0 - a_hi), zero_), -1)
        may_reach = pad3 & (Pprev * torch.exp(grow - rel_f) > T_EPS)
        del pair_dec, term_dec, E, reach, fac, P, grow, a_hi

        fb = torch.where(blended, 1.0 - alpha, one)
        Pb = torch.cumprod(fb, -1)
        Tb = torch.cat([torch.ones_like(Pb[..., :1]), Pb[..., :-1]], -1)       # T before each pair
        Tf = Pb[..., -1]                                                      # [nt, 256]
        vis = torch.where(blended, alpha * Tb, torch.zeros((), dtype=f8, device=dev))
        cg = col[gid][:, None, :, :]                                           # [nt, 1, L, 3]
        o_pix = (vis[..., None] * cg).sum(2) + Tf[..., None] * bg              # [nt, 256, 3]
        # error scale: each term's own alpha error plus the errors of the factors in front of it
        ue = eps / U
        amp_f = torch.where(blended, ue * alpha / (1.0 - alpha) + 2.0, torch.zeros((), dtype=f8, device=dev))
        ampc = torch.cumsum(amp_f, -1)
        amp_term = ampc - amp_f + ue                                           # front factors + own alpha
        Ao = (vis[..., None] * cg.abs()).sum(2) + Tf[..., None] * bg.abs()
        Bo = ((vis * amp_term)[..., None] * cg.abs()).sum(2) + (Tf * ampc[..., -1])[..., None] * bg.abs()
        nb = blended.sum(-1)
        last = torch.where(blended, kk.expand_as(blended), torch.full_like(kk, -1).expand_as(blended)).amax(-1)
        fidx = torch.where(last >= 0, s[:, None] + last, torch.zeros_like(last))
        bT = Tf * ampc[..., -1]
        if clamp:
            bound = clamp_margin * U * ((nb + 8)[..., None].to(f8) * Ao + Bo)
            pix_ok &= torch.all((o_pix - 1.0).abs() > bound, -1)
            st = o_pix > 1.0
        else:
            st = torch.zeros_like(o_pix, dtype=torch.bool)
        pix_ok |= ~inimg
        # an undecided pixel can change the contribution of every pair there that may blend, and only those: a pair
        # whose sigma < 0 or alpha < 1/255 is certain contributes nothing whatever the pixel's other decisions
        taint = (may_reach & possible & ~pix_ok[..., None]).any(1)             # [nt, L]
        if bool(taint.any()):
            bad.index_add_(0, gid[pad], taint[pad].to(f8))

        yy, xx = Yc[inimg], Xc[inimg]
        out[yy, xx] = torch.where(st, torch.ones((), dtype=f8, device=dev), o_pix)[inimg]
        fT[yy, xx] = Tf[inimg]
        fI[yy, xx] = fidx[inimg]
        nbl[yy, xx] = nb[inimg]
        A_out[yy, xx] = Ao[inimg]
        B_out[yy, xx] = Bo[inimg]
        A_T[yy, xx] = Tf[inimg]
        B_T[yy, xx] = bT[inimg]
        cert[yy, xx] = pix_ok[inimg]
        sat[yy, xx] = st[inimg]
        if not bwd:
            continue

        # ---- backward (raster_bwd.cu semantics) ----
        zero = torch.zeros((), dtype=f8, device=dev)
        vo = vout_img[Yc, Xc] * inimg[..., None]                                # [nt, 256, 3]
        vo = torch.where(st, zero, vo)
        voa = voa_img[Yc, Xc] * inimg if voa_img is not None else torch.zeros_like(Tf)
        a2 = au.clamp(max=0.99)
        ra = torch.where(blended, 1.0 / (1.0 - a2), one)
        rev = torch.flip(torch.cumprod(torch.flip(ra, [-1]), -1), [-1])         # prod_{j >= k} 1/(1-alpha_j)
        Tk = Tf[..., None] * rev
        fac2 = torch.where(blended, a2 * Tk, zero)                            # alpha T
        d = (cg * vo[:, :, None, :]).sum(-1)                                    # rgb . v_out  [nt, 256, L]
        dabs = (cg.abs() * vo[:, :, None, :].abs()).sum(-1)
        q0 = Tf * ((bg * vo).sum(-1) - voa)
        q0abs = Tf * ((bg * vo).abs().sum(-1) + voa.abs())
        behind = torch.flip(torch.cumsum(torch.flip(d * fac2, [-1]), -1), [-1]) - d * fac2   # sum_{j > k}
        behind_abs = torch.flip(torch.cumsum(torch.flip(dabs * fac2, [-1]), -1), [-1]) - dabs * fac2
        Bq = q0[..., None] + behind
        v_alpha = d * Tk - ra * Bq
        m_alpha = dabs * Tk + ra * (q0abs[..., None] + behind_abs)
        amp_b = ampc[..., -1:] + ue + 2.0 * nb[..., None].to(f8)               # all factors + own alpha
        w = torch.where(blended, au * v_alpha, zero)
        wm = torch.where(blended, au * m_alpha, zero)
        del behind, behind_abs, Bq, v_alpha, m_alpha, rev, Tk

        def acc(name, val, mag):
            """Sum a per-pair contribution [nt, 256, L, k] over the tile's pixels into the Gaussians' rows."""
            v = val.sum(1).reshape(nt * L, -1)
            m_ = mag.sum(1).reshape(nt * L, -1)
            mb = (mag * amp_b[..., None]).sum(1).reshape(nt * L, -1)
            sel = pad.reshape(-1)
            g = gid.reshape(-1)[sel]
            res[name].index_add_(0, g, v[sel])
            res["A_" + name].index_add_(0, g, m_[sel])
            res["B_" + name].index_add_(0, g, mb[sel])

        ab, bb, cb = a.abs(), b.abs(), c.abs()
        acc("v_xy", torch.stack([-w * (a * dx + b * dy), -w * (b * dx + c * dy)], -1),
            torch.stack([wm * (ab * dx.abs() + bb * dy.abs()), wm * (bb * dx.abs() + cb * dy.abs())], -1))
        acc("v_conic", torch.stack([-0.5 * w * dx * dx, -0.5 * w * dx * dy, -0.5 * w * dy * dy], -1),
            torch.stack([0.5 * wm * dx * dx, 0.5 * wm * (dx * dy).abs(), 0.5 * wm * dy * dy], -1))
        ws = (wm / o.clamp_min(1e-30))
        acc("v_opacity", torch.where(o > 0, w / o.clamp_min(1e-30), zero)[..., None], ws[..., None])
        acc("v_colors", fac2[..., None] * vo[:, :, None, :], fac2[..., None] * vo[:, :, None, :].abs())

    if gs.shape[0]:
        gl = gs[_list_positions(bins, lens)]
        ntl = torch.zeros(N, dtype=f8, device=dev).index_add_(0, gl, torch.ones_like(gl, dtype=f8))
    else:
        ntl = torch.zeros(N, dtype=f8, device=dev)
    res.update(out_img=out, final_Ts=fT, final_idx=fI, n_blend=nbl, A_out=A_out, B_out=B_out, A_T=A_T, B_T=B_T,
               pix_cert=cert, gauss_cert=bad == 0, sat=sat, n_tiles=ntl)
    return res


def _list_positions(bins, lens):
    """Positions of all list entries, tile by tile (tile_bins rows may not be contiguous or ordered)."""
    total = int(lens.sum())
    starts = torch.repeat_interleave(bins[:, 0], lens)
    first = torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)
    return starts + torch.arange(total, device=bins.device) - first


def forward_autograd(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background, img_h, img_w):
    """The forward of blend() written with differentiable torch ops, for the autograd check: returns (out_img [H,W,3],
    out_alpha = 1 - final_Ts [H,W]), both functions of xys / conics / colors / opacities.  Which pairs blend is decided
    without gradient; the derivatives are those of the smooth blend on that selection, which is what the backward
    implements wherever no alpha reaches the 0.99 clamp."""
    dev = xys.device
    f8 = torch.float64
    H, W = int(img_h), int(img_w)
    tx_n = (W + TILE - 1) // TILE
    gs = gaussian_ids_sorted.to(dev).long()
    bins = tile_bins.to(dev).long().reshape(-1, 2)
    lens = (bins[:, 1] - bins[:, 0]).clamp_min(0)
    bg = torch.as_tensor(background).to(dev, f8).reshape(3)
    op = opacities.reshape(-1)
    out = bg.expand(H, W, 3).clone()
    oa = torch.zeros(H, W, dtype=f8, device=dev)
    lx = torch.arange(256, device=dev) % TILE
    ly = torch.arange(256, device=dev) // TILE
    tiles = torch.nonzero(lens > 0).reshape(-1)
    for t in tiles.tolist():
        s, L = int(bins[t, 0]), int(lens[t])
        gid = gs[s:s + L]
        X = (t % tx_n) * TILE + lx
        Y = (t // tx_n) * TILE + ly
        inimg = (X < W) & (Y < H)
        dx = xys[gid, 0][None, :] - X[:, None].to(f8)
        dy = xys[gid, 1][None, :] - Y[:, None].to(f8)
        a, b, c = conics[gid, 0][None], conics[gid, 1][None], conics[gid, 2][None]
        sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
        alpha = torch.clamp(op[gid][None] * torch.exp(-sigma), max=0.999)
        with torch.no_grad():
            valid = (sigma >= 0) & (alpha >= ALPHA_MIN)
            P = torch.cumprod(torch.where(valid, 1.0 - alpha, torch.ones_like(alpha)), -1)
            blended = valid & (P > T_EPS)
        fb = torch.where(blended, 1.0 - alpha, torch.ones_like(alpha))
        Pb = torch.cumprod(fb, -1)
        Tb = torch.cat([torch.ones_like(Pb[:, :1]), Pb[:, :-1]], -1)
        vis = torch.where(blended, alpha * Tb, torch.zeros_like(alpha))
        o_pix = vis @ colors[gid] + Pb[:, -1:] * bg
        out = out.index_put((Y[inimg], X[inimg]), o_pix[inimg])
        oa = oa.index_put((Y[inimg], X[inimg]), 1.0 - Pb[:, -1][inimg])
    return out, oa
