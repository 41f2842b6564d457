"""Float64 restatement of the fisheye projection (DESIGN D27; gsb_project_forward_fisheye /
gsb_project_backward_fisheye in csrc/project.cu) with a per-element error bound and a certificate of its decisions.

The map.  t = V (p, 1); r = |t.xy|, theta = atan2(r, t.z), theta_d = theta (1 + k1 theta^2 + .. + k4 theta^8);
(u, v) = (fx, fy) theta_d / r t.xy + (cx, cy) - 0.5.  The EWA covariance takes J = d(u, v)/dt at t, then the pinhole's
0.3 blur, conic, radius, tile box and anti-aliased opacity.  A Gaussian is culled where t.z <= clip or theta > theta_lim.

The tree.  `_forward_tree` evaluates the kernel's own operation tree on project_f64's R type (value plus first-order
running error bound): g = theta_d / r and h = (t.z q - g) / r^2 above the small-r switch r < 0.1f t.z, the series
G = 1 + c1 rho^2 + .. + c4 rho^8 (g = G / t.z, h = H / t.z^3) below it.  The device's atan2f adds its documented 2 ulp
(<= 4 u |result|); the series' first dropped term (c5 rho^10, and 10 c5 rho^8 in H) is added to the bound, so the
values are those of the exact map to within the bound, and the bound holds the kernel per element.

The certificate.  A Gaussian is certified when t.z vs clip, theta vs theta_lim, r vs 0.1f t.z (the branch), det vs 0,
the ceil of the radius and the four tile-box truncations each lie clear of their threshold by the operand's bound.

The backward is torch autograd of the differentiable map (`forward_map`, J itself by autograd with create_graph), so
it checks the kernel's hand-written second derivatives independently.
"""
import math

import numpy as np
import torch

import project_f64 as pf
from project_f64 import C03, C01, F8, TILE, R, U, _covariance, _trunc_box, _view, f32, rexp, rmax, sqrtf

ATAN2_ULP = 4.0          # device atan2f: 2 ulp <= 4 u |result| (CUDA C Programming Guide, maximum ulp error table)
RHO = f32(0.1)           # FISH_RHO: the small-r switch
C1_3, C5_3, C14_15, C1_7, C7_3, C19_9, C818_945, C1_9, C02 = (f32(np.float32(a) / np.float32(b)) for a, b in (
    (1, 3), (5, 3), (14, 15), (1, 7), (7, 3), (19, 9), (818, 945), (1, 9), (1, 5)))


def series_c5(k):
    """The first coefficient the kernel's series drops (exact rationals of model D27)."""
    k1, k2, k3, k4 = k
    return -1.0 / 11.0 + 141.0 / 175.0 * k1 - 457.0 / 189.0 * k2 + 56.0 / 15.0 * k3 - 3.0 * k4


def ratan2(y, x):
    v = torch.atan2(y.v, x.v)
    n2 = y.v * y.v + x.v * x.v
    return R(v, (x.v.abs() * y.b + y.v.abs() * x.b) / n2 + ATAN2_ULP * U * v.abs())


class FishCam:
    """The kernels' scalar arguments as the fp32 values they receive."""

    def __init__(self, viewmat, fx, fy, cx, cy, k, theta_lim, img_h, img_w, clip_thresh=0.01):
        self.V = np.asarray(viewmat, np.float32).reshape(16)
        self.fx, self.fy, self.cx, self.cy = f32(fx), f32(fy), f32(cx), f32(cy)
        self.k = tuple(f32(x) for x in k)
        self.theta_lim = f32(theta_lim)
        self.H, self.W = int(img_h), int(img_w)
        self.clip = f32(clip_thresh)
        self.tiles_x, self.tiles_y = (self.W + TILE - 1) // TILE, (self.H + TILE - 1) // TILE


def _fisheye_terms(k, tx, ty, tz, second=False, alt=None):
    """fisheye_terms<second> on R: (r, theta, g, h, q, series branch mask, |r - 0.1f t.z| certified), and with
    `second` w, m and qz, the second derivatives the backward's J VJP needs.  Below the switch the series' first
    dropped terms are added to the bounds: c5 rho^10 in G, 10 c5 rho^8 in H and 80 c5 rho^6 in W.  alt "series_sign":
    the sign of H's rho^2 term flipped, for the sensitivity checks."""
    k1, k2, k3, k4 = k
    r2 = tx * tx + ty * ty
    r = sqrtf(r2)
    r = R(r.v, torch.where(r2.v > 0, r.b, r2.b.sqrt()))      # on the axis: |sqrt(x) - 0| <= sqrt(|x|)
    theta = ratan2(r, tz)
    t2 = theta * theta
    kr = [R.of(x, tz.v) for x in k]
    D = 1.0 + t2 * (3.0 * kr[0] + t2 * (5.0 * kr[1] + t2 * (7.0 * kr[2] + t2 * (9.0 * kr[3]))))
    n2 = r2 + tz * tz
    q = D / n2
    # series
    c1 = R.of(k1, tz.v) - C1_3
    c2 = R.of(k2, tz.v) - k1 + C02
    c3 = R.of(k3, tz.v) - R.of(C5_3, tz.v) * k2 + R.of(C14_15, tz.v) * k1 - C1_7
    c4 = R.of(k4, tz.v) - R.of(C7_3, tz.v) * k3 + R.of(C19_9, tz.v) * k2 - R.of(C818_945, tz.v) * k1 + C1_9
    iz = 1.0 / tz
    iz2 = iz * iz
    p2 = r2 * iz2
    G = 1.0 + p2 * (c1 + p2 * (c2 + p2 * (c3 + p2 * c4)))
    Ht = p2 * (4.0 * c2 + p2 * (6.0 * c3 + p2 * (8.0 * c4)))
    H = 2.0 * c1 - Ht if alt == "series_sign" else 2.0 * c1 + Ht
    c5 = abs(series_c5(k))
    gs, hs = G * iz, H * (iz2 * iz)
    gs = R(gs.v, gs.b + c5 * p2.v ** 5 / tz.v.abs())
    hs = R(hs.v, hs.b + 10.0 * c5 * p2.v ** 4 / tz.v.abs() ** 3)
    # closed form (r > 0 there)
    rs = R(torch.where(r.v > 0, r.v, 1.0), r.b)
    r2s = R(torch.where(r2.v > 0, r2.v, 1.0), r2.b)
    td = theta * (1.0 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4))))
    gd = td / rs
    hd = (tz * q - gd) / r2s
    sw = RHO * tz
    series = r.v < sw.v
    d_switch = (r.v - sw.v).abs() > (r.b + sw.b)
    g = R(torch.where(series, gs.v, gd.v), torch.where(series, gs.b, gd.b))
    h = R(torch.where(series, hs.v, hd.v), torch.where(series, hs.b, hd.b))
    out = dict(r=r, r2=r2, theta=theta, g=g, h=h, q=q, series=series, d_switch=d_switch)
    if second:
        W = 8.0 * c2 + p2 * (24.0 * c3 + p2 * (48.0 * c4))
        ws = W * ((iz2 * iz2) * iz)
        ws = R(ws.v, ws.b + 80.0 * c5 * p2.v ** 3 / tz.v.abs() ** 5)
        ms = (3.0 * hs + r2 * ws) / tz
        E = 6.0 * kr[0] + t2 * (20.0 * kr[1] + t2 * (42.0 * kr[2] + t2 * (72.0 * kr[3])))
        md = (E * tz * (theta / rs) - 2.0 * D) / (n2 * n2)
        wd = (tz * md - 3.0 * hd) / r2s
        m = R(torch.where(series, ms.v, md.v), torch.where(series, ms.b, md.b))
        out.update(w=R(torch.where(series, ws.v, wd.v), torch.where(series, ws.b, wd.b)), m=m,
                   qz=(-(2.0 * q + r2 * m)) / tz)
    return out


def _forward_tree(cam, p, a, q, glob_scale, second=False, alt=None):
    """project_forward_kernel<ACT, AA, false, true>'s tree on R (with `second` also the backward's w, m, qz)."""
    V = [float(x) for x in cam.V]
    tx, ty, tz = _view(V, p)
    cv = _covariance(q, a, glob_scale, True)
    C = cv["C"]
    f = _fisheye_terms(cam.k, tx, ty, tz, second, alt)
    g, h, qq = f["g"], f["h"], f["q"]
    fx, fy = cam.fx, cam.fy
    xy = tx * ty
    J = [[fx * (g + (tx * tx) * h), fx * (xy * h), -(fx * (tx * qq))],
         [fy * (xy * h), fy * (g + (ty * ty) * h), -(fy * (ty * qq))]]
    T = [[J[r][0] * V[c] + J[r][1] * V[4 + c] + J[r][2] * V[8 + c] for c in range(3)] for r in range(2)]
    TV = [[T[r][0] * C[0][c] + T[r][1] * C[1][c] + T[r][2] * C[2][c] for c in range(3)] for r in range(2)]
    cxx0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2]
    cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2]
    cyy0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2]
    cxx, cyy = cxx0 + C03, cyy0 + C03
    det = cxx * cyy - cxy * cxy
    inv_det = 1.0 / det
    conic = [cyy * inv_det, -cxy * inv_det, cxx * inv_det]
    b = 0.5 * (cxx + cyy)
    sq = sqrtf(rmax(b * b - det, C01))
    r3 = 3.0 * sqrtf(rmax(b + sq, b - sq))
    pxc = fx * (g * tx) + cam.cx - 0.5
    pyc = fy * (g * ty) + cam.cy - 0.5
    comp = sqrtf(rmax((cxx0 * cyy0 - cxy * cxy) / det, 0.0))
    return dict(cv, t=(tx, ty, tz), f=f, Jf=J, T=T, det=det, conic=conic, r3=r3, xy=(pxc, pyc), comp=comp)


def _backward_tree(cam, f, q, glob_scale, conic, v_xy, v_depth, v_conic, dS=None, extra=None, alt=None):
    """project_backward_kernel<.., FISH>'s tree on R from a forward tree built with `second`: project_f64's vS and
    cov2d chain and its v_scale / v_quat, and between them the fisheye's J^T (v_u, v_v) plus sum_rc vJ_rc dJ_rc / dt,
    in the kernel's order.  extra: receives vt, vT and vh (0: no projmat).  alt "no_Jderiv": w, m and qz taken as 0."""
    V = [float(x) for x in cam.V]
    fx, fy = cam.fx, cam.fy
    tx, ty, tz = f["t"]
    ft, Jf = f["f"], f["Jf"]
    vV, vT = pf._cov2d_chain(f["T"], f["C"], pf._vS(conic, v_conic, dS))
    A = [[(fx if r == 0 else fy) * (vT[r][0] * V[4 * c] + vT[r][1] * V[4 * c + 1] + vT[r][2] * V[4 * c + 2])
          for c in range(3)] for r in range(2)]
    h, qq = ft["h"], ft["q"]
    w, m, qz = (R(torch.zeros_like(tz.v)),) * 3 if alt == "no_Jderiv" else (ft["w"], ft["m"], ft["qz"])
    xx, yy, xy = tx * tx, ty * ty, tx * ty
    hx, hy, S = h + xx * w, h + yy * w, A[0][1] + A[1][0]
    qxm, qym, xym = qq + xx * m, qq + yy * m, xy * m
    vx, vy = v_xy
    vtx = (Jf[0][0] * vx + Jf[1][0] * vy + A[0][0] * (tx * (2.0 * h + hx)) + S * (ty * hx) + A[1][1] * (tx * hy)
           - A[0][2] * qxm - A[1][2] * xym)
    vty = (Jf[0][1] * vx + Jf[1][1] * vy + A[0][0] * (ty * hx) + S * (tx * hy) + A[1][1] * (ty * (2.0 * h + hy))
           - A[0][2] * xym - A[1][2] * qym)
    vtz = (v_depth + Jf[0][2] * vx + Jf[1][2] * vy - A[0][0] * qxm - S * xym - A[1][1] * qym
           - (A[0][2] * tx + A[1][2] * ty) * qz)
    vm = [V[c] * vtx + V[4 + c] * vty + V[8 + c] * vtz for c in range(3)]
    if extra is not None:
        z = R(torch.zeros_like(tz.v))
        extra.update(vt=(vtx, vty, vtz), vT=vT, vh=(z, z, z))
    vs, vq = pf._scale_quat(f, q, glob_scale, True, vV)
    return vm, vs, vq


def _t(a, dev):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev, F8)


def forward_map(cam, means, scales, quats, logits, aa=False, alt=None, V=None):
    """The fisheye projection as a differentiable float64 map: xys [N,2], depths [N], conics [N,3], opacities [N].
    alt, a known wrong convention for the sensitivity checks: "no_half" (no -0.5), "theta" (theta in place of
    theta_d), "eps" (gsplat's r + eps).  V: the view matrix as a float64 [4,4] tensor (default cam.V)."""
    dev = means.device
    if V is None:
        V = torch.as_tensor(cam.V, device=dev).to(F8).reshape(4, 4)
    t = means @ V[:3, :3].T + V[:3, 3]
    qn = quats / quats.norm(dim=-1, keepdim=True)
    w, x, y, z = qn.unbind(-1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                      2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                      2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    M = Rm * torch.exp(scales)[:, None, :]
    cov3 = M @ M.transpose(1, 2)
    with torch.enable_grad():
        tt = t if t.requires_grad else t.detach().requires_grad_()
        uv = pixel_map(tt, cam.k, cam.fx, cam.fy, cam.cx, cam.cy, alt)
        J = torch.stack([torch.autograd.grad(uv[:, i].sum(), tt, create_graph=True)[0] for i in range(2)], 1)
    T = J @ V[:3, :3]
    cov2 = T @ cov3 @ T.transpose(1, 2)
    cxx0, cxy, cyy0 = cov2[:, 0, 0], cov2[:, 0, 1], cov2[:, 1, 1]
    cxx, cyy = cxx0 + C03, cyy0 + C03
    det = cxx * cyy - cxy * cxy
    conic = torch.stack([cyy / det, -cxy / det, cxx / det], -1)
    o = torch.sigmoid(logits)
    if aa:
        o = o * torch.sqrt(torch.clamp((cxx0 * cyy0 - cxy * cxy) / det, min=0.0))
    return uv, t[:, 2], conic, o


def pixel_map(t, k, fx, fy, cx, cy, alt=None):
    """(u, v) of view-space points t [N,3] (float64, differentiable, finite with finite derivatives at r = 0)."""
    k1, k2, k3, k4 = k
    tx, ty, tz = t.unbind(-1)
    r2 = tx * tx + ty * ty
    small = r2 < (1e-4 * tz) ** 2
    r = torch.sqrt(torch.where(small, torch.ones_like(r2), r2))
    if alt == "eps":
        r = r + 1e-4 * tz
    theta = torch.atan2(r, tz)
    t2 = theta * theta
    td = theta if alt == "theta" else theta * (1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4))))
    p2 = r2 / (tz * tz)
    c = [k1 - 1 / 3, k2 - k1 + 1 / 5, k3 - 5 / 3 * k2 + 14 / 15 * k1 - 1 / 7,
         k4 - 7 / 3 * k3 + 19 / 9 * k2 - 818 / 945 * k1 + 1 / 9, series_c5(k)]
    G = 1 + p2 * (c[0] + p2 * (c[1] + p2 * (c[2] + p2 * (c[3] + p2 * c[4]))))
    g = torch.where(small, G / tz, td / r)
    half = 0.0 if alt == "no_half" else 0.5
    return torch.stack([fx * g * tx + cx - half, fy * g * ty + cy - half], -1)


def forward_outputs(cam, f, n, dev):
    """The forward outputs of a fisheye forward tree f: cov3d, xys, depths, radii, conics, num_tiles_hit with bounds
    B_<name>, kept, cert and the decisions' flags (front, in_fov, series)."""
    tx, ty, tz = f["t"]
    th = f["f"]["theta"]
    front = tz.v > cam.clip
    in_fov = th.v <= cam.theta_lim
    vis = front & in_fov
    d_front = (tz.v - cam.clip).abs() > tz.b
    d_fov = (th.v - cam.theta_lim).abs() > th.b
    d_det = f["det"].v.abs() > f["det"].b
    has_conic = vis & (f["det"].v != 0)
    r3 = f["r3"]
    radius = torch.ceil(r3.v)
    d_ceil = torch.ceil(r3.v - r3.b) == torch.ceil(r3.v + r3.b)
    pxc, pyc = f["xy"]
    tr = R(radius / TILE)
    box, d_box = [], torch.ones(n, dtype=torch.bool, device=dev)
    for arg, lim_n in (((pxc / 16.0) - tr, cam.tiles_x), ((pxc / 16.0) + tr + 1.0, cam.tiles_x),
                       ((pyc / 16.0) - tr, cam.tiles_y), ((pyc / 16.0) + tr + 1.0, cam.tiles_y)):
        big = has_conic & ((arg.v.abs() + arg.b) >= 2.0 ** 31)
        assert not bool(big.any()), "a tile-box operand reaches 2^31: out of scope"
        box.append(_trunc_box(arg.v, lim_n))
        d_box &= _trunc_box(arg.v - arg.b, lim_n) == _trunc_box(arg.v + arg.b, lim_n)
    area = (box[1] - box[0]) * (box[3] - box[2])
    kept = has_conic & (area > 0)
    cert = d_front & (~front | (d_fov & (~in_fov | (f["f"]["d_switch"] & d_det & d_ceil & d_box))))
    z = torch.zeros((), dtype=F8, device=dev)
    out = dict(kept=kept, front=front, in_fov=in_fov, cert=cert, series=vis & f["f"]["series"])
    stack = pf.stack_masked

    out["cov3d"], out["B_cov3d"] = stack(f["cov3d"], vis)
    out["conics"], out["B_conics"] = stack(f["conic"], has_conic)
    out["xys"], out["B_xys"] = stack([pxc, pyc], kept)
    out["depths"], out["B_depths"] = torch.where(kept, tz.v, z), torch.where(kept, tz.b, z)
    out["radii"] = torch.where(kept, radius, z).to(torch.int64)
    out["num_tiles_hit"] = torch.where(kept, area, torch.zeros_like(area))
    return out


def project(cam, means, scales, quats, logits, aa=False, v_xy=None, v_depth=None, v_conic=None, v_opacity=None,
            device=None):
    """The float64 reference of gsb_project_forward_fisheye and, with cotangents, of gsb_project_backward_fisheye.
    Returns the forward outputs (xys, depths, radii, conics, num_tiles_hit, cov3d, opacities) with bounds B_<name>,
    kept, cert, the decision flags, and with cotangents v_mean3d, v_scale, v_quat, v_opacity_logits (autograd)."""
    dev = device if device is not None else (means.device if torch.is_tensor(means) else "cpu")
    m, a, q, ol = _t(means, dev), _t(scales, dev), _t(quats, dev), _t(logits, dev).reshape(-1)
    n = m.shape[0]
    f = _forward_tree(cam, [R(m[:, i]) for i in range(3)], [R(a[:, i]) for i in range(3)],
                      [R(q[:, i]) for i in range(4)], 1.0)
    out = forward_outputs(cam, f, n, dev)
    kept = out["kept"]
    z = torch.zeros((), dtype=F8, device=dev)
    o = 1.0 / (1.0 + rexp(-R(ol)))
    if aa:
        comp = f["comp"]
        o = R(torch.where(kept, (o * comp).v, z), torch.where(kept, (o * comp).b, z))
    out["opacities"], out["B_opacities"] = o.v, o.b
    if v_xy is None:
        return out
    ins = [x.detach().clone().requires_grad_() for x in (m, a, q, ol)]
    with torch.enable_grad():
        uv, depth, conic, op = forward_map(cam, *ins, aa=aa)
        keep = kept[:, None]
        loss = (torch.where(keep, uv, 0) * _t(v_xy, dev)).sum() + (torch.where(keep, conic, 0) * _t(v_conic, dev)).sum()
        if v_depth is not None:
            loss = loss + (torch.where(kept, depth, 0) * _t(v_depth, dev)).sum()
        if v_opacity is not None:
            loss = loss + (torch.where(kept | (not aa), op, 0) * _t(v_opacity, dev)).sum()
        gr = torch.autograd.grad(loss, ins, allow_unused=True)
    names = ("v_mean3d", "v_scale", "v_quat", "v_opacity_logits")
    for nm, gv, x in zip(names, gr, ins):
        out[nm] = torch.zeros_like(x) if gv is None else torch.nan_to_num(gv)
    return out


def random_fisheye_gaussians(cam, n, seed, frac_axis=0.05, frac_switch=0.1, frac_out=0.08, frac_behind=0.04,
                             px=(0.3, 0.1)):
    """Gaussians in a fisheye camera's view (fp32 means, log-scales, raw quats, logits): directions out to theta_lim,
    some exactly on the axis (t.x = t.y = 0), some either side of the small-r switch rho = 0.1, some beyond theta_lim
    and some behind the camera; footprints from px[0] pixels to px[1] of the image width."""
    rng = np.random.default_rng(seed)
    tz_dist = np.exp(rng.uniform(np.log(0.5), np.log(20.0), n))
    theta = np.sqrt(rng.uniform(0, 1, n)) * cam.theta_lim * 0.999
    u = rng.uniform(size=n)
    ax = u < frac_axis
    sw = (u >= frac_axis) & (u < frac_axis + frac_switch)
    out = (u >= frac_axis + frac_switch) & (u < frac_axis + frac_switch + frac_out)
    theta[ax] = 0.0
    theta[sw] = np.arctan(0.1 * np.exp(rng.uniform(-0.05, 0.05, sw.sum())))
    hi = 0.5 * np.pi - 1e-3       # t.z > 0: fields of view of 180 degrees or more are out of scope
    theta[out] = rng.uniform(min(cam.theta_lim * 1.001, hi - 1e-3), hi, out.sum())
    phi = rng.uniform(0, 2 * np.pi, n)
    d = np.stack([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)], -1)
    t = d * tz_dist[:, None]
    beh = rng.uniform(size=n) < frac_behind
    t[beh, 2] = -np.abs(t[beh, 2]) - 0.05
    t[ax, 0] = 0.0
    t[ax, 1] = 0.0
    V = cam.V.reshape(4, 4).astype(np.float64)
    means = (t - V[:3, 3]) @ V[:3, :3]
    if np.array_equal(cam.V.reshape(4, 4), np.eye(4, dtype=np.float32)):
        means = t
    dist = np.linalg.norm(t, axis=1)
    px = np.exp(rng.uniform(np.log(px[0]), np.log(px[1] * cam.W), (n, 3)))
    scales = np.log(px * dist[:, None] / cam.fx)
    quats = rng.standard_normal((n, 4)) * np.exp(rng.uniform(np.log(0.5), np.log(2.0), (n, 1)))
    logits = rng.normal(0, 2, n)
    return (means.astype(np.float32), scales.astype(np.float32), quats.astype(np.float32),
            logits.astype(np.float32))


def fisheye_camera(W, H, seed, k=(0.05, -0.02, 0.004, -0.0005), identity=False):
    """A FishCam with a rotated and translated view, fx != fy, an off-centre principal point, and fx chosen so that
    theta_lim lands near the image edge."""
    from opensplat_b200.model import fisheye_theta_limit
    rng = np.random.default_rng(seed)
    th = fisheye_theta_limit(*k)
    k1, k2, k3, k4 = k
    tdl = th * (1 + k1 * th ** 2 + k2 * th ** 4 + k3 * th ** 6 + k4 * th ** 8)
    fx = 0.5 * W / tdl
    V = np.eye(4)
    if not identity:
        ax = rng.standard_normal(3)
        ax /= np.linalg.norm(ax)
        ang = rng.uniform(0.3, 1.2)
        Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        V[:3, :3] = np.eye(3) + math.sin(ang) * Kx + (1 - math.cos(ang)) * Kx @ Kx
        V[:3, 3] = rng.uniform(-1, 1, 3)
    return FishCam(V.astype(np.float32), fx, fx * 1.03, 0.5 * W + 3.7, 0.5 * H - 2.2, k, th, H, W)
