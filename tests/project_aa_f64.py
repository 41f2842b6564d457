"""Float64 reference of the anti-aliased activated projection (DESIGN D19: gsb_project_forward_activated_aa and
gsb_project_backward_activated_aa[_acc]), on top of tests/project_f64.py.

The map.  opacities = sigmoid(logit) * comp, comp = sqrt(max(0, det0 / det)) where radii > 0 and 0 elsewhere, with
det0 = cxx0 cyy0 - cxy^2 the determinant of the screen covariance T cov3d T^T before the 0.3 px^2 blur and det the
one after it; every other output is that of the activated projection.  `vjp_aa` is torch autograd of an independently
written map, sigmoid(l) * sqrt(clamp_min(det S0 / det(S0 + 0.3 I), 0)) chained onto project_f64.forward_map; where
comp = 0 (det0 <= 0) the comp term contributes nothing (the chosen subgradient).

The bound.  `_comp_tree` follows the forward kernel's operations in order (the three sums before the blur from the
forward tree's T and cov3d, det0, the ratio, sqrtf) and the backward is project_f64's _backward_tree with the comp
term `comp_dS` added to vS before the T / J / clamp chain, evaluated as the kernel does, and
v_logit = ((v comp) o) (1 - o).  The tree's values must equal autograd's, which pins its restatement.

The certificate adds one decision to project_f64's: det0 / det > 0 (the fmaxf), clear of 0 by its bound or exact
(bound 0, as for a constructed det0 == 0)."""
import torch

import project_f64 as pf
from project_f64 import C03, F8, R, rexp, sqrtf

ALTS = ("offdiag_full", "comp_eps", "no_comp_in_vlogit", "swap_dets")


def _cov2d0(f):
    """cxx0, cxy, cyy0: the kernel's three sums before `+ 0.3f`, from the forward tree's T and cov3d."""
    T, C = f["T"], f["C"]
    TV = [[T[r][0] * C[0][c] + T[r][1] * C[1][c] + T[r][2] * C[2][c] for c in range(3)] for r in range(2)]
    cxx0 = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2]
    cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2]
    cyy0 = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2]
    return cxx0, cxy, cyy0


def _comp_tree(f, alt=None):
    """(comp, pos, ratio, (cxx0, cxy, cyy0)) on R; pos = ratio > 0, where comp = sqrtf(ratio) (else exactly 0)."""
    cxx0, cxy, cyy0 = _cov2d0(f)
    det0 = cxx0 * cyy0 - cxy * cxy
    ratio = f["det"] / det0 if alt == "swap_dets" else det0 / f["det"]
    pos = ratio.v > 0
    safe = R(torch.where(pos, ratio.v, torch.ones_like(ratio.v)), torch.where(pos, ratio.b, torch.zeros_like(ratio.b)))
    c = sqrtf(safe)
    zero = torch.zeros_like(ratio.v)
    return R(torch.where(pos, c.v, zero), torch.where(pos, c.b, zero)), pos, ratio, (cxx0, cxy, cyy0)


def comp_dS(f, kept, oe, vo, alt=None):
    """The comp term the backward kernel adds to vS, (mask, d00, d01, d11) on R: k = 0.5 (v_o oe) / comp, id = 1 / det,
    (a, b, c, e) = (cyy0, cxy, cxx0, 0.3) id; mask = ratio > 0 on `kept`.  oe: the opacity comp multiplies, sigmoid(l)
    (times c3 under the 3-D filter).  alt "comp_eps" / "offdiag_full": ALTS."""
    comp, pos, _, (cxx0, cxy, cyy0) = _comp_tree(f, alt)
    pos = pos & kept
    safe = R(torch.where(pos, comp.v, torch.ones_like(comp.v)), comp.b)
    k = 0.5 * (R(vo) * oe) / (safe + pf.f32(1e-6) if alt == "comp_eps" else safe)
    idet = 1.0 / f["det"]
    ea, eb, ec, ee = cyy0 * idet, cxy * idet, cxx0 * idet, C03 * idet
    d00 = k * (C03 * (ea * ea + eb * eb + ee * ea))
    d01 = k * (C03 * (eb * (ea + ec + ee)))
    d11 = k * (C03 * (ec * ec + eb * eb + ee * ec))
    return pos, d00, (2.0 * d01 if alt == "offdiag_full" else d01), d11


# ------------------------------------------------------------------------------------------------ autograd map
def comp_map(cam, means, scales, quats, glob_scale=1.0):
    """comp of the activated projection as a differentiable float64 map, written from the definition: S0 = T cov3d T^T
    with T = J V (fov clamp as the reference's min / max), comp = sqrt(clamp_min(det S0 / det(S0 + 0.3 I), 0)), its
    gradient taken as 0 where the ratio is <= 0.  Returns (comp, ratio)."""
    dev = means.device
    V = torch.as_tensor(cam.V, device=dev).to(F8).reshape(4, 4)
    t = means @ V[:3, :3].T + V[:3, 3]
    Rm = pf._rotmat(quats / quats.norm(dim=-1, keepdim=True))
    M = Rm * (glob_scale * torch.exp(scales))[:, None, :]
    tz = t[:, 2]
    lim = torch.tensor([cam.lim_x, cam.lim_y], dtype=F8, device=dev)
    tt = tz[:, None] * torch.minimum(lim, torch.maximum(-lim, t[:, :2] / tz[:, None]))
    zero = torch.zeros_like(tz)
    J = torch.stack([cam.fx / tz, zero, -cam.fx * tt[:, 0] / tz ** 2,
                     zero, cam.fy / tz, -cam.fy * tt[:, 1] / tz ** 2], -1).reshape(-1, 2, 3)
    T = J @ V[:3, :3]
    S0 = T @ M @ M.transpose(1, 2) @ T.transpose(1, 2)
    a, b, c = S0[:, 0, 0], S0[:, 0, 1], S0[:, 1, 1]
    ratio = (a * c - b * b) / ((a + C03) * (c + C03) - b * b)
    pos = ratio > 0
    comp = torch.where(pos, torch.sqrt(torch.where(pos, ratio, 1.0).clamp_min(0)), 0.0)
    return comp, ratio


def vjp_aa(cam, means, scales, quats, logits, v_xy, v_depth, v_conic, v_opacity, glob_scale=1.0, kept=None):
    """Autograd of the anti-aliased map: (v_mean3d, v_scale, v_quat, v_opacity_logits), float64, comp taken as 0
    outside `kept` (radii > 0)."""
    ins = [x.detach().to(F8).clone().requires_grad_() for x in (means, scales, quats, logits)]
    with torch.enable_grad():
        xy, tz, conic, _, _ = pf.forward_map(cam, *ins[:3], glob_scale, True, None)
        comp, _ = comp_map(cam, *ins[:3], glob_scale)
        if kept is not None:
            comp = torch.where(kept, comp, 0.0)
        loss = (torch.where(torch.isfinite(xy), xy, 0) * v_xy).sum() + \
            (torch.where(torch.isfinite(conic), conic, 0) * v_conic).sum() + (tz * v_depth).sum()
        if v_opacity is not None:
            loss = loss + (torch.sigmoid(ins[3]) * comp * v_opacity).sum()
        g = torch.autograd.grad(loss, ins, allow_unused=True)
    return [x if x is not None else torch.zeros_like(a) for x, a in zip(g, ins)]


# ------------------------------------------------------------------------------------------------ the reference
def project_aa(cam, means, scales, quats, opacity_logits, glob_scale=1.0, v_xy=None, v_depth=None, v_conic=None,
               v_opacity=None, device=None, alt=None):
    """project_f64.project(act=True) for the anti-aliased entry points: the same keys, with opacities / B_opacities =
    sigmoid * comp, v_* from vjp_aa and their trees, and cert including the comp decision.  Also: comp, B_comp,
    comp_pos (ratio > 0 on a kept Gaussian).  alt: one of ALTS, a known wrong convention applied to the tree (for the
    sensitivity checks): "offdiag_full" (the off-diagonal cotangent not per entry), "comp_eps" (gsplat's comp + 1e-6
    in the backward's denominator), "no_comp_in_vlogit", "swap_dets" (det / det0)."""
    dev = device if device is not None else (means.device if torch.is_tensor(means) else "cpu")
    m, a, q = pf._t(means, dev), pf._t(scales, dev), pf._t(quats, dev)
    n = m.shape[0]
    ol = pf._t(opacity_logits, dev).reshape(n)
    out = pf.project(cam, m, a, q, glob_scale, act=True, opacity_logits=ol, device=dev)
    f = pf._forward_tree(cam, [R(m[:, i]) for i in range(3)], [R(a[:, i]) for i in range(3)],
                         [R(q[:, i]) for i in range(4)], glob_scale, True, "cuda")
    kept = out["radii"] > 0
    comp, pos, ratio, _ = _comp_tree(f, alt)
    z = torch.zeros((), dtype=F8, device=dev)
    comp = R(torch.where(kept, comp.v, z), torch.where(kept, comp.b, z))
    pos = pos & kept
    d_comp = (ratio.v.abs() > ratio.b) | (ratio.b == 0)
    out["cert"] = out["cert"] & (~kept | d_comp)
    out["comp"], out["B_comp"], out["comp_pos"] = comp.v, comp.b, pos
    o = 1.0 / (1.0 + rexp(-R(ol)))
    oc = o * comp
    out["opacities"], out["B_opacities"] = oc.v, oc.b
    if v_xy is None:
        return out

    vx, vc = pf._t(v_xy, dev).reshape(n, 2), pf._t(v_conic, dev).reshape(n, 3)
    vd = pf._t(v_depth, dev).reshape(n) if v_depth is not None else torch.zeros(n, dtype=F8, device=dev)
    vo = pf._t(v_opacity, dev).reshape(n) if v_opacity is not None else None
    g = vjp_aa(cam, m, a, q, ol, vx, vd, vc, vo, glob_scale, kept)
    dS = comp_dS(f, kept, o, vo, alt) if vo is not None else None
    vm, vs, vq = pf._backward_tree(cam, f, [R(q[:, i]) for i in range(4)], glob_scale, True, f["conic"],
                                   [R(vx[:, 0]), R(vx[:, 1])], R(vd), [R(vc[:, i]) for i in range(3)], dS)

    def stack(rs, mask):
        return (torch.stack([torch.where(mask, r.v, z) for r in rs], -1),
                torch.stack([torch.where(mask, r.b, z) for r in rs], -1))

    for name, rs, gv in (("v_mean3d", vm, g[0]), ("v_scale", vs, g[1]), ("v_quat", vq, g[2])):
        out["re_" + name], out["B_" + name] = stack(rs, kept)
        out[name] = torch.where(kept[:, None], gv, z)
    if vo is not None:
        vol = (R(vo) * o * (1.0 - o)) if alt == "no_comp_in_vlogit" else (R(vo) * comp * o * (1.0 - o))
    else:
        vol = R(torch.zeros(n, dtype=F8, device=dev))
    out["re_v_opacity_logits"], out["B_v_opacity_logits"] = vol.v, vol.b
    out["v_opacity_logits"] = g[3]
    return out
