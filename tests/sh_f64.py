"""Float64 restatement of the SH colour kernels (csrc/sh.cu) with a per-element error bound and a certificate of the
colour clamp.

The forward follows sh_forward_kernel's tree: the view direction v = means - cam_pos (one fp32 subtraction per
component) or the given viewdirs; norm = sqrtf((vx vx + vy vy) + vz vz) and three divides; the six second-order
products; the 25 bases exactly as sh_basis writes them (constants as the kernel's fp32 literals); the accumulation
c += Y[b] coef[b] over b < nb = min((degrees_to_use + 1)^2, K), starting from Y[0] coef[0]; then + bias and the clamp
rgbs = clamp_min(c + bias, 0) (model.cpp:192).  The backward is torch autograd of that map with respect to the
coefficients, written as a plain float64 formula (textbook polynomial bases of the normalised direction), not as the
kernel's tree; the multi-view backward is scale * sum over the views.  The clamp's gradient passes where
c + bias >= 0, as torch's clamp_min does (D17).

The bound.  `project_f64.R` evaluates the same tree on value-plus-bound numbers: each fp32 operation adds u |result|
to the propagated bound of its operands.  sh.cu is built with the default --fmad=true, so ptxas may contract a
multiply and an add into one fused operation; the first-order bound of a separately rounded multiply-add is at least
that of the fused one, so the bound holds whether or not it contracts.  The tree's values are those of the exact map,
so they must equal the autograd values to float64 precision: that pins the restatement of the tree, and the bound B
then holds the kernels per element, |kernel - reference| <= C B.

The certificate.  A channel's clamp decision is certified when |c + bias| > B, or when its fp32 value is determined:
at degrees_to_use = 0 the kernel forms s = fl(fl(Y0 coef0) + bias) whatever ptxas contracts (the only candidate is
fma(Y0, coef0, 0), the same rounded product).  `sh` evaluates that s in fp32 and takes the decision from it, as the
reference's own fp32 clamp_min does.  That makes a constructed tie checkable: featuresDc = -1.7724538f gives
fl(0.28209479f * c) = -0.5 exactly, so s = 0 and the gradient passes (D17), though the float64 product is below -0.5.
"""
import numpy as np
import torch

from project_f64 import F8, U, R, f32, rwhere, sqrtf

C0 = f32(0.28209479177387814)
C1 = f32(0.4886025119029199)
C2 = [f32(x) for x in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                       0.5462742152960396)]
C3 = [f32(x) for x in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                       -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]
C4 = [f32(x) for x in (2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892,
                       0.10578554691520431, -0.6690465435572892, 0.47308734787878004, -1.7701307697799304,
                       0.6258357354491761)]
TIE_DC = f32(-1.7724538)          # fl(C0 * TIE_DC) == -0.5: with bias 0.5, an exact clamp tie at degrees_to_use 0


def num_bases(degree):
    return (degree + 1) ** 2


def _t(a, dev):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev, F8)


# ------------------------------------------------------------------------------------------------ kernel tree
def _basis_tree(nb, vx, vy, vz):
    """sh_basis on R, in its order: a list of nb R values."""
    Y = [R(torch.full_like(vx.v, C0))]
    if nb <= 1:
        return Y
    norm = sqrtf(vx * vx + vy * vy + vz * vz)
    x, y, z = vx / norm, vy / norm, vz / norm
    xx, xy, xz, yy, yz, zz = x * x, x * y, x * z, y * y, y * z, z * z
    Y += [-C1 * y, C1 * z, -C1 * x]
    if nb <= 4:
        return Y
    Y += [C2[0] * xy, C2[1] * yz, C2[2] * (2.0 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy)]
    if nb <= 9:
        return Y
    Y += [C3[0] * y * (3.0 * xx - yy), C3[1] * xy * z, C3[2] * y * (4.0 * zz - xx - yy),
          C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy), C3[4] * x * (4.0 * zz - xx - yy), C3[5] * z * (xx - yy),
          C3[6] * x * (xx - 3.0 * yy)]
    if nb <= 16:
        return Y
    Y += [C4[0] * xy * (xx - yy), C4[1] * yz * (3.0 * xx - yy), C4[2] * xy * (7.0 * zz - 1.0),
          C4[3] * yz * (7.0 * zz - 3.0), C4[4] * (zz * (35.0 * zz - 30.0) + 3.0), C4[5] * xz * (7.0 * zz - 3.0),
          C4[6] * (xx - yy) * (7.0 * zz - 1.0), C4[7] * xz * (xx - 3.0 * yy),
          C4[8] * (xx * (xx - 3.0 * yy) - yy * (3.0 * xx - yy))]
    return Y


def _dir_tree(viewdirs=None, means=None, cam_pos=None):
    if cam_pos is None:
        return [R(viewdirs[:, i]) for i in range(3)]
    return [R(means[:, i]) - R(torch.full_like(means[:, i], float(cam_pos[i]))) for i in range(3)]


# ------------------------------------------------------------------------------------------------ plain map
def _plain_basis(nb, d):
    """The real SH bases of degree <= 4 as textbook polynomials of the unit direction (float64, differentiable)."""
    x, y, z = d.unbind(-1)
    Y = [torch.full_like(x, C0)]
    if nb > 1:
        Y += [-C1 * y, C1 * z, -C1 * x]
    if nb > 4:
        Y += [C2[0] * x * y, C2[1] * y * z, C2[2] * (3 * z * z - 1), C2[3] * x * z, C2[4] * (x * x - y * y)]
    if nb > 9:
        Y += [C3[0] * (3 * x * x * y - y ** 3), C3[1] * x * y * z, C3[2] * y * (5 * z * z - 1),
              C3[3] * (5 * z ** 3 - 3 * z), C3[4] * x * (5 * z * z - 1), C3[5] * z * (x * x - y * y),
              C3[6] * (x ** 3 - 3 * x * y * y)]
    if nb > 16:
        Y += [C4[0] * (x ** 3 * y - x * y ** 3), C4[1] * (3 * x * x * y * z - y ** 3 * z),
              C4[2] * x * y * (7 * z * z - 1), C4[3] * y * z * (7 * z * z - 3), C4[4] * (35 * z ** 4 - 30 * z * z + 3), C4[5] * x * z * (7 * z * z - 3),
              C4[6] * (x * x - y * y) * (7 * z * z - 1), C4[7] * (x ** 3 * z - 3 * x * y * y * z),
              C4[8] * (x ** 4 - 6 * x * x * y * y + y ** 4)]
    return torch.stack(Y, -1)


def _plain_colour(nb, v, coeffs):
    d = v / v.norm(dim=-1, keepdim=True) if nb > 1 else v
    return torch.einsum("nb,nbc->nc", _plain_basis(nb, d), coeffs[:, :nb, :])


# ------------------------------------------------------------------------------------------------ the reference
def sh(degree, degrees_to_use, coeffs, viewdirs=None, means=None, cam_pos=None, bias=None, v_colors=None,
       device=None, alt=None):
    """The float64 reference of one view.  coeffs [N,K,3] (K = (degree + 1)^2); the direction is viewdirs [N,3], or
    means [N,3] - cam_pos [3] formed in fp32 as the *_cam / *_split kernels do.  bias None: the plain colours
    (gsb_sh_forward); else rgbs = clamp_min(colours + bias, 0).  Returns float64 tensors on `device`: colors
    (rgbs when bias is given) and B_colors; s (colours + bias) and B_s; cert [N,3] (the clamp decision certified; all
    True without bias); mask [N,3] (the clamp passes the gradient: s >= 0); tie [N,3] (the determined fp32 s is 0);
    and with v_colors [N,3]: v_coeffs [N,K,3] from autograd, re_v_coeffs (the bound's evaluation) and B_v_coeffs.
    alt: "tie_blocked" takes the clamp's gradient as s > 0, the convention before D17 (for the sensitivity checks)."""
    dev = device if device is not None else (coeffs.device if torch.is_tensor(coeffs) else "cpu")
    co = _t(coeffs, dev)
    n, K = co.shape[0], co.shape[1]
    assert K == num_bases(degree) and 0 <= degrees_to_use <= degree
    nb = min(num_bases(degrees_to_use), K)
    vd = _t(viewdirs, dev) if cam_pos is None else None
    m = _t(means, dev) if cam_pos is not None else None
    cp = [float(c) for c in np.asarray(cam_pos, np.float32).reshape(3)] if cam_pos is not None else None
    Y = _basis_tree(nb, *_dir_tree(vd, m, cp))
    col = []
    for ch in range(3):
        c = Y[0] * R(co[:, 0, ch])
        for b in range(1, nb):
            c = c + Y[b] * R(co[:, b, ch])
        col.append(c)
    out = dict()
    z = torch.zeros((), dtype=F8, device=dev)
    if bias is None:
        out["colors"] = torch.stack([c.v for c in col], -1)
        out["B_colors"] = torch.stack([c.b for c in col], -1)
        out["cert"] = torch.ones((n, 3), dtype=torch.bool, device=dev)
        mask = out["cert"]
        out["tie"] = ~mask
    else:
        s = [c + f32(bias) for c in col]
        sv, sb = torch.stack([x.v for x in s], -1), torch.stack([x.b for x in s], -1)
        out["s"], out["B_s"] = sv, sb
        out["colors"] = torch.where(sv > 0, sv, z)
        out["B_colors"] = torch.where(sv > 0, sb, z)      # |max(a, 0) - max(b, 0)| <= |a - b|
        if nb == 1:
            # the fp32 s of the kernel: fl(fl(Y0 coef0) + bias), evaluated here in the same order
            s32 = (torch.tensor(C0, dtype=torch.float32) * co[:, 0, :].float().cpu()
                   + torch.tensor(f32(bias), dtype=torch.float32)).to(dev, F8)
            out["cert"] = torch.ones((n, 3), dtype=torch.bool, device=dev)
            dec = s32
        else:
            out["cert"] = sv.abs() > sb
            dec = sv
        out["tie"] = dec == 0
        mask = dec >= 0
        if alt == "tie_blocked":
            mask = dec > 0
    out["mask"] = mask
    if v_colors is None:
        return out
    vc = _t(v_colors, dev).reshape(n, 3)
    vm = torch.where(mask, vc, z)
    out["v_coeffs"] = vjp(nb, co, vm, vd, m, cp)
    re, bb = _vjp_tree(Y, K, [R(vm[:, ch]) for ch in range(3)])
    out["re_v_coeffs"], out["B_v_coeffs"] = re, bb
    return out


def vjp(nb, co, v_masked, viewdirs=None, means=None, cam_pos=None):
    """Autograd of the plain map: d <colours, v_masked> / d coeffs (float64 [N,K,3]).  The clamp's gradient enters
    through v_masked (the cotangent where the clamp passes it, else 0)."""
    v = viewdirs if cam_pos is None else means - torch.tensor(cam_pos, dtype=F8, device=means.device)
    c = co.detach().clone().requires_grad_()
    with torch.enable_grad():
        (g,) = torch.autograd.grad((_plain_colour(nb, v, c) * v_masked).sum(), [c])
    return g


def _vjp_tree(Y, K, v):
    """sh_backward_kernel's row[3b + ch] = Y[b] * v[ch] (0 for b >= nb), as [N,K,3] value and bound."""
    n = Y[0].v.shape[0]
    val = torch.zeros((n, K, 3), dtype=F8, device=Y[0].v.device)
    bnd = torch.zeros_like(val)
    for b, yb in enumerate(Y):
        for ch in range(3):
            p = yb * v[ch]
            val[:, b, ch], bnd[:, b, ch] = p.v, p.b
    return val, bnd


def sh_multiview(degree, degrees_to_use, coeffs, means, cams, v_rgbs, scale, bias=0.5, device=None):
    """The multi-view SH backward: the forward of every view (rgbs = clamp_min(SH(means - cams[r]) + bias, 0)) and
    v_coeffs = scale * sum_r d <rgbs_r, v_rgbs[r]> / d coeffs, the clamp's gradient included.  The bound follows
    sh_backward_multiview_kernel: row = fmaf(Y_r[b], v_r, row) over the views in order, skipping a view whose three
    masked cotangents are 0, then scale * row.  Returns views (the per-view `sh` dicts: colors, B_colors, cert, mask,
    tie), v_coeffs, re_v_coeffs, B_v_coeffs, and cert_v [N,3]: every view's clamp decision of that channel certified."""
    dev = device if device is not None else (coeffs.device if torch.is_tensor(coeffs) else "cpu")
    co, m = _t(coeffs, dev), _t(means, dev)
    cams = np.asarray(cams.cpu() if torch.is_tensor(cams) else cams, np.float32).reshape(-1, 3)
    vr = _t(v_rgbs, dev)
    n, K = co.shape[0], co.shape[1]
    nb = min(num_bases(degrees_to_use), K)
    views, total = [], torch.zeros((n, K, 3), dtype=F8, device=dev)
    row = [[R(torch.zeros(n, dtype=F8, device=dev)) for _ in range(3)] for _ in range(nb)]
    cert_v = torch.ones((n, 3), dtype=torch.bool, device=dev)
    z = torch.zeros((), dtype=F8, device=dev)
    for r in range(cams.shape[0]):
        o = sh(degree, degrees_to_use, co, means=m, cam_pos=cams[r], bias=bias, device=dev)
        views.append(o)
        cert_v &= o["cert"]
        vm = torch.where(o["mask"], vr[r], z)
        total += vjp(nb, co, vm, means=m, cam_pos=[float(c) for c in cams[r]])
        Y = _basis_tree(nb, *_dir_tree(means=m, cam_pos=[float(c) for c in cams[r]]))
        live = (vm != 0).any(-1)
        for b in range(nb):
            for ch in range(3):
                acc = Y[b] * R(vm[:, ch]) + row[b][ch]
                row[b][ch] = rwhere(live, acc, row[b][ch])
    re = torch.zeros((n, K, 3), dtype=F8, device=dev)
    bb = torch.zeros_like(re)
    for b in range(nb):
        for ch in range(3):
            p = f32(scale) * row[b][ch]
            re[:, b, ch], bb[:, b, ch] = p.v, p.b
    return dict(views=views, v_coeffs=f32(scale) * total, re_v_coeffs=re, B_v_coeffs=bb, cert_v=cert_v)
