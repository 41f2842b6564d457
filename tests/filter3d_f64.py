"""Restatement of Mip-Splatting's 3-D smoothing filter (DESIGN D24: csrc/filter3d.cu and the F3D mode of
csrc/project.cu), in numpy fp32 in the kernels' operation order and in float64.

- `filter_fp32` is gsb_filter3d_compute operation for operation (fp32, no contraction), so the kernel must equal it
  bit for bit.  `filter_f64` is the same definition in float64, with a certificate: a (Gaussian, camera) decision
  counts as certified when every quantity it compares lies further than a relative bound from its threshold, and a
  Gaussian is certified when all its decisions are.
- `filtered_map` is the filtered projection as a float64 torch map, built on project_f64.forward_map and
  project_aa_f64.comp_map (imported, not edited): the effective log-scales log(e^2 + f^2) / 2 and the opacity
  sigmoid(l) c3 [comp].  Autograd of it is the VJP; `vjp_terms` writes the kernel's closed forms for the scale and
  opacity-logit gradients, which the CPU tests pin against autograd.
- `reset_f64` and `bake_f64` are the filter-aware opacity reset and the bake, in float64."""
import numpy as np
import torch

F4, F8 = np.float32, torch.float64
EPS32 = 2.0 ** -24


def camera_rows(cameras):
    """filter3d.camera_table on the host, as numpy float32 [C, 18]."""
    from opensplat_b200.filter3d import camera_table
    return camera_table(cameras, "cpu").numpy()


def filter_fp32(means, table, near=0.2, margin=0.15, variance=0.2, alt=None):
    """gsb_filter3d_compute in numpy fp32, the kernel's operation order.  means [n,3] float32, table [C,18].
    alt: a wrong convention for the sensitivity checks ("euclid", "min_focal", "no_margin", "unseen_zero")."""
    p = np.asarray(means, F4)
    t = np.asarray(table, F4)
    n = p.shape[0]
    near, margin = F4(near), F4(margin)
    d = np.full(n, np.inf, F4)
    with np.errstate(all="ignore"):
        for c in t:
            V = c[:12]
            fx, fy, cx, cy, W, H = c[12:18]
            tz = ((V[8] * p[:, 0] + V[9] * p[:, 1]) + V[10] * p[:, 2]) + V[11]
            tx = ((V[0] * p[:, 0] + V[1] * p[:, 1]) + V[2] * p[:, 2]) + V[3]
            ty = ((V[4] * p[:, 0] + V[5] * p[:, 1]) + V[6] * p[:, 2]) + V[7]
            u = fx * (tx / tz) + cx
            v = fy * (ty / tz) + cy
            m = F4(0) if alt == "no_margin" else margin
            xlo, xhi = -(m * W), (F4(1) + m) * W
            ylo, yhi = -(m * H), (F4(1) + m) * H
            seen = (tz > near) & (u >= xlo) & (u <= xhi) & (v >= ylo) & (v <= yhi)
            z = np.sqrt(tx * tx + ty * ty + tz * tz).astype(F4) if alt == "euclid" else tz
            d = np.where(seen & (z < d), z, d).astype(F4)
        fxs = t[:, 12]
        F = fxs.min() if alt == "min_focal" else fxs.max()
        S = F4(np.sqrt(np.float64(F4(variance))))
        seen = np.isfinite(d)
        if not seen.any():
            return np.zeros(n, F4)
        d = np.where(seen, d, F4(0) if alt == "unseen_zero" else d[seen].max()).astype(F4)
        return ((d / F).astype(F4) * S).astype(F4)


def filter_f64(means, table, near=0.2, margin=0.15, variance=0.2, rel=1e-5):
    """(f [n] float64, certified [n] bool): the definition in float64 from the fp32 inputs.  A decision (z > near,
    the four window edges, and which camera gives the least z) is certified when its two sides differ by more than
    rel times their magnitude, far above the kernel's few-ulp rounding."""
    p = np.asarray(means, np.float64)
    t = np.asarray(table, np.float32).astype(np.float64)
    n = p.shape[0]
    near, margin = float(F4(near)), float(F4(margin))
    d = np.full(n, np.inf)
    cert = np.ones(n, bool)
    zs = []
    with np.errstate(all="ignore"):
        for c in t:
            V = c[:12].reshape(3, 4)
            fx, fy, cx, cy, W, H = c[12:18]
            x, y, z = (p @ V[:, :3].T + V[:, 3]).T
            u, v = fx * (x / z) + cx, fy * (y / z) + cy
            lo_x, hi_x, lo_y, hi_y = -margin * W, (1 + margin) * W, -margin * H, (1 + margin) * H
            seen = (z > near) & (u >= lo_x) & (u <= hi_x) & (v >= lo_y) & (v <= hi_y)
            scale_u, scale_v = np.abs(fx * x / z) + abs(cx) + W, np.abs(fy * y / z) + abs(cy) + H
            near_ok = z - near > rel * (np.abs(z) + 1)       # the window decides only in front of the near plane
            cert &= ~(np.abs(z - near) <= rel * (np.abs(z) + 1))
            for a, b, s in ((u, lo_x, scale_u), (u, hi_x, scale_u), (v, lo_y, scale_v), (v, hi_y, scale_v)):
                cert &= ~(near_ok & (np.abs(a - b) <= rel * s))
            zs.append(np.where(seen, z, np.inf))
            d = np.minimum(d, np.where(seen, z, np.inf))
    zs = np.stack(zs, 1) if zs else np.full((n, 1), np.inf)
    # the least z must be clear of the runner-up, or the two give the same fp32 z anyway
    srt = np.sort(zs, 1)
    if srt.shape[1] > 1:
        both = np.isfinite(srt[:, 1])
        gap = np.abs(np.where(both, srt[:, 1], 0.0) - np.where(both, srt[:, 0], 0.0))
        cert &= ~(both & (gap <= rel * np.abs(np.where(both, srt[:, 0], 0.0))))
    F = t[:, 12].max()
    S = float(F4(np.sqrt(float(F4(variance)))))      # the kernel's S, exact in both
    seen = np.isfinite(d)
    if not seen.any():
        return np.zeros(n), cert
    d = np.where(seen, d, d[seen].max())
    return d / F * S, cert


def mip_splatting_filter(means, cams, variance=0.2):
    """An independent float64 transcription of Mip-Splatting's compute_3D_filter: cams is a list of (R, T, fx, fy,
    W, H) with xyz_cam = xyz @ R + T (R the transposed world-to-camera rotation, as its cameras store it) and the
    principal point at (W / 2, H / 2); near 0.2 and margin 0.15 are its constants."""
    xyz = np.asarray(means, np.float64)
    distance = np.full(xyz.shape[0], 100000.0)
    valid_points = np.zeros(xyz.shape[0], bool)
    focal_length = 0.0
    for R, T, fx, fy, W, H in cams:
        xyz_cam = xyz @ R + T
        z = xyz_cam[:, 2]
        valid_depth = z > 0.2
        x = xyz_cam[:, 0] / z * fx + W / 2.0
        y = xyz_cam[:, 1] / z * fy + H / 2.0
        in_screen = (x >= -0.15 * W) & (x <= W * 1.15) & (y >= -0.15 * H) & (y <= 1.15 * H)
        valid = in_screen & valid_depth
        distance[valid] = np.minimum(distance[valid], z[valid])
        valid_points = valid_points | valid
        if focal_length < fx:
            focal_length = fx
    distance[~valid_points] = distance[valid_points].max()
    return distance / focal_length * (variance ** 0.5)


# ------------------------------------------------------------------------------------------------ the projection
def effective(scales, logits, f, alt=None):
    """(effective log-scales [n,3], c3 [n], sigmoid(l) c3 [n]) as float64 torch (differentiable in scales and logits).
    alt: "scale_add" (sigma = e + f), "logscale_add" (a + f), "no_sqrt" (c3 = prod r^2), "sqrt_twice"
    (c3 = prod sqrt(r))."""
    e = torch.exp(scales)
    f = f[:, None]
    if alt == "scale_add":
        sig = e + f
    elif alt == "logscale_add":
        sig = torch.exp(scales + f)
    else:
        sig = torch.sqrt(e * e + f * f)
    r = e / sig
    c3 = {"no_sqrt": (r * r).prod(-1), "sqrt_twice": torch.sqrt(r).prod(-1)}.get(alt, r.prod(-1))
    return torch.log(sig), c3, torch.sigmoid(logits) * c3


def filtered_map(cam, means, scales, quats, logits, f, aa=False, kept=None, alt=None):
    """The filtered activated projection as a float64 map: (xys, depths, conics, opacities).  cam: a project_f64.Cam.
    Under aa the opacity is (sigmoid(l) c3) comp with comp from the filtered covariance, 0 outside `kept`."""
    import project_aa_f64 as paa
    import project_f64 as pf
    a_eff, c3, o = effective(scales, logits, f, alt)
    xy, tz, conic, _, _ = pf.forward_map(cam, means, a_eff, quats, 1.0, True)
    if aa:
        comp, _ = paa.comp_map(cam, means, a_eff, quats)
        if kept is not None:
            comp = torch.where(kept, comp, 0.0)
        o = o * comp
    return xy, tz, conic, o


def filtered_vjp(cam, means, scales, quats, logits, f, v_xy, v_depth, v_conic, v_opacity, aa=False, kept=None,
                 alt=None):
    """Autograd of filtered_map: (v_means, v_log_scales, v_quats, v_logits), float64."""
    ins = [torch.as_tensor(x).detach().to(F8).clone().requires_grad_() for x in (means, scales, quats, logits)]
    f = torch.as_tensor(f).to(F8)
    with torch.enable_grad():
        xy, tz, conic, o = filtered_map(cam, *ins, f, aa, kept, alt)
        loss = (torch.where(torch.isfinite(xy), xy, 0) * v_xy).sum() + \
            (torch.where(torch.isfinite(conic), conic, 0) * v_conic).sum() + (tz * v_depth).sum() + \
            (o * v_opacity).sum()
        g = torch.autograd.grad(loss, ins, allow_unused=True)
    return [x if x is not None else torch.zeros_like(a) for x, a in zip(g, ins)]


def vjp_terms(scales, logits, f, v_sigma, v_opacity, comp=None, cancel=False):
    """The kernel's closed forms in float64 numpy: v_a_k = v_sigma_k e_k r_k + v_o o_eff (f / sigma_k)^2 and
    v_l = v_o c3 [comp] o (1 - o).  v_sigma: the cotangent of sigma_k.  cancel: write (f / sigma)^2 as 1 - r^2."""
    e = np.exp(np.asarray(scales, np.float64))
    f = np.asarray(f, np.float64)[:, None]
    sig = np.sqrt(e * e + f * f)
    r = e / sig
    c3 = r.prod(-1)
    o = 1.0 / (1.0 + np.exp(-np.asarray(logits, np.float64)))
    k = c3 if comp is None else c3 * comp
    o_eff = o * k
    share = (1.0 - r * r) if cancel else (f / sig) ** 2
    v_a = v_sigma * e * r + (v_opacity * o_eff)[:, None] * share
    v_l = v_opacity * k * o * (1.0 - o)
    return v_a, v_l


def c3_fp32(scales, f):
    """The projection's fp32 c3 at glob_scale 1: r_k = e_k / sqrtf(e_k e_k + f f), c3 = (r_0 r_1) r_2."""
    e = np.exp(np.asarray(scales, F4)).astype(F4)
    f = np.asarray(f, F4)[:, None]
    r = (e / np.sqrt((e * e + f * f).astype(F4)).astype(F4)).astype(F4)
    return ((r[:, 0] * r[:, 1]).astype(F4) * r[:, 2]).astype(F4)


def reset_f64(logits, scales, f, reset_value, max_logit, c3=None):
    """gsb_reset_opacity_filter3d: min(l, logit(r / c3)) where r / c3 < 1, l where >= 1, min(l, max_logit) where
    c3 == 1 (c3 the fp32 value, the logit in fp64 rounded once).  c3: the device's fp32 c3 if given (numpy's expf
    differs from the device's by an ulp here and there, which logit(r / c3) amplifies by 1 / (1 - r / c3))."""
    l = np.asarray(logits, F4).reshape(-1)
    c3 = c3_fp32(scales, f) if c3 is None else np.asarray(c3, F4)
    with np.errstate(all="ignore"):
        q = np.float64(F4(reset_value)) / c3.astype(np.float64)
        lim = (np.log(q) - np.log1p(-q)).astype(F4)
    out = np.where(q < 1.0, np.minimum(l, lim), l)
    return np.where(c3 == F4(1), np.minimum(l, F4(max_logit)), out).astype(F4)


def bake_f64(scales, logits, f):
    """gsb_filter3d_bake in float64 from the definitions: (log(e^2 + f^2) / 2, logit(sigmoid(l) c3)), unrounded."""
    a = np.asarray(scales, np.float64)
    f = np.asarray(f, np.float64)[:, None]
    e = np.exp(a)
    sig2 = e * e + f * f
    c3 = np.sqrt(e * e / sig2).prod(-1)
    p = c3 / (1.0 + np.exp(-np.asarray(logits, np.float64).reshape(-1)))
    return 0.5 * np.log(sig2), np.log(p) - np.log1p(-p)
