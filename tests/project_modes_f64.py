"""Float64 reference of every cell of the activated projection's mode matrix (project_forward_kernel /
project_backward_kernel of csrc/project.cu), with a per-element error bound and a certificate of the decisions.

The modes are pinhole ("act"), pinhole-AA ("aa"), the 3-D filter ("f3d", "f3d_aa") and the fisheye camera ("fish",
"fish_aa"); the backward adds ACC (prior + vjp, one rounding) and CAMGRAD (the camera gradient, summed per block).
Every mode runs on the shared trees of project_f64 (R: a float64 value and a first-order bound of the fp32 evaluation
in the kernel's order): the pinhole forward tree (with the filter's sigma_k in place of s_k under F3D), the fisheye
forward tree, project_f64's vS / cov2d / v_scale / v_quat chain in the backward, project_aa_f64's comp and dS, and
pose_f64's camera-gradient terms and sums.  Each mode adds only its own terms here, in the kernel's order:
  * F3D: opacity o c3 [comp]; v_logit = v_o c3 [comp] o (1 - o); v_scale gains r_k (in _scale_quat) and, for every
    Gaussian with f > 0 (culled ones included), the opacity's share v_o o_eff (f / sigma_k)^2;
  * FISH: opacity o [comp], v_logit = v_o [comp] o (1 - o) from the logits, and the fisheye camera chain.
`forward_trees` / `backward_trees` evaluate the trees in any float dtype: in float64 they give the reference and its
bound, in float32 they are an fp32 restatement of the kernel (the CPU tests hold it within C B of the reference).
`autograd` is torch autograd of each mode's map, written from the definitions, which pins the trees' values."""
import numpy as np
import torch

import pose_f64 as pose
import project_aa_f64 as paa
import project_f64 as pf
import project_fisheye_f64 as pff
from project_f64 import F8, R, f32, rexp, rwhere

MODES = ("act", "aa", "f3d", "f3d_aa", "fish", "fish_aa")
# known wrong conventions, for the sensitivity checks: the F3D opacity share of v_scale dropped; (f / sigma)^2 written
# as 1 - r^2; glob_scale left out of s; c3 applied twice (under AA); the F3D camera terms on the unfiltered
# covariance; the fisheye J's derivative terms (w, m, qz) dropped; the sign of one series term flipped
ALTS = ("no_share", "share_cancel", "no_glob_scale", "c3_twice", "unfiltered_camgrad", "no_Jderiv", "series_sign")
FWD = ("cov3d", "xys", "depths", "conics", "opacities")
GRADS = ("v_mean3d", "v_scale", "v_quat", "v_opacity_logits")


def flags(mode):
    """(aa, f3d, fish) of a mode name."""
    return mode.endswith("aa"), mode.startswith("f3d"), mode.startswith("fish")


class Scene:
    """One projection call's inputs as the kernel receives them (fp32): cam (project_f64.Cam, or
    project_fisheye_f64.FishCam for the fisheye modes), means [N,3], log-scales [N,3], raw quats [N,4], logits [N],
    glob_scale, and the F3D filter f3 [N] (or None)."""

    def __init__(self, cam, means, scales, quats, logits, glob_scale, f3=None):
        self.cam = cam
        self.means, self.scales, self.quats = (np.asarray(x, np.float32) for x in (means, scales, quats))
        self.logits = np.asarray(logits, np.float32).reshape(-1)
        self.f3 = None if f3 is None else np.asarray(f3, np.float32).reshape(-1)
        self.glob_scale = f32(glob_scale)
        self.n = self.means.shape[0]


def _cols(x, dtype, dev):
    t = torch.as_tensor(np.asarray(x)).to(dev, dtype)
    return [R(t[:, i]) for i in range(t.shape[1])] if t.dim() == 2 else R(t)


def _mask(m, r):
    return rwhere(m, r, 0.0)


# ------------------------------------------------------------------------------------------------ the trees
def forward_trees(mode, sc, dtype=F8, device="cpu", alt=None):
    """The forward tree of `mode` on R over inputs of `dtype`: dict(f, p, q, o, oe, comp, ratio); oe is the opacity
    comp multiplies (o, or o c3 under F3D), comp is unmasked (the caller applies radii > 0)."""
    aa, f3d, fish = flags(mode)
    p, a, q = (_cols(x, dtype, device) for x in (sc.means, sc.scales, sc.quats))
    gs = 1.0 if alt == "no_glob_scale" else sc.glob_scale
    if fish:
        f = pff._forward_tree(sc.cam, p, a, q, gs, second=True, alt=alt)
    else:
        f = pf._forward_tree(sc.cam, p, a, q, gs, True, "cuda", _cols(sc.f3, dtype, device) if f3d else None)
    o = 1.0 / (1.0 + rexp(-_cols(sc.logits, dtype, device)))
    oe = o * f["c3"] if f3d else o
    if f3d and aa and alt == "c3_twice":
        oe = oe * f["c3"]
    out = dict(f=f, p=p, q=q, o=o, oe=oe)
    if aa:
        out["comp"], _, out["ratio"], _ = paa._comp_tree(f)
    return out


def backward_trees(mode, sc, fw, cot, kept, alt=None):
    """The backward tree of `mode` from forward_trees' fw: dict(v_mean3d, v_scale, v_quat (lists of R),
    v_opacity_logits (R), terms (the 24 camera-gradient terms)), as the kernel writes them for radii > 0 on `kept`
    and 0 (or the opacity's terms) elsewhere.  cot: v_xy [N,2], v_depth [N] or None, v_conic [N,3], v_opacity [N] or
    None, in the inputs' dtype."""
    aa, f3d, fish = flags(mode)
    f, o, oe, q = fw["f"], fw["o"], fw["oe"], fw["q"]
    dt, dev = o.v.dtype, o.v.device
    vx = _cols(cot["v_xy"], dt, dev)
    vc = _cols(cot["v_conic"], dt, dev)
    vd = _cols(cot["v_depth"], dt, dev) if cot.get("v_depth") is not None else R(torch.zeros_like(o.v))
    vo = _cols(cot["v_opacity"], dt, dev).v if cot.get("v_opacity") is not None else None
    gs = 1.0 if alt == "no_glob_scale" else sc.glob_scale
    comp = _mask(kept, fw["comp"]) if aa else None
    dS = paa.comp_dS(f, kept, oe, vo) if (aa and vo is not None) else None

    def chain(f):
        extra = {}
        if fish:
            vm, vs, vq = pff._backward_tree(sc.cam, f, q, gs, f["conic"], vx, vd, vc, dS, extra, alt)
        else:
            vm, vs, vq = pf._backward_tree(sc.cam, f, q, gs, True, f["conic"], vx, vd, vc, dS, extra)
        return vm, vs, vq, pose.camgrad_terms(f, fw["p"], extra)

    vm, vs, vq, terms = chain(f)
    if alt == "unfiltered_camgrad":
        fu = pf._forward_tree(sc.cam, fw["p"], _cols(sc.scales, dt, dev), q, gs, True, "cuda")
        terms = chain(fu)[3]
    vm, vs, vq = ([_mask(kept, x) for x in xs] for xs in (vm, vs, vq))
    if vo is None:
        vl = R(torch.zeros_like(o.v))
    else:
        k = R(vo) * f["c3"] if f3d else R(vo)
        if f3d and aa and alt == "c3_twice":
            k = k * f["c3"]
        vl = ((k * comp if aa else k) * o) * (1.0 - o)
        if f3d and alt != "no_share":
            f3 = f["f3"]
            vo_ = R(vo) * (oe * comp if aa else oe)
            if alt == "share_cancel":
                fsh = [1.0 - r * r for r in f["fr"]]
            else:
                fsh = [(f3 / g) * (f3 / g) for g in f["s"]]
            vs = [rwhere(f3.v > 0, x + vo_ * sh, x) for x, sh in zip(vs, fsh)]
    return dict(v_mean3d=vm, v_scale=vs, v_quat=vq, v_opacity_logits=vl, terms=terms)


# ------------------------------------------------------------------------------------------------ the reference
def reference(mode, sc, device="cpu", cot=None, kept=None):
    """Every output of `mode` in float64 on `device`, as project_f64.project's keys: the forward outputs with bounds
    B_<name>, radii, num_tiles_hit, kept (radii > 0) and cert; with cot, the four VJP outputs (values of the tree, 0
    outside `kept` -- the radii the backward is given, default the reference's) with bounds, and the camera gradient
    GV, GP with bounds BV, BP."""
    aa, f3d, fish = flags(mode)
    fw = forward_trees(mode, sc, F8, device)
    f = fw["f"]
    m = torch.as_tensor(sc.means).to(device, F8)
    out = pff.forward_outputs(sc.cam, f, sc.n, device) if fish else pf.forward_outputs(sc.cam, f, m)
    kf = out["kept"]
    op = fw["oe"]
    if aa:
        ratio = fw["ratio"]
        out["cert"] = out["cert"] & (~kf | (ratio.v.abs() > ratio.b) | (ratio.b == 0))
        op = _mask(kf, op * _mask(kf, fw["comp"]))
    out["opacities"], out["B_opacities"] = op.v, op.b
    out["fw"] = fw
    if cot is None:
        return out
    kb = kf if kept is None else kept
    bw = backward_trees(mode, sc, fw, cot, kb)
    for nm in GRADS[:3]:
        out[nm], out["B_" + nm] = pf.stack_masked(bw[nm], torch.ones_like(kb))
    out["v_opacity_logits"], out["B_v_opacity_logits"] = bw["v_opacity_logits"].v, bw["v_opacity_logits"].b
    out["GV"], out["GP"], out["BV"], out["BP"] = pose.camgrad_sum(bw["terms"], kb)
    out["terms"] = bw["terms"]
    return out


# ------------------------------------------------------------------------------------------------ autograd
def _f3d_map(cam, m, a, q, l, f3, gs, aa):
    """The filtered projection from the definitions: sigma_k = sqrt((gs e_k)^2 + f^2) builds the covariance
    (forward_map at glob_scale 1 on log sigma), opacity sigmoid(l) c3 [comp], c3 = prod(gs e_k / sigma_k)."""
    s = gs * torch.exp(a)
    sig = torch.sqrt(s * s + (f3 * f3)[:, None])
    xy, tz, conic, _, _ = pf.forward_map(cam, m, torch.log(sig), q, 1.0, True)
    # c3 = prod s_k / sigma_k as exp(-sum log1p((f / s_k)^2) / 2): float64 autograd of s / sigma itself cancels at f << s
    o = torch.sigmoid(l) * torch.exp(-0.5 * torch.log1p((f3[:, None] / s) ** 2).sum(-1))
    if aa:
        o = o * paa.comp_map(cam, m, torch.log(sig), q)[0]
    return xy, tz, conic, o


def autograd(mode, sc, cot, kept):
    """Float64 autograd of `mode`'s map for the cotangents: (v_mean3d, v_scale, v_quat, v_opacity_logits, G_V, G_P),
    the pixel-centre, depth, conic and (under AA) comp terms taken over `kept`, the opacity's other terms over every
    Gaussian, as the kernel does; G_V, G_P the camera gradient (for fisheye G_P is 0)."""
    aa, f3d, fish = flags(mode)
    t = lambda x: torch.as_tensor(np.asarray(x), dtype=F8)
    ins = [t(x).clone().requires_grad_() for x in (sc.means, sc.scales, sc.quats, sc.logits)]
    lc = pose._leaf_cam(sc.cam, torch.device("cpu")) if not fish else None
    V = torch.tensor(sc.cam.V, dtype=F8).reshape(4, 4).requires_grad_() if fish else None
    kept = torch.as_tensor(kept).cpu()
    gs = sc.glob_scale
    with torch.enable_grad():
        m, a, q, l = ins
        if fish:
            xy, tz, conic, o = pff.forward_map(sc.cam, m, a + np.log(gs), q, l, aa, V=V)
        elif f3d:
            xy, tz, conic, o = _f3d_map(lc, m, a, q, l, t(sc.f3), gs, aa)
        else:
            xy, tz, conic, _, _ = pf.forward_map(lc, m, a, q, gs, True)
            o = torch.sigmoid(l)
            if aa:
                o = o * paa.comp_map(lc, m, a, q, gs)[0]
        if aa:
            o = torch.where(kept, o, 0.0)
        k2 = kept[:, None]
        loss = torch.where(k2, xy * t(cot["v_xy"]), 0.0).sum() + torch.where(k2, conic * t(cot["v_conic"]), 0.0).sum()
        if cot.get("v_depth") is not None:
            loss = loss + torch.where(kept, tz * t(cot["v_depth"]), 0.0).sum()
        if cot.get("v_opacity") is not None:
            loss = loss + (o * t(cot["v_opacity"])).sum()
        leaves = ins + ([V] if fish else [lc.V, lc.P])
        g = torch.autograd.grad(loss, leaves, allow_unused=True)
    g = [torch.zeros_like(x) if gx is None else torch.nan_to_num(gx) for gx, x in zip(g, leaves)]
    GV = g[4].reshape(4, 4)
    GP = torch.zeros(4, 4, dtype=F8) if fish else g[5].reshape(4, 4)
    return g[0], g[1], g[2], g[3], GV, GP


# ------------------------------------------------------------------------------------------------ scenes
def _filter(rng, scales, gs):
    """A 3-D filter over three regimes, a third each: f = 0 exactly, f << s (1e-4 .. 1e-2 of the mean scale) and
    f >> s: f is the Gaussian's smallest scale and its log-scales drop by log 1 .. log 1e3 (c3 down to about 1e-9),
    so that the filtered footprint stays within that of the scene.  Edits `scales` in place; returns f [N] float32."""
    n = scales.shape[0]
    e = gs * np.exp(scales.astype(np.float64))
    u = rng.integers(0, 3, n)
    f = np.where(u == 1, e.mean(1) * np.exp(rng.uniform(np.log(1e-4), np.log(1e-2), n)), e.min(1))
    big = u == 2
    scales[big] -= rng.uniform(0.0, np.log(1e3), (int(big.sum()), 1)).astype(np.float32)
    return np.where(u == 0, 0.0, f).astype(np.float32)


def scene(mode, n, seed, W=320, H=200, glob_scale=1.3):
    """A random scene for `mode` through a general camera: pinhole modes as project_f64.random_gaussians (a tenth near
    the clip plane, 3 % beyond the fov clamp), fisheye modes as project_fisheye_f64.random_fisheye_gaussians (on the
    axis, either side of the series switch, beyond theta_lim and behind the camera) with footprints of 1 px to 5 % of
    the width; logits in [-8, 8].  Wider footprints, sub-pixel needles (comp near 0) and log-scales out to -12 and 3
    are edge_scene's: their radii and comp are certified less often."""
    _, f3d, fish = flags(mode)
    rng = np.random.default_rng(seed)
    if fish:
        cam = pff.fisheye_camera(W, H, seed)
        m, s, q, l = pff.random_fisheye_gaussians(cam, n, seed, px=(1.0, 0.05))
    else:
        cam = pf.camera_from_setup(pf.general_camera(W, H, seed))
        m, s, q = pf.random_gaussians(cam, n, seed, frac_out=0.03, act=True)
        l = rng.uniform(-8, 8, n).astype(np.float32)
    return Scene(cam, m, s, q, l, glob_scale, _filter(rng, s, f32(glob_scale)) if f3d else None)


def edge_scene(mode, seed, n=3000, glob_scale=0.7):
    """Constructed edges for `mode`, on an identity-view camera where t is exact in fp32.  Every mode: log-scales from
    -12 to 3 on a fifth of the Gaussians (comp near 0 under AA at the small end), logits from -30 to 30.  Pinhole:
    Gaussians exactly on the fov clamp (the D16 ties) and t.z one fp32 step above, at, and below clip_thresh.
    Fisheye: Gaussians on the axis, either side of the series switch, a relative 1e-6 .. 1e-3 either side of
    theta_lim and behind the camera.  F3D: the three filter regimes."""
    _, f3d, fish = flags(mode)
    rng = np.random.default_rng(seed)
    if fish:
        cam = pff.fisheye_camera(256, 192, seed, identity=True)
        m, s, q, _ = pff.random_fisheye_gaussians(cam, n, seed, frac_axis=0.1, frac_switch=0.2)
        k = 64
        th = cam.theta_lim * (1.0 + np.array([-1.0, 1.0]).repeat(k // 2) * np.exp(rng.uniform(np.log(1e-6),
                                                                                                np.log(1e-3), k)))
        ph = rng.uniform(0, 2 * np.pi, k)
        d = rng.uniform(1.0, 5.0, k)[:, None]
        te = (np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1) * d).astype(np.float32)
        m = np.concatenate([m, te])
        s = np.concatenate([s, np.log(rng.uniform(0.5, 5.0, (k, 3)) * d / cam.fx).astype(np.float32)])
        q = np.concatenate([q, rng.standard_normal((k, 4)).astype(np.float32)])
    else:
        from opensplat_b200.model import Camera
        cam = pf.camera_from_setup(Camera(128, 96, 100.0, 80.0, 71.0, 43.0,
                                             np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32)))
        mt, st, qt = pf.tie_gaussians(cam, seed)
        clip = np.float32(cam.clip)
        zs = np.array([np.nextafter(clip, np.float32(1)), clip, np.nextafter(clip, np.float32(0))], np.float32)
        mc = np.stack([np.zeros(3), np.zeros(3), zs], -1).astype(np.float32)
        sc_ = np.full((3, 3), np.log(1e-3), np.float32)
        mg, sg, qg = pf.random_gaussians(cam, n, seed, act=True)
        m = np.concatenate([mt, mc, mg])
        s = np.concatenate([np.log(st), sc_, sg]).astype(np.float32)
        q = np.concatenate([qt, rng.standard_normal((3, 4)).astype(np.float32), qg])
    nn = m.shape[0]
    k = nn // 5
    idx = rng.permutation(nn)[:k]
    s[idx] = rng.uniform(-12, 3, (k, 3)).astype(np.float32)
    l = rng.uniform(-30, 30, nn).astype(np.float32)
    return Scene(cam, m, s, q, l, glob_scale, _filter(rng, s, f32(glob_scale)) if f3d else None)


def cotangent_sets(n, seed, dtype=np.float32):
    """Random (v_xy, v_depth, v_conic, v_opacity), and v_conic with v_opacity alone (the conic-only set exposes the
    clamp and J terms that the pixel-centre path would hide)."""
    rng = np.random.default_rng(seed)
    c = dict(v_xy=rng.standard_normal((n, 2)).astype(dtype), v_depth=rng.standard_normal(n).astype(dtype),
             v_conic=rng.standard_normal((n, 3)).astype(dtype), v_opacity=rng.standard_normal(n).astype(dtype))
    return c, dict(c, v_xy=np.zeros_like(c["v_xy"]), v_depth=np.zeros_like(c["v_depth"]))
