"""Float64 restatement of the camera gradient of the activated projection backward (CAMGRAD of csrc/project.cu,
gsb_project_camera_grad_reduce) and of the pose chain (csrc/pose.cu), DESIGN D22, on top of tests/project_f64.py and
tests/project_aa_f64.py.

The camera gradient.  `camgrad_autograd` is torch autograd of project_f64.forward_map (with project_aa_f64.comp_map
for the anti-aliased opacity) with the viewmat and the projmat as leaf tensors, summed over the Gaussians with
radii > 0.  `camgrad_tree` restates the kernel's per-Gaussian terms on project_f64.R along its operation tree (the
backward tree up to vt and vT, then the 24 terms in the kernel's order); its values must equal autograd's, which pins
the tree.  The kernel sums each term in fp32 over a warp shuffle tree (depth 5) and then over the 8 warps in order
(depth 7), and the blocks' partials in fp64 before one rounding, so with the per-term bounds B_i
    |kernel - reference| <= C (sum B_i + g12 sum (|t_i| + B_i)) + g64 sum |t_i| + u |reference|,
g12 = 12u / (1 - 12u) with u = 2^-24, g64 = n u64 / (1 - n u64) with u64 = 2^-53 for the fp64 sum (n the block count
plus the shuffle depth, a generous depth), and C = 2 as in project_f64 for the first-order propagation.

The pose chain.  `pose_apply` forms the corrected view and centre from the definition (view' = Delta^-1 view, centre'
= centre + R t) in float64; `pose_grad` is torch autograd of e -> <G_V, view'(e)> + <G_P, proj view'(e)>, the
loss's first-order dependence on e through both matrices the projection reads.  `ALTS` are known wrong conventions,
for the sensitivity checks."""
import copy

import numpy as np
import torch

import project_aa_f64 as paa
import project_f64 as pf
from project_f64 import F8, R, rexp

U = pf.U
U64 = 2.0 ** -53
C = 2.0
TREE_DEPTH = 12                       # 5 shuffle levels + 7 sequential warp sums
CG_ROW = 24                           # the terms of one partial row: viewmat rows 0..2, projmat rows 0, 1, 3
ALTS = ("left", "columns", "no_fold", "no_JvT", "centre_unmoved")


def gamma(k, u=U):
    return k * u / (1.0 - k * u)


# ------------------------------------------------------------------------------------------------ camera gradient
def _leaf_cam(cam, dev):
    """A copy of the project_f64.Cam whose V and P are float64 leaf tensors (forward_map / comp_map read them)."""
    c = copy.copy(cam)
    c.V = torch.tensor(cam.V, dtype=F8, device=dev).requires_grad_()
    c.P = torch.tensor(cam.P, dtype=F8, device=dev).requires_grad_()
    return c


def camgrad_autograd(cam, means, scales, quats, logits, v_xy, v_conic, v_opacity=None, aa=False, kept=None):
    """(G_V [4,4], G_P [4,4]) float64: autograd of the activated (aa: anti-aliased) projection's loss
    <v_xy, xy> + <v_conic, conic> (+ <v_opacity, opacity> when aa) w.r.t. viewmat and projmat, over `kept`."""
    dev = torch.device("cpu")
    m, a, q, ol = (pf._t(x, dev) for x in (means, scales, quats, logits))
    vx, vc = pf._t(v_xy, dev).reshape(-1, 2), pf._t(v_conic, dev).reshape(-1, 3)
    kept = torch.ones(m.shape[0], dtype=torch.bool) if kept is None else torch.as_tensor(kept).cpu()
    lc = _leaf_cam(cam, dev)
    with torch.enable_grad():
        xy, _, conic, _, _ = pf.forward_map(lc, m, a, q, 1.0, True)
        k2 = kept[:, None]
        loss = torch.where(k2, xy * vx, 0.0).sum() + torch.where(k2, conic * vc, 0.0).sum()
        if aa and v_opacity is not None:
            comp, _ = paa.comp_map(lc, m, a, q)
            loss = loss + torch.where(kept, torch.sigmoid(ol) * comp * pf._t(v_opacity, dev), 0.0).sum()
        gv, gp = torch.autograd.grad(loss, [lc.V, lc.P], allow_unused=True)
    gv = torch.zeros(16, dtype=F8) if gv is None else gv
    gp = torch.zeros(16, dtype=F8) if gp is None else gp
    return gv.reshape(4, 4).detach(), gp.reshape(4, 4).detach()


def camgrad_terms(f, p, extra, alt=None):
    """The kernel's 24 terms per Gaussian on R, viewmat rows 0..2 then projmat rows 0, 1, 3 (each 4 floats), from the
    forward tree f, the means p and the backward tree's vt, vT, vh (`extra` of project_f64._backward_tree).  Row r of
    the viewmat gets vt_r (p, 1) plus column c's J^T vT: the pinhole's J00, J11 and (J02, J12), or the fisheye's full
    J (f["Jf"]), whose projmat rows are 0.  alt "no_JvT": the J^T vT columns dropped."""
    vt, vT, vh = extra["vt"], extra["vT"], extra["vh"]
    terms = []
    for r in range(3):
        row = [vt[r] * p[c] for c in range(3)] + [vt[r]]
        if alt != "no_JvT":
            for c in range(3):
                if "Jf" in f:
                    Jf = f["Jf"]
                    row[c] = row[c] + (Jf[0][r] * vT[0][c] + Jf[1][r] * vT[1][c])
                elif r == 0:
                    row[c] = row[c] + f["J"][0] * vT[0][c]
                elif r == 1:
                    row[c] = row[c] + f["J"][2] * vT[1][c]
                else:
                    row[c] = row[c] + (f["J"][1] * vT[0][c] + f["J"][3] * vT[1][c])
        terms += row
    for h in vh:
        terms += [h * p[c] for c in range(3)] + [h]
    return terms


def camgrad_sum(terms, kept):
    """The kernel's sums of the per-Gaussian terms over `kept`: (G_V, G_P, B_V, B_P), float64 [4,4] each on the terms'
    device (the bound as in the module docstring; row 3 of G_V and row 2 of G_P are 0 with bound 0)."""
    n = kept.shape[0]
    z = torch.zeros((), dtype=F8, device=kept.device)
    val = torch.stack([torch.where(kept, t.v, z).sum() for t in terms])
    bsum = torch.stack([torch.where(kept, t.b, z).sum() for t in terms])
    asum = torch.stack([torch.where(kept, t.v.abs(), z).sum() for t in terms])
    nb = (n + 255) // 256
    bound = C * (bsum + gamma(TREE_DEPTH) * (asum + bsum)) + gamma(nb + 5, U64) * (asum + bsum) + U * val.abs()
    GV, GP, BV, BP = (torch.zeros((4, 4), dtype=F8, device=kept.device) for _ in range(4))
    GV[:3] = val[:12].reshape(3, 4)
    BV[:3] = bound[:12].reshape(3, 4)
    GP[[0, 1, 3]] = val[12:].reshape(3, 4)
    BP[[0, 1, 3]] = bound[12:].reshape(3, 4)
    return GV, GP, BV, BP


def camgrad_tree(cam, means, scales, quats, logits, v_xy, v_conic, v_opacity=None, aa=False, kept=None, alt=None):
    """The kernel's sums on the tree: (G_V, G_P, B_V, B_P), float64 [4,4] each (the bound as in the module docstring;
    row 3 of G_V and row 2 of G_P are 0 with bound 0), over `kept`."""
    dev = torch.device("cpu")
    m, a, q, ol = (pf._t(x, dev) for x in (means, scales, quats, logits))
    n = m.shape[0]
    vx, vc = pf._t(v_xy, dev).reshape(n, 2), pf._t(v_conic, dev).reshape(n, 3)
    kept = torch.ones(n, dtype=torch.bool) if kept is None else torch.as_tensor(kept).cpu()
    p = [R(m[:, i]) for i in range(3)]
    qr = [R(q[:, i]) for i in range(4)]
    f = pf._forward_tree(cam, p, [R(a[:, i]) for i in range(3)], qr, 1.0, True, "cuda")
    dS = None
    if aa and v_opacity is not None:
        o = 1.0 / (1.0 + rexp(-R(ol)))
        dS = paa.comp_dS(f, kept, o, pf._t(v_opacity, dev).reshape(n))
    extra = {}
    pf._backward_tree(cam, f, qr, 1.0, True, f["conic"], [R(vx[:, 0]), R(vx[:, 1])], R(torch.zeros(n, dtype=F8)),
                      [R(vc[:, i]) for i in range(3)], dS, extra)
    return camgrad_sum(camgrad_terms(f, p, extra, alt), kept)


# ------------------------------------------------------------------------------------------------ pose chain
def rot6d(d, alt=None):
    """Rd (float64 [3,3]) of the 6-D offset d [6]: rows b1, b2, b3 (alt "columns": the columns)."""
    a = d + torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0], dtype=F8)
    a1, a2 = a[:3], a[3:]
    b1 = a1 / torch.sqrt((a1 * a1).sum())
    w = a2 - (b1 * a2).sum() * b1
    b2 = w / torch.sqrt((w * w).sum())
    b3 = torch.stack([b1[1] * b2[2] - b1[2] * b2[1], b1[2] * b2[0] - b1[0] * b2[2], b1[0] * b2[1] - b1[1] * b2[0]])
    Rd = torch.stack([b1, b2, b3])
    return Rd.T if alt == "columns" else Rd


def delta(e, alt=None):
    """Delta = [[Rd, t], [0, 1]], float64 [4,4]."""
    D = torch.eye(4, dtype=F8)
    D = D.index_put((torch.arange(3)[:, None], torch.arange(3)[None, :]), rot6d(e[3:9], alt))
    return D.index_put((torch.arange(3), torch.full((3,), 3)), e[0:3])


def pose_apply(e, view, centre, alt=None):
    """(view', centre') in float64: the camera [R|T] Delta, i.e. view' = Delta^-1 view and centre' = T + R t
    (alt "left": Delta [R|T], the correction in the world frame; "centre_unmoved": centre' = T)."""
    e, view, centre = (torch.as_tensor(x, dtype=F8).reshape(-1) for x in (e, view, centre))
    view = view.reshape(4, 4)
    Di = torch.linalg.inv(delta(e, alt))
    vp = view @ Di if alt == "left" else Di @ view
    cam = torch.linalg.inv(vp)                      # camera-to-world of view'
    c = centre if alt == "centre_unmoved" else cam[:3, 3]
    return vp, c


def pose_grad(e, view, proj, G_V, G_P, alt=None):
    """d/de of <G_V, view'(e)> + <G_P, proj view'(e)> by float64 autograd (alt "no_fold": the G_P term dropped)."""
    e = torch.as_tensor(e, dtype=F8).reshape(-1).clone().requires_grad_()
    view, proj = (torch.as_tensor(x, dtype=F8).reshape(4, 4) for x in (view, proj))
    with torch.enable_grad():
        vp, _ = pose_apply(e, view, torch.zeros(3, dtype=F8), alt if alt in ("left", "columns") else None)
        loss = (torch.as_tensor(G_V, dtype=F8) * vp).sum()
        if alt != "no_fold":
            loss = loss + (torch.as_tensor(G_P, dtype=F8) * (proj @ vp)).sum()
        (g,) = torch.autograd.grad(loss, [e])
    return g


def random_pose(seed, rot=0.02, trans=0.05):
    """A small correction e [9] (float32 values), as learning produces."""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.normal(0, trans, 3), rng.normal(0, rot, 6)]).astype(np.float32)
