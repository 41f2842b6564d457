"""Float64 restatement of the projection kernels (P1 / P2 of csrc/project.cu) with a per-element error bound and a
certificate of the kernels' decisions.

The forward follows the CUDA semantics that project.cu implements: view transform; cull unless t.z > clip_thresh;
M = R(q / |q|) S with S = glob_scale * scale (exp of the log-scale for the activated variant), cov3d = M M^T; the fov
clamp min(lim, max(-lim, t.x / t.z)) with lim = 1.3f * (float)(0.5 W / fx), as the kernel forms it; J, T = J V, cov2d
= T cov3d T^T + 0.3 I; det != 0 and the conic; radius = ceil(3 sqrt(max(v1, v2))); rw = 1 / (h.w + 1e-6), xy =
0.5 W ndc + cx - 0.5; the tile box of gsb_tile_bbox and area > 0.  cov3d is written for every Gaussian with
t.z > clip_thresh and the conic for every one with det != 0, even when the box is empty; everything else of a culled
Gaussian is 0.  The backward is torch autograd of that map (`vjp`), not a restatement of the kernel's hand-written VJP;
at an exact fov-clamp tie autograd splits the gradient of min / max in half, which is the reference's convention (D16).

The bound.  `R` is a value-plus-bound type over float64 tensors: a first-order running-error evaluation of an fp32
computation.  Each fp32 operation adds u |result| (u = 2^-24) to the propagated bounds of its operands; the device's
expf adds 2 ulp (<= 4 u |result|).  project.cu is compiled with --fmad=false, so every operation rounds on its own,
and `_forward_tree` / `_backward_tree` apply R along the kernel's own operation tree, in its order.  Their values are
those of the exact (float64) map, so they must equal the autograd values to float64 precision: that pins the
restatement of the tree, and the bound B then holds the kernels per element, |kernel - reference| <= C B.

The certificate.  A Gaussian is certified when each of its decisions lies clear of its threshold by the bound of the
operand: t.z vs clip_thresh, q = t / t.z vs +-lim (x and y), det vs 0, the ceil of the radius, the four truncations
of the tile box.  A decision is also certified where the fp32 evaluation of its operand (computed here in the
kernel's order: t and q) equals the float64 one exactly -- then kernel and reference take it the same way, which is
what makes a constructed exact tie, or t.z exactly at clip_thresh, checkable.  On certified Gaussians any correct fp32
implementation of the kernel's tree has the reference's radii and num_tiles_hit exactly.

Radii at or above 2^31 px are out of scope: the device's float -> int conversion saturates there and C's is undefined;
`project` asserts that no tile-box operand reaches 2^31.
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
F8 = torch.float64
TILE = 16
EXP_ULP = 4.0            # device expf: 2 ulp <= 4 u |result|


def f32(x):
    """The fp32 value of a Python number, as a Python float (exact in float64)."""
    return float(np.float32(x))


C03, C1E6, C01 = f32(0.3), f32(1e-6), f32(0.1)


class R:
    """A float64 value v and a bound b on the error of the fp32 evaluation that produced it (first order)."""
    __slots__ = ("v", "b")

    def __init__(self, v, b=None):
        self.v = v
        self.b = torch.zeros_like(v) if b is None else b

    @staticmethod
    def of(x, like):
        if isinstance(x, R):
            return x
        return R(torch.as_tensor(x, dtype=F8, device=like.device))

    def _r(self, v, b):
        return R(v, b + U * v.abs())

    def __add__(self, o):
        o = R.of(o, self.v)
        return self._r(self.v + o.v, self.b + o.b)

    def __radd__(self, o):
        return R.of(o, self.v) + self

    def __sub__(self, o):
        o = R.of(o, self.v)
        return self._r(self.v - o.v, self.b + o.b)

    def __rsub__(self, o):
        return R.of(o, self.v) - self

    def __mul__(self, o):
        o = R.of(o, self.v)
        return self._r(self.v * o.v, self.v.abs() * o.b + o.v.abs() * self.b)

    def __rmul__(self, o):
        return R.of(o, self.v) * self

    def __truediv__(self, o):
        o = R.of(o, self.v)
        v = self.v / o.v
        return self._r(v, (self.b + v.abs() * o.b) / o.v.abs())

    def __rtruediv__(self, o):
        return R.of(o, self.v) / self

    def __neg__(self):
        return R(-self.v, self.b)


def sqrtf(a):
    v = torch.sqrt(a.v)
    return R(v, a.b / (2 * v) + U * v)


def rexp(a):
    v = torch.exp(a.v)
    return R(v, v * a.b + EXP_ULP * U * v)


def rmin(a, o):
    """fminf: 1-Lipschitz in each operand, so the larger bound covers whichever operand the fp32 comparison picks."""
    o = R.of(o, a.v)
    return R(torch.minimum(a.v, o.v), torch.maximum(a.b, o.b))


def rmax(a, o):
    o = R.of(o, a.v)
    return R(torch.maximum(a.v, o.v), torch.maximum(a.b, o.b))


def rwhere(m, a, o):
    a, o = R.of(a, m), R.of(o, m)
    return R(torch.where(m, a.v, o.v), torch.where(m, a.b, o.b))


# -------------------------------------------------------------------------------------------------------- camera
class Cam:
    """The kernels' scalar arguments, held as the fp32 values the kernel receives."""

    def __init__(self, viewmat, projmat, fx, fy, cx, cy, img_h, img_w, clip_thresh=0.01):
        self.V = np.asarray(viewmat, np.float32).reshape(16)
        self.P = np.asarray(projmat, np.float32).reshape(16)
        self.fx, self.fy, self.cx, self.cy = f32(fx), f32(fy), f32(cx), f32(cy)
        self.H, self.W = int(img_h), int(img_w)
        self.clip = f32(clip_thresh)
        self.tiles_x, self.tiles_y = (self.W + TILE - 1) // TILE, (self.H + TILE - 1) // TILE
        # project_forward_impl: `0.5 * img_w / fx` in double, narrowed; then 1.3f * that in fp32
        self.lim_x = float(np.float32(1.3) * np.float32(0.5 * self.W / self.fx))
        self.lim_y = float(np.float32(1.3) * np.float32(0.5 * self.H / self.fy))
        # the reference's CPU back end forms 0.5f * W / fx in fp32 (gsplat_cpu.cpp:64-65)
        self.lim_x_cpu = float(np.float32(1.3) * (np.float32(0.5) * np.float32(self.W) / np.float32(self.fx)))
        self.lim_y_cpu = float(np.float32(1.3) * (np.float32(0.5) * np.float32(self.H) / np.float32(self.fy)))

    def args(self):
        """(viewmat, projmat, fx, fy, cx, cy, H, W) for the oracle and the kernels."""
        return (self.V.reshape(4, 4), self.P.reshape(4, 4), self.fx, self.fy, self.cx, self.cy, self.H, self.W)


def camera_from_setup(cam, downscale=1.0, clip_thresh=0.01):
    """A Cam from model.camera_setup: the full projection is proj @ view, formed in fp32 as the trainer does."""
    from opensplat_b200.model import camera_setup
    H, W, (fx, fy, cx, cy), view, proj, _ = camera_setup(cam, downscale)
    return Cam(view.numpy(), (proj @ view).numpy(), fx, fy, cx, cy, H, W, clip_thresh)


# ------------------------------------------------------------------------------------------------ operation trees
def _t(a, dev):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev, F8)


def _quat_to_rotmat(qw, qx, qy, qz):
    s = 1.0 / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz)
    w, x, y, z = qw * s, qx * s, qy * s, qz * s
    return [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)],
            [2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x)],
            [2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]]


def _filter3d_scales(s, f3):
    """filter3d_scales of project.cu on R: sigma_k = sqrtf(s_k s_k + f f), r_k = s_k / sigma_k, c3 = (r_0 r_1) r_2."""
    ff = f3 * f3
    sig = [sqrtf(x * x + ff) for x in s]
    fr = [x / g for x, g in zip(s, sig)]
    return sig, fr, fr[0] * fr[1] * fr[2]


def _covariance(q, a, glob_scale, act, f3=None):
    """R(q / |q|), e (exp of the log-scales under act), s = glob_scale e, and M = R S, cov3d = M M^T on R; with the
    3-D filter f3 (an R over [N]) S holds sigma_k and the dict also fr (r_k), c3 and f3."""
    Rm = _quat_to_rotmat(*q)
    e = [rexp(x) if act else x for x in a]
    s = [glob_scale * x for x in e]
    out = dict(Rm=Rm, e=e)
    if f3 is not None:
        s, fr, c3 = _filter3d_scales(s, f3)
        out.update(fr=fr, c3=c3, f3=f3)
    M = [[Rm[r][c] * s[c] for c in range(3)] for r in range(3)]
    C = [[M[r][0] * M[c][0] + M[r][1] * M[c][1] + M[r][2] * M[c][2] for c in range(3)] for r in range(3)]
    out.update(s=s, M=M, C=C, cov3d=[C[0][0], C[0][1], C[0][2], C[1][1], C[1][2], C[2][2]])
    return out


def _view(V, p):
    px, py, pz = p
    return (V[0] * px + V[1] * py + V[2] * pz + V[3], V[4] * px + V[5] * py + V[6] * pz + V[7],
            V[8] * px + V[9] * py + V[10] * pz + V[11])


def _forward_tree(cam, p, a, q, glob_scale, act, d3, f3=None):
    """project_forward_kernel's tree on R.  p [3] means, a [3] (log-)scales, q [4] raw quaternion, each R over [N];
    f3: the F3D mode's filter (an R over [N]), or None."""
    V, P = [float(x) for x in cam.V], [float(x) for x in cam.P]
    px, py, pz = p
    tx, ty, tz = _view(V, p)
    cv = _covariance(q, a, glob_scale, act, f3)
    C = cv["C"]
    lim_x, lim_y = (cam.lim_x, cam.lim_y) if d3 == "cuda" else (cam.lim_x_cpu, cam.lim_y_cpu)
    qx, qy = tx / tz, ty / tz
    cqx, cqy = rmin(rmax(qx, -lim_x), lim_x), rmin(rmax(qy, -lim_y), lim_y)
    ttx, tty = tz * cqx, tz * cqy
    rz = 1.0 / tz
    rz2 = rz * rz
    fx, fy = cam.fx, cam.fy
    J00, J02, J11, J12 = fx * rz, -fx * ttx * rz2, fy * rz, -fy * tty * rz2
    T = [[J00 * V[c] + J02 * V[8 + c] for c in range(3)], [J11 * V[4 + c] + J12 * V[8 + c] for c in range(3)]]
    TV = [[T[r][0] * C[0][c] + T[r][1] * C[1][c] + T[r][2] * C[2][c] for c in range(3)] for r in range(2)]
    cxx = TV[0][0] * T[0][0] + TV[0][1] * T[0][1] + TV[0][2] * T[0][2] + C03
    cxy = TV[0][0] * T[1][0] + TV[0][1] * T[1][1] + TV[0][2] * T[1][2]
    cyy = TV[1][0] * T[1][0] + TV[1][1] * T[1][1] + TV[1][2] * T[1][2] + C03
    det = cxx * cyy - cxy * cxy
    inv_det = 1.0 / det
    conic = [cyy * inv_det, -cxy * inv_det, cxx * inv_det]
    b = 0.5 * (cxx + cyy)
    sq = sqrtf(rmax(b * b - det, C01))
    v1, v2 = b + sq, b - sq
    r3 = 3.0 * sqrtf(rmax(v1, v2))
    hx = P[0] * px + P[1] * py + P[2] * pz + P[3]
    hy = P[4] * px + P[5] * py + P[6] * pz + P[7]
    hw = P[12] * px + P[13] * py + P[14] * pz + P[15]
    rw = 1.0 / (hw + C1E6) if d3 == "cuda" else 1.0 / rmax(hw, C1E6)
    ndcx, ndcy = hx * rw, hy * rw
    cx, cy = (cam.cx, cam.cy) if d3 == "cuda" else (0.5 * cam.W, 0.5 * cam.H)
    pxc = 0.5 * float(cam.W) * ndcx + cx - 0.5
    pyc = 0.5 * float(cam.H) * ndcy + cy - 0.5
    return dict(cv, t=(tx, ty, tz), q=(qx, qy), cq=(cqx, cqy), tt=(ttx, tty), rz=(rz, rz2), J=(J00, J02, J11, J12),
                T=T, det=det, conic=conic, r3=r3, h=(hx, hy, hw), rw=rw, xy=(pxc, pyc), lim=(lim_x, lim_y))


def _vS(conic, v_conic, dS=None):
    """v_Sigma = -X G X from the conic and its cotangent, plus the anti-aliased dS = (mask, d00, d01, d11) where given
    (project_aa_f64.comp_dS), in the kernel's order."""
    A, B, Cc = conic
    gA, gB, gC = v_conic[0], 0.5 * v_conic[1], v_conic[2]
    xg00, xg01 = A * gA + B * gB, A * gB + B * gC
    xg10, xg11 = B * gA + Cc * gB, B * gB + Cc * gC
    vS00 = -(xg00 * A + xg01 * B)
    vS01 = -(xg00 * B + xg01 * Cc)
    vS11 = -(xg10 * B + xg11 * Cc)
    if dS is not None:
        mask, d00, d01, d11 = dS
        vS00 = rwhere(mask, vS00 + d00, vS00)
        vS01 = rwhere(mask, vS01 - d01, vS01)
        vS11 = rwhere(mask, vS11 + d11, vS11)
    return vS00, vS01, vS11


def _cov2d_chain(T, Cs, vS):
    """(vV, vT): cov2d = T cov3d T^T taken back to cov3d and to T."""
    vS00, vS01, vS11 = vS
    vST = [[vS00 * T[0][c] + vS01 * T[1][c] for c in range(3)], [vS01 * T[0][c] + vS11 * T[1][c] for c in range(3)]]
    vV = [[T[0][r] * vST[0][c] + T[1][r] * vST[1][c] for c in range(3)] for r in range(3)]
    vT = [[2.0 * (vST[r][0] * Cs[0][c] + vST[r][1] * Cs[1][c] + vST[r][2] * Cs[2][c]) for c in range(3)]
          for r in range(2)]
    return vV, vT


def _scale_quat(f, q, glob_scale, act, vV):
    """(v_scale, v_quat) from vV = d/d cov3d: M = R S, the log-scale's exp under act, and the F3D factor r_k where the
    forward tree carries the filter (S then holds sigma_k)."""
    M, Rm, e, s = f["M"], f["Rm"], f["e"], f["s"]
    vM = [[2.0 * (vV[r][0] * M[0][c] + vV[r][1] * M[1][c] + vV[r][2] * M[2][c]) for c in range(3)] for r in range(3)]
    vs = [glob_scale * (Rm[0][c] * vM[0][c] + Rm[1][c] * vM[1][c] + Rm[2][c] * vM[2][c]) for c in range(3)]
    if act:
        vs = [vs[c] * e[c] for c in range(3)]
    if "fr" in f:
        vs = [vs[c] * f["fr"][c] for c in range(3)]
    vR = [[vM[r][c] * s[c] for c in range(3)] for r in range(3)]
    qw_, qx_, qy_, qz_ = q
    nq = sqrtf(qw_ * qw_ + qx_ * qx_ + qy_ * qy_ + qz_ * qz_)
    inv = 1.0 / nq
    w, x, y, z = qw_ * inv, qx_ * inv, qy_ * inv, qz_ * inv
    gw = 2.0 * (x * (vR[2][1] - vR[1][2]) + y * (vR[0][2] - vR[2][0]) + z * (vR[1][0] - vR[0][1]))
    gx = 2.0 * (-2.0 * x * (vR[1][1] + vR[2][2]) + y * (vR[1][0] + vR[0][1]) + z * (vR[2][0] + vR[0][2])
                + w * (vR[2][1] - vR[1][2]))
    gy = 2.0 * (x * (vR[1][0] + vR[0][1]) - 2.0 * y * (vR[0][0] + vR[2][2]) + z * (vR[2][1] + vR[1][2])
                + w * (vR[0][2] - vR[2][0]))
    gz = 2.0 * (x * (vR[2][0] + vR[0][2]) + y * (vR[2][1] + vR[1][2]) - 2.0 * z * (vR[0][0] + vR[1][1])
                + w * (vR[1][0] - vR[0][1]))
    dot = w * gw + x * gx + y * gy + z * gz
    vq = [(gw - w * dot) * inv, (gx - x * dot) * inv, (gy - y * dot) * inv, (gz - z * dot) * inv]
    return vs, vq


def _backward_tree(cam, f, q, glob_scale, act, conic, v_xy, v_depth, v_conic, dS=None, extra=None):
    """project_backward_kernel's tree on R, from the forward tree's intermediates (the kernel recomputes the same
    values in the same order) and the forward's conic (which carries the forward's bound).  dS: the anti-aliased
    term added to vS (project_aa_f64.comp_dS).  extra: a dict that receives vt, vT and vh, the camera gradient's
    inputs."""
    V, P = [float(x) for x in cam.V], [float(x) for x in cam.P]
    fx, fy = cam.fx, cam.fy
    hx, hy, hw = f["h"]
    rw = f["rw"]
    vndcx, vndcy = (0.5 * float(cam.W)) * v_xy[0], (0.5 * float(cam.H)) * v_xy[1]
    vhx, vhy = vndcx * rw, vndcy * rw
    vhw = -(vndcx * hx + vndcy * hy) * rw * rw
    vm = [P[c] * vhx + P[4 + c] * vhy + P[12 + c] * vhw for c in range(3)]
    vtz = v_depth
    vV, vT = _cov2d_chain(f["T"], f["C"], _vS(conic, v_conic, dS))
    ttx, tty = f["tt"]
    cqx, cqy = f["cq"]
    qx, qy = f["q"]
    rz, rz2 = f["rz"]
    rz3 = rz2 * rz
    vJ00 = vT[0][0] * V[0] + vT[0][1] * V[1] + vT[0][2] * V[2]
    vJ02 = vT[0][0] * V[8] + vT[0][1] * V[9] + vT[0][2] * V[10]
    vJ11 = vT[1][0] * V[4] + vT[1][1] * V[5] + vT[1][2] * V[6]
    vJ12 = vT[1][0] * V[8] + vT[1][1] * V[9] + vT[1][2] * V[10]
    vttx, vtty = -fx * rz2 * vJ02, -fy * rz2 * vJ12
    vtz = vtz + (-fx * rz2 * vJ00 + 2.0 * fx * ttx * rz3 * vJ02 - fy * rz2 * vJ11 + 2.0 * fy * tty * rz3 * vJ12)
    vt = []
    for qq, cq, vtt, lim in ((qx, cqx, vttx, f["lim"][0]), (qy, cqy, vtty, f["lim"][1])):
        tie = (qq.v == lim) | (qq.v == -lim)
        clamped = ~((qq.v > -lim) & (qq.v < lim))
        h = 0.5 * vtt
        vt.append(rwhere(tie, h, rwhere(clamped, 0.0, vtt)))
        vtz = rwhere(tie, vtz + cq * h, rwhere(clamped, vtz + cq * vtt, vtz))
    vtx, vty = vt
    vm = [vm[c] + (V[c] * vtx + V[4 + c] * vty + V[8 + c] * vtz) for c in range(3)]
    if extra is not None:
        extra.update(vt=(vtx, vty, vtz), vT=vT, vh=(vhx, vhy, vhw))
    vs, vq = _scale_quat(f, q, glob_scale, act, vV)
    return vm, vs, vq


# ------------------------------------------------------------------------------------------------ autograd map
def _rotmat(qn):
    w, x, y, z = qn.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def forward_map(cam, means, scales, quats, glob_scale=1.0, act=False, opacity_logits=None, d3="cuda", alt=None):
    """The projection as a differentiable float64 map of (means, scales, quats[, opacity_logits]):
    returns xys [N,2], depths [N], conics [N,3], cov3d [N,6], opacities [N] (or None).
    d3: "cuda" -> rw = 1/(w + 1e-6) and xy = 0.5 W ndc + cx - 0.5; "cpu" -> the reference's CPU back end, rw =
    1/max(w, 1e-6), its fp32 lim and xy = 0.5 ((ndc + 1) W - 1) (cx, cy ignored).
    alt: a known wrong gradient convention, for the sensitivity checks: "no_d8" (clamp sub-gradient dropped), "no_d11"
    (normalisation Jacobian dropped), "no_d12" (perspective-divide term dropped), "JVt" (T = J V^T), "full_clamp"
    (at a tie, the clamped branch)."""
    dev = means.device
    V = torch.as_tensor(cam.V, device=dev).to(F8).reshape(4, 4)
    P = torch.as_tensor(cam.P, device=dev).to(F8).reshape(4, 4)
    t = means @ V[:3, :3].T + V[:3, 3]
    qn = quats / quats.norm(dim=-1, keepdim=True)
    if alt == "no_d11":
        qn = quats + (qn - quats).detach()
    Rm = _rotmat(qn)
    s = glob_scale * (torch.exp(scales) if act else scales)
    M = Rm * s[:, None, :]
    cov3 = M @ M.transpose(1, 2)
    tz = t[:, 2]
    lim = torch.tensor([cam.lim_x, cam.lim_y] if d3 == "cuda" else [cam.lim_x_cpu, cam.lim_y_cpu], dtype=F8,
                       device=dev)
    qv = t[:, :2] / tz[:, None]
    cq = torch.minimum(lim, torch.maximum(-lim, qv))        # the reference's min / max: a tie splits the gradient
    if alt == "no_d8":
        cq = qv + (cq - qv).detach()
    elif alt == "full_clamp":
        cq = torch.where((qv >= lim) | (qv <= -lim), cq.detach(), qv)
    tt = tz[:, None] * cq
    rz = 1.0 / tz
    zero = torch.zeros_like(rz)
    J = torch.stack([cam.fx * rz, zero, -cam.fx * tt[:, 0] * rz * rz,
                     zero, cam.fy * rz, -cam.fy * tt[:, 1] * rz * rz], -1).reshape(-1, 2, 3)
    T = J @ (V[:3, :3].T if alt == "JVt" else V[:3, :3])
    cov2 = T @ cov3 @ T.transpose(1, 2)
    cxx, cxy, cyy = cov2[:, 0, 0] + C03, cov2[:, 0, 1], cov2[:, 1, 1] + C03
    det = cxx * cyy - cxy * cxy
    conic = torch.stack([cyy / det, -cxy / det, cxx / det], -1)
    hom = means @ P[:, :3].T + P[:, 3]
    rw = 1.0 / (hom[:, 3] + C1E6) if d3 == "cuda" else 1.0 / hom[:, 3].clamp_min(C1E6)
    if alt == "no_d12":
        rw = rw.detach()
    cx, cy = (cam.cx, cam.cy) if d3 == "cuda" else (0.5 * cam.W, 0.5 * cam.H)
    xy = torch.stack([0.5 * cam.W * hom[:, 0] * rw + cx - 0.5, 0.5 * cam.H * hom[:, 1] * rw + cy - 0.5], -1)
    c6 = cov3.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]]
    opac = torch.sigmoid(opacity_logits) if opacity_logits is not None else None
    return xy, tz, conic, c6, opac


def vjp(cam, means, scales, quats, v_xy, v_depth, v_conic, glob_scale=1.0, act=False, opacity_logits=None,
        v_opacity=None, d3="cuda", alt=None):
    """Autograd of forward_map for the cotangents: (v_mean3d, v_scale, v_quat, v_opacity_logits or None), float64,
    for every Gaussian (the caller masks the culled ones)."""
    dev = means.device
    ins = [x.detach().to(F8).clone().requires_grad_() for x in (means, scales, quats)]
    ol = opacity_logits.detach().to(F8).clone().requires_grad_() if opacity_logits is not None else None
    with torch.enable_grad():
        xy, tz, conic, _, opac = forward_map(cam, *ins, glob_scale, act, ol, d3, alt)
        loss = (torch.where(torch.isfinite(xy), xy, 0) * v_xy).sum() + (torch.where(torch.isfinite(conic), conic, 0)
                                                                         * v_conic).sum()
        if v_depth is not None:
            loss = loss + (tz * v_depth).sum()
        if opac is not None and v_opacity is not None:
            loss = loss + (opac * v_opacity).sum()
        args = ins + ([ol] if ol is not None else [])
        g = torch.autograd.grad(loss, args, allow_unused=True)
    g = [x if x is not None else torch.zeros_like(a) for x, a in zip(g, args)]
    return g[0], g[1], g[2], (g[3] if ol is not None else None)


# ------------------------------------------------------------------------------------------------ the reference
def _trunc_box(x, n):
    return (torch.trunc(x).clamp(0, n)).to(torch.int64)


def _exact32(cam, means):
    """t and q as the kernel evaluates them in fp32 (same order, every operation rounded), float64 on return."""
    V = [torch.tensor(float(v), dtype=torch.float32, device=means.device) for v in cam.V]
    m = means.to(torch.float32)
    px, py, pz = m[:, 0], m[:, 1], m[:, 2]
    tx = V[0] * px + V[1] * py + V[2] * pz + V[3]
    ty = V[4] * px + V[5] * py + V[6] * pz + V[7]
    tz = V[8] * px + V[9] * py + V[10] * pz + V[11]
    return tz.to(F8), (tx / tz).to(F8), (ty / tz).to(F8)


def stack_masked(rs, mask):
    """(values, bounds) of a list of R as [N, len] float64, 0 (bound 0) outside mask."""
    z = torch.zeros((), dtype=F8, device=mask.device)
    return (torch.stack([torch.where(mask, r.v.to(F8), z) for r in rs], -1),
            torch.stack([torch.where(mask, r.b.to(F8), z) for r in rs], -1))


def forward_outputs(cam, f, m, d3="cuda"):
    """The forward outputs of a forward tree f (pinhole, any mode): cov3d, xys, depths, radii, conics, num_tiles_hit
    with bounds B_<name>, kept, cert and the decisions' flags.  m: the means (float64 [N,3])."""
    dev, n = m.device, m.shape[0]
    tx, ty, tz = f["t"]
    front = tz.v > cam.clip
    tz32, qx32, qy32 = _exact32(cam, m)
    exact_tz = tz32 == tz.v
    d_front = ((tz.v - cam.clip).abs() > tz.b) | exact_tz
    qx, qy = f["q"]
    lim_x, lim_y = f["lim"]

    def d_q(qq, q32, lim):
        return (((qq.v - lim).abs() > qq.b) & ((qq.v + lim).abs() > qq.b)) | (q32 == qq.v)

    d_det = f["det"].v.abs() > f["det"].b
    has_conic = front & (f["det"].v != 0)
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
    kept = has_conic & (area > 0) if d3 == "cuda" else has_conic       # the CPU back end has no tile cull
    cert = d_front & (~front | (d_q(qx, qx32, lim_x) & d_q(qy, qy32, lim_y) & d_det & (d_ceil & d_box)))
    assert not bool((front & ~(f["det"].v > 0)).any()), "cov2d + 0.3 I is positive definite"

    z = torch.zeros((), dtype=F8, device=dev)
    out = dict(kept=kept, front=front, cert=cert, exact_tz=exact_tz,
               tie_x=front & ((qx.v == lim_x) | (qx.v == -lim_x)), tie_y=front & ((qy.v == lim_y) | (qy.v == -lim_y)),
               clamp_x=front & (qx.v.abs() > lim_x), clamp_y=front & (qy.v.abs() > lim_y))
    stack = stack_masked
    out["cov3d"], out["B_cov3d"] = stack(f["cov3d"], front)
    out["conics"], out["B_conics"] = stack(f["conic"], has_conic)
    out["xys"], out["B_xys"] = stack([pxc, pyc], kept)
    out["depths"], out["B_depths"] = torch.where(kept, tz.v, z), torch.where(kept, tz.b, z)
    out["radii"] = torch.where(kept, radius, z).to(torch.int64)
    out["num_tiles_hit"] = torch.where(kept, area, torch.zeros_like(area))
    return out


def project(cam, means, scales, quats, glob_scale=1.0, act=False, opacity_logits=None, v_xy=None, v_depth=None,
            v_conic=None, v_opacity=None, d3="cuda", device=None):
    """The float64 reference of gsb_project_forward[_activated] and, with cotangents, gsb_project_backward[_activated].
    Inputs are the kernels' fp32 inputs (numpy or torch); everything returned is float64 (radii / num_tiles_hit
    int64) on `device` (default: that of `means`).  Keys: the forward outputs cov3d, xys, depths, radii, conics,
    num_tiles_hit (and opacities) with bounds B_<name>; kept (radii > 0); cert; the decisions' own flags
    (exact_tz, tie_x, tie_y, clamp_x, clamp_y); with v_xy / v_conic given, v_mean3d, v_scale, v_quat (and
    v_opacity_logits) from autograd, their bounds B_<name>, and re_<name>, the values of the bound's evaluation."""
    dev = device if device is not None else (means.device if torch.is_tensor(means) else "cpu")
    m, a, q = _t(means, dev), _t(scales, dev), _t(quats, dev)
    n = m.shape[0]
    ol = _t(opacity_logits, dev).reshape(n) if opacity_logits is not None else None
    f = _forward_tree(cam, [R(m[:, i]) for i in range(3)], [R(a[:, i]) for i in range(3)],
                      [R(q[:, i]) for i in range(4)], glob_scale, act, d3)
    out = forward_outputs(cam, f, m, d3)
    tz = f["t"][2]
    kept = out["kept"]
    z = torch.zeros((), dtype=F8, device=dev)

    def stack(rs, mask):
        v = torch.stack([torch.where(mask, r.v, z) for r in rs], -1)
        b = torch.stack([torch.where(mask, r.b, z) for r in rs], -1)
        return v, b

    if act:
        o = 1.0 / (1.0 + rexp(-R(ol)))
        out["opacities"], out["B_opacities"] = o.v, o.b
    if v_xy is None:
        return out

    vx, vc = _t(v_xy, dev).reshape(n, 2), _t(v_conic, dev).reshape(n, 3)
    vd = _t(v_depth, dev).reshape(n) if v_depth is not None else None
    vo = _t(v_opacity, dev).reshape(n) if (act and v_opacity is not None) else None
    g = vjp(cam, m, a, q, vx, vd, vc, glob_scale, act, ol, vo, d3)
    vm, vs, vq = _backward_tree(cam, f, [R(q[:, i]) for i in range(4)], glob_scale, act, f["conic"],
                                [R(vx[:, 0]), R(vx[:, 1])], R(vd) if vd is not None else R(torch.zeros_like(tz.v)),
                                [R(vc[:, i]) for i in range(3)])
    for name, rs, gv in (("v_mean3d", vm, g[0]), ("v_scale", vs, g[1]), ("v_quat", vq, g[2])):
        out["re_" + name], out["B_" + name] = stack(rs, kept)
        out[name] = torch.where(kept[:, None], gv, z)
    if act:
        # v o (1 - o) from the saved (fp32, bounded) opacity; where fp32 sigmoid rounds to 1 the kernel's 1 - o is 0
        # and so is its gradient, and the bound of 1 - o (that of o, >= u) covers the exact o (1 - o) ~ e^-x it drops
        o = R(out["opacities"], out["B_opacities"])
        vol = (R(vo) * o * (1.0 - o)) if vo is not None else R(torch.zeros_like(tz.v))
        out["re_v_opacity_logits"], out["B_v_opacity_logits"] = vol.v, vol.b
        out["v_opacity_logits"] = g[3] if vo is not None else torch.zeros_like(tz.v)
    return out


# ------------------------------------------------------------------------------------------------ scenes
def general_camera(W, H, seed, fx_ratio=1.17, downscale=1.0):
    """A model.Camera with a rotated and translated camToWorld, fx != fy and an off-centre principal point."""
    from opensplat_b200.model import Camera
    rng = np.random.default_rng(seed)
    ax = rng.standard_normal(3)
    ax /= np.linalg.norm(ax)
    ang = rng.uniform(0.3, 1.2)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    Rw = np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K
    c2w = np.eye(4)
    c2w[:3, :3] = Rw
    c2w[:3, 3] = rng.uniform(-2, 2, 3)
    fx = 0.9 * max(W, H) + 1.0
    return Camera(W, H, fx, fx * fx_ratio, 0.5 * W + 0.137 * W, 0.5 * H - 0.091 * H, c2w.astype(np.float32))


def view_to_world(cam, t):
    """World points whose view-space position is t (float64), as fp32."""
    V = cam.V.reshape(4, 4).astype(np.float64)
    return ((t - V[:3, 3]) @ V[:3, :3]).astype(np.float32)      # V[:3,:3] is a rotation: its inverse is its transpose


def random_gaussians(cam, n, seed, near=(0.02, 0.2), frac_near=0.1, frac_out=0.06, q_norm=(0.5, 2.0),
                     px_std=(0.05, 40.0), act=False):
    """Gaussians in the camera's view: t.z log-uniform in [0.3, 30] (a fraction frac_near in `near`), t.x / t.z and
    t.y / t.z uniform inside +-1.1 lim, or (frac_out of them) up to 2.5 lim beyond the fov clamp on any side and in
    the corners, with footprints of 0.1 to 0.5 image width, some of which reach into the image; the others have
    standard deviations log-uniform in px_std pixels.  Raw quaternions with norms log-uniform in q_norm.
    Returns (means, scales, quats) fp32 -- scales are log-scales when act."""
    rng = np.random.default_rng(seed)
    tz = np.exp(rng.uniform(np.log(0.3), np.log(30.0), n))
    k = rng.uniform(size=n) < frac_near
    tz[k] = rng.uniform(near[0], near[1], k.sum())
    lim = np.array([cam.lim_x, cam.lim_y])
    qv = rng.uniform(-1.1, 1.1, (n, 2)) * lim
    o = rng.uniform(size=n) < frac_out
    qv[o] = rng.uniform(-2.5, 2.5, (o.sum(), 2)) * lim
    s = np.exp(rng.uniform(np.log(px_std[0]), np.log(px_std[1]), (n, 3))) * (tz / cam.fx)[:, None]
    s[o] = rng.uniform(0.03, 0.12, (o.sum(), 3)) * (lim[0] * tz[o])[:, None]    # 3 sigma: 0.1 to 0.5 image width
    t = np.stack([qv[:, 0] * tz, qv[:, 1] * tz, tz], -1)
    quats = rng.standard_normal((n, 4)) * np.exp(rng.uniform(np.log(q_norm[0]), np.log(q_norm[1]), (n, 1)))
    sc = np.log(s) if act else s
    return view_to_world(cam, t), sc.astype(np.float32), quats.astype(np.float32)


def tie_gaussians(cam, seed, tz=2.0):
    """Gaussians exactly on the fov clamp (t.x / t.z == +-lim_x, t.y / t.z == +-lim_y, and corners), for a camera
    with an identity view rotation and zero translation, so that t and q are exact in fp32.  Wide enough to be
    visible.  Returns (means, scales, quats)."""
    V = cam.V.reshape(4, 4)
    assert np.array_equal(V, np.eye(4, dtype=np.float32)), "ties need the identity view"
    rng = np.random.default_rng(seed)
    lx, ly = cam.lim_x, cam.lim_y
    pts = []
    for sx, sy in ((1, None), (-1, None), (None, 1), (None, -1), (1, 1), (-1, 1), (1, -1), (-1, -1)):
        for _ in range(3):
            x = sx * lx * tz if sx is not None else rng.uniform(-0.8, 0.8) * lx * tz
            y = sy * ly * tz if sy is not None else rng.uniform(-0.8, 0.8) * ly * tz
            pts.append([x, y, tz])
    t = np.array(pts, np.float32)
    n = t.shape[0]
    assert np.all(t[:, 2] == np.float32(tz))
    s = (rng.uniform(0.3, 0.8, (n, 3)) * tz).astype(np.float32)
    quats = (rng.standard_normal((n, 4)) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    return t, s, quats
