"""Float64 restatement of the small streaming kernels of csrc/fused.cu -- Adam (plain and segmented), the parameter
activations, the densification statistics and the MSE loss -- with a per-element error bound and a certificate of the
kernels' decisions.  Bounds use project_f64.R: a first-order running-error evaluation of the kernel's fp32 tree, each
operation adding u |result| (u = 2^-24).  Where a result can be subnormal or underflow, each rounding here also adds
ETA = 2^-150 (half the smallest subnormal spacing), which R alone does not.

Adam.  The value is one step of libtorch's torch::optim::Adam (model.cpp), restated from the fp32 state the kernel
started with (so errors never compound across steps), with the scalars formed as libtorch forms them: bc1 = 1 - b1^t
and bc2 = 1 - b2^t in double, and every scalar operand narrowed to float by ATen:
    m' = b1 m + (1 - b1) g,  v' = b2 v + (1 - b2) g^2,  p' = p - (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps)
with b1 = 0.9f, 1 - b1 = fl(0.1), b2 = 0.999f, 1 - b2 = fl(0.001), lr / bc1 and sqrt(bc2) rounded from double, eps =
1e-8f.  The bound follows adam_update's tree: m' = fmaf(1 - b1, g, b1 m), v' = fmaf(g, (1 - b2) g, b2 v), den =
fmaf(sqrtf(v'), 1 / sqrt(bc2), eps), q = __fdividef(m', den) at 2 ulp, then the FMUL by lr * (1 / bc1) and the FSUB.
The kernel forms its scalars in fp32 -- 1.f - b1 = 0.10000002f, 1.f - b2, lr * (1.f / bc1), 1.f / sqrtf(bc2) -- and
each is charged its distance to libtorch's, as loss_f64 charges C1 / C2.  Errors propagate to first order through
1 / den and m' / den^2.
__fdividef's 2-ulp bound holds for denominators in [2^-126, 2^126]: den >= eps = 1e-8 > 2^-126, and a finite v' is at
most FLT_MAX, so den <= sqrt(FLT_MAX) / sqrt(1 - b2) + eps < 6e20 < 2^126 for the b2 and eps in use (asserted in
`adam`).  The one decision is the overflow of v' (|g| above about 5.8e20 from a zero state): where the exact v' lies
above the overflow threshold by more than its bound the kernel must write v' = inf and leave p unchanged (q = m' / inf
= 0), exactly, as libtorch does; where it lies below by more than its bound the bound holds.  Only elements within
the bound of the threshold are uncertified.  The segmented kernel runs the same step, each element taking lr_head
where e % row_floats < head_floats, e counted from its segment's start, and lr_rest elsewhere.

Activations (activate_forward_kernel / activate_backward_kernel, model.cpp:148-150,176-177,200).  The values are the
reference's op sequence in float64 -- exp, q / |q|, sigmoid, normalize(means - cam) -- and the VJPs autograd of it.
fused.cu is built with --fmad=true; the bound takes every operation rounded on its own, which dominates the fused
ones (as loss_f64 notes).  The device's expf is charged 2 ulp (EXP_ULP).  Decisions: where exp(s) exceeds FLT_MAX by
more than 4 u, scales must be +inf (and the VJP v * inf, as also where v * scale itself overflows); where exp(-x) does, the opacity must be exactly 0 and its
VJP exactly 0.  Within 4 u of the threshold an element is uncertified.  The quaternion bound is restricted to norms
whose squares stay normal ([2^-63, 2^63]); outside it the kernel's |q|^2 underflows into the subnormals or overflows
(|q| >= 2^64 gives |q|^2 = inf, so 1 / |q| = 0 and the quaternion and its VJP come out 0, and a zero quaternion gives
NaN), which `activate` records in `q_in_range` without bounding.

Densification statistics (densify_stats_kernel / densify_stats_init_kernel, model.cpp:317-337).  |v_xy| =
sqrtf(gx^2 + gy^2) is bounded; vis_counts is exact; max_2d_size = fmaxf(old, (float)r / max(H, W)) is bit-exact,
the IEEE division restated with float32 numpy division (a rounded float64 quotient could round twice).  Update leaves
rows with radii <= 0 alone; init sets every row: |v_xy| and 1 also for invisible Gaussians (the reference's quirk),
and max_2d_size 0 there.

MSE (mse_loss_grad_kernel).  v_img = fl(fl(2 inv_count) fl(a - b)) is reproduced bit for bit in float32.  The loss
is an fp32 sum: per-thread chains of ceil(n4 / stride) float4 terms (4-term sums) plus the scalar tail, the 5 + 3
levels of the shuffle tree, the multiply by inv_count and one atomic per block (8 SMs blocks, in any order); a sum of
depth d errs by at most d u sum |terms|."""
import math

import numpy as np
import torch

from project_f64 import EXP_ULP, F8, U, R, f32

ETA = 2.0 ** -150
FLT_MAX = float(np.finfo(np.float32).max)
OVF = 2.0 ** 128 * (1.0 - 2.0 ** -25)    # the smallest real that rounds to +inf in fp32
LN_OVF = math.log(OVF)


def _t(a, dev, dt=F8):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev, dt)


def _rd(v, b):
    """One fp32 rounding of exact value v with propagated bound b."""
    return R(v, b + U * v.abs() + ETA)


def rmul(a, o):
    return _rd(a.v * o.v, a.v.abs() * o.b + o.v.abs() * a.b)


def radd(a, o):
    return _rd(a.v + o.v, a.b + o.b)


def rsub(a, o):
    return _rd(a.v - o.v, a.b + o.b)


def rfma(a, o, c):
    """fmaf(a, o, c): one rounding."""
    return _rd(a.v * o.v + c.v, a.v.abs() * o.b + o.v.abs() * a.b + c.b)


def rdiv(a, o, ulp=1.0):
    """a / o, correctly rounded (ulp = 1: u) or within `ulp` ulp (<= 2 ulp u |result| each)."""
    v = a.v / o.v
    b = (a.b + v.abs() * o.b) / o.v.abs()
    return R(v, b + (U if ulp == 1.0 else 2.0 * ulp * U) * v.abs() + ETA)


def rsqrt_(a):
    """sqrtf (IEEE): first order a.b / (2 sqrt a), never more than sqrt(a.b)."""
    v = torch.sqrt(a.v)
    lin = torch.where(v > 0, a.b / (2 * v.clamp_min(1e-300)), torch.full_like(v, math.inf))
    return R(v, torch.minimum(lin, torch.sqrt(a.b)) + U * v + ETA)


def rexp_(a):
    v = torch.exp(a.v)
    return R(v, v * a.b + EXP_ULP * U * v + ETA)


def const(x, like, b=0.0):
    return R(torch.full_like(like, float(x)), torch.full_like(like, float(b)))


# ------------------------------------------------------------------------------------------------ Adam
B1, B2, EPS = 0.9, 0.999, 1e-8


def adam_scalars(t, b1=B1, b2=B2, eps=EPS):
    """(libtorch's scalars, the kernel's fp32 scalars) of step t.  libtorch: bc1, bc2 in double; ATen narrows the
    scalar operands to float.  Kernel: the host passes fl(bc1), fl(bc2) and forms 1.f / bc1 and 1.f / sqrtf(bc2)."""
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    b1f, b2f = np.float32(b1), np.float32(b2)
    lt = dict(b1=f32(b1), c1=f32(1.0 - b1), b2=f32(b2), c2=f32(1.0 - b2), eps=f32(eps), bc1=bc1,
              isb=1.0 / f32(math.sqrt(bc2)))
    k = dict(b1=float(b1f), c1=float(np.float32(1) - b1f), b2=float(b2f), c2=float(np.float32(1) - b2f),
             eps=f32(eps), inv_bc1=float(np.float32(1) / np.float32(bc1)),
             isb=float(np.float32(1) / np.sqrt(np.float32(bc2))))
    return lt, k


def adam(p, g, m, v, lr, t, b1=B1, b2=B2, eps=EPS, device=None, alt=None):
    """The float64 reference of one gsb_adam_step / gsb_adam_step_segments step from the fp32 state (p, g, m, v) (flat
    numpy or torch).  lr: a Python float or a float64 tensor of per-element rates (Python doubles; the kernel gets them
    narrowed).  Returns float64 tensors p, m, v (libtorch's step) with bounds B_p, B_m, B_v; ovf (v' overflows: v'
    must be inf and p unchanged, exactly); cert (the overflow decision is clear of its threshold); re_p, the value of
    the bound's evaluation.  alt, a known wrong convention: "eps_in_sqrt", "bc2_unsqrt" (bc2 not square-rooted),
    "no_bc" (no bias correction)."""
    dev = device if device is not None else (p.device if torch.is_tensor(p) else "cpu")
    p, g, m, v = (_t(x, dev) for x in (p, g, m, v))
    lr = _t(lr, dev) if torch.is_tensor(lr) or isinstance(lr, np.ndarray) else torch.full_like(p, float(lr))
    lt, k = adam_scalars(t, b1, b2, eps)
    assert math.sqrt(FLT_MAX) * k["isb"] + k["eps"] < 2.0 ** 126 and k["eps"] >= 2.0 ** -126, "__fdividef range"
    vinf = torch.isinf(v)
    v0 = torch.where(vinf, torch.zeros_like(v), v)
    # value: libtorch's step (float64 over the exact fp32 scalars)
    m1 = lt["b1"] * m + lt["c1"] * g
    v1 = lt["b2"] * v0 + lt["c2"] * g * g
    bc1, isb = lt["bc1"], lt["isb"]
    if alt == "no_bc":
        bc1, isb = 1.0, 1.0
    elif alt == "bc2_unsqrt":
        isb = 1.0 / f32(1.0 - b2 ** t)
    step = torch.as_tensor(lr / bc1, dtype=torch.float32).to(F8)           # -step_size narrowed by addcdiv_
    den = (torch.sqrt(v1 + lt["eps"]) * isb) if alt == "eps_in_sqrt" else (torch.sqrt(v1) * isb + lt["eps"])
    p1 = p - step * (m1 / den)
    # bound along adam_update's tree, the kernel's scalars charged their distance to libtorch's
    z = torch.zeros_like(p)
    c1 = const(lt["c1"], p, abs(k["c1"] - lt["c1"]))
    c2 = const(lt["c2"], p, abs(k["c2"] - lt["c2"]))
    Rg, Rm, Rv = R(g), R(m), R(v0)
    rm = rfma(c1, Rg, rmul(const(lt["b1"], p), Rm))
    rv = rfma(Rg, rmul(c2, Rg), rmul(const(lt["b2"], p), Rv))
    kstep = torch.as_tensor(torch.as_tensor(lr, dtype=torch.float32) * np.float32(k["inv_bc1"]), dtype=torch.float32)
    s = R(step, (kstep.to(F8) - step).abs())
    den_r = rfma(rsqrt_(rv), const(lt["isb"], p, abs(k["isb"] - lt["isb"])), const(lt["eps"], p))
    q = rdiv(rm, den_r, ulp=2.0)
    rp = rsub(R(p), rmul(s, q))
    ovf = vinf | (rv.v >= OVF)
    cert = vinf | ((rv.v - OVF).abs() > rv.b)
    inf = torch.full_like(p, math.inf)
    out = dict(p=torch.where(ovf, p, p1), m=m1, v=torch.where(ovf, inf, v1), B_p=torch.where(ovf, z, rp.b),
               B_m=rm.b, B_v=torch.where(ovf, z, rv.b), ovf=ovf, cert=cert, re_p=torch.where(ovf, p, rp.v))
    return out


def segment_rates(n_total, segments, device="cpu"):
    """Per-element rates (float64; NaN outside every segment) and the in-segment mask of a gsb_adam_segment table
    [(offset, count, row_floats, head_floats, lr_head, lr_rest)]: element e of a segment (counted from its start)
    takes lr_head where e % row_floats < head_floats."""
    lr = torch.full((n_total,), math.nan, dtype=F8, device=device)
    for o, c, row, head, lh, lrest in segments:
        e = torch.arange(c, device=device)
        lr[o:o + c] = torch.where(e % row < head, torch.tensor(float(lh), dtype=F8, device=device),
                                  torch.tensor(float(lrest), dtype=F8, device=device))
    return lr, ~torch.isnan(lr)


def segment_rates_alt(n_total, segments, alt, device="cpu"):
    """Known wrong rate conventions: "head_whole_row" (lr_head on every float of a row with a head), "buffer_rows"
    (rows counted from the buffer start), "per_float4" (one rate per float4, from its first lane)."""
    lr = torch.full((n_total,), math.nan, dtype=F8, device=device)
    for o, c, row, head, lh, lrest in segments:
        e = torch.arange(c, device=device)
        if alt == "head_whole_row":
            pick = torch.full_like(e, head > 0, dtype=torch.bool)
        elif alt == "buffer_rows":
            pick = (e + o) % row < head
        elif alt == "per_float4":
            pick = (e - e % 4) % row < head
        lr[o:o + c] = torch.where(pick, torch.tensor(float(lh), dtype=F8, device=device),
                                  torch.tensor(float(lrest), dtype=F8, device=device))
    return lr


def synthetic_segments(seed, scale=1):
    """8 segments over one flat buffer, two of them (chosen by the seed) empty, rows of 1 to 48 floats, heads of 0, 1, 3 or the whole
    row, counts that are multiples of neither 4 nor the row (about `scale` x 100 rows each), starts on 16-byte
    boundaries with padding between segments, lr_head / lr_rest >= 10.  Returns (table, total floats)."""
    rng = np.random.default_rng(seed)
    rows = [(1, 1), (3, 1), (4, 3), (5, 0), (7, 3), (12, 12), (27, 3), (48, 3)]
    segs, o = [], 4
    for k, (row, head) in enumerate(rows):
        c = 0 if k in (seed % 8, (seed + 3) % 8) else int(row * rng.integers(20, 200) * scale + rng.integers(1, row + 3))
        if c and c % 4 == 0:
            c += 1
        lh = float(10.0 ** rng.uniform(-3, -2))
        segs.append((o, c, row, head, lh, lh / float(rng.uniform(10, 30))))
        o += (c + 3) // 4 * 4 + 4 * int(rng.integers(0, 3))
    return segs, o + 4


def adam_plain(p, g, m, v, lr, t, b1=B1, b2=B2, eps=EPS):
    """The libtorch formula, written plainly in float64 (for pinning `adam`)."""
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    m1 = f32(b1) * m + f32(1.0 - b1) * g
    v1 = f32(b2) * v + f32(1.0 - b2) * g * g
    step = torch.as_tensor(lr / bc1, dtype=torch.float32).to(F8) if torch.is_tensor(lr) else f32(lr / bc1)
    return p - step * m1 / (torch.sqrt(v1) / f32(math.sqrt(bc2)) + f32(eps)), m1, v1


# ------------------------------------------------------------------------------------------------ activations
def act_map(means, log_scales, raw_quats, logits, cam):
    """The reference's op sequence (model.cpp:148-150,176-177,200) in float64 torch, differentiable."""
    d = means - cam
    return (torch.exp(log_scales), raw_quats / raw_quats.norm(dim=-1, keepdim=True), torch.sigmoid(logits),
            d / d.norm(dim=-1, keepdim=True))


def activate(means, log_scales, raw_quats, logits, cam, v_scales=None, v_quats=None, v_opac=None, device=None,
             alt=None):
    """The float64 reference of gsb_activate_forward and (with cotangents) gsb_activate_backward.  Inputs are the
    kernels' fp32 inputs; logits [n].  The backward takes the forward's fp32 outputs scales / opacities, as the kernel
    does; their bounds carry into the VJP's.  Returns float64: scales, quats, opacities, viewdirs with B_ bounds;
    s_ovf (scales must be +inf), o_zero (opacity and its VJP must be exactly 0), cert_s / cert_o / cert_vls (those
    decisions and the overflow of v_log_scales certified), q_in_range (|q|^2 normal: the quaternion bound applies); with cotangents v_log_scales, v_raw_quats,
    v_logits (autograd) with B_ bounds and re_ the bound's evaluation.  alt, a known wrong convention: "sig_oo"
    (o^2), "sig_o1po" (o (1 + o)), "q_no_proj" (the quaternion VJP without -q^ (q^ . g))."""
    dev = device if device is not None else (means.device if torch.is_tensor(means) else "cpu")
    mu, s, q, x = (_t(a, dev) for a in (means, log_scales, raw_quats, logits))
    x = x.reshape(-1)
    c = _t(cam, dev).reshape(3)
    n = mu.shape[0]
    out = {}
    # scales = expf(s)
    es = [rexp_(R(s[:, i])) for i in range(3)]
    ev = torch.stack([e.v for e in es], -1)
    eb = torch.stack([e.b for e in es], -1)
    s_ovf = ev * (1 - EXP_ULP * U) > FLT_MAX
    out["cert_s"] = s_ovf | (ev * (1 + EXP_ULP * U) < FLT_MAX)
    out["s_ovf"] = s_ovf
    out["scales"] = torch.where(s_ovf, math.inf, ev)
    out["B_scales"] = torch.where(s_ovf, 0.0, eb)
    # quats = q / sqrtf(sum q^2)
    qs = [R(q[:, i]) for i in range(4)]
    ss = radd(radd(radd(rmul(qs[0], qs[0]), rmul(qs[1], qs[1])), rmul(qs[2], qs[2])), rmul(qs[3], qs[3]))
    inv = rdiv(const(1.0, ss.v), rsqrt_(ss))
    h = [rmul(qi, inv) for qi in qs]
    nrm2 = (q * q).sum(-1)
    out["q_in_range"] = (nrm2 >= 2.0 ** -126) & (nrm2 <= FLT_MAX)
    out["quats"] = torch.stack([hi.v for hi in h], -1)
    out["B_quats"] = torch.stack([hi.b for hi in h], -1)
    # opacity = 1 / (1 + expf(-x))
    e = rexp_(R(-x))
    o_zero = e.v * (1 - EXP_ULP * U) > FLT_MAX
    out["cert_o"] = o_zero | (e.v * (1 + EXP_ULP * U) < FLT_MAX)
    out["o_zero"] = o_zero
    o = rdiv(const(1.0, x), radd(const(1.0, x), e))
    out["opacities"] = torch.where(o_zero, 0.0, o.v)
    out["B_opacities"] = torch.where(o_zero, 0.0, o.b)
    # viewdirs = d / sqrtf(|d|^2), d = means - cam
    d = [rsub(R(mu[:, i]), const(float(c[i]), mu[:, i])) for i in range(3)]
    dn = rdiv(const(1.0, d[0].v), rsqrt_(radd(radd(rmul(d[0], d[0]), rmul(d[1], d[1])), rmul(d[2], d[2]))))
    vd = [rmul(di, dn) for di in d]
    out["viewdirs"] = torch.stack([r.v for r in vd], -1)
    out["B_viewdirs"] = torch.stack([r.b for r in vd], -1)
    # the plain map (pins the trees' values)
    sc, qn, op, vdir = act_map(mu, s, q, x, c)
    out["plain"] = dict(scales=sc, quats=qn, opacities=op, viewdirs=vdir)
    if v_scales is None:
        return out

    vs, vq, vo = _t(v_scales, dev), _t(v_quats, dev), _t(v_opac, dev).reshape(-1)
    # autograd of the reference's ops
    with torch.enable_grad():
        ins = [a.clone().requires_grad_() for a in (s, q, x)]
        sc, qn, op, _ = act_map(mu, *ins, c)
        if alt == "q_no_proj":
            qn = ins[1] / ins[1].norm(dim=-1, keepdim=True).detach()
        loss = (torch.where(s_ovf, 0.0, sc) * vs).sum() + (qn * vq).sum() + (op * vo).sum()
        gs, gq, gx = torch.autograd.grad(loss, ins)
    if alt in ("sig_oo", "sig_o1po"):
        sg = torch.sigmoid(x)
        gx = vo * sg * (sg if alt == "sig_oo" else (1 + sg))
    # v_log_scales = v_scales * scales (the forward's fp32 output)
    S = R(torch.where(s_ovf, 0.0, ev), torch.where(s_ovf, 0.0, eb))
    vls = rmul(R(vs), S)
    p_ovf = s_ovf | (vls.v.abs() - vls.b >= OVF)           # the product overflows: v * scale rounds to +-inf
    out["cert_vls"] = p_ovf | (vls.v.abs() + vls.b < OVF)
    out["v_log_scales"] = torch.where(p_ovf, vs * math.inf, gs)
    out["re_v_log_scales"], out["B_v_log_scales"] = torch.where(p_ovf, vs * math.inf, vls.v), torch.where(
        p_ovf, 0.0, vls.b)
    # v_raw_quats = (g - h (h . g)) * inv
    gv = [R(vq[:, i]) for i in range(4)]
    dot = radd(radd(radd(rmul(h[0], gv[0]), rmul(h[1], gv[1])), rmul(h[2], gv[2])), rmul(h[3], gv[3]))
    vr = [rmul(rsub(gv[i], rmul(h[i], dot)), inv) for i in range(4)]
    out["v_raw_quats"] = gq
    out["re_v_raw_quats"] = torch.stack([r.v for r in vr], -1)
    out["B_v_raw_quats"] = torch.stack([r.b for r in vr], -1)
    # v_logits = v * o * (1 - o), from the forward's fp32 opacity (bounded)
    O = R(out["opacities"], out["B_opacities"])
    vl = rmul(rmul(R(vo), O), rsub(const(1.0, x), O))
    out["v_logits"] = torch.where(o_zero, 0.0, gx)
    out["re_v_logits"] = torch.where(o_zero, 0.0, vl.v)
    out["B_v_logits"] = torch.where(o_zero, 0.0, vl.b)
    return out


# ------------------------------------------------------------------------------------------------ densification
def densify_stats(v_xy, radii, img_h, img_w, state=None, device=None, alt=None):
    """The float64 reference of gsb_densify_stats_update (state = (xys_grad_norm, vis_counts, max_2d_size), fp32) or,
    with state None, gsb_densify_stats_init.  Returns float64 xys_grad_norm with B_xys_grad_norm, and vis_counts and
    max_2d_size, which the kernels must match exactly.  alt: "min_hw" (max_2d_size over min(H, W)), "init_visible"
    (init writes visible rows only, leaving the state it is given)."""
    dev = device if device is not None else (v_xy.device if torch.is_tensor(v_xy) else "cpu")
    vx = _t(v_xy, dev).reshape(-1, 2)
    r = _t(radii, dev, torch.int64).reshape(-1)
    vis = r > 0
    hw = min(img_h, img_w) if alt == "min_hw" else max(img_h, img_w)
    q32 = (r.to(torch.float32).cpu().numpy() / np.float32(hw)).astype(np.float32)     # IEEE fp32 division
    q = torch.as_tensor(q32, device=dev).to(F8)
    gx, gy = R(vx[:, 0]), R(vx[:, 1])
    nr = rsqrt_(radd(rmul(gx, gx), rmul(gy, gy)))
    plain = torch.sqrt(vx[:, 0] ** 2 + vx[:, 1] ** 2)
    if state is None and alt != "init_visible":
        return dict(xys_grad_norm=nr.v, B_xys_grad_norm=nr.b, vis_counts=torch.ones_like(nr.v),
                    max_2d_size=torch.where(vis, q.clamp_min(0.0), 0.0), plain=plain)
    if state is None:
        raise ValueError("init_visible needs the state it leaves")
    gn, vc, ms = (_t(x, dev).reshape(-1) for x in state)
    if alt == "init_visible":
        return dict(xys_grad_norm=torch.where(vis, nr.v, gn), B_xys_grad_norm=torch.where(vis, nr.b, 0.0),
                    vis_counts=torch.where(vis, 1.0, vc), max_2d_size=torch.where(vis, q.clamp_min(0.0), ms),
                    plain=plain)
    acc = radd(R(gn), nr)
    return dict(xys_grad_norm=torch.where(vis, acc.v, gn), B_xys_grad_norm=torch.where(vis, acc.b, 0.0),
                vis_counts=torch.where(vis, vc + 1, vc), max_2d_size=torch.where(vis, torch.maximum(ms, q), ms),
                plain=torch.where(vis, gn + plain, gn))


# ------------------------------------------------------------------------------------------------ MSE
def mse(img, target, inv_count, sms, aligned=True, device=None, alt=None):
    """The float64 reference of gsb_mse_loss_grad over flat fp32 img / target of n floats, with inv_count the fp32
    the kernel gets and sms the device's SM count (the grid is 8 sms blocks of 256 threads).  Returns v_img, bit-exact
    (float32 tensor), and loss (a Python float, inv_count * sum (a - b)^2 in float64) with its bound B_loss.
    aligned: all pointers 16-byte aligned (the float4 path runs).  alt "no_two": v_img = inv_count (a - b)."""
    dev = device if device is not None else (img.device if torch.is_tensor(img) else "cpu")
    a = _t(img, dev, torch.float32).reshape(-1)
    b = _t(target, dev, torch.float32).reshape(-1)
    n = a.numel()
    ic = torch.tensor(f32(inv_count), dtype=torch.float32, device=dev)
    s = ic if alt == "no_two" else torch.tensor(2.0, dtype=torch.float32, device=dev) * ic
    d32 = a - b
    v = s * d32
    d = a.to(F8) - b.to(F8)
    sq = float((d * d).sum())
    stride = 8 * sms * 256
    n4 = n // 4 if aligned else 0
    chain = -(-n4 // stride) + -(-(n - 4 * n4) // stride)
    depth = 2 + 1 + 3 + chain + 5 + 3 + 8 * sms     # d, d^2, the float4's 3 adds, the chain, the tree, the atomics
    loss = f32(inv_count) * sq
    return dict(v_img=v, loss=loss, B_loss=(depth + 1) * U * loss + 8 * sms * ETA, depth=depth)
