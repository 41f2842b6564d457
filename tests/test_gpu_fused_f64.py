"""The kernels of csrc/fused.cu element by element against the float64 reference of tests/fused_f64.py: Adam
(gsb_adam_step and gsb_adam_step_segments), the activations (gsb_activate_forward / _backward and
ops.ActivateGaussians), the densification statistics (gsb_densify_stats_update / _init) and gsb_mse_loss_grad.

Every output element must lie within C B of the reference, where B is the reference's first-order running-error bound
of the kernel's own operation tree; C = 2 covers the second-order terms B drops.  Decisions the reference documents
are checked exactly where certified (Adam's v' overflow: v' = inf and p unchanged; exp overflow: +inf; sigmoid
saturation: opacity and VJP exactly 0) and the few uncertified elements are left out and counted.  Counts, maxima and
the MSE gradient are bit-exact.  Sentinels surround every output buffer and the padding between segments, and must
come back bit for bit.  Adam cases reach every path of adam_kernel: the two-float4 loop and its one-float4
remainder (n / 4 around multiples of the grid stride 8 SMs x 256, taken from the device), the scalar tail, and the
scalar path of a misaligned pointer.  The worst err/bound ratio and the certified fraction of each case are printed
(-s)."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import fused_f64 as ff
from opensplat_b200 import capi, ops, parallel
from opensplat_b200.model import LEARNING_RATES
from opensplat_b200.trainer import adam_segments

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_ = 2.0
SENT = 12345.678
G = 4                     # sentinel floats on each side of a buffer (16 bytes: keeps the buffer's alignment)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stride():
    return 8 * sms() * 256


class Guarded:
    """n floats `off` floats past a 16-byte boundary, with G + off sentinels before and G after."""

    def __init__(self, n, off=0, init=None):
        self.base = torch.full((n + 2 * G + off,), SENT, device=DEV)
        self.n, self.lo = n, G + off
        self.t = self.base[self.lo:self.lo + n]
        if init is not None:
            self.t.copy_(init)

    def intact(self):
        return bool((self.base[:self.lo] == SENT).all()) and bool((self.base[self.lo + self.n:] == SENT).all())


class Worst:
    def __init__(self, name):
        self.name, self.r, self.unc, self.tot = name, {}, 0, 0

    def check(self, tag, got, want, bound, mask=None):
        got = got.double().reshape(want.shape)
        err = (got - want).abs()
        bound = C_ * bound
        m = torch.isfinite(want) if mask is None else (mask & torch.isfinite(want))
        if bool(m.any()):
            self.r[tag] = max(self.r.get(tag, 0.0), float((err[m] / bound[m].clamp_min(1e-300)).max()))
        over = ((err > bound) | torch.isnan(got)) & m
        if bool(over.any()):
            i = tuple(torch.nonzero(over)[0].tolist())
            pytest.fail(f"{self.name} {tag}{list(i)}: kernel {float(got[i])!r} reference {float(want[i])!r} "
                        f"bound {float(bound[i]):.3e}")

    def exact(self, tag, got, want, mask=None):
        got = got.double().reshape(want.shape)
        same = (got == want) | (torch.isnan(got) & torch.isnan(want))
        if mask is not None:
            same = same | ~mask
        if not bool(same.all()):
            i = tuple(torch.nonzero(~same)[0].tolist())
            pytest.fail(f"{self.name} {tag}{list(i)}: kernel {float(got[i])!r} expected {float(want[i])!r} exactly")

    def cert(self, c):
        self.unc += int((~c).sum())
        self.tot += c.numel()

    def report(self, extra=""):
        frac = 1.0 - self.unc / max(self.tot, 1)
        print(f"\n{self.name}: {extra}certified {frac:.7f} ({self.unc} not); worst err/bound "
              + " ".join(f"{k}={v:.3f}" for k, v in sorted(self.r.items())))


# ------------------------------------------------------------------------------------------------ Adam
def adam_inputs(n, seed, kind="mix"):
    """Device fp32 (p, g, m, v).  mix: |g| log-uniform in [1e-30, 1e19] with random signs, 5 % exact zeros and 0.1 %
    past the overflow of v' (1e21 .. 1e30); a state as after some steps.  zero: p random, g = m = v = 0."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    U_ = lambda a, b: torch.rand(n, device=DEV, generator=gen, dtype=torch.float64) * (b - a) + a
    sgn = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.5, -1.0, 1.0).double()
    p = torch.randn(n, device=DEV, generator=gen, dtype=torch.float64) * 10.0 ** U_(-3, 1)
    if kind == "zero":
        z = torch.zeros(n, device=DEV)
        return p.float(), z, z.clone(), z.clone()
    g = sgn * 10.0 ** U_(-30, 19)
    g = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.05, 0.0, g)
    g = torch.where(torch.rand(n, device=DEV, generator=gen) < 0.001, sgn * 10.0 ** U_(21, 30), g)
    m = 0.1 * g.clamp(-1e19, 1e19) * 10.0 ** U_(-1, 1)
    v = 1e-3 * g.clamp(-1e19, 1e19) ** 2 * 10.0 ** U_(-1, 1)
    return p.float(), g.float(), m.float(), v.float()


def next_grad(n, seed, t):
    """The gradient of a later step: the mix, with the first 1/8 of the floats large at the first step and tiny
    after it (m stays far from 0 while v' ~ 0 relative to it)."""
    _, g, _, _ = adam_inputs(n, seed * 7919 + t)
    k = max(1, n // 8)
    g[:k] = 1e3 if t == 1 else 1e-30
    return g


def run_adam(name, n, steps, offs=(0, 0, 0, 0), seed=0, kind="mix"):
    L = capi.lib()
    p0, g0, m0, v0 = adam_inputs(n, seed, kind)
    if kind == "mix":
        m0.zero_(), v0.zero_()
    P, Gr, M, V = (Guarded(n, o, x) for o, x in zip(offs, (p0, g0, m0, v0)))
    w = Worst(name)
    for i, t in enumerate(steps):
        if i and kind == "mix":
            Gr.t.copy_(next_grad(n, seed, i))
        before = [x.t.clone() for x in (P, Gr, M, V)]
        r = ff.adam(*before, 1.6e-4, t, device=DEV)
        capi.check(L.gsb_adam_step(n, capi.ptr(P.t), capi.ptr(Gr.t), capi.ptr(M.t), capi.ptr(V.t), 1.6e-4, 0.9,
                                   0.999, 1e-8, 1.0 - 0.9 ** t, 1.0 - 0.999 ** t, capi.stream()))
        c = r["cert"]
        w.cert(c)
        ok = c & ~r["ovf"]
        w.check("p", P.t, r["p"], r["B_p"], ok)
        w.check("m", M.t, r["m"], r["B_m"], c)
        w.check("v", V.t, r["v"], r["B_v"], ok)
        w.exact("p.ovf", P.t, before[0].double(), c & r["ovf"])
        w.exact("v.ovf", V.t, r["v"], c & r["ovf"])
        if kind == "zero":
            assert torch.equal(P.t, before[0]) and torch.equal(M.t, before[2]) and torch.equal(V.t, before[3])
        assert torch.equal(Gr.t, before[1]), "the gradient is read only"
        assert all(x.intact() for x in (P, Gr, M, V)), "a sentinel changed"
    torch.cuda.synchronize()
    w.report()
    return w


T_ALL = (1, 2, 10, 1000, 30000)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8, 1023])
def test_adam_small(n):
    run_adam(f"adam n={n}", n, T_ALL, seed=n)
    run_adam(f"adam n={n} zero state and gradient", n, (1, 30000), seed=n, kind="zero")


@pytest.mark.parametrize("k,r", [("s-1", 3), ("s", 0), ("s+1", 1), ("2s", 2), ("2s+1", 3), ("5s+3", 1)])
def test_adam_grid_stride_paths(k, r):
    """n / 4 at stride - 1, stride, stride + 1, 2 stride, 2 stride + 1 and 5 stride + 3: threads run the two-float4
    loop zero to three times, with and without the one-float4 remainder, plus a scalar tail of r floats."""
    s = stride()
    n4 = {"s-1": s - 1, "s": s, "s+1": s + 1, "2s": 2 * s, "2s+1": 2 * s + 1, "5s+3": 5 * s + 3}[k]
    run_adam(f"adam n/4={n4} (+{r})", 4 * n4 + r, (1, 1000), seed=n4)


def test_adam_fifty_million():
    t0 = time.time()
    run_adam("adam n=50000017", 50_000_017, (10,), seed=5)
    print(f"{time.time() - t0:.1f} s")


@pytest.mark.parametrize("which", [0, 1, 2, 3])
@pytest.mark.parametrize("off", [1, 2, 3])
def test_adam_misaligned(which, off):
    """One of the four pointers off a 16-byte boundary: the whole buffer takes the scalar path."""
    offs = [0, 0, 0, 0]
    offs[which] = off
    run_adam(f"adam misaligned ptr {which} by {off}", 100_003, T_ALL, offs=tuple(offs), seed=10 * which + off)


# ------------------------------------------------------------------------------------------------ segmented Adam
def run_segments(name, segs, total, steps=(1, 10, 30000), seed=0):
    L = capi.lib()
    lr, inside = ff.segment_rates(total, segs, device=DEV)
    p0, g0, _, _ = adam_inputs(total, seed)
    z = torch.zeros(total, device=DEV)
    P, Gr, M, V = (Guarded(total, 0, x) for x in (p0, g0, z, z))
    for x in (P, Gr, M, V):
        x.t[~inside] = SENT                         # padding between segments
    table = (capi.AdamSegment * len(segs))(*[capi.AdamSegment(*sg) for sg in segs])
    w = Worst(name)
    lr0 = torch.where(inside, lr, 0.0)
    for i, t in enumerate(steps):
        if i:
            g = next_grad(total, seed, i)
            Gr.t[inside] = g[inside]
        before = [x.t.clone() for x in (P, Gr, M, V)]
        r = ff.adam(*before, lr0, t, device=DEV)
        capi.check(L.gsb_adam_step_segments(len(segs), C.addressof(table), capi.ptr(P.t), capi.ptr(Gr.t),
                                            capi.ptr(M.t), capi.ptr(V.t), 0.9, 0.999, 1e-8, 1.0 - 0.9 ** t,
                                            1.0 - 0.999 ** t, capi.stream()))
        c = r["cert"] & inside
        w.cert(r["cert"][inside])
        ok = c & ~r["ovf"]
        w.check("p", P.t, r["p"], r["B_p"], ok)
        w.check("m", M.t, r["m"], r["B_m"], c)
        w.check("v", V.t, r["v"], r["B_v"], ok)
        w.exact("p.ovf", P.t, before[0].double(), c & r["ovf"])
        for x in (P, Gr, M, V):
            assert bool((x.t[~inside] == SENT).all()), "padding between segments changed"
            assert x.intact(), "a sentinel changed"
    torch.cuda.synchronize()
    w.report()


@pytest.mark.parametrize("n", [1, 7, 1000, 4097])
@pytest.mark.parametrize("k", [1, 4, 16])
def test_adam_segments_trainer_table(n, k):
    offs, total = parallel.flat_layout(n, k)
    lr = dict(LEARNING_RATES)
    lr["means"] = 1.3e-4                            # a scheduled means rate, as the trainer passes it
    run_segments(f"segments trainer n={n} K={k}", adam_segments(offs, lr), total, seed=n * 31 + k)


def test_adam_segments_trainer_table_three_million():
    t0 = time.time()
    offs, total = parallel.flat_layout(3_000_000, 16)
    lr = dict(LEARNING_RATES)
    lr["means"] = 1.3e-4
    run_segments("segments trainer n=3000000 K=16", adam_segments(offs, lr), total, steps=(10,), seed=3)
    print(f"{time.time() - t0:.1f} s")


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("scale", [1, 300])
def test_adam_segments_synthetic(seed, scale):
    segs, total = ff.synthetic_segments(seed, scale)
    run_segments(f"segments synthetic seed={seed} x{scale}", segs, total, seed=seed)


def test_adam_segments_argument_checks():
    """Nine segments, and a segment offset off a 16-byte boundary, are refused before any launch."""
    L = capi.lib()
    buf = [torch.full((4096,), 0.5, device=DEV) for _ in range(4)]
    good = (0, 100, 3, 1, 1e-2, 1e-3)
    for segs in ([good] * 9, [good, (102, 10, 1, 1, 1e-2, 1e-3)]):
        table = (capi.AdamSegment * len(segs))(*[capi.AdamSegment(*sg) for sg in segs])
        code = L.gsb_adam_step_segments(len(segs), C.addressof(table), *[capi.ptr(b) for b in buf], 0.9, 0.999,
                                        1e-8, 0.1, 0.001, capi.stream())
        assert code == -1
    torch.cuda.synchronize()
    assert all(bool((b == 0.5).all()) for b in buf)


# ------------------------------------------------------------------------------------------------ activations
def act_inputs(n, seed):
    """Log-scales in [-30, 88] (2 % in [89, 100], past the overflow of expf); raw quaternions with norms 1e-15 ..
    1e15, a quarter axis-aligned; logits in +-[0, 100] with exact zeros; means 1e-6 .. 1e6 from the camera."""
    rng = np.random.default_rng(seed)
    ls = rng.uniform(-30, 88, (n, 3))
    big = rng.uniform(size=(n, 3)) < 0.02
    ls[big] = rng.uniform(89, 100, int(big.sum()))
    q = rng.standard_normal((n, 4))
    ax = rng.uniform(size=n) < 0.25
    q[ax] = 0.0
    q[ax, rng.integers(0, 4, int(ax.sum()))] = rng.choice([-1.0, 1.0], int(ax.sum()))
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * 10.0 ** rng.uniform(-15, 15, (n, 1))
    x = rng.uniform(-100, 100, n)
    x[rng.uniform(size=n) < 0.03] = 0.0
    cam = np.array([0.3, -2.7, 4.1], np.float32)
    d = rng.standard_normal((n, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True) * 10.0 ** rng.uniform(-6, 6, (n, 1))
    means = cam.astype(np.float64) + d
    vs, vq, vo = rng.standard_normal((n, 3)), rng.standard_normal((n, 4)), rng.standard_normal(n)
    return [torch.as_tensor(np.asarray(a, np.float32)).to(DEV) for a in (means, ls, q, x, cam, vs, vq, vo)]


def check_activations(w, tag, r, scales, quats, opac, vd):
    w.cert(r["cert_s"])
    w.cert(r["cert_o"])
    ok_s = r["cert_s"] & ~r["s_ovf"]
    w.check(tag + "scales", scales, r["scales"], r["B_scales"], ok_s)
    w.exact(tag + "scales.inf", scales, r["scales"], r["cert_s"] & r["s_ovf"])
    w.check(tag + "quats", quats, r["quats"], r["B_quats"], r["q_in_range"][:, None])
    ok_o = r["cert_o"] & ~r["o_zero"]
    w.check(tag + "opac", opac, r["opacities"], r["B_opacities"], ok_o)
    w.exact(tag + "opac.0", opac, r["opacities"], r["cert_o"] & r["o_zero"])
    w.check(tag + "viewdirs", vd, r["viewdirs"], r["B_viewdirs"])


def check_vjp(w, tag, r, vls, vrq, vl):
    cs, co = r["cert_s"] & r["cert_vls"], r["cert_o"]
    w.check(tag + "v_log_scales", vls, r["v_log_scales"], r["B_v_log_scales"], cs & torch.isfinite(r["v_log_scales"]))
    w.exact(tag + "v_log_scales.inf", vls, r["v_log_scales"], cs & ~torch.isfinite(r["v_log_scales"]))
    w.check(tag + "v_raw_quats", vrq, r["v_raw_quats"], r["B_v_raw_quats"], r["q_in_range"][:, None])
    w.check(tag + "v_logits", vl, r["v_logits"], r["B_v_logits"], co & ~r["o_zero"])
    w.exact(tag + "v_logits.0", vl, r["v_logits"], co & r["o_zero"])


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1_000_003])
def test_activations(n):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    means, ls, q, x, cam, vs, vq, vo = act_inputs(n, n)
    r = ff.activate(means, ls, q, x, cam, vs, vq, vo, device=DEV)
    w = Worst(f"activate n={n}")
    out = [Guarded(k * n) for k in (3, 4, 1, 3)]
    capi.check(L.gsb_activate_forward(n, P(means), P(ls), P(q), P(x), P(cam), *[P(o.t) for o in out], s))
    scales, quats, opac, vd = out[0].t.view(n, 3), out[1].t.view(n, 4), out[2].t, out[3].t.view(n, 3)
    check_activations(w, "", r, scales, quats, opac, vd)
    grads = [Guarded(k * n) for k in (3, 4, 1)]
    capi.check(L.gsb_activate_backward(n, P(scales.contiguous()), P(q), P(opac), P(vs), P(vq), P(vo),
                                       *[P(gd.t) for gd in grads], s))
    check_vjp(w, "", r, grads[0].t.view(n, 3), grads[1].t.view(n, 4), grads[2].t)
    assert all(o.intact() for o in out + grads), "a sentinel changed"
    # ops.ActivateGaussians: the same kernels through autograd
    lg, qg, xg = (t.clone().requires_grad_() for t in (ls, q, x.view(n, 1)))
    so, qo, oo, vdo = ops.ActivateGaussians.apply(means, lg, qg, xg, cam)
    check_activations(w, "op.", r, so.detach(), qo.detach(), oo.detach().view(n), vdo)
    torch.autograd.backward([so, qo, oo], [vs, vq, vo.view(n, 1)])
    check_vjp(w, "op.", r, lg.grad, qg.grad, xg.grad.view(n))
    torch.cuda.synchronize()
    w.report()


def test_activation_quaternions_outside_the_bounded_range():
    """Norms whose squares leave the normal range are not bounded; what the kernel does there is recorded: |q|^2 = inf
    gives a zero quaternion and a zero VJP, a zero quaternion gives NaN."""
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    q = torch.tensor([[1e20, 0, 0, 0], [3e19, -3e19, 3e19, 3e19], [0, 0, 0, 0]], device=DEV)
    n = q.shape[0]
    one = torch.ones((n, 3), device=DEV)
    out = [torch.empty((n, k), device=DEV) for k in (3, 4, 1, 3)]
    capi.check(L.gsb_activate_forward(n, P(one), P(one), P(q), P(one[:, 0].contiguous()),
                                      P(torch.zeros(3, device=DEV)), *[P(o) for o in out], s))
    g = [torch.empty((n, k), device=DEV) for k in (3, 4, 1)]
    capi.check(L.gsb_activate_backward(n, P(out[0]), P(q), P(out[2]), P(one), P(torch.ones((n, 4), device=DEV)),
                                       P(one[:, 0].contiguous()), *[P(x) for x in g], s))
    quats, vq = out[1].cpu(), g[1].cpu()
    print(f"\nquaternions outside the bounded range: {quats.tolist()} VJP {vq.tolist()}")
    assert bool((quats[:2] == 0).all()) and bool((vq[:2] == 0).all())
    assert bool(torch.isnan(quats[2]).all())


# ------------------------------------------------------------------------------------------------ densification
def stats_inputs(n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    mag = 10.0 ** (torch.rand((n, 1), device=DEV, generator=gen) * 30 - 15)
    v = torch.randn((n, 2), device=DEV, generator=gen) * mag
    v[torch.rand(n, device=DEV, generator=gen) < 0.03] = 0.0
    r = torch.randint(-1, 5000, (n,), device=DEV, generator=gen, dtype=torch.int32)
    r[torch.rand(n, device=DEV, generator=gen) < 0.2] = 0
    return v.float().contiguous(), r


@pytest.mark.parametrize("n", [1, 257, 100_003])
@pytest.mark.parametrize("H,W", [(300, 480), (481, 299), (2160, 3840)])
def test_densify_stats(n, H, W):
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    w = Worst(f"densify stats n={n} {H}x{W}")
    v, r = stats_inputs(n, n + H)
    st = [Guarded(n, 0, torch.full((n,), 7.0, device=DEV)) for _ in range(3)]
    capi.check(L.gsb_densify_stats_init(n, P(v), P(r), H, W, *[P(x.t) for x in st], s))
    ref = ff.densify_stats(v, r, H, W, device=DEV)
    w.check("init.norm", st[0].t, ref["xys_grad_norm"], ref["B_xys_grad_norm"])
    w.exact("init.counts", st[1].t, ref["vis_counts"])
    w.exact("init.max2d", st[2].t, ref["max_2d_size"])
    for call in range(4):                            # accumulating calls
        v, r = stats_inputs(n, 1000 * call + n + H)
        state = [x.t.clone() for x in st]
        capi.check(L.gsb_densify_stats_update(n, P(v), P(r), H, W, *[P(x.t) for x in st], s))
        ref = ff.densify_stats(v, r, H, W, state=state, device=DEV)
        w.check("upd.norm", st[0].t, ref["xys_grad_norm"], ref["B_xys_grad_norm"])
        w.exact("upd.counts", st[1].t, ref["vis_counts"])
        w.exact("upd.max2d", st[2].t, ref["max_2d_size"])
    assert all(x.intact() for x in st), "a sentinel changed"
    torch.cuda.synchronize()
    w.report()


# ------------------------------------------------------------------------------------------------ MSE
def run_mse(name, n, offs=(0, 0, 0), kind="random", seed=0):
    L = capi.lib()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.rand(n, device=DEV, generator=gen)
    b = a.clone() if kind == "equal" else torch.rand(n, device=DEV, generator=gen)
    A, Bt = Guarded(n, offs[0], a), Guarded(n, offs[1], b)
    V = Guarded(n, offs[2])
    loss = torch.full((1,), 7.0, device=DEV)                 # the call overwrites, never accumulates
    capi.check(L.gsb_mse_loss_grad(n, capi.ptr(A.t), capi.ptr(Bt.t), capi.ptr(V.t), capi.ptr(loss), 1.0 / n,
                                   capi.stream()))
    ref = ff.mse(a, b, 1.0 / n, sms(), aligned=not any(offs), device=DEV)
    w = Worst(name)
    w.exact("v_img", V.t, ref["v_img"].double())
    w.check("loss", loss, torch.tensor([ref["loss"]], dtype=torch.float64, device=DEV),
            torch.tensor([ref["B_loss"]], dtype=torch.float64, device=DEV))
    if kind == "equal":
        assert bool((V.t == 0).all()) and float(loss) == 0.0
    assert A.intact() and Bt.intact() and V.intact(), "a sentinel changed"
    torch.cuda.synchronize()
    w.report(f"depth {ref['depth']}; ")


@pytest.mark.parametrize("H,W", [(1, 1), (1, 5), (3, 7), (17, 16), (123, 77), (540, 960), (1080, 1920),
                                 (2160, 3840)])
def test_mse_images(H, W):
    for kind in ("random", "equal"):
        run_mse(f"mse {H}x{W} {kind}", H * W * 3, kind=kind, seed=H * W)


@pytest.mark.parametrize("n4,r", [(1000, 0), (1000, 1), (1000, 2), (1000, 3), ("3s", 2), ("3s+5", 3)])
def test_mse_remainders(n4, r):
    """n % 4 in {0, 1, 2, 3}, and per-thread chains of three and four float4 terms."""
    n4 = {"3s": 3 * stride(), "3s+5": 3 * stride() + 5}.get(n4, n4)
    run_mse(f"mse n={4 * n4 + r}", 4 * n4 + r, seed=n4 + r)


@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("off", [1, 3])
def test_mse_misaligned(which, off):
    offs = [0, 0, 0]
    offs[which] = off
    run_mse(f"mse misaligned ptr {which} by {off}", 100_003, offs=tuple(offs), seed=which + off)


def test_mse_empty_zeroes_the_loss():
    loss = torch.full((1,), 7.0, device=DEV)
    capi.check(capi.lib().gsb_mse_loss_grad(0, None, None, None, capi.ptr(loss), 1.0, capi.stream()))
    assert float(loss) == 0.0
