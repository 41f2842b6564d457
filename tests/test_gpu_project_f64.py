"""The projection kernels Gaussian by Gaussian against the float64 reference of tests/project_f64.py.

Every case runs the five C entry points (gsb_project_forward[_activated], gsb_project_backward[_activated][_acc])
and the autograd operators ops.ProjectGaussians / ops.ProjectGaussiansActivated.  On the Gaussians the reference
certifies (every decision clear of its threshold by its bound, or taken on an operand that is exact in fp32), with
no flip allowance and no aggregate norm:
  * radii and num_tiles_hit match exactly;
  * every float output and every gradient component lies within C u-bound, |kernel - reference| <= C B, where B is the
    reference's first-order running-error bound of the kernel's own operation tree (fp32 operations rounded one by
    one, --fmad=false; device expf 2 ulp).  C = 2 covers the second-order terms B drops and the u |exact| it charges
    where the kernel's rounding is u |computed|.  B is 0 where the output is exactly 0 (culled Gaussians, the written
    cov3d / conic rules): those must match exactly;
  * the accumulating backward returns prior + vjp with one rounding: |acc - (prior + ref)| <= C B + u |prior + ref|;
    culled Gaussians keep their prior bit for bit; v_opacity_logits is written for every Gaussian.
Backward passes run with two cotangent sets: random (v_xy, v_depth, v_conic), and v_conic alone, which is what makes
the fov clamp's gradient visible against the pixel-centre path.  Generic cases must certify >= 99 % of their
Gaussians; the worst err/bound ratio of each case is printed (run with -s)."""
import time

import numpy as np
import pytest
import torch

import project_f64 as pf
from opensplat_b200 import capi, ops
from opensplat_b200.model import Camera

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = pf.U
C = 2.0
GRADS = ("v_mean3d", "v_scale", "v_quat")


def cu(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype).contiguous()


class Worst:
    def __init__(self, name):
        self.name, self.r = name, {}

    def check(self, tag, got, r, key, cert, prior=None):
        got = got.double().reshape(r[key].shape)
        want = r[key] if prior is None else prior.double().reshape(r[key].shape) + r[key]
        bound = C * r["B_" + key]
        if prior is not None:
            bound = bound + U * (want.abs() + bound)     # the rounding of prior + kernel vjp
        err = (got - want).abs()
        m = cert if err.dim() == 1 else cert[:, None].expand_as(err)
        if bool(m.any()):
            self.r[tag + key] = max(self.r.get(tag + key, 0.0), float((err[m] / bound[m].clamp_min(1e-300)).max()))
        over = (err > bound) & m
        if bool(over.any()):
            i = torch.nonzero(over)[0].tolist()
            pytest.fail(f"{self.name} {tag}{key}{i}: kernel {float(got[tuple(i)])!r} reference "
                        f"{float(want[tuple(i)])!r} bound {float(bound[tuple(i)]):.3e}")

    def report(self, cert):
        print(f"\n{self.name}: certified {float(cert.double().mean()) if cert.numel() else 1.0:.5f}; worst err/bound "
              + " ".join(f"{k}={v:.3f}" for k, v in sorted(self.r.items())))


def _exact(name, got, want, cert):
    got, want = got.long().reshape(-1), want.reshape(-1)
    bad = (got != want) & cert
    assert not bool(bad.any()), f"{name}: differs at certified {torch.nonzero(bad)[:8].reshape(-1).tolist()}"


def _cotangents(n, seed, act):
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = dict(v_xy=torch.randn((n, 2), device=DEV, generator=g), v_depth=torch.randn((n,), device=DEV, generator=g),
             v_conic=torch.randn((n, 3), device=DEV, generator=g))
    if act:
        c["v_opacity"] = torch.randn((n,), device=DEV, generator=g)
    z = dict(c, v_xy=torch.zeros_like(c["v_xy"]), v_depth=torch.zeros_like(c["v_depth"]))
    return [c, z]


def run_case(name, cam, means, scales, quats, glob_scale, act=False, logits=None, min_cert=0.99, seed=0, priors=True):
    """Forward, backward (both cotangent sets), the accumulating backward (activated) and the autograd operator."""
    t0 = time.time()
    n = means.shape[0]
    m, s, q = cu(means), cu(scales), cu(quats)
    ol = cu(logits) if act else None
    V, P = cu(cam.V.reshape(4, 4)), cu(cam.P.reshape(4, 4))
    L, ptr, st = capi.lib(), capi.ptr, capi.stream()
    tb = ops.tile_bounds(cam.W, cam.H)
    r = pf.project(cam, m, s, q, glob_scale, act=act, opacity_logits=ol, device=DEV)
    cert = r["cert"]
    frac = float(cert.double().mean()) if n else 1.0
    assert frac >= min_cert, f"{name}: certified {frac:.4f}"
    w = Worst(name)
    if act:
        out = dict(cov3d=torch.empty((n, 6), device=DEV), xys=torch.empty((n, 2), device=DEV),
                   depths=torch.empty((n,), device=DEV), radii=torch.empty((n,), dtype=torch.int32, device=DEV),
                   conics=torch.empty((n, 3), device=DEV), num_tiles_hit=torch.empty((n,), dtype=torch.int32,
                                                                                      device=DEV),
                   opacities=torch.empty((n,), device=DEV))
        capi.check(L.gsb_project_forward_activated(
            n, ptr(m), ptr(s), glob_scale, ptr(q), ptr(ol), ptr(V), ptr(P), cam.fx, cam.fy, cam.cx, cam.cy, cam.H,
            cam.W, tb[0], tb[1], cam.clip, ptr(out["cov3d"]), ptr(out["xys"]), ptr(out["depths"]), ptr(out["radii"]),
            ptr(out["conics"]), ptr(out["num_tiles_hit"]), ptr(out["opacities"]), st))
    else:
        out = dict(zip(("cov3d", "xys", "depths", "radii", "conics", "num_tiles_hit"), ops.project_gaussians_forward(
            m, s, glob_scale, q, V, P, cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W, tb, cam.clip)))
    _exact(name + " radii", out["radii"], r["radii"], cert)
    _exact(name + " num_tiles_hit", out["num_tiles_hit"], r["num_tiles_hit"], cert)
    for k in ("cov3d", "xys", "depths", "conics") + (("opacities",) if act else ()):
        w.check("fwd.", out[k], r, k, cert)

    g = torch.Generator(device=DEV).manual_seed(seed + 99)
    for ci, c in enumerate(_cotangents(n, seed, act)):
        rb = pf.project(cam, m, s, q, glob_scale, act=act, opacity_logits=ol, device=DEV, **c)
        tag = f"bwd{ci}."
        if act:
            vo = c["v_opacity"]
            outs = [torch.empty((n, 3), device=DEV), torch.empty((n, 3), device=DEV), torch.empty((n, 4), device=DEV),
                    torch.empty((n,), device=DEV)]
            args = (n, ptr(m), ptr(s), glob_scale, ptr(q), ptr(out["opacities"]), ptr(V), ptr(P), cam.fx, cam.fy,
                    cam.H, cam.W, ptr(out["radii"]), ptr(out["conics"]), ptr(c["v_xy"]), ptr(c["v_depth"]),
                    ptr(c["v_conic"]), ptr(vo))
            capi.check(L.gsb_project_backward_activated(*args, *[ptr(o) for o in outs], st))
            for k, o in zip(GRADS + ("v_opacity_logits",), outs):
                w.check(tag, o, rb, k, cert)
            if priors:
                # priors of the scale of the VJP and up to 1e6 times larger
                prior = [torch.randn(o.shape, device=DEV, generator=g) * (o.abs().mean() + 1e-30)
                         * torch.exp(torch.empty(o.shape, device=DEV).uniform_(0, 14, generator=g)) for o in outs]
                acc = [p.clone() for p in prior]
                capi.check(L.gsb_project_backward_activated_acc(*args, *[ptr(o) for o in acc], st))
                for k, a, p in zip(GRADS + ("v_opacity_logits",), acc, prior):
                    w.check(tag + "acc.", a, rb, k, cert, prior=p)
                culled = out["radii"] <= 0
                for a, p in zip(acc[:3], prior[:3]):
                    assert torch.equal(a[culled], p[culled]), f"{name}: a culled Gaussian's prior changed"
        else:
            got = ops.project_gaussians_backward(m, s, glob_scale, q, V, P, cam.fx, cam.fy, cam.cx, cam.cy, cam.H,
                                                 cam.W, out["cov3d"], out["radii"], out["conics"], c["v_xy"],
                                                 c["v_depth"], c["v_conic"])
            for k, o in zip(GRADS, got):
                w.check(tag, o, rb, k, cert)

        # the autograd operator: same forward, the same VJP through torch's graph
        mg, sg, qg = (x.clone().requires_grad_() for x in (m, s, q))
        if act:
            og = ol.clone().reshape(n, 1).requires_grad_()
            xys, depths, _, conics, _, _, opac = ops.ProjectGaussiansActivated.apply(
                mg, sg, glob_scale, qg, og, V, P, cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W, tb, cam.clip)
            loss = (opac.reshape(n) * c["v_opacity"]).sum()
        else:
            xys, depths, _, conics, _, _ = ops.ProjectGaussians.apply(
                mg, sg, glob_scale, qg, V, P, cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W, tb, cam.clip)
            loss = 0.0
        if n:
            ((xys * c["v_xy"]).sum() + (depths * c["v_depth"]).sum() + (conics * c["v_conic"]).sum() + loss).backward()
            for k, o in zip(GRADS, (mg.grad, sg.grad, qg.grad)):
                w.check(tag + "op.", o, rb, k, cert)
            if act:
                w.check(tag + "op.", og.grad, rb, "v_opacity_logits", cert)
    torch.cuda.synchronize()
    w.report(cert)
    print(f"{name}: n={n} {time.time() - t0:.1f} s")
    return r


# ------------------------------------------------------------------------------------------------------ cases
def _general(W, H, seed):
    return pf.camera_from_setup(pf.general_camera(W, H, seed))


@pytest.mark.parametrize("n,W,H", [(0, 17, 33), (1, 17, 33), (255, 1920, 1080), (256, 1, 1), (257, 3840, 2160),
                                   (65537, 1920, 1080), (65537, 17, 33)])
@pytest.mark.parametrize("act", [False, True])
def test_counts_and_image_sizes(n, W, H, act):
    """Ragged counts around the 256-thread block and image sizes from one pixel to 4K, with a general camera:
    rotated and translated, fx != fy, off-centre principal point; a third of the Gaussians beyond the fov clamp on any
    side or corner, a tenth with t.z in (0.02, 0.2], raw quaternions; glob_scale 1.3."""
    cam = _general(W, H, seed=n + W)
    m, s, q = pf.random_gaussians(cam, n, seed=n + H, act=act)
    ol = np.random.default_rng(n).uniform(-30, 30, n).astype(np.float32)
    run_case(f"{'act ' if act else ''}n={n} {W}x{H}", cam, m, s, q, 1.3, act=act, logits=ol, seed=n)


def test_c2_size():
    """1M Gaussians at 1920x1080 with a camera_setup camera, through the activated entry points the trainer runs."""
    cam = _general(1920, 1080, seed=3)
    n = 1_000_000
    m, s, q = pf.random_gaussians(cam, n, seed=4, act=True)
    ol = np.random.default_rng(5).uniform(-8, 8, n).astype(np.float32)
    run_case("C2 1M 1920x1080", cam, m, s, q, 1.0, act=True, logits=ol, seed=5)


def _axis_cam(W=128, H=96, clip=0.01):
    """camera_setup's y / z flip makes this camToWorld the identity view: t = mean exactly in fp32."""
    return pf.camera_from_setup(Camera(W, H, 100.0, 80.0, 0.5 * W + 7.0, 0.5 * H - 5.0,
                                       np.diag([1.0, -1.0, -1.0, 1.0]).astype(np.float32)), clip_thresh=clip)


@pytest.mark.parametrize("glob_scale", [0.7, 1.3])
def test_geometry_edges(glob_scale):
    """Constructed edges on the identity-view camera, where t and t / t.z are exact in fp32:
      * Gaussians exactly on +-lim in x, in y and in the corners (the D16 tie), and beyond the clamp on every side;
      * t.z one fp32 step above clip_thresh (kept), exactly at it (culled: the test is strict >), 0 and negative;
      * scales of 1e-4 (the 0.3 dilation dominates), needles of anisotropy up to 1e4, footprints covering every tile;
      * quaternion norms from 1e-3 to 1e3.
    Certified: every Gaussian whose decisions are clear by their bounds or exact.  The clip cases are exact and all
    certified; the ties' q decisions are exact, but their radii (hundreds of px through the clamped J) and the needles'
    are conditioned badly enough that the ceil is certified for only part of them: at least 90 % overall and half of
    the ties."""
    cam = _axis_cam()
    rng = np.random.default_rng(int(glob_scale * 10))
    mt, st, qt = pf.tie_gaussians(cam, seed=1)
    clip = np.float32(cam.clip)
    zs = np.array([np.nextafter(clip, np.float32(1)), clip, 0.0, -1.0, np.nextafter(clip, np.float32(1)), clip],
                  np.float32)
    mc = np.stack([np.zeros(6), np.zeros(6), zs], -1).astype(np.float32)
    mc[4:, 0] = np.float32(0.25 * cam.lim_x * float(zs[4]))
    sc = np.full((6, 3), 1e-4, np.float32)
    qc = rng.standard_normal((6, 4)).astype(np.float32)
    n = 3000
    mg, sg, qg = pf.random_gaussians(cam, n, seed=2, q_norm=(1e-3, 1e3))
    k = n // 6
    sg[:k] = 1e-4                                                             # the dilation dominates
    sg[k:2 * k, 0] *= np.exp(rng.uniform(0, np.log(1e4), k)).astype(np.float32)   # needles, anisotropy up to 1e4
    sg[k:2 * k, 1:] *= 0.3
    mg[2 * k:2 * k + 20] = np.array([0.0, 0.0, 3.0], np.float32) + rng.uniform(-0.2, 0.2, (20, 3)).astype(np.float32)
    sg[2 * k:2 * k + 20] = 5.0                                               # covers every tile
    means, scales, quats = (np.concatenate(x) for x in ((mt, mc, mg), (st, sc, sg), (qt, qc, qg)))
    r = run_case(f"geometry gs={glob_scale}", cam, means, scales, quats, glob_scale, min_cert=0.9, seed=7)
    nt = mt.shape[0]
    cert, kept = r["cert"].cpu(), r["kept"].cpu()
    print(f"ties certified {int(cert[:nt].sum())} of {nt}")
    assert bool(cert[nt:nt + 6].all()) and int(cert[:nt].sum()) >= nt // 2
    assert bool(kept[:nt].all()) and int((r["tie_x"] | r["tie_y"]).sum()) >= nt
    assert kept[nt:nt + 6].tolist() == [True, False, False, False, True, False]
    covers = r["num_tiles_hit"].cpu()[nt + 6 + 2 * k:nt + 6 + 2 * k + 20]
    assert bool((covers == cam.tiles_x * cam.tiles_y).all())


def test_activated_ranges():
    """Log-scales in [-12, 3] and opacity logits in [-30, 30].  Where fp32 sigmoid rounds to 1 the kernel's 1 - o is 0
    and so is its v_opacity_logits, as the reference's own fp32 autograd gives; the reference's bound of 1 - o (that of
    o, >= u) covers the exact o (1 - o) ~ e^-x that this drops.  Log-scales up to 3 make radii of 1e3 to 1e6 px,
    whose ceil lies within its bound of an integer for about a quarter of the Gaussians: at least 70 % certified."""
    cam = _general(640, 360, seed=8)
    n = 20000
    m, _, q = pf.random_gaussians(cam, n, seed=9, q_norm=(1e-3, 1e3))
    rng = np.random.default_rng(10)
    ls = rng.uniform(-12, 3, (n, 3)).astype(np.float32)
    ol = rng.uniform(-30, 30, n).astype(np.float32)
    r = run_case("activated ranges", cam, m, ls, q, 1.0, act=True, logits=ol, seed=10, min_cert=0.7)
    assert float((r["opacities"] > 1 - 2 ** -25).double().mean()) > 0.2           # sigmoid rounds to 1 in fp32
