"""The SH colour kernels and the fused SSIM / L1 loss element by element against the float64 references of
tests/sh_f64.py and tests/loss_f64.py.

Every output element must lie within C u-bound of the reference, |kernel - reference| <= C B, where B is the
reference's first-order running-error bound of the kernel's own operation tree; C = 2 covers the second-order terms
B drops and the u |exact| it charges where the kernel's rounding is u |computed|.  B is 0 where the output is exactly 0
(a clamped colour, a masked gradient, a basis above degrees_to_use): those must match exactly.  On every channel whose
clamp decision is certified (|colour + 0.5| > B, or the fp32 value determined at degrees_to_use 0, which is how the
constructed ties are checked) the kernel's mask -- rgbs > 0 or rgbs == -0 (D17) -- must equal the reference's
colour + 0.5 >= 0 exactly.  Generic SH cases must certify >= 99 % of their channels.  The loss has one decision,
sgn(y - x), exact in fp32, so every element is checked.  The worst err/bound ratio of each case is printed (-s).

SH entry points: gsb_sh_forward / _backward, _rgb, _rgb_cam, _split (through ops.SphericalHarmonicsRgb),
_rgb_cam_multiview, gsb_mask_rgb_grad followed by gsb_sh_backward_multiview and _multiview_cams, gsb_exchange_gradients
and _cams at world 1 with a geometry prefix, and ops.SphericalHarmonics.  Loss: gsb_ssim_l1_loss and ops.MainLoss."""
import time

import numpy as np
import pytest
import torch

import loss_f64 as lf
import sh_f64 as sf
from opensplat_b200 import capi, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 2.0


def cu(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, torch.float32).contiguous()


def shifted(shape, off):
    """An uninitialised fp32 tensor of `shape` whose data pointer is `off` floats past a 256-B aligned allocation."""
    n = int(np.prod(shape))
    return torch.full((n + off,), float("nan"), device=DEV)[off:].view(shape)


class Worst:
    def __init__(self, name):
        self.name, self.r = name, {}

    def check(self, tag, got, want, bound, mask=None):
        got = got.double().reshape(want.shape)
        err = (got - want).abs()
        bound = C * bound
        m = torch.ones_like(err, dtype=torch.bool) if mask is None else mask.expand_as(err)
        if bool(m.any()):
            self.r[tag] = max(self.r.get(tag, 0.0), float((err[m] / bound[m].clamp_min(1e-300)).max()))
        over = ((err > bound) | torch.isnan(got)) & m
        if bool(over.any()):
            i = tuple(torch.nonzero(over)[0].tolist())
            pytest.fail(f"{self.name} {tag}{list(i)}: kernel {float(got[i])!r} reference {float(want[i])!r} "
                        f"bound {float(bound[i]):.3e}")

    def report(self, extra=""):
        print(f"\n{self.name}: {extra}worst err/bound " + " ".join(f"{k}={v:.3f}" for k, v in sorted(self.r.items())))


def kernel_mask(rgbs):
    return (rgbs > 0) | ((rgbs == 0) & torch.signbit(rgbs))


def check_mask(name, rgbs, r):
    got, cert = kernel_mask(rgbs.reshape(r["mask"].shape)), r["cert"]
    bad = (got != r["mask"]) & cert
    assert not bool(bad.any()), f"{name}: clamp mask differs at certified {torch.nonzero(bad)[:8].tolist()}"
    ties = r["tie"] & cert
    assert bool(torch.signbit(rgbs.reshape(ties.shape)[ties]).all()), f"{name}: a tie is not written as -0"


# ------------------------------------------------------------------------------------------------------ SH inputs
def sh_inputs(n, degree, seed, kind="generic"):
    """(coeffs [n,K,3], means [n,3], cam [3], v_rgb [n,3]).  kinds:
      generic   standard-normal coefficients, means in a unit box, camera 4 units away;
      straddle  colours within about +-0.3 of the clamp, so each channel is clamped or not independently;
      far       means around 1e4 with the camera 3 units away (cancellation in means - cam);
      axis      means - cam along the axes and the diagonals (exactly zero direction components);
      ties      straddle, plus featuresDc = -1.7724538f on random channels: an exact tie at degrees_to_use 0."""
    rng = np.random.default_rng(seed)
    K = sf.num_bases(degree)
    co = rng.standard_normal((n, K, 3)).astype(np.float32)
    means = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    cam = np.array([0.7, -3.1, 2.2], np.float32)
    if kind in ("straddle", "ties"):
        co[:, 1:] *= np.float32(0.05)
        co[:, 0] = ((rng.uniform(-0.3, 0.3, (n, 3)) - 0.5) / sf.C0).astype(np.float32)
    if kind == "ties":
        t = rng.uniform(size=(n, 3)) < 0.3
        co[:, 0][t] = sf.TIE_DC
    if kind == "far":
        cam = np.array([1e4, -1e4, 1e4], np.float32)
        means = (cam + rng.uniform(-3, 3, (n, 3))).astype(np.float32)
    if kind == "axis":
        dirs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 1, 0], [0, 1, -1],
                         [1, 1, 1]], np.float32)
        d = dirs[rng.integers(0, len(dirs), n)] * rng.uniform(0.5, 4, (n, 1)).astype(np.float32)
        cam = np.array([0.0, 0.0, 0.0], np.float32)
        means = d.astype(np.float32)
    v = rng.standard_normal((n, 3)).astype(np.float32)
    return co, means, cam, v


def run_sh_case(name, degree, use, co, means, cam, v, off=0, min_cert=0.99):
    """Every single-view entry point on one input set."""
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    n, K = co.shape[0], co.shape[1]
    w = Worst(name)
    co_d = shifted((n, K, 3), off)
    co_d.copy_(cu(co))
    m_d, cam_d, v_d = cu(means), cu(cam), cu(v)
    vd = (means - cam).astype(np.float32)          # what the viewdirs entry points receive: the same fp32 subtraction
    vd_d = cu(vd)

    # plain SH: gsb_sh_forward / gsb_sh_backward and ops.SphericalHarmonics
    r0 = sf.sh(degree, use, co_d, viewdirs=vd_d, v_colors=v_d, device=DEV)
    col = torch.empty((n, 3), device=DEV)
    capi.check(L.gsb_sh_forward(n, degree, use, P(vd_d), P(co_d), P(col), s))
    w.check("fwd.", col, r0["colors"], r0["B_colors"])
    vco = shifted((n, K, 3), off)
    capi.check(L.gsb_sh_backward(n, degree, use, P(vd_d), P(v_d), P(vco), s))
    w.check("bwd.", vco, r0["v_coeffs"], r0["B_v_coeffs"])
    cg = co_d.clone().requires_grad_()
    out = ops.SphericalHarmonics.apply(use, vd_d, cg)
    (out * v_d).sum().backward()
    w.check("op.fwd.", out.detach(), r0["colors"], r0["B_colors"])
    w.check("op.bwd.", cg.grad, r0["v_coeffs"], r0["B_v_coeffs"])

    # fused clamp, view directions given: gsb_sh_forward_rgb / _backward_rgb
    r1 = sf.sh(degree, use, co_d, viewdirs=vd_d, bias=0.5, v_colors=v_d, device=DEV)
    frac = float(r1["cert"].double().mean())
    assert frac >= min_cert, f"{name}: certified {frac:.4f}"
    cm = r1["cert"][:, None, :]
    rgb = torch.empty((n, 3), device=DEV)
    capi.check(L.gsb_sh_forward_rgb(n, degree, use, P(vd_d), P(co_d), 0.5, P(rgb), s))
    w.check("rgb.fwd.", rgb, r1["colors"], r1["B_colors"])
    check_mask(name + " rgb", rgb, r1)
    capi.check(L.gsb_sh_backward_rgb(n, degree, use, P(vd_d), P(rgb), P(v_d), P(vco), s))
    w.check("rgb.bwd.", vco, r1["v_coeffs"], r1["B_v_coeffs"], cm)

    # camera variants: the direction formed in the kernel
    r2 = sf.sh(degree, use, co_d, means=m_d, cam_pos=cam, bias=0.5, v_colors=v_d, device=DEV)
    cm2 = r2["cert"][:, None, :]
    capi.check(L.gsb_sh_forward_rgb_cam(n, degree, use, P(m_d), P(cam_d), P(co_d), 0.5, P(rgb), s))
    w.check("cam.fwd.", rgb, r2["colors"], r2["B_colors"])
    check_mask(name + " cam", rgb, r2)
    capi.check(L.gsb_sh_backward_rgb_cam(n, degree, use, P(m_d), P(cam_d), P(rgb), P(v_d), P(vco), s))
    w.check("cam.bwd.", vco, r2["v_coeffs"], r2["B_v_coeffs"], cm2)
    rgbm = torch.empty((1, n, 3), device=DEV)
    capi.check(L.gsb_sh_forward_rgb_cam_multiview(n, degree, use, P(m_d), 1, P(cam_d), P(co_d), 0.5, P(rgbm), s))
    assert torch.equal(rgbm[0], rgb) and torch.equal(torch.signbit(rgbm[0]), torch.signbit(rgb))

    # split (featuresDc, featuresRest) through the autograd operator
    if K > 1:
        dc = co_d[:, 0].contiguous().requires_grad_()
        rest = co_d[:, 1:].contiguous().requires_grad_()
        out = ops.SphericalHarmonicsRgb.apply(use, m_d, cam_d, dc, rest)
        w.check("split.fwd.", out.detach(), r2["colors"], r2["B_colors"])
        check_mask(name + " split", out.detach(), r2)
        (out * v_d).sum().backward()
        w.check("split.bwd.", torch.cat([dc.grad[:, None], rest.grad], 1), r2["v_coeffs"], r2["B_v_coeffs"], cm2)
    torch.cuda.synchronize()
    w.report(f"certified {frac:.5f}; ")
    return r2


@pytest.mark.parametrize("n", [1, 127, 128, 129])
@pytest.mark.parametrize("degree", [0, 1, 2, 3, 4])
def test_sh_counts_and_degrees(n, degree):
    for use in range(degree + 1):
        for kind in ("generic", "straddle"):
            co, means, cam, v = sh_inputs(n, degree, 100 * n + 10 * degree + use, kind)
            run_sh_case(f"SH n={n} deg={degree} use={use} {kind}", degree, use, co, means, cam, v,
                        min_cert=0.99 if n > 100 else 0.0)


@pytest.mark.parametrize("degree,use", [(3, 3), (4, 2)])
def test_sh_million(degree, use):
    co, means, cam, v = sh_inputs(1_000_003, degree, 7 + degree)
    t0 = time.time()
    run_sh_case(f"SH n=1000003 deg={degree} use={use}", degree, use, co, means, cam, v)
    print(f"{time.time() - t0:.1f} s")


@pytest.mark.parametrize("degree", [1, 3])
@pytest.mark.parametrize("use", [0, 1])
def test_sh_misaligned_pointers(degree, use):
    """Coefficients and coefficient gradients one float past an aligned address: K = 4 and 16 leave the 128-bit
    span path for the scalar loads and stores."""
    co, means, cam, v = sh_inputs(1000 + 129, degree, 40 + degree, "straddle")
    run_sh_case(f"SH misaligned deg={degree} use={use}", degree, use, co, means, cam, v, off=1)


@pytest.mark.parametrize("kind", ["far", "axis", "straddle"])
@pytest.mark.parametrize("degree", [2, 4])
def test_sh_geometry_edges(kind, degree):
    co, means, cam, v = sh_inputs(5000, degree, 3 + degree, kind)
    for use in range(degree + 1):
        run_sh_case(f"SH {kind} deg={degree} use={use}", degree, use, co, means, cam, v)


@pytest.mark.parametrize("degree", [0, 3])
def test_sh_exact_ties(degree):
    """featuresDc = -1.7724538f at degrees_to_use 0: colour + 0.5 is exactly 0 in fp32, the kernels write -0 and
    pass the gradient there (D17).  With the fix reverted, these are the cases that fail."""
    co, means, cam, v = sh_inputs(3000, degree, 11 + degree, "ties")
    r = run_sh_case(f"SH ties deg={degree}", degree, 0, co, means, cam, v)
    assert int((r["tie"] & r["cert"]).sum()) > 1000 and bool(r["cert"].all())


# ------------------------------------------------------------------------------------------------ multi-view SH
def _multiview_inputs(n, degree, views, seed):
    co, means, _, _ = sh_inputs(n, degree, seed, "straddle")
    rng = np.random.default_rng(seed + 1)
    cams = (rng.standard_normal((views, 3)) * 3 + np.array([0, 0, -6])).astype(np.float32)
    v = rng.standard_normal((views, n, 3)).astype(np.float32)
    v[rng.uniform(size=(views, n)) < 0.3] = 0.0            # not visible in that view
    if views > 1:
        v[views // 2] = 0.0                                # a view whose cotangents are all zero
    co[:7, 0] = sf.TIE_DC                                  # exact ties (at degrees_to_use 0)
    return co, means, cams, v


@pytest.mark.parametrize("degree,views", [(3, 1), (3, 2), (3, 8), (3, 9), (3, 17), (4, 4), (4, 5)])
@pytest.mark.parametrize("use_sel", ["full", "zero"])
def test_sh_multiview(degree, views, use_sel):
    """gsb_sh_forward_rgb_cam_multiview, then gsb_mask_rgb_grad on the B slots and the multi-view VJP through
    gsb_sh_backward_multiview, _multiview_cams, gsb_exchange_gradients and _cams (world 1, with a geometry prefix that
    must come back times scale).  The straddling colours mask some channels of a Gaussian and not others."""
    use = degree if use_sel == "full" else 0
    n = 3001
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    co, means, cams, v = _multiview_inputs(n, degree, views, 31 * views + degree)
    K = co.shape[1]
    scale = 1.0 / views
    r = sf.sh_multiview(degree, use, cu(co), cu(means), cams, cu(v), scale, device=DEV)
    w = Worst(f"multiview deg={degree} use={use} views={views}")
    co_d, m_d, cams_d = cu(co), cu(means), cu(cams)
    rgbs = torch.empty((views, n, 3), device=DEV)
    capi.check(L.gsb_sh_forward_rgb_cam_multiview(n, degree, use, P(m_d), views, P(cams_d), P(co_d), 0.5, P(rgbs), s))
    cert_all = torch.ones(n, dtype=torch.bool, device=DEV)
    for i, rv in enumerate(r["views"]):
        w.check("fwd.", rgbs[i], rv["colors"], rv["B_colors"])
        check_mask(w.name + f" view {i}", rgbs[i], rv)
        cert_all &= rv["cert"].all(-1)
    frac = float(r["cert_v"].double().mean())
    assert frac >= 0.99, frac
    vm = cu(v)
    capi.check(L.gsb_mask_rgb_grad(n * views, P(rgbs), P(vm), s))
    part = (vm[:, :, 0] == 0) & (vm[:, :, 1] == 0) & (vm[:, :, 2] != 0)
    assert int(part.sum()) > 50                      # Gaussians with only the last channel live in a view
    ptrs = torch.tensor([vm[i].data_ptr() for i in range(views)], dtype=torch.int64, device=DEV)
    cam_ptrs = torch.tensor([cams_d[i].data_ptr() for i in range(views)], dtype=torch.int64, device=DEV)
    cm = r["cert_v"][:, None, :]
    for tag in ("mv", "mv_cams", "ex", "ex_cams"):
        out = torch.full((n, K, 3), float("nan"), device=DEV)
        cams_arg = cam_ptrs.data_ptr() if tag.endswith("cams") else P(cams_d)
        if tag.startswith("mv"):
            fn = L.gsb_sh_backward_multiview_cams if tag.endswith("cams") else L.gsb_sh_backward_multiview
            capi.check(fn(n, degree, use, P(m_d), views, cams_arg, ptrs.data_ptr(), scale, P(out), s))
        else:
            geom = torch.randn(4 * 1001, device=DEV)
            g0 = geom.clone()
            gp = torch.tensor([geom.data_ptr()], dtype=torch.int64, device=DEV)
            fn = L.gsb_exchange_gradients_cams if tag.endswith("cams") else L.gsb_exchange_gradients
            capi.check(fn(n, degree, use, P(m_d), views, cams_arg, ptrs.data_ptr(), scale, P(out), 0, 1, geom.numel(),
                          gp.data_ptr(), None, s))
            assert torch.equal(geom, g0 * np.float32(scale)), tag
        w.check(tag + ".", out, r["v_coeffs"], r["B_v_coeffs"], cm)
    torch.cuda.synchronize()
    w.report(f"certified {frac:.5f}; ")


# ------------------------------------------------------------------------------------------------------ loss
def loss_images(kind, H, W, seed):
    rng = np.random.default_rng(seed)
    if kind == "ties":
        return lf.tie_images(H, W, seed)
    if kind == "const_same":
        a = np.full((H, W, 3), 0.5, np.float32)
        return a, a.copy()
    if kind == "const_diff":
        return np.full((H, W, 3), 0.7, np.float32), np.full((H, W, 3), 0.2, np.float32)
    if kind == "checker":
        i, j = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        gt = np.repeat(((i + j) % 2).astype(np.float32)[..., None], 3, -1)
        rend = np.repeat((((i // 2) + (j // 2)) % 2).astype(np.float32)[..., None], 3, -1)
        return rend, gt
    gt = rng.uniform(0, 1, (H, W, 3)).astype(np.float32)
    if kind == "equal":
        return gt.copy(), gt
    rend = np.clip(gt + 0.15 * rng.standard_normal((H, W, 3)).astype(np.float32), 0, 1).astype(np.float32)
    return rend, gt


def run_loss_case(H, W, kind, weight):
    rend, gt = loss_images(kind, H, W, H * 7 + W)
    r_d, g_d = cu(rend), cu(gt)
    ref = lf.loss(r_d, g_d, weight, device=DEV)
    L = capi.lib()
    wsb = L.gsb_ssim_workspace_bytes(H, W)
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device=DEV)
    off = (-ws.data_ptr()) % 256
    v = torch.full((H, W, 3), float("nan"), device=DEV)
    out = torch.empty(3, device=DEV)
    capi.check(L.gsb_ssim_l1_loss(H, W, capi.ptr(r_d), capi.ptr(g_d), float(weight), capi.ptr(v), capi.ptr(out),
                                  ws.data_ptr() + off, wsb, capi.stream()))
    w = Worst(f"loss {H}x{W} {kind} w={weight}")
    w.check("v.", v, ref["v_rendered"], ref["B_v_rendered"])
    for i, k in enumerate(("loss", "l1", "ssim")):
        w.check(k, out[i:i + 1], torch.tensor([ref[k]], dtype=torch.float64, device=DEV),
                torch.tensor([ref["B_" + k]], dtype=torch.float64, device=DEV))
    rg = r_d.clone().requires_grad_()
    lo = ops.MainLoss.apply(rg, g_d, weight)
    lo.backward()
    w.check("op.loss", lo.detach().reshape(1), torch.tensor([ref["loss"]], dtype=torch.float64, device=DEV),
            torch.tensor([ref["B_loss"]], dtype=torch.float64, device=DEV))
    w.check("op.v.", rg.grad, ref["v_rendered"], ref["B_v_rendered"])
    torch.cuda.synchronize()
    w.report()


SMALL = [(1, 1), (1, 37), (37, 1), (5, 7), (11, 11), (15, 17), (16, 16), (17, 16), (31, 33), (45, 70), (270, 480)]
KINDS = ["random", "ties", "const_same", "const_diff", "checker", "equal"]


@pytest.mark.parametrize("H,W", SMALL)
@pytest.mark.parametrize("weight", [0.0, 0.2, 1.0])
def test_loss_sizes_and_contents(H, W, weight):
    for kind in KINDS:
        run_loss_case(H, W, kind, weight)


@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("weight", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("kind", ["random", "ties"])
def test_loss_full_size(H, W, weight, kind):
    t0 = time.time()
    run_loss_case(H, W, kind, weight)
    print(f"{time.time() - t0:.1f} s")
