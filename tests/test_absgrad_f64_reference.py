"""CPU: the float64 reference of AbsGS's absolute screen-space gradient (tests/absgrad_f64.py, DESIGN D25) against
an independent restatement, its defining properties and the failure it exists for; RefineConfig's defaults,
GaussianModel's refusal of absgrad and the argument checks of gsb_rasterize_backward_absgrad (no kernel runs)."""
import ctypes as C

import numpy as np
import pytest
import torch

import absgrad_f64 as af
import blend_f64 as bf
from opensplat_b200 import capi
from opensplat_b200.densify import RefineConfig

F8 = torch.float64


def _bins(xys, radii, H, W):
    """Sorted lists (depth order = index order) and tile_bins of every Gaussian over its tile box, in float64 numpy."""
    tx, ty = (W + 15) // 16, (H + 15) // 16
    lists = [[] for _ in range(tx * ty)]
    for g in range(xys.shape[0]):
        x, y, r = float(xys[g, 0]), float(xys[g, 1]), int(radii[g])
        x0, x1 = max(0, int(np.floor((x - r) / 16))), min(tx, int(np.floor((x + r) / 16)) + 1)
        y0, y1 = max(0, int(np.floor((y - r) / 16))), min(ty, int(np.floor((y + r) / 16)) + 1)
        for j in range(y0, y1):
            for i in range(x0, x1):
                lists[j * tx + i].append(g)
    gs, bins = [], []
    for lst in lists:
        bins.append((len(gs), len(gs) + len(lst)))
        gs.extend(lst)
    return torch.tensor(gs, dtype=torch.int64), torch.tensor(bins, dtype=torch.int64)


def _case(seed, n, W, H, s=(0.8, 4.0), opac=(0.05, 0.9)):
    rng = np.random.default_rng(seed)
    xys = np.stack([rng.uniform(-2, W + 2, n), rng.uniform(-2, H + 2, n)], -1)
    sm = rng.uniform(*s, n)
    sn = sm * rng.uniform(0.3, 1.0, n)
    th = rng.uniform(0, np.pi, n)
    ct, st = np.cos(th), np.sin(th)
    sxx, syy, sxy = ct * ct * sm ** 2 + st * st * sn ** 2, st * st * sm ** 2 + ct * ct * sn ** 2, ct * st * (sm ** 2 - sn ** 2)
    det = sxx * syy - sxy * sxy
    con = np.stack([syy / det, -sxy / det, sxx / det], -1)
    gs, bins = _bins(xys, np.ceil(3 * sm), H, W)
    t = lambda a: torch.tensor(np.asarray(a), dtype=F8)
    return dict(gs=gs, bins=bins, xys=t(xys), conics=t(con), colors=t(rng.uniform(0, 1, (n, 3))),
                opac=t(rng.uniform(*opac, n)), bg=t([0.3, 0.6, 0.2]), v_out=t(rng.uniform(-1, 1, (H, W, 3))),
                voa=t(rng.uniform(-1, 1, (H, W))), depths=t(rng.uniform(0.5, 5.0, n)),
                vd=t(rng.uniform(-1, 1, (H, W))), H=H, W=W)


def _ref(c, depth=False, voa=True):
    return af.absgrad(c["gs"], c["bins"], c["xys"], c["conics"], c["colors"], c["opac"], c["bg"], c["H"], c["W"],
                      c["v_out"], c["voa"] if voa else None, depths=c["depths"] if depth else None,
                      v_output_depth=c["vd"] if depth else None)


@pytest.mark.parametrize("depth", [False, True])
@pytest.mark.parametrize("seed,n,W,H", [(0, 12, 9, 7), (1, 20, 18, 17)])
def test_equals_per_pixel_autograd(seed, n, W, H, depth):
    """v_xy_abs = sum over pixels p of |d(v_out_p . out_p + v_alpha_p alpha_p [+ v_depth_p depth_p]) / d xy|, each
    pixel's gradient taken by autograd through blend_f64.forward_autograd (the depth map as a blend of z with
    background 0).  Opacities stay below 0.99, where the forward and backward alpha clamps do not bind."""
    c = _case(seed, n, W, H)
    r = _ref(c, depth=depth)
    xys = c["xys"].clone().requires_grad_()
    out, oa = bf.forward_autograd(c["gs"], c["bins"], xys, c["conics"], c["colors"], c["opac"], c["bg"], H, W)
    per_pixel = (out * c["v_out"]).sum(-1) + oa * c["voa"]
    if depth:
        z3 = c["depths"][:, None].expand(-1, 3)
        od, _ = bf.forward_autograd(c["gs"], c["bins"], xys, c["conics"], z3, c["opac"], torch.zeros(3, dtype=F8), H,
                                    W)
        per_pixel = per_pixel + od[..., 0] * c["vd"]
    want = torch.zeros(n, 2, dtype=F8)
    for y in range(H):
        for x in range(W):
            g, = torch.autograd.grad(per_pixel[y, x], xys, retain_graph=True, allow_unused=True)
            if g is not None:
                want += g.abs()
    assert float(want.abs().max()) > 0
    torch.testing.assert_close(r["v_xy_abs"], want, rtol=1e-10, atol=1e-14)
    # and the signed sum over the same pairs is blend_f64's v_xy
    torch.testing.assert_close(r["v_xy_pairs"], r["v_xy"], rtol=1e-10, atol=1e-14)


def test_single_pixel_gaussians_give_abs_v_xy():
    """Gaussians so small that each blends exactly one pixel: the sum of absolute values is the absolute sum."""
    rng = np.random.default_rng(3)
    H, W, n = 20, 24, 30
    px = rng.permutation(H * W)[:n]
    xys = np.stack([px % W + rng.uniform(-0.2, 0.2, n), px // W + rng.uniform(-0.2, 0.2, n)], -1)
    s = rng.uniform(0.15, 0.25, n)
    con = np.stack([1 / s ** 2, np.zeros(n), 1 / s ** 2], -1)
    gs, bins = _bins(xys, np.ones(n), H, W)
    t = lambda a: torch.tensor(np.asarray(a), dtype=F8)
    c = dict(gs=gs, bins=bins, xys=t(xys), conics=t(con), colors=t(rng.uniform(0, 1, (n, 3))),
             opac=t(rng.uniform(0.2, 0.9, n)), bg=t([0.1, 0.2, 0.3]), v_out=t(rng.uniform(-1, 1, (H, W, 3))),
             voa=t(rng.uniform(-1, 1, (H, W))), H=H, W=W)
    r = _ref(c)
    assert int(r["n_blend"].sum()) == n and int(r["n_blend"].max()) == 1      # one pixel per Gaussian
    assert float(r["v_xy"].abs().min()) > 0
    torch.testing.assert_close(r["v_xy_abs"], r["v_xy"].abs(), rtol=1e-12, atol=0)


@pytest.mark.parametrize("depth", [False, True])
def test_abs_sum_bounds_abs_v_xy(depth):
    """Componentwise v_xy_abs >= |v_xy| (up to float64 rounding of the two sums), and strictly above it for Gaussians
    that cover several pixels."""
    c = _case(7, 80, 40, 33, s=(1.0, 6.0))
    r = _ref(c, depth=depth)
    slack = 1e-12 * r["A_v_xy_abs"]
    assert bool((r["v_xy_abs"] >= r["v_xy"].abs() - slack).all())
    assert float((r["v_xy_abs"] - r["v_xy"].abs()).max()) > 0.1 * float(r["v_xy_abs"].max())
    assert bool((r["B_v_xy_abs"] >= 0).all()) and bool((r["A_v_xy_abs"] >= r["v_xy_abs"] * (1 - 1e-12)).all())


def test_cancellation_case():
    """One Gaussian centred on a pixel over a target that is mirror-symmetric about that centre (alternating dark and
    bright columns, and rows): each pixel pulls the mean one way, its mirror image the other way, so v_xy cancels to
    rounding while v_xy_abs is large -- the Gaussian AbsGS splits and the plain statistic never does."""
    H = W = 33
    cx = cy = 16.0
    sd = 4.0
    t = lambda a: torch.tensor(np.asarray(a), dtype=F8)
    xys, con = t([[cx, cy]]), t([[1 / sd ** 2, 0.0, 1 / sd ** 2]])
    gs, bins = _bins(np.array([[cx, cy]]), [int(3 * sd)], H, W)
    X, Y = np.meshgrid(np.arange(W), np.arange(H))
    target = ((X - 16) % 2 == 0) ^ ((Y - 16) % 2 == 0)
    target = t(np.repeat(target[..., None], 3, -1).astype(np.float64))
    c = dict(gs=gs, bins=bins, xys=xys, conics=con, colors=t([[0.5, 0.5, 0.5]]), opac=t([0.8]),
             bg=t([0.0, 0.0, 0.0]), H=H, W=W, voa=None)
    fwd = bf.blend(gs, bins, xys, con, c["colors"], c["opac"], c["bg"], H, W)
    c["v_out"] = 2.0 * (fwd["out_img"] - target) / target.numel()            # the gradient of the MSE
    r = _ref(c, voa=False)
    v, va = float(r["v_xy"].abs().max()), float(r["v_xy_abs"].min())
    assert v <= 1e-12 * va
    # the statistic (norm x 0.5 max(W, H), one view): far above the absgrad threshold, far below the plain one
    scale = 0.5 * max(H, W)
    assert float(r["v_xy_abs"].norm()) * scale > 10 * 0.0008 and float(r["v_xy"].norm()) * scale < 1e-3 * 0.0002


def test_config_defaults_and_model_refusal():
    c = RefineConfig()
    assert c.absgrad is False and c.densify_grad_thresh == 0.0002
    assert RefineConfig(absgrad=True, densify_grad_thresh=0.0008).absgrad
    from opensplat_b200.model import GaussianModel
    with pytest.raises(ValueError, match="absgrad"):
        GaussianModel({}, RefineConfig(absgrad=True), device="cpu")


P = C.c_void_p(256)      # any 256-byte aligned address: every call below is rejected before it is used


def test_capi_argument_checks():
    L = capi.lib()
    fn = L.gsb_rasterize_backward_absgrad

    def call(flags=0, record_depths=None, v_output_depth=None, v_depths=None, v_xy_abs=P, m=4):
        # a 20x20 image: 2x2 tiles
        return fn(20, 20, 2, 2, 3, m, P, None, P, P, P, P, P, P, P, P, None, P, P, P, P, P, flags, record_depths,
                  v_output_depth, v_depths, v_xy_abs, None)

    assert call(v_xy_abs=None) != 0                          # no output
    assert call(v_xy_abs=C.c_void_p(260)) != 0               # not 8-byte aligned
    assert call(record_depths=P) != 0                        # depth pointers without v_depths
    assert call(v_output_depth=P) != 0
    assert call(v_depths=P) != 0                             # depth without record_depths (m > 0)
    assert call(flags=2) != 0                                # unknown flag
    assert call(flags=0x100) != 0
    for code in (call(v_xy_abs=None), call(flags=2)):
        assert code != 0 and L.gsb_last_error()
