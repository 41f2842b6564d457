"""Pins tests/depth_f64.py, the float64 reference of the depth and opacity maps (DESIGN D18) the GPU depth tests are
held to (CPU only):
  * against the reference's own numbers (tests/golden/depth_*.npz, made by tests/golden/make_golden_depth.py) at the
    tolerances of the operator-chain test: image, depth and alpha maps, and the gradients w.r.t. xys, conics, colours,
    opacities and the view-space depths of one weighted sum of the three;
  * it is not satisfied by wrong conventions: depth normalised by alpha, the background colour as background depth,
    and depth accumulated for the pair that terminates a pixel (blending it before the termination test);
  * against its own autograd: where every alpha stays below the 0.99 clamp, the depth gradient is the exact
    derivative of the depth map."""
import numpy as np
import pytest
import torch

import blend_f64 as bf
import depth_f64 as df
from oracle import oracle as orc
from util import load_golden, rel_l2, image_close

CASES = [("depth_tight_100x72", 2e-3), ("depth_bg_quat_128x96", 2e-3), ("depth_opaque_96x96", 2e-2)]


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(dtype) if dtype is not None else t


def _golden_case(name):
    g = load_golden(name)
    fx, fy, cx, cy = g["intrins"]
    H, W = [int(v) for v in g["hw"]]
    p = orc.project_forward(g["means"], g["scales"], 1.0, g["quats"], g["viewmat"], g["projmat"], fx, fy, cx, cy, H, W)
    cum, _ = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(g["ref_xys"], p["depths"], p["radii"], cum, H, W)
    return g, b, H, W


def _reference(g, b, H, W, **kw):
    return df.blend_depth(_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), _t(g["ref_xys"]), _t(g["ref_conics"]),
                          _t(g["colors"]), _t(g["opacities"]), _t(g["ref_z"]), _t(g["background"]), H, W,
                          v_output=_t(g["wgt"]), v_output_depth=_t(g["wgt_depth"]), v_output_alpha=_t(g["wgt_alpha"]),
                          **kw)


def _maps_close(r, g, gtol, depth=None):
    """(image, depth, alpha) against the golden at the chain test's image tolerance (the depth map relative to its
    largest value: it is not in [0, 1])."""
    frac = 1e-3 if gtol < 1e-2 else 1e-2
    depth = r["out_depth"] if depth is None else depth
    scale = float(np.abs(g["ref_depth"]).max())
    return (image_close(r["out_img"].numpy(), g["ref_img"], tol=5e-5, frac=frac)[0],
            image_close((depth / scale).numpy()[..., None], g["ref_depth"][..., None] / scale, tol=5e-5,
                        frac=frac)[0],
            image_close(r["out_alpha"].numpy()[..., None], g["ref_alpha"][..., None], tol=5e-5, frac=frac)[0])


@pytest.mark.parametrize("name,gtol", CASES)
def test_matches_reference_golden(name, gtol):
    g, b, H, W = _golden_case(name)
    r = _reference(g, b, H, W)
    assert all(_maps_close(r, g, gtol))
    for k, ref in (("v_xy", "ref_v_xy"), ("v_conic", "ref_v_conic"), ("v_colors", "ref_v_colors"),
                   ("v_opacity", "ref_v_opacity"), ("v_depths", "ref_v_z")):
        got = r[k].numpy().reshape(g[ref].shape)
        assert rel_l2(got, g[ref]) <= gtol, (k, rel_l2(got, g[ref]))
    assert float(np.abs(g["ref_v_z"]).max()) > 0 and float(r["out_depth"].max()) > 1.0


def _depth_forward(gs, bins, xys, conics, opac, z, H, W, blend_terminating=False):
    """The depth map written with plain torch ops per tile; blend_terminating=True accumulates the depth of the pair
    that terminates a pixel as well (the termination test placed after the blend)."""
    f8 = torch.float64
    tx_n = (W + bf.TILE - 1) // bf.TILE
    bins = bins.long().reshape(-1, 2)
    lens = (bins[:, 1] - bins[:, 0]).clamp_min(0)
    out = torch.zeros(H, W, dtype=f8)
    lx, ly = torch.arange(256) % bf.TILE, torch.arange(256) // bf.TILE
    for t in torch.nonzero(lens > 0).reshape(-1).tolist():
        s, L = int(bins[t, 0]), int(lens[t])
        gid = gs[s:s + L].long()
        X, Y = (t % tx_n) * bf.TILE + lx, (t // tx_n) * bf.TILE + ly
        inimg = (X < W) & (Y < H)
        dx = xys[gid, 0][None, :] - X[:, None].to(f8)
        dy = xys[gid, 1][None, :] - Y[:, None].to(f8)
        a, b, c = conics[gid, 0][None], conics[gid, 1][None], conics[gid, 2][None]
        sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
        alpha = torch.clamp(opac[gid][None] * torch.exp(-sigma), max=0.999)
        valid = (sigma >= 0) & (alpha >= bf.ALPHA_MIN)
        P = torch.cumprod(torch.where(valid, 1.0 - alpha, torch.ones_like(alpha)), -1)
        Pprev = torch.cat([torch.ones_like(P[:, :1]), P[:, :-1]], -1)
        blended = valid & ((Pprev > bf.T_EPS) if blend_terminating else (P > bf.T_EPS))
        Pb = torch.cumprod(torch.where(blended, 1.0 - alpha, torch.ones_like(alpha)), -1)
        Tb = torch.cat([torch.ones_like(Pb[:, :1]), Pb[:, :-1]], -1)
        d = (torch.where(blended, alpha * Tb, torch.zeros_like(alpha)) * z[gid][None]).sum(-1)
        out = out.index_put((Y[inimg], X[inimg]), d[inimg])
    return out


@pytest.mark.parametrize("name,gtol", CASES)
def test_wrong_conventions_do_not_match(name, gtol):
    g, b, H, W = _golden_case(name)
    r = _reference(g, b, H, W)
    # normalised depth: depth / alpha
    a = r["out_alpha"]
    normalised = torch.where(a > 0, r["out_depth"] / a.clamp_min(1e-30), torch.zeros_like(a))
    assert not _maps_close(r, g, gtol, depth=normalised)[1]
    # the forward restated per tile reproduces the map; with the terminating pair blended it does not (opaque case:
    # the only one whose pixels terminate)
    args = (_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), _t(g["ref_xys"], torch.float64),
            _t(g["ref_conics"], torch.float64), _t(g["opacities"], torch.float64).reshape(-1),
            _t(g["ref_z"], torch.float64), H, W)
    assert torch.allclose(_depth_forward(*args), r["out_depth"], rtol=0, atol=1e-12)
    if "opaque" in name:
        assert not _maps_close(r, g, gtol, depth=_depth_forward(*args, blend_terminating=True))[1]
    if float(np.abs(g["background"]).max()) > 0:
        # background depth = background colour
        rb = _reference(g, b, H, W, depth_background=g["background"][0])
        assert not _maps_close(rb, g, gtol)[1]


def test_depth_gradient_is_the_autograd_derivative():
    """Opacities below 0.99: the explicit v_depths and the depth map's share of v_xy / v_conic / v_opacity are the
    derivatives of the depth map written with torch ops."""
    g, b, H, W = _golden_case("depth_tight_100x72")
    vd = _t(g["wgt_depth"], torch.float64)
    r = df.blend_depth(_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), _t(g["ref_xys"]), _t(g["ref_conics"]),
                       _t(g["colors"]), _t(g["opacities"]), _t(g["ref_z"]), _t(g["background"]), H, W,
                       v_output=torch.zeros(H, W, 3, dtype=torch.float64), v_output_depth=vd)
    xy, con, op, z = (_t(g[k], torch.float64).reshape(s).requires_grad_()
                      for k, s in (("ref_xys", (-1, 2)), ("ref_conics", (-1, 3)), ("opacities", (-1,)), ("ref_z", (-1,))))
    d = _depth_forward(_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), xy, con, op, z, H, W)
    (d * vd).sum().backward()
    auto = {"v_depths": z.grad.reshape(-1, 1), "v_xy": xy.grad,
            "v_conic": con.grad * torch.tensor([1.0, 0.5, 1.0], dtype=torch.float64),
            "v_opacity": op.grad.reshape(-1, 1)}
    for k, gr in auto.items():
        err = (r[k] - gr).abs()
        assert bool((err <= 1e-10 * r["A_" + k] + 1e-300).all()), (k, float((err / r["A_" + k]).nan_to_num().max()))
        assert float(gr.abs().max()) > 0
