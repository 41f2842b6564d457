"""Pins tests/blend_f64.py, the float64 blend reference the GPU blend tests are held to (CPU only):
  * against its own autograd: where every alpha stays below the 0.99 clamp its explicit backward is the exact
    derivative of its forward;
  * against the fp32 oracle (oracle/gsplat_oracle.c) on the pixels and Gaussians it certifies, with no flip allowance;
  * against the reference's own numbers (tests/golden/chain_*.npz) at the tolerances of the operator-chain test."""
import numpy as np
import pytest
import torch

import blend_f64 as bf
from oracle import oracle as orc
from opensplat_b200.scene import make_scene
from util import load_golden, rel_l2, image_close

U = bf.U
# fp32 oracle vs float64: the oracle's expf is correctly rounded to within an ulp and its sums run in list order, so
# the error model needs less headroom than the kernels' (ex2.approx / rcp.approx, reordered sums)
C_ORC = 4.0


def _scene_2d(n, W, H, scale, opacity, seed, colors=(0.0, 1.0)):
    sc = make_scene(n, W, H, scale=scale, sh_degree=0, opacity=opacity, seed=seed)
    p = orc.project_forward(sc["means"], sc["scales"], 1.0, sc["quats"], sc["viewmat"], sc["projmat"], sc["fx"],
                            sc["fy"], sc["cx"], sc["cy"], H, W)
    cum, m = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], cum, H, W)
    rng = np.random.default_rng(seed + 7)
    col = rng.uniform(colors[0], colors[1], (n, 3)).astype(np.float32)
    return p, b, col, sc["opacities"]


def _t(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(dtype) if dtype is not None else t


def _ref(p, b, col, op, bg, H, W, **kw):
    return bf.blend(_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), _t(p["xys"]), _t(p["conics"]), _t(col), _t(op),
                    _t(np.asarray(bg, np.float32)), H, W, **kw)


@pytest.mark.parametrize("seed", [0, 1])
def test_explicit_backward_is_the_autograd_derivative(seed):
    """Opacities below 0.99: the 0.99 clamp of the backward never acts, so the explicit backward (T rebuilt from
    T_final back to front, v_output_alpha term, v_conic's 1/2 on the off-diagonal) is the derivative of the forward."""
    W, H, n = 37, 35, 300
    p, b, col, op = _scene_2d(n, W, H, 0.8, (0.3, 0.95), seed)
    rng = np.random.default_rng(seed)
    bg = np.array([0.3, 0.1, 0.7], np.float32)
    vo = rng.uniform(-1, 1, (H, W, 3))
    voa = rng.uniform(-1, 1, (H, W))
    r = _ref(p, b, col, op, bg, H, W, v_output=_t(vo), v_output_alpha=_t(voa))
    assert int(r["n_blend"].sum()) > 500 and float(r["final_Ts"].min()) < 0.05   # many pairs, some near-opaque pixels
    xy, con, c, o = (_t(a, torch.float64).requires_grad_() for a in (p["xys"], p["conics"], col, op))
    out, oa = bf.forward_autograd(_t(b["gaussian_ids_sorted"]), _t(b["tile_bins"]), xy, con, c, o, _t(bg), H, W)
    assert torch.allclose(out, r["out_img"], rtol=0, atol=1e-13)
    assert torch.allclose(1 - oa, r["final_Ts"], rtol=0, atol=1e-13)
    ((out * _t(vo)).sum() + (oa * _t(voa)).sum()).backward()
    auto = {"v_xy": xy.grad, "v_conic": con.grad * torch.tensor([1.0, 0.5, 1.0], dtype=torch.float64),
            "v_colors": c.grad, "v_opacity": o.grad.reshape(-1, 1)}
    for k, g in auto.items():
        err = (r[k] - g).abs()
        assert bool((err <= 1e-10 * r["A_" + k] + 1e-300).all()), (k, float((err / r["A_" + k]).nan_to_num().max()))
        assert float(g.abs().max()) > 0


@pytest.mark.parametrize("seed,W,H,n,scale,opacity,exp_mode", [
    (0, 64, 48, 300, 0.3, (0.05, 0.35), 0),
    (1, 70, 50, 800, 0.2, (0.004, 0.02), 1),     # faint: alpha near 1/255 over much of each footprint
    (2, 48, 40, 200, 0.8, (0.9, 1.0), 0),        # opaque: both clamps, early termination
])
def test_certified_pixels_and_gaussians_match_oracle(seed, W, H, n, scale, opacity, exp_mode):
    p, b, col, op = _scene_2d(n, W, H, scale, opacity, seed)
    bg = np.array([0.2, 0.5, 0.1], np.float32)
    rng = np.random.default_rng(seed + 1)
    vo = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    r = _ref(p, b, col, op, bg, H, W, v_output=_t(vo))
    f = orc.rasterize_forward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"], p["conics"], col, op, bg,
                              exp_mode=exp_mode)
    cert = r["pix_cert"].numpy()
    assert cert.mean() >= 0.99, cert.mean()
    assert np.array_equal(f["final_idx"][cert], r["final_idx"].numpy()[cert])
    nb = r["n_blend"].numpy()[..., None] + 8.0
    bound = C_ORC * U * (nb * r["A_out"].numpy() + r["B_out"].numpy())
    d = np.abs(f["out_img"] - r["out_img"].numpy())
    assert (d[cert] <= bound[cert]).all(), (d[cert] / bound[cert]).max()
    bT = C_ORC * U * (nb[..., 0] * r["A_T"].numpy() + r["B_T"].numpy())
    assert (np.abs(f["final_Ts"] - r["final_Ts"].numpy())[cert] <= bT[cert]).all()
    g = orc.rasterize_backward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"], p["conics"], col, op, bg,
                               f["final_Ts"], f["final_idx"], vo, exp_mode=exp_mode)
    gc = r["gauss_cert"].numpy()
    assert gc.mean() >= 0.95, gc.mean()
    for k in ("v_xy", "v_conic", "v_colors", "v_opacity"):
        err = np.abs(g[k] - r[k].numpy())[gc]
        bd = C_ORC * U * (r["B_" + k].numpy() + (8 + r["n_tiles"].numpy()[:, None]) * r["A_" + k].numpy())[gc]
        assert (err <= bd).all(), (k, (err / bd).max())


@pytest.mark.parametrize("name,gtol,itol", [("chain_tight_100x72", 2e-3, 5e-5), ("chain_bg_quat_128x96", 2e-3, 5e-5),
                                            ("chain_opaque_96x96", 2e-2, 5e-5)])
def test_matches_reference_golden(name, gtol, itol):
    """The reference's own image and gradients for these inputs; the opaque case has the D5 fringe (the reference's
    CPU back end blends only inside +-(3 sqrt(cov) + 2) px, the tile blend down to alpha = 1/255)."""
    g = load_golden(name)
    fx, fy, cx, cy = g["intrins"]
    H, W = [int(v) for v in g["hw"]]
    p = orc.project_forward(g["means"], g["scales"], 1.0, g["quats"], g["viewmat"], g["projmat"], fx, fy, cx, cy, H, W)
    cum, _ = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(g["ref_xys"], p["depths"], p["radii"], cum, H, W)
    q = dict(xys=g["ref_xys"], conics=g["ref_conics"])
    r = _ref(q, b, g["colors"], g["opacities"], g["background"], H, W, v_output=_t(g["wgt"]))
    ok, stats = image_close(r["out_img"].numpy(), g["ref_img"], tol=itol, frac=1e-3 if gtol < 1e-2 else 1e-2)
    assert ok, stats
    for k in ("v_xy", "v_conic", "v_colors", "v_opacity"):
        assert rel_l2(r[k].numpy(), g["ref_" + k]) <= gtol, k
