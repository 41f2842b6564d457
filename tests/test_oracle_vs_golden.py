"""Pins oracle/gsplat_oracle.c (plain-C restatement with CUDA tile semantics) against vectors
produced by the REFERENCE ITSELF (tests/golden/make_golden.py -> oracle/_ref).  CPU only.

Tolerances (SURVEY.md 8c, justified there): integer artefacts exact; projection |dxy| <= 2e-4 px
(D3: 1/(w+1e-6) vs 1/clamp(w)), conics rel 1e-4; rasterize on identical inputs: image 1e-5 with
isolated alpha-threshold flips <= 1/255; raster grads rel-L2 1e-4 (tight) / 2e-3 (opaque, D5 fringe);
projection grads rel-L2 1e-4.
"""
import numpy as np
import pytest
from oracle import oracle as orc
from util import load_golden, rel_l2, image_close

CASES = [("chain_tight_100x72", 1e-4), ("chain_bg_quat_128x96", 1e-4), ("chain_opaque_96x96", 5e-3)]


def _project(g):
    fx, fy, cx, cy = g["intrins"]
    H, W = [int(v) for v in g["hw"]]
    return orc.project_forward(g["means"], g["scales"], 1.0, g["quats"], g["viewmat"], g["projmat"],
                               fx, fy, cx, cy, H, W), (fx, fy, cx, cy, H, W)


@pytest.mark.parametrize("name,_", CASES)
def test_projection_forward_matches_reference(name, _):
    g = load_golden(name)
    p, _ = _project(g)
    vis = p["radii"] > 0
    assert vis.mean() > 0.9
    assert np.abs(p["xys"][vis] - g["ref_xys"][vis]).max() <= 2e-4
    cscale = np.abs(g["ref_conics"][vis]).max(axis=-1, keepdims=True)  # off-diagonals cancel to ~0
    assert (np.abs(p["conics"][vis] - g["ref_conics"][vis]) / cscale).max() <= 1e-4
    assert np.array_equal(p["depths"][vis], g["ref_depths"][vis])  # w == 1: NDC z == view z, exact
    # radius formula is shared (helpers.cuh:68-72 == gsplat_cpu.cpp:111-115); allow rare ceil() flips
    assert (p["radii"][vis] != g["ref_radii"][vis]).mean() <= 2e-3


@pytest.mark.parametrize("name,gtol", CASES)
def test_rasterize_forward_backward_match_reference(name, gtol):
    """Rasterize operator on IDENTICAL inputs (the reference's own xys/conics)."""
    g = load_golden(name)
    p, (fx, fy, cx, cy, H, W) = _project(g)
    cum, m = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(g["ref_xys"], p["depths"], p["radii"], cum, H, W)
    assert b["isect_ids"].shape[0] == m
    f = orc.rasterize_forward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], g["ref_xys"], g["ref_conics"],
                              g["colors"], g["opacities"], g["background"])
    # opaque case: D5 fringe (CPU blends inside +-(3*sqrt(cov)+2) px only, tiles blend up to alpha<1/255)
    ok, stats = image_close(f["out_img"], g["ref_img"], tol=1e-5, frac=1e-3 if gtol < 1e-3 else 1e-2)
    assert ok, stats
    r = orc.rasterize_backward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], g["ref_xys"], g["ref_conics"],
                               g["colors"], g["opacities"], g["background"], f["final_Ts"], f["final_idx"],
                               g["wgt"])
    assert rel_l2(r["v_colors"], g["ref_v_colors"]) <= gtol
    assert rel_l2(r["v_opacity"], g["ref_v_opacity"]) <= gtol
    assert rel_l2(r["v_xy"], g["ref_v_xy"]) <= gtol
    assert rel_l2(r["v_conic"], g["ref_v_conic"]) <= gtol


@pytest.mark.parametrize("name,_", CASES + [("projection_general", None), ("projection_ties", None)])
def test_projection_backward_matches_reference_autograd(name, _):
    """projection_*: general cameras (fov clamp, perspective divide, rotation in T = J V, glob_scale 1.3) and exact
    fov-clamp ties (D16); their cotangents are zero for the Gaussians the CUDA semantics cull."""
    g = load_golden(name)
    fx, fy, cx, cy = g["intrins"]
    H, W = [int(v) for v in g["hw"]]
    gs = float(g.get("glob_scale", 1.0))
    p = orc.project_forward(g["means"], g["scales"], gs, g["quats"], g["viewmat"], g["projmat"], fx, fy, cx, cy, H, W,
                            float(g.get("clip_thresh", 0.01)))
    r = orc.project_backward(g["means"], g["scales"], gs, g["quats"], g["viewmat"], g["projmat"],
                             fx, fy, cx, cy, H, W, p["radii"], p["conics"], g.get("v_xy", g.get("ref_v_xy")), None,
                             g.get("v_conic", g.get("ref_v_conic")))
    assert rel_l2(r["v_mean3d"], g["ref_v_means"]) <= 1e-4
    assert rel_l2(r["v_scale"], g["ref_v_scales"]) <= 1e-4
    assert rel_l2(r["v_quat"], g["ref_v_quats"]) <= 1e-4


def test_full_chain_image_close():
    g = load_golden("chain_tight_100x72")
    p, (fx, fy, cx, cy, H, W) = _project(g)
    cum, m = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], cum, H, W)
    f = orc.rasterize_forward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"], p["conics"],
                              g["colors"], g["opacities"], g["background"])
    ok, stats = image_close(f["out_img"], g["ref_img"], tol=5e-5, frac=2e-3)
    assert ok, stats


@pytest.mark.parametrize("name", ["sh_deg3", "sh_deg4"])
def test_sh_matches_reference(name):
    g = load_golden(name)
    deg = int(g["degree"])
    K = (deg + 1) ** 2
    for d in range(deg + 1):
        col = orc.sh_forward(d, g["viewdirs"], g["coeffs"])
        assert np.abs(col - g[f"ref_colors_d{d}"]).max() <= 2e-5
        vc = orc.sh_backward(d, K, g["viewdirs"], g["wgt"])
        assert np.abs(vc - g[f"ref_v_coeffs_d{d}"]).max() <= 2e-6
        nb = (d + 1) ** 2
        assert np.all(vc[:, nb:, :] == 0)


def test_tile_semantics_edge_cases():
    # empty scene: all tiles (0,0), image == background
    H, W = 40, 50
    z = np.zeros((0,), np.int32)
    bins = np.zeros((((W + 15) // 16) * ((H + 15) // 16), 2), np.int32)
    f = orc.rasterize_forward(H, W, z, bins, np.zeros((0, 2)), np.zeros((0, 3)), np.zeros((0, 3)),
                              np.zeros((0, 1)), [0.2, 0.4, 0.6])
    assert np.allclose(f["out_img"], [0.2, 0.4, 0.6]) and np.all(f["final_Ts"] == 1) and np.all(f["final_idx"] == 0)
    # behind-camera / near-clipped Gaussians are culled: radii == 0, num_tiles_hit == 0
    view = np.eye(4, dtype=np.float32)
    p = orc.project_forward(np.array([[0, 0, -1.0], [0, 0, 0.005], [0, 0, 2.0]], np.float32),
                            np.full((3, 3), 0.1, np.float32), 1.0, np.array([[1, 0, 0, 0]] * 3, np.float32),
                            view, view, 25.0, 25.0, 25.0, 20.0, H, W)
    assert list(p["radii"][:2]) == [0, 0] and p["radii"][2] > 0 and p["num_tiles_hit"][2] > 0
    # key layout: tile id in the high 32 bits, depth bits in the low 32 (forward.cu:132-137)
    cum, m = orc.cumsum(p["num_tiles_hit"])
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], cum, H, W)
    assert np.all((b["isect_ids"] & 0xFFFFFFFF) == np.float32(2.0).view(np.int32))
    assert np.all(np.diff(b["isect_ids_sorted"]) >= 0)


def test_main_loss_matches_reference():
    """(1-w) L1 + w (1 - SSIM) and its gradient: numpy restatement vs the reference's SSIM class + autograd."""
    g = load_golden("loss_45x70")
    r = orc.main_loss(g["rendered"], g["gt"], float(g["ssim_weight"]))
    assert abs(r["loss"] - float(g["ref_loss"])) <= 1e-6
    assert rel_l2(r["v_rendered"], g["ref_v_rendered"]) <= 1e-5
    # the reference's window is the asymmetric staircase of ssim.cpp:41-47, not a centred Gaussian
    w = orc.ssim_window()
    assert abs(w.sum() - 1) < 1e-6 and w[10] > w[0] and abs(w[9] - w[10]) < 1e-12 and w[0] != w[10]
