"""GPU parity: the sm_90a kernels, called through the C ABI (opensplat_b200.capi / ops), against
  (a) oracle/gsplat_oracle.c on the same seeded inputs (stage by stage),
  (b) the committed golden vectors produced by the reference itself (tests/golden).
Integer artefacts (radii, num_tiles_hit, M, keys, permutation, tile bins) must be BIT-EXACT.
Floating point tolerances are those of SURVEY.md 8c and are written next to each assert."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from opensplat_b200 import ops
from opensplat_b200.scene import make_scene
from util import load_golden, rel_l2, image_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def cu(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV)


def npy(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------------------------------------- SH
@pytest.mark.parametrize("name", ["sh_deg3", "sh_deg4"])
def test_sh_vs_golden_and_oracle(name):
    g = load_golden(name)
    deg = int(g["degree"])
    K = (deg + 1) ** 2
    for d in range(deg + 1):
        col = ops.compute_sh_forward(deg, d, cu(g["viewdirs"]), cu(g["coeffs"]))
        assert np.abs(npy(col) - g[f"ref_colors_d{d}"]).max() <= 2e-5          # vs reference
        assert np.abs(npy(col) - orc.sh_forward(d, g["viewdirs"], g["coeffs"])).max() <= 5e-6  # vs oracle
        vc = ops.compute_sh_backward(deg, d, cu(g["viewdirs"]), cu(g["wgt"]))
        assert np.abs(npy(vc) - g[f"ref_v_coeffs_d{d}"]).max() <= 2e-6
        assert np.all(npy(vc)[:, (d + 1) ** 2:, :] == 0)


@pytest.mark.parametrize("n,deg", [(1, 0), (127, 1), (129, 2), (1000, 3), (257, 4)])
def test_sh_ragged_sizes(n, deg):
    rng = np.random.default_rng(n)
    K = (deg + 1) ** 2
    vd = rng.standard_normal((n, 3)).astype(np.float32)
    co = rng.standard_normal((n, K, 3)).astype(np.float32)
    vcol = rng.standard_normal((n, 3)).astype(np.float32)
    col = ops.compute_sh_forward(deg, deg, cu(vd), cu(co))
    assert np.abs(npy(col) - orc.sh_forward(deg, vd, co)).max() <= 1e-5
    vc = ops.compute_sh_backward(deg, deg, cu(vd), cu(vcol))
    assert np.abs(npy(vc) - orc.sh_backward(deg, K, vd, vcol)).max() <= 3e-6


def test_sh_fused_rgb_variants():
    from opensplat_b200 import capi
    g = load_golden("sh_deg3")
    n = g["viewdirs"].shape[0]
    vd, co, w = cu(g["viewdirs"]), cu(g["coeffs"]).requires_grad_(), cu(g["wgt"])
    ref = torch.clamp_min(ops.SphericalHarmonics.apply(3, vd, co) + 0.5, 0.0)
    (ref * w).sum().backward()
    L = capi.lib()
    rgbs = torch.empty((n, 3), device=DEV)
    vco = torch.empty((n, 16, 3), device=DEV)
    capi.check(L.gsb_sh_forward_rgb(n, 3, 3, capi.ptr(vd), capi.ptr(co.detach()), 0.5, capi.ptr(rgbs), capi.stream()))
    capi.check(L.gsb_sh_backward_rgb(n, 3, 3, capi.ptr(vd), capi.ptr(rgbs), capi.ptr(w), capi.ptr(vco), capi.stream()))
    assert torch.equal(rgbs, ref.detach()) and torch.equal(vco, co.grad)
    assert float((rgbs == 0).float().mean()) > 0.05   # the clamp is active on this data


@pytest.mark.parametrize("n,deg,use", [(1000, 3, 3), (129, 3, 1), (5003, 2, 2), (64, 0, 0), (300, 4, 4)])
def test_sh_split_variant_matches_cat_sh_clamp(n, deg, use):
    """gsb_sh_forward_split / _backward_split (featuresDc + featuresRest read where they lie, view direction formed in
    the kernel, + 0.5 and clamp fused) against the reference's op sequence cat -> SphericalHarmonics -> clamp_min
    (model.cpp:176-177,186-192) through autograd."""
    rng = np.random.default_rng(n + deg)
    K = (deg + 1) ** 2
    means = cu(rng.uniform(-1, 1, (n, 3)).astype(np.float32))
    cam = cu(np.array([0.3, -0.2, -8.0], np.float32))
    dc = cu(rng.standard_normal((n, 3)).astype(np.float32)).requires_grad_()
    rest = cu((0.3 * rng.standard_normal((n, K - 1, 3))).astype(np.float32)).requires_grad_()
    w = cu(rng.standard_normal((n, 3)).astype(np.float32))
    vd = means - cam
    vd = vd / vd.norm(dim=-1, keepdim=True)
    ref = torch.clamp_min(ops.SphericalHarmonics.apply(use, vd, torch.cat([dc[:, None, :], rest], 1)) + 0.5, 0.0)
    (ref * w).sum().backward()
    g_dc, g_rest = dc.grad.clone(), rest.grad.clone()
    dc.grad = rest.grad = None
    got = ops.SphericalHarmonicsRgb.apply(use, means, cam, dc, rest)
    (got * w).sum().backward()
    assert float((got - ref).abs().max()) <= 3e-6
    assert float((got == 0).float().mean()) > 0.02 or deg == 0      # the clamp is active
    # a clamp decision may flip where SH + 0.5 is within rounding of 0; everywhere else the gradients agree
    same = ((got > 0) == (ref > 0)).all(dim=-1)
    assert float(same.float().mean()) > 0.999
    assert float((dc.grad - g_dc)[same].abs().max()) <= 3e-6
    if K > 1:
        assert float((rest.grad - g_rest)[same].abs().max()) <= 3e-6
        assert float(rest.grad[:, (use + 1) ** 2 - 1:, :].abs().sum()) == 0.0     # bases above degreesToUse get 0


# ------------------------------------------------------------------------------- projection + bins
def _scene(n, W, H, scale, opacity=(0.05, 0.35), seed=0, **kw):
    return make_scene(n, W, H, scale=scale, sh_degree=0, opacity=opacity, seed=seed, **kw)


def _project_gpu(sc):
    tb = ops.tile_bounds(sc["W"], sc["H"])
    return ops.project_gaussians_forward(cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]),
                                         cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"], sc["fy"], sc["cx"],
                                         sc["cy"], sc["H"], sc["W"], tb)


def _project_orc(sc):
    return orc.project_forward(sc["means"], sc["scales"], 1.0, sc["quats"], sc["viewmat"], sc["projmat"],
                               sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["H"], sc["W"])


@pytest.mark.parametrize("n,W,H,scale", [(5000, 256, 256, 0.3), (20000, 500, 300, 0.2), (3, 33, 17, 1.0)])
def test_projection_forward_bit_exact(n, W, H, scale):
    sc = _scene(n, W, H, scale, seed=n)
    # push some Gaussians behind the near plane / off screen to exercise the culls
    sc["means"][: n // 10, 2] = -9.0
    sc["means"][n // 10: n // 5, 0] = 5.0
    cov3d, xys, depths, radii, conics, nth = _project_gpu(sc)
    o = _project_orc(sc)
    assert np.array_equal(npy(radii), o["radii"])                 # bit-exact
    assert np.array_equal(npy(nth), o["num_tiles_hit"])           # bit-exact
    # the float chain is correctly-rounded op-for-op on both sides -> also bit-exact
    assert np.array_equal(npy(xys), o["xys"])
    assert np.array_equal(npy(depths), o["depths"])
    assert np.array_equal(npy(conics), o["conics"])
    assert np.array_equal(npy(cov3d), o["cov3d"])
    assert (o["radii"] == 0).sum() >= n // 5


@pytest.mark.parametrize("n,W,H,scale", [(4000, 256, 256, 0.3), (30000, 640, 360, 0.15), (50, 48, 40, 2.0)])
def test_binning_bit_exact(n, W, H, scale):
    sc = _scene(n, W, H, scale, seed=7 * n)
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    o = _project_orc(sc)
    cum = ops.cumsum_tiles_hit(nth)
    ocum, m = orc.cumsum(o["num_tiles_hit"])
    assert np.array_equal(npy(cum), ocum) and int(cum[-1]) == m
    tb = ops.tile_bounds(W, H)
    isect, gids, ks, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, tb, return_index=True)
    ob = orc.bin_and_sort(o["xys"], o["depths"], o["radii"], ocum, H, W)
    assert np.array_equal(npy(isect), ob["isect_ids"])
    assert np.array_equal(npy(gids), ob["gaussian_ids"])
    assert np.array_equal(npy(ks), ob["isect_ids_sorted"])
    assert np.array_equal(npy(idx), ob["sorted_index"])           # stable: ties keep ascending index
    assert np.array_equal(npy(gs), ob["gaussian_ids_sorted"])
    assert np.array_equal(npy(bins), ob["tile_bins"])


def _bucket_exact(xys, depths, radii, conics, colors, opac, tb, cull, want_index=True):
    """Two-phase fast path with exact capacities (phase 1 once with zero capacities to learn M / longest list)."""
    n = xys.shape[0]
    _, _, stats0, _ = ops.bucket_tile_ranges(xys, radii, conics, colors, opac, tb, 0, 0, cull=cull)
    m, max_len, ovf, _ = (int(v) for v in stats0.tolist())
    assert ovf == (1 if m > 0 else 0)
    bins, cum, stats, ws = ops.bucket_tile_ranges(xys, radii, conics, colors, opac, tb, m, max_len, cull=cull)
    assert [int(v) for v in stats.tolist()] == [m, max_len, 0, 0]
    rec, idx, gs = ops.bucket_sort_pack(n, m, max_len, depths, radii, cum, tb, bins, stats, ws, cull=cull,
                                        want_index=want_index)
    return m, max_len, bins, cum, stats, rec, idx, gs


@pytest.mark.parametrize("n,W,H,scale", [(4000, 256, 256, 0.3), (30000, 640, 360, 0.15), (50, 48, 40, 2.0),
                                         (200_000, 1024, 576, 0.05), (1_000_000, 1920, 1080, 0.02)])
def test_bucket_binning_matches_generic_sort(n, W, H, scale):
    """The two-level fast path (tile bucket + in-smem depth sort + fused pack), WITHOUT culling, must give the same
    cum_tiles_hit, tile_bins and the same per-tile order as cumsum + emit + global 64-bit sort + bin edges
    (bit-exact), and the same records -- up to the full C2 size the bench runs."""
    sc = _scene(n, W, H, scale, seed=3 * n, opacity=(0.05, 0.95) if n >= 1_000_000 else (0.05, 0.35))
    if n == 4000:   # duplicate depths: ties must resolve to ascending unsorted slot (stable order)
        sc["means"][:, 2] = np.round(sc["means"][:, 2] * 8) / 8
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    cum = ops.cumsum_tiles_hit(nth)
    tb = ops.tile_bounds(W, H)
    rng = np.random.default_rng(5)
    colors = cu(rng.uniform(0, 1, (n, 3)).astype(np.float32))
    opac = cu(sc["opacities"])
    m, max_len, bins_b, cum_b, stats, rec_b, idx_b, gs_b = _bucket_exact(xys, depths, radii, conics, colors, opac, tb,
                                                                        cull=False)
    assert m == int(cum[-1]) and torch.equal(cum_b, cum)
    isect, gids, ks, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, tb, return_index=True)
    assert torch.equal(bins_b, bins)
    assert int((bins[:, 1] - bins[:, 0]).max()) == max_len
    assert torch.equal(idx_b, idx) and torch.equal(gs_b, gs)
    bg = cu(np.zeros(3, np.float32))
    out, fT, fI, rec = ops.rasterize_forward(tb, (W, H, 1), gs, idx, bins, xys, conics, colors, opac, bg)
    assert torch.equal(rec_b[: m * 48], rec[: m * 48])
    out_b, fT_b, fI_b = ops.rasterize_forward_packed(tb, (W, H, 1), m, bins_b, rec_b, bg, stats)
    assert torch.equal(out, out_b) and torch.equal(fI, fI_b)


@pytest.mark.parametrize("n,W,H,scale,opac", [(4000, 256, 256, 0.3, (0.05, 0.35)), (30000, 640, 360, 0.15, (0.01, 0.99)),
                                              (50, 48, 40, 2.0, (0.3, 0.6)), (200_000, 1024, 576, 0.05, (0.05, 0.95)),
                                              (1_000_000, 1920, 1080, 0.02, (0.05, 0.95))])
def test_culled_binning_is_the_generic_lists_minus_untouched_pairs(n, W, H, scale, opac):
    """cull = 1 (what RasterizeGaussians uses): every tile list is the reference's list minus pairs whose extent box
    misses the tile, in the same order; image, final_Ts and all four gradients are BIT-identical to the
    unculled path (the dropped pairs contribute exactly nothing)."""
    sc = _scene(n, W, H, scale, seed=3 * n + 1, opacity=opac)
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    cum = ops.cumsum_tiles_hit(nth)
    tb = ops.tile_bounds(W, H)
    rng = np.random.default_rng(6)
    colors = cu(rng.uniform(0, 1, (n, 3)).astype(np.float32))
    op = cu(sc["opacities"])
    bg = cu(np.array([0.2, 0.1, 0.3], np.float32))
    m0, _, bins0, cum0, st0, rec0, idx0, gs0 = _bucket_exact(xys, depths, radii, conics, colors, op, tb, cull=False)
    m1, len1, bins1, cum1, st1, rec1, idx1, gs1 = _bucket_exact(xys, depths, radii, conics, colors, op, tb, cull=True)
    assert 0 < m1 <= m0
    if n >= 30000:
        assert m1 < 0.95 * m0          # the cull does remove pairs on these scenes
    # per tile: the culled Gaussian list is a subsequence of the reference's list
    b0, b1, g0, g1 = npy(bins0), npy(bins1), npy(gs0), npy(gs1)
    lens1 = b1[:, 1] - b1[:, 0]
    assert lens1.sum() == m1 and lens1.max() == len1
    for t in np.random.default_rng(0).choice(b0.shape[0], size=min(200, b0.shape[0]), replace=False):
        full, kept = g0[b0[t, 0]:b0[t, 1]], g1[b1[t, 0]:b1[t, 1]]
        it = iter(full.tolist())
        assert all(any(x == y for y in it) for x in kept.tolist()), f"tile {t}: not a subsequence"
    # cum of the culled path counts the kept pairs per Gaussian
    per_g = np.bincount(g1[:m1], minlength=n)
    assert np.array_equal(np.diff(np.concatenate([[0], npy(cum1)])), per_g)
    out0, fT0, fI0 = ops.rasterize_forward_packed(tb, (W, H, 1), m0, bins0, rec0, bg, st0)
    out1, fT1, fI1 = ops.rasterize_forward_packed(tb, (W, H, 1), m1, bins1, rec1, bg, st1)
    assert torch.equal(out0, out1) and torch.equal(fT0, fT1)
    v_out = cu(rng.uniform(-1, 1, (H, W, 3)).astype(np.float32))
    ga = ops.rasterize_backward(H, W, n, m0, bins0, conics, op, rec0, cum0, bg, fT0, fI0, v_out)
    gb = ops.rasterize_backward(H, W, n, m1, bins1, conics, op, rec1, cum1, bg, fT1, fI1, v_out)
    for a, b in zip(ga, gb):
        assert torch.equal(a, b)


def test_tile_order_is_a_longest_first_permutation_and_changes_nothing():
    """gsb_bucket_tile_ranges' tile order: a permutation of the tile ids in which list lengths never increase by more
    than one 1/64 length bucket; image and gradients are bit-identical with and without it."""
    n, W, H = 60_000, 640, 360
    sc = _scene(n, W, H, 0.12, seed=31, opacity=(0.05, 0.9))
    sc["means"][: n // 2, :2] *= 0.4                 # uneven coverage: long lists in the centre, short at the border
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    tb = ops.tile_bounds(W, H)
    T = tb[0] * tb[1]
    rng = np.random.default_rng(8)
    colors, op = cu(rng.uniform(0, 1, (n, 3)).astype(np.float32)), cu(sc["opacities"])
    bg = cu(np.zeros(3, np.float32))
    m, max_len, bins, cum, stats, rec, _, _ = _bucket_exact(xys, depths, radii, conics, colors, op, tb, cull=True)
    order = npy(bins.tile_order)
    assert np.array_equal(np.sort(order), np.arange(T))
    lens = (npy(bins)[:, 1] - npy(bins)[:, 0])[order]
    bucket = lens.astype(np.int64) * 64 // (max_len + 1)
    assert np.all(np.diff(bucket) <= 0) and bucket[0] == bucket.max() and lens.max() == max_len
    a = ops.rasterize_forward_packed(tb, (W, H, 1), m, bins, rec, bg, stats)                      # ordered (default)
    b = ops.rasterize_forward_packed(tb, (W, H, 1), m, bins.clone(), rec, bg, stats)              # identity order
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    v = cu(rng.uniform(-1, 1, (H, W, 3)).astype(np.float32))
    g1 = ops.rasterize_backward(H, W, n, m, bins, conics, op, rec, cum, bg, a[1], a[2], v, tile_order=bins.tile_order)
    g2 = ops.rasterize_backward(H, W, n, m, bins, conics, op, rec, cum, bg, a[1], a[2], v)
    for x, y in zip(g1, g2):
        assert torch.equal(x, y)


def test_capacity_overflow_is_flagged_and_leaves_pack_and_blend_untouched():
    """Capacities smaller than the frame needs: stats[2] = 1 and neither the sort/pack nor the blend kernel touch
    their outputs; the operator redoes the frame with larger capacities and gives the same image."""
    n, W, H = 20000, 320, 200
    sc = _scene(n, W, H, 0.2, seed=77)
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    tb = ops.tile_bounds(W, H)
    colors = cu(np.random.default_rng(1).uniform(0, 1, (n, 3)).astype(np.float32))
    op = cu(sc["opacities"])
    bg = cu(np.zeros(3, np.float32))
    m, max_len, bins, cum, stats, rec, _, _ = _bucket_exact(xys, depths, radii, conics, colors, op, tb, cull=True)
    ref, _, _ = ops.rasterize_forward_packed(tb, (W, H, 1), m, bins, rec, bg, stats)
    for m_cap, len_cap in ((m - 1, max_len), (m, max_len - 1), (m // 2, 64)):
        b2, c2, st2, ws2 = ops.bucket_tile_ranges(xys, radii, conics, colors, op, tb, m_cap, len_cap)
        assert [int(v) for v in st2.tolist()] == [m, max_len, 1, 0]
        rec2 = torch.full((capi_records_bytes(m_cap),), 0xAB, dtype=torch.uint8, device=DEV)
        from opensplat_b200 import capi
        off = (-ws2.data_ptr()) % 256
        capi.check(capi.lib().gsb_bucket_sort_pack(n, m_cap, len_cap, capi.ptr(depths), capi.ptr(radii), capi.ptr(c2),
                                                   1, tb[0], tb[1], capi.ptr(b2), capi.ptr(st2), ws2.data_ptr() + off,
                                                   ws2.numel() - off, capi.ptr(rec2), None, None, capi.stream()))
        assert bool((rec2 == 0xAB).all())
        out = torch.full((H, W, 3), -7.0, device=DEV)
        fT, fI = torch.empty((H, W), device=DEV), torch.empty((H, W), dtype=torch.int32, device=DEV)
        capi.check(capi.lib().gsb_rasterize_forward_packed(H, W, tb[0], tb[1], m_cap, capi.ptr(b2), None, capi.ptr(st2),
                                                           capi.ptr(bg), capi.ptr(rec2), capi.ptr(out), capi.ptr(fT),
                                                           capi.ptr(fI), 0, capi.stream()))
        assert bool((out == -7.0).all())
    # operator level: plans start too small (fresh plan), the result must not depend on it
    ops._plans.clear()
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colors, op, H, W, bg)
    assert torch.equal(img, ref)
    ops._plans[torch.device(DEV).index].m_cap = 17     # force one more overflow + redo
    img2 = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colors, op, H, W, bg)
    assert torch.equal(img2, ref)


def capi_records_bytes(m):
    from opensplat_b200 import capi
    return capi.lib().gsb_raster_records_bytes(m)


def test_sort_stability_with_duplicate_keys():
    # many identical (tile, depth) keys: the permutation must be the stable one
    rng = np.random.default_rng(0)
    m = 100_003
    keys = (rng.integers(0, 37, m).astype(np.int64) << 32) | rng.integers(0, 5, m).astype(np.int64)
    ks, idx = ops.sort_intersects(cu(keys), 37)
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(npy(idx), order.astype(np.int32))
    assert np.array_equal(npy(ks), keys[order])


@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 100_000, 1_000_003])
def test_cumsum_sizes(n):
    rng = np.random.default_rng(n)
    a = rng.integers(0, 9, n).astype(np.int32)
    cum = ops.cumsum_tiles_hit(cu(a))
    assert np.array_equal(npy(cum), np.cumsum(a, dtype=np.int64).astype(np.int32))


# ---------------------------------------------------------------------------------- rasterization
def _raster_both(sc, colors, background, exp_mode=1):
    n, W, H = sc["means"].shape[0], sc["W"], sc["H"]
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    cum = ops.cumsum_tiles_hit(nth)
    m = int(cum[-1])
    tb = ops.tile_bounds(W, H)
    _, _, _, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, tb, return_index=True)
    bg = cu(np.asarray(background, np.float32))
    out, fT, fI, rec = ops.rasterize_forward(tb, (W, H, 1), gs, idx, bins, xys, conics, cu(colors),
                                             cu(sc["opacities"]), bg)
    o = orc.rasterize_forward(H, W, npy(gs), npy(bins), npy(xys), npy(conics), colors, sc["opacities"],
                              background, exp_mode=exp_mode)
    st = dict(n=n, m=m, tb=tb, gs=gs, bins=bins, idx=idx, xys=xys, conics=conics, cum=cum, bg=bg, rec=rec)
    return (out, fT, fI), o, st


@pytest.mark.parametrize("n,W,H,scale,opac,bg", [
    (3000, 256, 256, 0.35, (0.05, 0.35), [0, 0, 0]),
    (2000, 200, 120, 0.5, (0.3, 0.95), [0.6130, 0.0101, 0.3984]),   # ragged tiles + magenta background
    (6000, 128, 128, 0.6, (0.7, 0.99), [1, 1, 1]),                  # saturating pixels: early termination
])
def test_rasterize_forward_backward_vs_oracle(n, W, H, scale, opac, bg):
    sc = _scene(n, W, H, scale, opacity=opac, seed=n + W)
    rng = np.random.default_rng(1)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    (out, fT, fI), o, st = _raster_both(sc, colors, bg)
    # image: 1e-5 on all but isolated alpha-threshold flips (<= 1/255); kernel uses ex2.approx
    ok, stats = image_close(npy(out), o["out_img"], tol=1e-5, frac=1e-3)
    assert ok, stats
    assert np.abs(npy(fT) - o["final_Ts"]).max() <= 4.5e-3
    assert (npy(fI) != o["final_idx"]).mean() <= 1e-3            # identical except at threshold flips
    if opac[0] >= 0.7:
        assert (o["final_Ts"] < 1e-3).mean() > 0.2                 # the early-out path really ran
    # backward on the oracle's own final_Ts/final_idx (identical inputs to both sides)
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    fTo, fIo = cu(o["final_Ts"]), cu(o["final_idx"])
    v = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"], st["cum"], st["bg"], fTo, fIo, cu(wgt))
    ob = orc.rasterize_backward(H, W, npy(st["gs"]), npy(st["bins"]), npy(st["xys"]), npy(st["conics"]), colors,
                                sc["opacities"], bg, o["final_Ts"], o["final_idx"], wgt, exp_mode=1)
    tol = 2e-4 if opac[1] < 0.9 else 2e-3   # fp32 re-association; 1/(1-alpha) amplifies when alpha -> 0.99
    for a, b in zip(v, (ob["v_xy"], ob["v_conic"], ob["v_colors"], ob["v_opacity"])):
        assert rel_l2(npy(a), b) <= tol
    # deterministic: bit-identical on a second run (no atomics)
    v2 = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"], st["cum"], st["bg"], fTo, fIo, cu(wgt))
    for a, b in zip(v, v2):
        assert torch.equal(a, b)


def test_backward_unblended_tiles_do_not_touch_other_tiles_rows():
    """ADVICE r1 (high): a non-empty tile in which no pixel blends anything (only alpha < 1/255 candidates or
    bbox-corner overlaps) has final_idx == 0 everywhere; the backward kernel must then zero only ITS OWN rows, not
    sorted indices 1..range.x-1 that belong to earlier tiles.  Sparse, mostly sub-threshold scene on a 1080p image
    (8160 tiles > resident warps, so earlier tiles have finished when a late one would overwrite their rows)."""
    n, W, H = 40_000, 1920, 1080
    sc = _scene(n, W, H, 0.08, opacity=(0.001, 0.0035), seed=123)         # all below 1/255 = 0.0039: never blend ...
    left = np.nonzero(sc["means"][:, 0] < 0)[0]
    sc["opacities"][left[::3]] = 0.6       # ... except a third of the left half: the right half's tiles blend nothing
    rng = np.random.default_rng(9)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    bg = [0.1, 0.2, 0.3]
    (out, fT, fI), o, st = _raster_both(sc, colors, bg)
    bins = npy(st["bins"])
    lens = bins[:, 1] - bins[:, 0]
    # tiles with a list starting at sorted index >= 2 in which NO pixel blended (the situation of the bug)
    tx, ty = st["tb"][0], st["tb"][1]
    blended_any = np.zeros(tx * ty, bool)
    fin = o["final_Ts"]
    for t in np.nonzero((lens > 0) & (bins[:, 0] >= 2))[0]:
        y0, x0 = (t // tx) * 16, (t % tx) * 16
        blended_any[t] = bool((fin[y0:y0 + 16, x0:x0 + 16] < 1.0).any())
    n_bug_tiles = int(((lens > 0) & (bins[:, 0] >= 2) & ~blended_any).sum())
    assert n_bug_tiles > 200, n_bug_tiles
    ok, stats = image_close(npy(out), o["out_img"], tol=1e-5, frac=1e-3)
    assert ok, stats
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    v = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"], st["cum"],
                               st["bg"], cu(o["final_Ts"]), cu(o["final_idx"]), cu(wgt))
    ob = orc.rasterize_backward(H, W, npy(st["gs"]), bins, npy(st["xys"]), npy(st["conics"]), colors,
                                sc["opacities"], bg, o["final_Ts"], o["final_idx"], wgt, exp_mode=1)
    for a, b in zip(v, (ob["v_xy"], ob["v_conic"], ob["v_colors"], ob["v_opacity"])):
        assert rel_l2(npy(a), b) <= 2e-4
    # and run to run (the overwrite was a race: it showed up as nondeterminism first)
    for _ in range(3):
        v2 = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"],
                                    st["cum"], st["bg"], cu(o["final_Ts"]), cu(o["final_idx"]), cu(wgt))
        for a, b in zip(v, v2):
            assert torch.equal(a, b)
    # the operator (culled fast path) gives the same gradients as the generic path
    colt, opt = cu(colors).requires_grad_(), cu(sc["opacities"]).requires_grad_()
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colt, opt, H, W, st["bg"])
    assert torch.equal(img, out)
    (img * cu(wgt)).sum().backward()
    assert rel_l2(npy(colt.grad), ob["v_colors"]) <= 1e-3 and rel_l2(npy(opt.grad), ob["v_opacity"]) <= 1e-3


def test_rasterize_v_output_alpha_term():
    n, W, H = 1500, 96, 96
    sc = _scene(n, W, H, 0.5, seed=11)
    rng = np.random.default_rng(2)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    (out, fT, fI), o, st = _raster_both(sc, colors, [0.2, 0.3, 0.4])
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    wa = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    v = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"], st["cum"], st["bg"], cu(o["final_Ts"]),
                               cu(o["final_idx"]), cu(wgt), cu(wa))
    ob = orc.rasterize_backward(H, W, npy(st["gs"]), npy(st["bins"]), npy(st["xys"]), npy(st["conics"]), colors,
                                sc["opacities"], [0.2, 0.3, 0.4], o["final_Ts"], o["final_idx"], wgt, wa, exp_mode=1)
    for a, b in zip(v, (ob["v_xy"], ob["v_conic"], ob["v_colors"], ob["v_opacity"])):
        assert rel_l2(npy(a), b) <= 2e-4


def test_projection_backward_vs_oracle():
    n, W, H = 5000, 256, 192
    sc = _scene(n, W, H, 0.3, seed=5)
    rng = np.random.default_rng(3)
    sc["quats"] = (sc["quats"] * rng.uniform(0.5, 2, (n, 1))).astype(np.float32)  # raw quats (D11)
    cov3d, xys, depths, radii, conics, nth = _project_gpu(sc)
    v_xy = rng.standard_normal((n, 2)).astype(np.float32)
    v_depth = rng.standard_normal((n,)).astype(np.float32)
    v_conic = rng.standard_normal((n, 3)).astype(np.float32)
    g = ops.project_gaussians_backward(cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]),
                                       cu(sc["projmat"]), sc["fx"], sc["fy"], sc["cx"], sc["cy"], H, W, cov3d,
                                       radii, conics, cu(v_xy), cu(v_depth), cu(v_conic))
    o = orc.project_backward(sc["means"], sc["scales"], 1.0, sc["quats"], sc["viewmat"], sc["projmat"],
                             sc["fx"], sc["fy"], sc["cx"], sc["cy"], H, W, npy(radii), npy(conics), v_xy, v_depth,
                             v_conic)
    # same formulas, both without FMA contraction: 1e-6 relative
    assert rel_l2(npy(g[0]), o["v_mean3d"]) <= 1e-6
    assert rel_l2(npy(g[1]), o["v_scale"]) <= 1e-6
    assert rel_l2(npy(g[2]), o["v_quat"]) <= 1e-6


def test_projection_backward_vs_torch_autograd_of_forward():
    """fp32 torch restatement of OUR forward formula, differentiated by autograd (general P*V camera,
    glob_scale != 1): checks the hand VJP is the exact gradient of the forward map."""
    n, W, H = 2000, 320, 200
    sc = _scene(n, W, H, 0.3, seed=9)
    dev = DEV
    means = cu(sc["means"]).double().requires_grad_()
    scales = cu(sc["scales"]).double().requires_grad_()
    quats = (cu(sc["quats"]) * 1.7).double().requires_grad_()
    V = cu(sc["viewmat"]).double()
    a = 0.3
    V[:3, :3] = torch.tensor([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], device=dev)
    fx, fy, cx, cy, gsc = sc["fx"] * 0.9, sc["fy"] * 1.1, W / 2 + 3.0, H / 2 - 2.0, 1.3
    fovx, fovy = 2 * np.arctan(W / (2 * fx)), 2 * np.arctan(H / (2 * fy))
    zn, zf = 0.001, 1000.0
    t, r = zn * np.tan(0.5 * fovy), zn * np.tan(0.5 * fovx)
    Pm = torch.tensor([[zn / r, 0, 0, 0], [0, zn / t, 0, 0], [0, 0, (zf + zn) / (zf - zn), -zf * zn / (zf - zn)],
                       [0, 0, 1, 0]], device=dev, dtype=torch.float64)
    P = Pm @ V

    def fwd(means, scales, quats):
        tview = means @ V[:3, :3].T + V[:3, 3]
        qn = quats / quats.norm(dim=-1, keepdim=True)
        w, x, y, z = qn.unbind(-1)
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                         2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                         2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
        M = R * (gsc * scales)[:, None, :]
        cov3 = M @ M.transpose(1, 2)
        tanx, tany = 0.5 * W / fx, 0.5 * H / fy
        tz = tview[:, 2]
        ttx = tz * torch.clamp(tview[:, 0] / tz, -1.3 * tanx, 1.3 * tanx)
        tty = tz * torch.clamp(tview[:, 1] / tz, -1.3 * tany, 1.3 * tany)
        rz = 1 / tz
        zero = torch.zeros_like(rz)
        J = torch.stack([fx * rz, zero, -fx * ttx * rz * rz, zero, fy * rz, -fy * tty * rz * rz], -1).reshape(-1, 2, 3)
        T = J @ V[:3, :3]
        cov2 = T @ cov3 @ T.transpose(1, 2)
        cxx, cxy, cyy = cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3
        det = cxx * cyy - cxy * cxy
        conic = torch.stack([cyy / det, -cxy / det, cxx / det], -1)
        hom = means @ P[:, :3].T + P[:, 3]
        rw = 1 / (hom[:, 3] + 1e-6)
        xy = torch.stack([0.5 * W * hom[:, 0] * rw + cx - 0.5, 0.5 * H * hom[:, 1] * rw + cy - 0.5], -1)
        return xy, tz, conic

    xy, tz, conic = fwd(means, scales, quats)
    rng = np.random.default_rng(4)
    v_xy, v_d, v_c = (cu(rng.standard_normal(s).astype(np.float32)) for s in [(n, 2), (n,), (n, 3)])
    (xy * v_xy.double()).sum().add((tz * v_d.double()).sum()).add((conic * v_c.double()).sum()).backward()
    tb = ops.tile_bounds(W, H)
    f32 = lambda t: t.detach().float().contiguous()
    cov3d, xys, depths, radii, conics, nth = ops.project_gaussians_forward(
        f32(means), f32(scales), gsc, f32(quats), f32(V), f32(P), fx, fy, cx, cy, H, W, tb)
    vis = npy(radii) > 0
    assert vis.mean() > 0.5
    assert np.abs(npy(xys)[vis] - npy(xy)[vis]).max() <= 2e-3 and rel_l2(npy(conics)[vis], npy(conic)[vis]) <= 1e-5
    g = ops.project_gaussians_backward(f32(means), f32(scales), gsc, f32(quats), f32(V), f32(P), fx, fy, cx, cy, H,
                                       W, cov3d, radii, conics, v_xy, v_d, v_c)
    assert rel_l2(npy(g[0])[vis], npy(means.grad)[vis]) <= 2e-4
    assert rel_l2(npy(g[1])[vis], npy(scales.grad)[vis]) <= 2e-4
    assert rel_l2(npy(g[2])[vis], npy(quats.grad)[vis]) <= 2e-4
    assert np.all(npy(g[0])[~vis] == 0) and np.all(npy(g[2])[~vis] == 0)


# ------------------------------------------------------- operators end to end vs the reference itself
@pytest.mark.parametrize("name,gtol,itol", [("chain_tight_100x72", 2e-3, 5e-5), ("chain_bg_quat_128x96", 2e-3, 5e-5),
                                            ("chain_opaque_96x96", 2e-2, 5e-5)])
def test_operator_chain_vs_reference_golden(name, gtol, itol):
    """ProjectGaussians -> RasterizeGaussians (autograd operators) against the reference CPU back end's
    outputs for the same inputs.  Full-chain tolerances (SURVEY 8c table, row 4): image 5e-5 away from
    alpha-threshold flips; gradients rel-L2 2e-3 (projection round-off D3 feeds the rasterizer; opaque
    case additionally has the D5 fringe)."""
    g = load_golden(name)
    fx, fy, cx, cy = [float(v) for v in g["intrins"]]
    H, W = [int(v) for v in g["hw"]]
    means, scales, quats = (cu(g[k]).requires_grad_() for k in ("means", "scales", "quats"))
    colors, opac = cu(g["colors"]).requires_grad_(), cu(g["opacities"]).requires_grad_()
    tb = ops.tile_bounds(W, H)
    xys, depths, radii, conics, nth, cov3d = ops.ProjectGaussians.apply(
        means, scales, 1.0, quats, cu(g["viewmat"]), cu(g["projmat"]), fx, fy, cx, cy, H, W, tb)
    xys.retain_grad()  # model.cpp:171 relies on this
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colors, opac, H, W, cu(g["background"]))
    ok, stats = image_close(npy(img), g["ref_img"], tol=itol, frac=1e-3 if gtol < 1e-2 else 1e-2)
    assert ok, stats
    (img * cu(g["wgt"])).sum().backward()
    assert rel_l2(npy(xys.grad), g["ref_v_xy"]) <= gtol
    assert rel_l2(npy(colors.grad), g["ref_v_colors"]) <= gtol
    assert rel_l2(npy(opac.grad), g["ref_v_opacity"]) <= gtol
    assert rel_l2(npy(means.grad), g["ref_v_means"]) <= gtol
    assert rel_l2(npy(scales.grad), g["ref_v_scales"]) <= gtol
    assert rel_l2(npy(quats.grad), g["ref_v_quats"]) <= gtol


def test_sh_operator_autograd():
    g = load_golden("sh_deg3")
    co = cu(g["coeffs"]).requires_grad_()
    col = ops.SphericalHarmonics.apply(2, cu(g["viewdirs"]), co)
    (col * cu(g["wgt"])).sum().backward()
    assert np.abs(npy(col) - g["ref_colors_d2"]).max() <= 2e-5
    assert np.abs(npy(co.grad) - g["ref_v_coeffs_d2"]).max() <= 2e-6


# ------------------------------------------------------------------------------------- edge cases
def test_empty_and_fully_culled():
    W, H = 70, 50
    tb = ops.tile_bounds(W, H)
    sc = _scene(64, W, H, 0.3, seed=1)
    sc["means"][:, 2] = -20.0   # everything behind the camera -> M == 0
    cov3d, xys, depths, radii, conics, nth = _project_gpu(sc)
    assert int(radii.abs().sum()) == 0 and int(nth.sum()) == 0
    colors = cu(np.full((64, 3), 0.5, np.float32)).requires_grad_()
    opac = cu(sc["opacities"]).requires_grad_()
    bg = cu(np.array([0.1, 0.2, 0.3], np.float32))
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colors, opac, H, W, bg)
    assert torch.allclose(img, bg.expand(H, W, 3))
    img.sum().backward()
    assert float(colors.grad.abs().sum()) == 0.0
    # n == 0 through the C ABI
    z = torch.zeros((0, 3), device=DEV)
    out = ops.project_gaussians_forward(z, z, 1.0, torch.zeros((0, 4), device=DEV), cu(sc["viewmat"]),
                                        cu(sc["projmat"]), 10., 10., 5., 5., H, W, tb)
    assert out[1].shape == (0, 2)


def test_one_gaussian_covering_every_tile():
    W, H = 160, 96
    sc = _scene(3, W, H, 30.0, opacity=(0.5, 0.6), seed=2)
    sc["means"][:, :2] = 0.0
    colors = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    (out, fT, fI), o, st = _raster_both(sc, colors, [0, 0, 0])
    assert st["m"] == 3 * st["tb"][0] * st["tb"][1]
    ok, stats = image_close(npy(out), o["out_img"], tol=1e-5)
    assert ok, stats


@pytest.mark.parametrize("n,expect_path", [(7000, "radix"), (24000, "generic")])
def test_very_long_tile_lists_take_radix_and_generic_paths(n, expect_path):
    """All Gaussians piled on one spot: a tile list longer than the bitonic (4096) / in-smem (16384) limits.
    The operator must still match the oracle (CTA radix sort, resp. the generic global radix sort fallback), and
    SplatPipeline, which takes the same path, must match the operator chain bit for bit."""
    from opensplat_b200 import capi
    from opensplat_b200.pipeline import SplatPipeline
    W, H = 64, 48
    sc = _scene(n, W, H, 0.5, opacity=(0.0045, 0.01), seed=n)
    # pile up around the centre of tile (2,1) (pixel 39.5, 23.5): every Gaussian lies inside that one tile, with a
    # footprint of a few pixels so that the operator's extent cull keeps (nearly) all of them
    sc["means"][:, 0] = 0.25 + sc["means"][:, 0] * 0.05
    sc["means"][:, 1] = sc["means"][:, 1] * 0.05
    rng = np.random.default_rng(1)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    tb = ops.tile_bounds(W, H)
    _, _, stats, _ = ops.bucket_tile_ranges(xys, radii, conics, cu(colors), cu(sc["opacities"]), tb, 0, 0)   # culled
    m, max_len = (int(v) for v in stats.tolist()[:2])
    cap = capi.lib().gsb_bucket_max_tile_len()
    assert (max_len > 4096 and max_len <= cap) if expect_path == "radix" else (max_len > cap), max_len
    colt, opt = cu(colors).requires_grad_(), cu(sc["opacities"]).requires_grad_()
    bg = cu(np.array([0.1, 0.2, 0.3], np.float32))
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, colt, opt, H, W, bg)
    o = _project_orc(sc)
    cum, _ = orc.cumsum(o["num_tiles_hit"])
    b = orc.bin_and_sort(o["xys"], o["depths"], o["radii"], cum, H, W)
    f = orc.rasterize_forward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], o["xys"], o["conics"], colors,
                              sc["opacities"], [0.1, 0.2, 0.3], exp_mode=1)
    ok, stats_ = image_close(npy(img), f["out_img"], tol=2e-5, frac=2e-3)
    assert ok, stats_
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    (img * cu(wgt)).sum().backward()
    r = orc.rasterize_backward(H, W, b["gaussian_ids_sorted"], b["tile_bins"], o["xys"], o["conics"], colors,
                               sc["opacities"], [0.1, 0.2, 0.3], f["final_Ts"], f["final_idx"], wgt, exp_mode=1)
    assert rel_l2(npy(colt.grad), r["v_colors"]) <= 1e-3 and rel_l2(npy(opt.grad), r["v_opacity"]) <= 1e-3
    # the same scene through SplatPipeline and through SphericalHarmonics -> ProjectGaussians -> RasterizeGaussians:
    # same inputs, same kernels, so the image and the gradients are bit-identical
    pipe = SplatPipeline(n, W, H, sh_degree=0)
    pipe.load_scene(sc)
    pipe.forward()
    pipe.backward()
    assert pipe._ordered == (expect_path == "radix")   # the generic fallback blends without the tile order
    coeffs, opac = cu(sc["coeffs"]).requires_grad_(), cu(sc["opacities"]).requires_grad_()
    rgbs = torch.clamp_min(ops.SphericalHarmonics.apply(0, cu(sc["viewdirs"]), coeffs) + 0.5, 0.0)
    xys, depths, radii, conics, nth, _ = ops.ProjectGaussians.apply(
        cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"],
        sc["fy"], sc["cx"], sc["cy"], H, W, tb)
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, rgbs, opac, H, W, torch.zeros(3, device=DEV))
    assert torch.equal(pipe.out_img, img)
    img.backward(pipe.v_img)
    assert torch.equal(opac.grad, pipe.g["opacities"]) and torch.equal(coeffs.grad, pipe.g["coeffs"])


def test_long_tile_lists_at_realistic_tile_counts():
    """Tile lists between 4096 and 16384 entries on EVERY one of 256 tiles (not one pile-up tile): the distribution
    sort with its largest shared-memory footprint, and -- with depth ties forced on half of the Gaussians -- the
    comparison-sort fallback (CTA radix above 4096) at a realistic tile count.  Fast path (no cull) == generic path bit
    for bit; operator image / gradients vs the oracle."""
    n, W, H = 500_000, 256, 256
    sc = _scene(n, W, H, 0.25, opacity=(0.002, 0.02), seed=4242)
    left = sc["means"][:, 0] < 0          # left half of the image: heavy depth ties -> clustered bins -> fallback sorts;
    sc["means"][left, 2] = np.round(sc["means"][left, 2] * 4) / 4   # right half: distinct depths -> distribution sort
    rng = np.random.default_rng(3)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    _, xys, depths, radii, conics, nth = _project_gpu(sc)
    cum = ops.cumsum_tiles_hit(nth)
    tb = ops.tile_bounds(W, H)
    colt, opt = cu(colors), cu(sc["opacities"])
    m, max_len, bins_b, cum_b, stats, rec_b, idx_b, gs_b = _bucket_exact(xys, depths, radii, conics, colt, opt, tb,
                                                                        cull=False)
    lens = npy(bins_b)[:, 1] - npy(bins_b)[:, 0]
    assert 4096 < max_len <= 16384 and (lens > 4096).mean() > 0.5, (max_len, float((lens > 4096).mean()))
    isect, gids, ks, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, tb, return_index=True)
    assert torch.equal(bins_b, bins) and torch.equal(idx_b, idx) and torch.equal(gs_b, gs)
    bg = cu(np.array([0.1, 0.2, 0.3], np.float32))
    out, fT, fI, rec = ops.rasterize_forward(tb, (W, H, 1), gs, idx, bins, xys, conics, colt, opt, bg)
    assert torch.equal(rec_b[: m * 48], rec[: m * 48])
    del isect, gids, ks, idx, rec_b, idx_b, gs_b
    cg, og = colt.clone().requires_grad_(), opt.clone().requires_grad_()
    img = ops.RasterizeGaussians.apply(xys, depths, radii, conics, nth, cg, og, H, W, bg)
    assert torch.equal(img, out)
    o = orc.rasterize_forward(H, W, npy(gs), npy(bins), npy(xys), npy(conics), colors, sc["opacities"], [0.1, 0.2, 0.3],
                              exp_mode=1)
    ok, st = image_close(npy(img), o["out_img"], tol=2e-5, frac=2e-3)
    assert ok, st
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    (img * cu(wgt)).sum().backward()
    r = orc.rasterize_backward(H, W, npy(gs), npy(bins), npy(xys), npy(conics), colors, sc["opacities"], [0.1, 0.2, 0.3],
                               o["final_Ts"], o["final_idx"], wgt, exp_mode=1)
    assert rel_l2(npy(cg.grad), r["v_colors"]) <= 1e-3 and rel_l2(npy(og.grad), r["v_opacity"]) <= 1e-3


def test_dense_overlap_parity_c5_like():
    """Config C5 in miniature: ~200 candidate splats per pixel, saturating tiles, long lists (bitonic 2048-4096)."""
    n, W, H = 100_000, 320, 192
    sc = _scene(n, W, H, 0.16, opacity=(0.05, 0.95), seed=55)
    rng = np.random.default_rng(2)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    (out, fT, fI), o, st = _raster_both(sc, colors, [0, 0, 0])
    assert st["m"] / (W * H / 256) > 1000          # > 1000 records per tile on average
    ok, stats = image_close(npy(out), o["out_img"], tol=2e-5, frac=2e-3)
    assert ok, stats
    wgt = rng.uniform(-1, 1, (H, W, 3)).astype(np.float32)
    v = ops.rasterize_backward(H, W, n, st["m"], st["bins"], st["conics"], cu(sc["opacities"]), st["rec"], st["cum"],
                               st["bg"], cu(o["final_Ts"]), cu(o["final_idx"]), cu(wgt))
    ob = orc.rasterize_backward(H, W, npy(st["gs"]), npy(st["bins"]), npy(st["xys"]), npy(st["conics"]), colors,
                                sc["opacities"], [0, 0, 0], o["final_Ts"], o["final_idx"], wgt, exp_mode=1)
    for a, b in zip(v, (ob["v_xy"], ob["v_conic"], ob["v_colors"], ob["v_opacity"])):
        assert rel_l2(npy(a), b) <= 2e-3


# ---------------------------------------------------------------- full-size properties (config C2)
@pytest.mark.parametrize("n,W,H,scale", [(1_000_000, 1920, 1080, 0.02)])
def test_full_size_properties_and_oracle(n, W, H, scale):
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=(0.05, 0.95), seed=0)
    tb = ops.tile_bounds(W, H)
    T = tb[0] * tb[1]
    coeffs, vd = cu(sc["coeffs"]), cu(sc["viewdirs"])
    col = ops.compute_sh_forward(3, 3, vd, coeffs)
    # SH is linear in the coefficients
    col2 = ops.compute_sh_forward(3, 3, vd, coeffs * 2)
    assert torch.equal(col2, col * 2)
    rgbs = torch.clamp_min(col + 0.5, 0.0)
    cov3d, xys, depths, radii, conics, nth = _project_gpu(sc)
    o = _project_orc(sc)
    assert np.array_equal(npy(radii), o["radii"]) and np.array_equal(npy(nth), o["num_tiles_hit"])
    cum = ops.cumsum_tiles_hit(nth)
    m = int(cum[-1])
    assert m == int(o["num_tiles_hit"].astype(np.int64).sum())
    isect, gids, ks, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, tb, return_index=True)
    ksn, idxn, binsn = npy(ks), npy(idx), npy(bins)
    assert np.all(np.diff(ksn) >= 0)                                   # sortedness
    assert np.array_equal(np.sort(idxn), np.arange(m, dtype=np.int32))  # a permutation
    assert np.array_equal(npy(isect)[idxn], ksn)                        # ... of the input keys
    nz = binsn[:, 1] > binsn[:, 0]
    assert (binsn[nz, 1] - binsn[nz, 0]).sum() == m                     # bins partition [0, M)
    tiles_of_keys = (ksn >> 32).astype(np.int64)
    assert np.array_equal(np.bincount(tiles_of_keys, minlength=T), (binsn[:, 1] - binsn[:, 0]))
    ob = orc.bin_and_sort(o["xys"], o["depths"], o["radii"], npy(cum), H, W)
    assert np.array_equal(ksn, ob["isect_ids_sorted"]) and np.array_equal(npy(gs), ob["gaussian_ids_sorted"])
    assert np.array_equal(binsn, ob["tile_bins"])
    bg = cu(np.zeros(3, np.float32))
    opac = cu(sc["opacities"])
    out, fT, fI, rec = ops.rasterize_forward(tb, (W, H, 1), gs, idx, bins, xys, conics, rgbs, opac, bg)
    assert bool(torch.isfinite(out).all()) and float(out.min()) >= 0.0
    orf = orc.rasterize_forward(H, W, npy(gs), binsn, npy(xys), npy(conics), npy(rgbs), sc["opacities"], [0, 0, 0],
                                exp_mode=1)
    ok, stats = image_close(npy(out), orf["out_img"], tol=2e-5, frac=1e-3)
    assert ok, stats
    rng = np.random.default_rng(0)
    wgt = cu(rng.uniform(-1, 1, (H, W, 3)).astype(np.float32))
    v = ops.rasterize_backward(H, W, n, m, bins, conics, opac, rec, cum, bg, fT, fI, wgt)
    v2 = ops.rasterize_backward(H, W, n, m, bins, conics, opac, rec, cum, bg, fT, fI, wgt * 2)
    for a, b in zip(v, v2):
        assert torch.equal(a * 2, b)                                    # backward is linear in v_output
    orb = orc.rasterize_backward(H, W, npy(gs), binsn, npy(xys), npy(conics), npy(rgbs), sc["opacities"], [0, 0, 0],
                                 npy(fT), npy(fI), npy(wgt), exp_mode=1)
    for a, b in zip(v, (orb["v_xy"], orb["v_conic"], orb["v_colors"], orb["v_opacity"])):
        assert rel_l2(npy(a), b) <= 1e-3


# ------------------------------------------------------------------------ training loss (SURVEY 8f row 2)
def test_main_loss_vs_reference_golden_and_oracle():
    g = load_golden("loss_45x70")
    rend = cu(g["rendered"]).requires_grad_()
    loss = ops.MainLoss.apply(rend, cu(g["gt"]), float(g["ssim_weight"]))
    loss.backward()
    assert abs(float(loss) - float(g["ref_loss"])) <= 2e-6                       # vs the reference itself
    assert rel_l2(npy(rend.grad), g["ref_v_rendered"]) <= 2e-5
    o = orc.main_loss(g["rendered"], g["gt"], float(g["ssim_weight"]))
    assert abs(float(loss) - o["loss"]) <= 2e-6 and rel_l2(npy(rend.grad), o["v_rendered"]) <= 2e-5


@pytest.mark.parametrize("H,W,w", [(16, 16, 0.2), (33, 50, 0.5), (270, 480, 0.2), (5, 7, 1.0)])
def test_main_loss_ragged_sizes_vs_oracle(H, W, w):
    rng = np.random.default_rng(H * W)
    gt = rng.uniform(0, 1, (H, W, 3)).astype(np.float32)
    rend = np.clip(gt + 0.2 * rng.standard_normal((H, W, 3)), 0, 1).astype(np.float32)
    r = cu(rend).requires_grad_()
    loss = ops.MainLoss.apply(r, cu(gt), w)
    (3.0 * loss).backward()
    o = orc.main_loss(rend, gt, w)
    assert abs(float(loss) - o["loss"]) <= 5e-6
    assert rel_l2(npy(r.grad), 3.0 * o["v_rendered"]) <= 5e-5


def test_fused_adam_matches_torch_adam():
    from opensplat_b200 import capi
    torch.manual_seed(0)
    n = 1_000_003
    p0 = torch.randn(n, device=DEV)
    p_ref = p0.clone().requires_grad_()
    opt = torch.optim.Adam([p_ref], lr=1e-2, foreach=False)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    L = capi.lib()
    for t in range(1, 6):
        g = torch.randn(n, device=DEV) * (0.1 * t)
        p_ref.grad = g.clone()
        opt.step()
        capi.check(L.gsb_adam_step(n, capi.ptr(p), capi.ptr(g), capi.ptr(m), capi.ptr(v), 1e-2, 0.9, 0.999, 1e-8,
                                   1 - 0.9 ** t, 1 - 0.999 ** t, capi.stream()))
    assert float((p - p_ref.detach()).abs().max()) <= 2e-6


def test_mse_loss_grad_matches_torch():
    from opensplat_b200 import capi
    H, W = 123, 77
    img = torch.rand(H, W, 3, device=DEV).requires_grad_()
    tgt = torch.rand(H, W, 3, device=DEV)
    ref = torch.nn.functional.mse_loss(img, tgt)
    ref.backward()
    v = torch.empty_like(tgt)
    loss = torch.full((1,), 7.0, device=DEV)   # the call must overwrite, not accumulate onto stale values
    cnt = H * W * 3
    capi.check(capi.lib().gsb_mse_loss_grad(cnt, capi.ptr(img.detach()), capi.ptr(tgt), capi.ptr(v), capi.ptr(loss),
                                            1.0 / cnt, capi.stream()))
    assert abs(float(loss) - float(ref)) <= 1e-6 and float((v - img.grad).abs().max()) <= 1e-9


def test_fused_activations_match_torch_autograd():
    """exp / normalize / sigmoid / view directions of Model::forward (model.cpp:148-150,176-177,200)."""
    torch.manual_seed(1)
    n = 50_001
    means = torch.randn(n, 3, device=DEV)
    ls, rq, ol = (torch.randn(n, k, device=DEV).requires_grad_() for k in (3, 4, 1))
    cam = torch.tensor([0.3, -0.2, -8.0], device=DEV)
    s_ref, q_ref, o_ref = torch.exp(ls), rq / rq.norm(2, dim=-1, keepdim=True), torch.sigmoid(ol)
    vd_ref = (means - cam) / (means - cam).norm(2, dim=-1, keepdim=True)
    w = [torch.randn_like(t) for t in (s_ref, q_ref, o_ref)]
    (s_ref * w[0]).sum().add((q_ref * w[1]).sum()).add((o_ref * w[2]).sum()).backward()
    ref_grads = [t.grad.clone() for t in (ls, rq, ol)]
    for t in (ls, rq, ol):
        t.grad = None
    s, q, o, vd = ops.ActivateGaussians.apply(means, ls, rq, ol, cam)
    (s * w[0]).sum().add((q * w[1]).sum()).add((o * w[2]).sum()).backward()
    for a, b in ((s, s_ref), (q, q_ref), (o, o_ref), (vd, vd_ref)):
        assert float((a - b).abs().max()) <= 2e-6 * max(1.0, float(b.abs().max()))
    for t, gref in zip((ls, rq, ol), ref_grads):
        assert rel_l2(npy(t.grad), npy(gref)) <= 2e-6


def test_densify_stats_update_matches_reference_logic():
    """Model::afterTrain model.cpp:317-337 restated with the same torch ops the reference uses."""
    from opensplat_b200 import capi
    torch.manual_seed(2)
    n, H, W = 20_000, 300, 480
    v_xy = torch.randn(n, 2, device=DEV)
    radii = torch.randint(-1, 40, (n,), device=DEV, dtype=torch.int32)
    gn, vc, ms = torch.rand(n, device=DEV), torch.rand(n, device=DEV).round(), torch.rand(n, device=DEV) * 0.05
    gn_r, vc_r, ms_r = gn.clone(), vc.clone(), ms.clone()
    vis = (radii > 0).flatten()
    grads = torch.linalg.vector_norm(v_xy, 2, dim=-1)
    vc_r[vis] = vc_r[vis] + 1
    gn_r[vis] = grads[vis] + gn_r[vis]
    ms_r[vis] = torch.maximum(ms_r[vis], radii[vis] / float(max(H, W)))
    capi.check(capi.lib().gsb_densify_stats_update(n, capi.ptr(v_xy), capi.ptr(radii), H, W, capi.ptr(gn), capi.ptr(vc),
                                                   capi.ptr(ms), capi.stream()))
    assert torch.allclose(gn, gn_r, rtol=1e-6, atol=1e-7) and torch.equal(vc, vc_r) and torch.allclose(ms, ms_r, rtol=1e-6)
