"""The kernels of csrc/densify.cu and csrc/export.cu against the float64 restatement of tests/scene_edit_f64.py,
through the C ABI and opensplat_b200.densify / opensplat_b200.export.

Classify: every certified decision must match the float64 one exactly, and everything downstream (src_map,
split_rank, counts) must be bit-exact against the numpy compaction; uncertified parents (within the bound of a
threshold) take the decision the kernel's own outputs show, and are counted.  means_scales, the keepCrs scales and
the .splat floats must lie within C x the bound of their kernel's fp32 operation tree; copies, gathers and the PLY
rows are bit-exact; .splat bytes are exact wherever certified.  Sizes reach the scan's second chunk of 1024 blocks
(n > 1 048 576) and the grid-stride loops of the gather and the PLY pack (more than 2^28 floats).  The worst
err/bound per quantity and the uncertified count per case are printed (-s)."""
import ctypes as Ct

import numpy as np
import pytest
import torch

import scene_edit_f64 as sf
from test_scene_edit_f64_reference import default_cfg, pattern_decisions
from util import scene_edit_inputs
from oracle import scene_edit as se

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = 12345.678
WORST = {}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def check_within(tag, got, x):
    got = np.asarray(got, np.float64).reshape(x.v.shape)
    err = np.abs(got - x.v)
    bound = sf.C * x.b
    ok = (err <= bound) | (got == x.v)
    if x.v.size:
        r = float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0))))
        WORST[tag] = max(WORST.get(tag, 0.0), r)
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        pytest.fail(f"{tag}{list(i)}: kernel {got[i]!r} reference {x.v[i]!r} bound {bound[i]:.3e}")


def report(tag, **kw):
    print(f"\n[{tag}] " + " ".join(f"{k}={v}" for k, v in kw.items()) +
          " worst err/bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


def run_classify(scales, opac, gn, vc, m2, max_dim, cfg, cs, ch, cc):
    from opensplat_b200 import densify
    n = len(scales)
    src, rank, counts = densify.classify(cu(scales), cu(opac), cu(gn), cu(vc), None if m2 is None else cu(m2),
                                         max_dim, cfg, cs, ch, cc)
    cnt = counts.cpu().numpy()
    return src[:int(cnt[4])].cpu().numpy(), rank[:n].cpu().numpy(), cnt


def expect_classify(got, d, n, tag):
    """Certified decisions from `d`, uncertified ones read back from the kernel; then bit-exact downstream."""
    src, rank, cnt = got
    k = sf.decisions_of(src, rank, n)
    c = d["cert"]
    for name in ("split", "keep_self", "keep_split", "keep_dup"):
        bad = np.nonzero(c & (k[name] != d[name]))[0]
        assert len(bad) == 0, f"{tag}: {name} differs at certified parent {bad[0]} ({len(bad)} parents)"
    dd = {name: np.where(c, d[name], k[name]) for name in ("split", "keep_self", "keep_split", "keep_dup")}
    dd["dup"] = d["dup"]
    w_src, w_rank, w_cnt = sf.compact(**dd)
    assert np.array_equal(src, w_src), tag
    assert np.array_equal(rank, w_rank), tag
    assert np.array_equal(cnt[:5], w_cnt[:5]) and cnt[6] == 0 and cnt[7] == 0, (tag, cnt, w_cnt)
    n_unc_dup = int((~c).sum())
    dups_cert = int((d["dup"] & c).sum())
    assert dups_cert <= cnt[5] <= dups_cert + n_unc_dup, (tag, cnt[5], dups_cert)
    if n_unc_dup == 0:
        assert cnt[5] == w_cnt[5]
    return int((~c).sum())


# ---- classify -----------------------------------------------------------------------------------------------------
def truth_table(edges):
    """The product of every input class.  edges=False: default thresholds, values far from them.  edges=True:
    thresholds equal to exactly computed quantities (expf(0) = 1, sigmoid(0) = 1/2, gn 512 with vc = 1 and max_dim
    1024, max2DSize equal to both screen thresholds)."""
    f = np.float32
    if edges:
        cfg = default_cfg(densify_size_thresh=1.0, cull_scale_thresh=1.0, cull_alpha_thresh=0.5, size_fac=1.0)
        s_cls = [0.0, -1.0, 1.0]                           # mx = 1 (equal), below, above; child = parent's
        o_cls = [0.0, -4.0, 3.0]                           # sigmoid == alpha threshold, below, above
    else:
        cfg = default_cfg()
        s_cls = [np.log(0.003), np.log(0.05), np.log(0.7), np.log(1.5)]   # small, split, huge self, huge child too
        o_cls = [-5.0, 3.0]
    t = sf.cfg32(cfg)
    g0 = f(t["densify_grad_thresh"]) / f(512)
    g_cls = [(g0, 1.0), (g0 * f(4), 1.0), (g0 / f(4), 1.0), (0.0, 0.0), (g0, 0.0)]   # equal, high, low, 0/0, x/0
    ss, cs = f(t["split_screen_size"]), f(t["cull_screen_size"])
    m_cls = [0.0, ss / f(2), ss, (ss + cs) / f(2), cs, cs * f(2)]
    G, S, O, M = np.meshgrid(np.arange(len(g_cls)), np.arange(len(s_cls)), np.arange(len(o_cls)),
                             np.arange(len(m_cls)), indexing="ij")
    G, S, O, M = (a.reshape(-1) for a in (G, S, O, M))
    gn = np.array([g_cls[i][0] for i in G], f)
    vc = np.array([g_cls[i][1] for i in G], f)
    sc = np.repeat(np.array(s_cls, f)[S][:, None], 3, 1)
    sc[::2, 1] -= f(0.5)                                   # the max is not always the first component
    return sc, np.array(o_cls, f)[O][:, None], gn, vc, np.array(m_cls, f)[M], cfg


@pytest.mark.parametrize("edges", [False, True])
def test_classify_truth_table(edges):
    sc, o, gn, vc, m2, cfg = truth_table(edges)
    n = len(gn)
    seen = dict.fromkeys(("split", "dup", "keep_self", "keep_split", "keep_dup"), 0)
    for flags in [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]:
        for m2d in (m2, None):
            d = sf.classify(sc, o, gn, vc, m2d, 1024, cfg, *flags)
            assert d["cert"].all(), (flags, np.nonzero(~d["cert"])[0][:5])
            expect_classify(run_classify(sc, o, gn, vc, m2d, 1024, cfg, *flags), d, n, f"{edges} {flags}")
            for k in seen:
                seen[k] += int(d[k].sum())
    assert all(0 < v < 16 * n for v in seen.values()), seen      # every outcome taken, none always


def pattern_inputs(n, seed):
    """Inputs whose decisions are far from every threshold, with per-block probabilities so that whole blocks are
    kept, split, duplicated or culled, and every mix in between."""
    f = np.float32
    rng = np.random.default_rng(seed)
    nb = -(-n // 1024)
    pb = rng.uniform(0, 1, (nb, 4))
    pb[rng.integers(0, nb, max(nb // 8, 1)), :] = 0.0
    pb[rng.integers(0, nb, max(nb // 8, 1)), :] = 1.0
    pb = pb[np.arange(n) // 1024]
    u = rng.uniform(0, 1, (n, 4))
    gn = np.where(u[:, 0] < pb[:, 0], f(1e-3), f(1e-8)).astype(f)
    scale = np.where(u[:, 1] < pb[:, 1], np.where(u[:, 1] < pb[:, 1] / 4, np.log(0.9), np.log(0.05)), np.log(0.003))
    sc = (scale[:, None] - rng.choice(np.array([0.0, 0.25]), (n, 3)) * np.array([0.0, 1.0, 1.0])).astype(f)
    o = np.where(u[:, 2] < pb[:, 2], f(3.0), f(-5.0)).astype(f)[:, None]
    m2 = np.where(u[:, 3] < pb[:, 3], rng.choice(np.array([0.1, 0.2], f), n), f(0.01)).astype(f)
    return sc, o, gn, np.ones(n, f), m2


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 300_000, 1_048_576, 1_048_577, 3_000_000])
def test_classify_block_and_chunk_boundaries(n):
    """1 048 577 is the first size whose scan of the per-block counts runs a second chunk of 1024 blocks."""
    sc, o, gn, vc, m2 = pattern_inputs(n, n)
    if n > 1_048_576:         # the second chunk holds a kept split parent
        sc[1_048_576], o[1_048_576], gn[1_048_576] = np.log(0.05), 3.0, 1e-3
    cfg = default_cfg()
    for flags in [(1, 1, 1), (0, 1, 0)]:
        d = sf.classify(sc, o, gn, vc, m2, 640, cfg, *flags)
        assert d["cert"].all()
        got = run_classify(sc, o, gn, vc, m2, 640, cfg, *flags)
        assert expect_classify(got, d, n, f"n={n} {flags}") == 0
        assert got[2][5] == int(d["dup"].sum())
    if n > 1_048_576:
        assert d["keep_split"][1_048_576]


@pytest.mark.parametrize("chk_screen,chk_huge", [(True, True), (False, True), (True, False), (False, False)])
def test_classify_at_scale_certified(chk_screen, chk_huge):
    """scene_edit_inputs at 300 000 Gaussians, statistics from three views: no parent is exempt from the checks."""
    n, H, W = 300_000, 720, 1280
    p, _, _, draws = scene_edit_inputs(n, 4, 77 + 2 * chk_screen + chk_huge, max(H, W))
    stats = None
    for v_xy, radii in draws:
        stats = se.densify_stats(stats, v_xy * (640.0 / 1280.0), radii * 2, H, W)
    gn, vc, m2 = (s.numpy() for s in stats)
    cfg = default_cfg()
    d = sf.classify(p["scales"], p["opacities"], gn, vc, m2, max(H, W), cfg, chk_screen, chk_huge, chk_screen)
    got = run_classify(p["scales"], p["opacities"], gn, vc, m2, max(H, W), cfg, chk_screen, chk_huge, chk_screen)
    unc = expect_classify(got, d, n, f"{chk_screen} {chk_huge}")
    print(f"\n[classify at scale screen={chk_screen} huge={chk_huge}] uncertified parents {unc} of {n}, "
          f"new_n {got[2][4]}, splits {got[2][0]}, dups {got[2][5]}")
    assert unc <= 10


# ---- means_scales -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mixed", "no_splits"])
def test_means_scales_within_bound(case):
    from opensplat_b200 import densify
    f = np.float32
    rng = np.random.default_rng(11)
    n = 200_000
    dec = pattern_decisions(n, 12)
    if case == "no_splits":
        dec["split"][:] = False
        dec["keep_split"][:] = False
        dec["keep_self"] |= ~dec["dup"] & (rng.uniform(0, 1, n) < 0.5)
    src, rank, cnt = sf.compact(**dec)
    p = scene_edit_inputs(n, 1, 13)[0]
    quats = (p["quats"] * (f(10.0) ** rng.uniform(-3, 3, (n, 1)))).astype(f)     # far from unit norm
    samples = rng.standard_normal((max(2 * int(cnt[0]), 1), 3)).astype(f)
    new_n, ns_ = int(cnt[4]), int(cnt[0])
    nm, ns = densify.means_scales(cu(src), cu(rank), new_n, ns_, cu(samples), cu(p["means"]), cu(p["scales"]),
                                  cu(quats), 1.6)
    wm, ws = sf.means_scales(src, rank, ns_, samples, p["means"], p["scales"], quats, 1.6)
    check_within("means", nm.cpu().numpy(), wm)
    check_within("scales", ns.cpu().numpy(), ws)
    kinds = src.view(np.uint32) >> 30
    copy = (kinds == 0) | (kinds == 3)
    assert np.array_equal(nm.cpu().numpy()[copy], wm.v[copy].astype(f))
    report(f"means_scales {case}", new_n=new_n, n_splits=ns_)


# ---- gather_rows --------------------------------------------------------------------------------------------------
def gather_guarded(src_map_dev, new_n, src_dev, zero_children, extra=64):
    rf = src_dev.numel() // src_dev.shape[0]
    from opensplat_b200 import capi
    dst = torch.full(((new_n + extra) * rf,), SENT, device=DEV)
    capi.check(capi.lib().gsb_densify_gather_rows(new_n, rf, capi.ptr(src_map_dev), capi.ptr(src_dev),
                                                  capi.ptr(dst), int(zero_children), capi.stream()))
    assert bool((dst[new_n * rf:] == SENT).all()), "gather wrote past new_n"
    return dst[:new_n * rf].view(new_n, rf)


def gather_expected(src_map_dev, src_dev, zero_children):
    e = src_map_dev.long() & 0xFFFFFFFF
    par, child = e & ((1 << 30) - 1), (e >> 30) != 0
    want = torch.index_select(src_dev.reshape(src_dev.shape[0], -1), 0, par)
    if zero_children:
        want[child] = 0
    return want


@pytest.mark.parametrize("rf", [1, 3, 4, 9, 24, 45, 48, 72])
@pytest.mark.parametrize("zero_children", [False, True])
def test_gather_rows_exact(rf, zero_children):
    n = 70_001
    src_map, _, cnt = sf.compact(**pattern_decisions(n, rf))
    new_n = int(cnt[4])
    src = torch.randn(n, rf, device=DEV)
    m = cu(src_map)
    got = gather_guarded(m, new_n, src, zero_children)
    assert torch.equal(got, gather_expected(m, src, zero_children))


def test_gather_rows_grid_stride():
    """6 000 000 rows x 45 floats (featuresRest at degree 3) = 2.7e8 > 2^28 elements: the grid of 2^20 blocks of 256
    threads takes a second pass of its grid-stride loop."""
    new_n, rf, n = 6_000_000, 45, 3_000_000
    assert new_n * rf > (1 << 28)
    g = torch.Generator(device=DEV).manual_seed(5)
    par = torch.randint(0, n, (new_n,), device=DEV, generator=g, dtype=torch.int64)
    kind = torch.randint(0, 4, (new_n,), device=DEV, generator=g, dtype=torch.int64)
    m = ((par | (kind << 30)) & 0xFFFFFFFF).to(torch.int64)
    m = torch.where(m >= (1 << 31), m - (1 << 32), m).to(torch.int32)
    src = torch.randn(n, rf, device=DEV, generator=g)
    for zc in (False, True):
        got = gather_guarded(m, new_n, src, zc)
        assert torch.equal(got, gather_expected(m, src, zc))
        del got
    torch.cuda.empty_cache()


# ---- PLY ------------------------------------------------------------------------------------------------------------
def unpack(rows, k, layout, keep, scale, tr):
    """gsb_unpack_ply_rows into either feature layout; returns a dict in the reference's layout (dc, rest)."""
    from opensplat_b200 import capi, export
    n = rows.shape[0]
    f32 = dict(dtype=torch.float32, device=DEV)
    o = {x: torch.empty(s, **f32) for x, s in (("means", (n, 3)), ("scales", (n, 3)), ("quats", (n, 4)),
                                                ("opacities", (n, 1)))}
    if layout == "merged":
        coeffs = torch.full((n, k, 3), SENT, **f32)
        dc, dcs, rest, rs = coeffs.data_ptr(), 3 * k, (coeffs.data_ptr() + 12 if k > 1 else None), 3 * k
    else:
        fdc, frest = torch.empty((n, 3), **f32), torch.empty((n, k - 1, 3), **f32)
        dc, dcs, rest, rs = fdc.data_ptr(), 3, (frest.data_ptr() if k > 1 else None), 3 * (k - 1)
    capi.check(capi.lib().gsb_unpack_ply_rows(n, k, capi.ptr(rows), int(keep), float(scale), export._crs(keep, tr),
                                              capi.ptr(o["means"]), Ct.c_void_p(dc), dcs,
                                              Ct.c_void_p(rest) if rest else None, rs, capi.ptr(o["opacities"]),
                                              capi.ptr(o["scales"]), capi.ptr(o["quats"]), capi.stream()))
    if layout == "merged":
        o["featuresDc"], o["featuresRest"] = coeffs[:, 0], coeffs[:, 1:]
    else:
        o["featuresDc"], o["featuresRest"] = fdc, frest
    return {x: t.cpu().numpy() for x, t in o.items()}


@pytest.mark.parametrize("layout", ["reference", "merged"])
@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
@pytest.mark.parametrize("keep", [False, True])
def test_ply_pack_unpack(layout, k, keep):
    from opensplat_b200 import export
    n = 5003
    scale, tr = (0.37, (12.5, -3.25, 100.0)) if keep else (1.0, (0.0, 0.0, 0.0))
    p = scene_edit_inputs(n, k, 30 + k)[0]
    d = {x: cu(v) for x, v in p.items()}
    if layout == "merged":
        d = {x: v for x, v in d.items() if x not in ("featuresDc", "featuresRest")}
        d["coeffs"] = torch.cat([cu(p["featuresDc"])[:, None], cu(p["featuresRest"])], 1).contiguous()
    rows = export.pack_ply_rows(d, keep, scale, tr)
    want, sc = sf.ply_rows(p["means"], p["featuresDc"], p["featuresRest"], p["opacities"], p["scales"], p["quats"],
                           keep, scale, tr)
    got = rows.cpu().numpy()
    cols = np.ones(want.shape[1], bool)
    if keep:
        cols[-7:-4] = False
        check_within("ply keepCrs scales", got[:, -7:-4], sc)
    assert np.array_equal(got[:, cols], want[:, cols])
    back = unpack(rows, k, layout, keep, scale, tr)
    for x in ("quats", "featuresDc", "featuresRest", "opacities"):
        assert np.array_equal(back[x], p[x].reshape(back[x].shape)), x
    if keep:
        lm, ls = sf.unpack_crs(got[:, 0:3], got[:, -7:-4], scale, tr)
        assert np.array_equal(back["means"], lm)
        check_within("ply load keepCrs scales", back["scales"], ls)
    else:   # the round trip is the identity
        assert np.array_equal(back["means"], p["means"]) and np.array_equal(back["scales"], p["scales"])


def test_ply_pack_grid_stride():
    """4.4 M Gaussians at degree 3: 62 floats a row, 2.7e8 > 2^28 elements, so the pack's grid-stride loop runs a
    second pass."""
    from opensplat_b200 import export
    n, k = 4_400_000, 16
    assert n * (14 + 3 * k) > (1 << 28)
    g = torch.Generator(device=DEV).manual_seed(9)
    p = {"means": torch.randn(n, 3, device=DEV, generator=g), "scales": torch.randn(n, 3, device=DEV, generator=g),
         "quats": torch.randn(n, 4, device=DEV, generator=g), "opacities": torch.randn(n, 1, device=DEV, generator=g),
         "coeffs": torch.randn(n, k, 3, device=DEV, generator=g)}
    rows = export.pack_ply_rows(p)
    want = torch.cat([p["means"], torch.zeros(n, 3, device=DEV), p["coeffs"][:, 0],
                      p["coeffs"][:, 1:].transpose(1, 2).reshape(n, -1), p["opacities"], p["scales"], p["quats"]], 1)
    assert torch.equal(rows, want)
    del rows, want
    torch.cuda.empty_cache()


# ---- .splat ---------------------------------------------------------------------------------------------------------
def splat_inputs(n, seed):
    """scene_edit_inputs plus rows on the u8 edges: quaternion components on exact byte values (q 128 + 128 integral),
    colours clamped at 0 and 1, and exact key ties."""
    f = np.float32
    p = scene_edit_inputs(n, 4, seed)[0]
    p["quats"][:64] = np.array([0.5, -0.5, 0.0, 127.0 / 128.0], f)
    p["featuresDc"][64:96] = f(10.0)
    p["featuresDc"][96:128] = f(-10.0)
    p["scales"][128:160], p["opacities"][128:160] = p["scales"][127], p["opacities"][127]
    return p


@pytest.mark.parametrize("keep", [False, True])
def test_splat_certified(keep):
    from opensplat_b200 import capi, export
    n = 200_000
    scale, tr = (0.37, (12.5, -3.25, 100.0)) if keep else (1.0, (0.0, 0.0, 0.0))
    p = splat_inputs(n, 40 + keep)
    d = {x: cu(v) for x, v in p.items()}
    keys = torch.empty(n, dtype=torch.int64, device=DEV)
    capi.check(capi.lib().gsb_splat_order_keys(n, capi.ptr(d["scales"]), capi.ptr(d["opacities"]), int(keep),
                                               float(scale), capi.ptr(keys), capi.stream()))
    kf = sf.decode_keys(keys.cpu().numpy())
    key = sf.splat_key(p["scales"], p["opacities"], keep, scale)
    check_within("splat key", kf, key)
    order = export.splat_order(d, keep, scale)
    o = order.cpu().numpy()
    assert np.array_equal(np.sort(o), np.arange(n))
    bad, ties, unc = sf.order_check(o, key, kf[o])
    assert bad == 0 and ties == 0, (bad, ties)
    rows = export.pack_splat_rows(d, keep, scale, tr, order=order).cpu().numpy()
    means = sf.crs_means(p["means"], scale, tr) if keep else p["means"]
    assert np.array_equal(rows[:, 0:12], means[o].astype("<f4").view(np.uint8).reshape(n, 12))
    e = sf.splat_scales(p["scales"], keep, scale)
    fs = rows[:, 12:24].copy().view("<f4")
    for c in range(3):
        check_within("splat scale", fs[:, c], e[c][o])
    rgb, a, q = sf.splat_bytes(p["featuresDc"], p["opacities"], p["quats"])
    unc_bytes = 0
    for tag, got, x in (("rgb", rows[:, 24:27], rgb[o]), ("alpha", rows[:, 27], a[o]), ("quat", rows[:, 28:32], q[o])):
        ok, cert = sf.byte_check(got, x)
        assert ok.all(), (tag, np.argwhere(~ok)[:3])
        unc_bytes += int((~cert).sum())
    rgb8, q8 = sf.splat_bytes_fp32(p["featuresDc"], p["quats"])
    assert np.array_equal(rows[:, 24:27], rgb8[o]) and np.array_equal(rows[:, 28:32], q8[o])
    assert (rows[:, 28:32][np.isin(o, np.arange(64))] == np.array([192, 64, 128, 255], np.uint8)).all()
    report(f"splat keep={keep}", uncertified_pairs=unc, uncertified_bytes=unc_bytes)

