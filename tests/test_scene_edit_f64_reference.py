"""Pins tests/scene_edit_f64.py -- the float64 restatement of csrc/densify.cu and csrc/export.cu -- on the CPU:
against the reference's own outputs (tests/golden/scene_edit_*.npz, made by the unmodified model.cpp) and the CPU
restatement oracle/scene_edit.py on every certified element, against the plain formulas in float64 torch, against
fp32 evaluations of the kernels' operation trees (the bounds must cover them), and shows that the checks reject each
wrong convention a kernel could adopt."""
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import scene_edit_f64 as sf  # noqa: E402
from oracle import scene_edit as se  # noqa: E402
from test_scene_edit_oracle import cfg_of, schedule  # noqa: E402
from util import load_golden, scene_edit_inputs  # noqa: E402

DENSIFY_CASES = ["scene_edit_densify_screen", "scene_edit_densify_huge", "scene_edit_densify_all"]
DB = 1024


def default_cfg(**kw):
    c = dict(densify_grad_thresh=0.0002, densify_size_thresh=0.01, split_screen_size=0.05, cull_alpha_thresh=0.1,
             cull_scale_thresh=0.5, cull_screen_size=0.15, size_fac=1.6)
    c.update(kw)
    return types.SimpleNamespace(**c)


def within(got, x):
    got = np.asarray(got, np.float64)
    return bool(np.all((np.abs(got - x.v) <= sf.C * x.b) | (got == x.v)))


def golden_refine(name):
    """Replays a golden case up to its refine step: (inputs, stats, cfg, max_dim, check flags, samples)."""
    g = load_golden(name)
    n, k, seed = int(g["n"]), int(g["k"]), int(g["seed"])
    H, W = (int(x) for x in g["hw"])
    cfg = cfg_of(g)
    p, m, v, draws = scene_edit_inputs(n, k, seed, max(H, W))
    stats = None
    for si, step in enumerate(int(s) for s in g["steps"]):
        if step < cfg.stop_split_at:
            stats = se.densify_stats(stats, *draws[si], H, W)
        refine, densify, _, chk_screen, chk_huge = schedule(cfg, step)
        if refine and densify:
            return g, p, m, v, [s.numpy() for s in stats], cfg, max(H, W), chk_screen, chk_huge
    raise AssertionError(name)


# ---- against the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", DENSIFY_CASES)
def test_refine_matches_reference_golden(name):
    """Certified decisions -> compaction -> gathered rows and means/scales reproduce Model::afterTrain's output."""
    g, p, m, v, (gn, vc, ms), cfg, max_dim, chk_screen, chk_huge = golden_refine(name)
    d = sf.classify(p["scales"], p["opacities"], gn, vc, ms, max_dim, cfg, chk_screen, chk_huge, chk_screen)
    assert d["cert"].all(), int((~d["cert"]).sum())
    src, rank, cnt = sf.compact(**d)
    par = (src.view(np.uint32) & ((1 << 30) - 1)).astype(np.int64)
    child = (src.view(np.uint32) >> 30) != 0
    for x in ("quats", "featuresDc", "featuresRest", "opacities"):
        np.testing.assert_array_equal(p[x][par], g["p_" + x], err_msg=x)
    for x in p:
        z = m[x][par].copy()
        z[child] = 0
        np.testing.assert_array_equal(z, g["m_" + x], err_msg="m_" + x)
    torch.manual_seed(int(g["seed_randn"]))
    samples = torch.randn(2 * int(cnt[0]), 3).numpy()
    nm, ns = sf.means_scales(src, rank, int(cnt[0]), samples, p["means"], p["scales"], p["quats"], cfg.size_fac)
    assert within(g["p_means"], nm) and within(g["p_scales"], ns)
    assert cnt[0] > 0 and cnt[3] > 0 and cnt[4] < len(p["means"]) + 2 * cnt[0] + cnt[5]


@pytest.mark.parametrize("chk_screen,chk_huge", [(True, True), (False, True), (True, False), (False, False)])
def test_classify_matches_oracle_on_certified_parents(chk_screen, chk_huge):
    """The inputs of the GPU at-scale test: every certified parent decides as the reference's ATen sequence does."""
    n, H, W = 300_000, 720, 1280
    p, m, v, draws = scene_edit_inputs(n, 4, 77 + 2 * chk_screen + chk_huge, max(H, W))
    stats = None
    for v_xy, radii in draws:
        stats = se.densify_stats(stats, v_xy * (640.0 / 1280.0), radii * 2, H, W)
    cfg = default_cfg()
    d = sf.classify(p["scales"], p["opacities"], *(s.numpy() for s in stats), max(H, W), cfg, chk_screen, chk_huge,
                    chk_screen)
    unc = int((~d["cert"]).sum())
    assert unc <= 10, unc
    _, _, _, oi = se.refine({"means": p["means"], "scales": p["scales"], "quats": p["quats"],
                             "opacities": p["opacities"]}, None, None, stats, max(H, W), cfg, chk_screen, chk_huge,
                            lambda k: torch.zeros(2 * k, 3))
    od = sf.decisions_of(oi["src_map"].numpy(), np.where(oi["splits"].numpy(), 0, -1), n)
    od["dup"] = oi["dups"].numpy()
    c = d["cert"]
    for k in ("split", "dup", "keep_self", "keep_split", "keep_dup"):
        assert np.array_equal(d[k][c], od[k][c]), k


@pytest.mark.parametrize("name", ["scene_edit_save", "scene_edit_save_crs"])
def test_writers_match_reference_golden(name):
    g = load_golden(name)
    n, k = int(g["n"]), int(g["k"])
    p = scene_edit_inputs(n, k, int(g["seed"]))[0]
    keep, scale, tr = bool(g["keep_crs"]), float(g["scale"]), tuple(float(x) for x in g["translation"])
    rows, sc = sf.ply_rows(p["means"], p["featuresDc"], p["featuresRest"], p["opacities"], p["scales"], p["quats"],
                           keep, scale, tr)
    hdr = se.ply_header(n, 3 * (k - 1), int(g["step"]))
    ref = np.frombuffer(g["ply"].tobytes()[len(hdr):], "<f4").reshape(n, -1)
    cols = np.ones(rows.shape[1], bool)
    if keep:
        cols[-7:-4] = False
        assert within(ref[:, -7:-4], sc)
    np.testing.assert_array_equal(rows[:, cols], ref[:, cols])
    # the loader on the reference's own file
    ld = {x: g["ld_" + x] for x in ("means", "scales")}
    if keep:
        lm, ls = sf.unpack_crs(ref[:, 0:3], ref[:, -7:-4], scale, tr)
        np.testing.assert_array_equal(lm, ld["means"])
        assert within(ld["scales"], ls)
    # .splat: the reference's file, row by row
    ref_rows = g["splat"].reshape(n, 32)
    means = sf.crs_means(p["means"], scale, tr) if keep else p["means"]
    lookup = {bytes(r): i for i, r in enumerate(means.astype("<f4").view(np.uint8).reshape(n, 12))}
    order = np.array([lookup[bytes(r[:12])] for r in ref_rows])
    assert sorted(order.tolist()) == list(range(n))
    key = sf.splat_key(p["scales"], p["opacities"], keep, scale)
    bad, _, _ = sf.order_check(order, key)
    assert bad == 0
    e = sf.splat_scales(p["scales"], keep, scale)
    fs = ref_rows[:, 12:24].copy().view("<f4")
    for c in range(3):
        assert within(fs[:, c], e[c][order])
    rgb, a, q = sf.splat_bytes(p["featuresDc"], p["opacities"], p["quats"])
    for got, x in ((ref_rows[:, 24:27], rgb[order]), (ref_rows[:, 27], a[order]), (ref_rows[:, 28:32], q[order])):
        ok, cert = sf.byte_check(got, x)
        assert ok.all() and cert.mean() > 0.99
    rgb8, q8 = sf.splat_bytes_fp32(p["featuresDc"], p["quats"])
    assert np.array_equal(ref_rows[:, 24:27], rgb8[order]) and np.array_equal(ref_rows[:, 28:32], q8[order])


# ---- against the plain formulas --------------------------------------------------------------------------------
def test_values_match_plain_float64_torch():
    rng = np.random.default_rng(3)
    n = 20_000
    p = scene_edit_inputs(n, 4, 5)[0]
    gn, vc = rng.uniform(0, 1e-5, n).astype(np.float32), rng.integers(1, 5, n).astype(np.float32)
    d = sf.classify(p["scales"], p["opacities"], gn, vc, None, 1280, default_cfg(), True, True, True)
    t = lambda a: torch.from_numpy(np.asarray(a)).double()
    s = t(p["scales"])
    fac = float(np.float32(1.6))
    ref = {"mx": s.exp().amax(-1), "avg": t(gn) / t(vc) * 0.5 * 1280, "sig": torch.sigmoid(t(p["opacities"])[:, 0]),
           "mxc": (s.exp() / fac).amax(-1)}
    for k, r in ref.items():
        assert torch.allclose(t(d[k].v), r, rtol=1e-12, atol=0), k
    # split children of every parent
    ar = np.arange(n, dtype=np.int64)
    src = np.concatenate([ar | (1 << 30), ar | (2 << 30)]).astype(np.uint32).view(np.int32)
    smp = rng.standard_normal((2 * n, 3)).astype(np.float32)
    nm, ns = sf.means_scales(src, ar.astype(np.int32), n, smp, p["means"], p["scales"], p["quats"], 1.6)
    q = torch.nn.functional.normalize(t(p["quats"]), dim=-1)
    R = se.quat_to_rotmat(q)
    ref_m = t(p["means"]).repeat(2, 1) + torch.bmm(R.repeat(2, 1, 1), (s.exp().repeat(2, 1) * t(smp))[..., None])[..., 0]
    assert torch.allclose(t(nm.v), ref_m, rtol=1e-12, atol=1e-15)
    assert torch.allclose(t(ns.v), (s - np.log(fac)).repeat(2, 1), rtol=1e-12, atol=1e-15)
    key = sf.splat_key(p["scales"], p["opacities"], True, 0.37)
    ref_k = (s.exp() / float(np.float32(0.37))).sum(-1) * torch.sigmoid(t(p["opacities"])[:, 0])
    assert torch.allclose(t(key.v), ref_k, rtol=1e-12)
    rgb, a, qq = sf.splat_bytes(p["featuresDc"], p["opacities"], p["quats"])
    assert torch.allclose(t(rgb.v), torch.clamp(t(p["featuresDc"]) * sf.SH_C0 + 0.5, 0, 1) * 255, rtol=1e-12)
    assert torch.allclose(t(a.v), torch.sigmoid(t(p["opacities"])[:, 0]) * 255, rtol=1e-12)
    assert torch.allclose(t(qq.v), torch.clamp(t(p["quats"]) * 128 + 128, 0, 255), rtol=1e-12)


def test_bounds_cover_fp32_evaluations():
    """numpy's fp32 evaluation of each kernel tree (its exp and log are within the device's ulp bounds) must lie
    within the certified bound; the bounds are also no looser than a few hundred ulp of the result."""
    f = np.float32
    rng = np.random.default_rng(4)
    n = 50_000
    p = scene_edit_inputs(n, 4, 6)[0]
    s, o, q = p["scales"], p["opacities"][:, 0], p["quats"] * f(10.0) ** rng.uniform(-3, 3, (n, 1)).astype(f)
    e = np.exp(s)
    mx = e.max(-1)
    key = ((e[:, 0] + e[:, 1]) + e[:, 2]) / (f(1) + np.exp(-o))
    k = sf.splat_key(s, o[:, None])
    assert within(key, k)
    d = sf.quantities(s, o, np.ones(n, f), np.ones(n, f), 640, 1.6)
    assert within(mx, d["mx"]) and within(f(1) / (f(1) + np.exp(-o)), d["sig"])
    assert within(np.exp(np.log(e / f(1.6))).max(-1), d["mxc"])
    smp = rng.standard_normal((2 * n, 3)).astype(f)
    ar = np.arange(n, dtype=np.int64)
    src = np.concatenate([ar | (1 << 30), ar | (2 << 30)]).astype(np.uint32).view(np.int32)
    nm, ns = sf.means_scales(src, ar.astype(np.int32), n, smp, p["means"], s, q, 1.6)
    got_m, got_s = kernel_means_scales_fp32(src, ar, n, smp, p["means"], s, q, f(1.6))
    assert within(got_m, nm) and within(got_s, ns)
    mag = np.abs(np.tile(p["means"], (2, 1))) + (np.exp(np.tile(s, (2, 1)).astype(np.float64)) * np.abs(smp)).sum(
        -1, keepdims=True)                                  # A = |m| + sum |e_k sample_k| (|R| <= 1)
    assert float(np.max(nm.b / mag)) < 100 * sf.U


def kernel_means_scales_fp32(src, rank, n_splits, smp, means, scales, quats, fac, normalise=True, row_of=None):
    """densify_means_scales_kernel in numpy fp32 for children-only maps (the conventions are switches)."""
    f = np.float32
    e = src.view(np.uint32)
    par, kind = (e & ((1 << 30) - 1)).astype(np.int64), (e >> 30).astype(np.int64)
    row = (kind - 1) * n_splits + rank[par] if row_of is None else row_of(kind, rank[par])
    ex = np.exp(scales[par])
    v = ex * smp[row]
    w, x, y, z = (quats[par, i].copy() for i in range(4))
    for _ in range(2 if normalise else 0):
        nrm = np.maximum(np.sqrt(w * w + x * x + y * y + z * z), f(1e-12))
        w, x, y, z = w / nrm, x / nrm, y / nrm, z / nrm
    r = [[f(1) - f(2) * (y * y + z * z), f(2) * (x * y - w * z), f(2) * (x * z + w * y)],
         [f(2) * (x * y + w * z), f(1) - f(2) * (x * x + z * z), f(2) * (y * z - w * x)],
         [f(2) * (x * z - w * y), f(2) * (y * z + w * x), f(1) - f(2) * (x * x + y * y)]]
    m = np.stack([means[par, a] + ((r[a][0] * v[:, 0] + r[a][1] * v[:, 1]) + r[a][2] * v[:, 2]) for a in range(3)], -1)
    return m, np.log(ex / fac)


# ---- the checks reject wrong conventions -------------------------------------------------------------------------
def flags_of(d):
    return (d["split"] * 1 | d["dup"] * 2 | d["keep_self"] * 4 | d["keep_split"] * 8 | d["keep_dup"] * 16).astype(np.int64)


def scan_scatter(d, carry_all_chunks=True, sample_major=True):
    """The three classify kernels on the host: per-block counts, the chunked scan of the block counts (1024 blocks
    per chunk), the scatter.  The switches are wrong conventions."""
    f = flags_of(d)
    n = len(f)
    nb = -(-n // DB)
    fp = np.zeros(nb * DB, np.int64)
    fp[:n] = f
    bits = np.stack([(fp & 1) != 0, (fp & 4) != 0, (fp & 8) != 0, (fp & 16) != 0], -1).astype(np.int64)
    per_block = bits.reshape(nb, DB, 4).sum(1)
    offsets = np.zeros((nb, 4), np.int64)
    carry = np.zeros(4, np.int64)
    for base in range(0, nb, DB):
        c = per_block[base:base + DB]
        offsets[base:base + DB] = carry + np.cumsum(c, 0) - c
        if carry_all_chunks or base == 0:
            carry = carry + c.sum(0)
    within_block = (np.cumsum(bits.reshape(nb, DB, 4), 1) - bits.reshape(nb, DB, 4)).reshape(-1, 4)[:n]
    rank = np.repeat(offsets, DB, 0)[:n] + within_block
    kself, ksplit, new_n = carry[1], carry[2], carry[1] + 2 * carry[2] + carry[3]
    src = np.full(max(int(new_n), 3 * n), -7, np.int64)
    i = np.arange(n, dtype=np.int64)
    m = (f & 4) != 0
    src[rank[m, 1]] = i[m]
    m = (f & 8) != 0
    if sample_major:
        src[kself + rank[m, 2]] = i[m] | (1 << 30)
        src[kself + ksplit + rank[m, 2]] = i[m] | (2 << 30)
    else:
        src[kself + 2 * rank[m, 2]] = i[m] | (1 << 30)
        src[kself + 2 * rank[m, 2] + 1] = i[m] | (2 << 30)
    m = (f & 16) != 0
    src[kself + 2 * ksplit + rank[m, 3]] = i[m] | (3 << 30)
    split_rank = np.where(f & 1, rank[:, 0], -1)
    counts = [carry[0], carry[1], carry[2], carry[3], new_n, int(d["dup"].sum()), 0, 0]
    return src[:new_n].astype(np.uint32).view(np.int32), split_rank.astype(np.int32), np.array(counts, np.int32)


def same_outputs(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def pattern_decisions(n, seed=0):
    """Decisions varying across blocks: each block draws its own probabilities."""
    rng = np.random.default_rng(seed)
    pb = rng.uniform(0, 1, (-(-n // DB), 4))[np.arange(n) // DB]
    u = rng.uniform(0, 1, (n, 4))
    split, dup = (u[:, 0] < pb[:, 0]), (u[:, 0] >= pb[:, 0]) & (u[:, 1] < pb[:, 1])
    keep = u[:, 2] < pb[:, 2]
    return {"split": split, "dup": dup, "keep_self": keep & ~split & (u[:, 3] < pb[:, 3]), "keep_split": split & keep,
            "keep_dup": dup & keep}


def test_host_scan_matches_compaction_and_rejects_wrong_carry():
    d = pattern_decisions(1_048_577 + 5000)
    want = sf.compact(**d)
    assert same_outputs(scan_scatter(d), want)
    assert not same_outputs(scan_scatter(d, carry_all_chunks=False), want)
    small = pattern_decisions(5000, 1)
    assert same_outputs(scan_scatter(small, carry_all_chunks=False), sf.compact(**small))  # one chunk: no carry
    assert not same_outputs(scan_scatter(small, sample_major=False), sf.compact(**small))


def classify_fixture():
    """Parents on the edges the mutations move: [0] avg == grad threshold exactly, [1] sigmoid == alpha threshold
    exactly (a duplicate), [2] a split parent whose own scale is huge but whose child's is not."""
    f = np.float32
    cfg = default_cfg(cull_alpha_thresh=0.5)
    t = sf.cfg32(cfg)
    scales = np.array([[-3, -3, -3], [-6, -6, -6], [np.log(0.6)] * 3], f)
    opac = np.array([[3.0], [0.0], [3.0]], f)
    gn = np.array([f(t["densify_grad_thresh"]) / f(512), 1e-3, 1e-3], f)
    return scales, opac, gn, np.ones(3, f), np.zeros(3, f), 1024, cfg


def test_classify_rejects_wrong_comparisons():
    scales, opac, gn, vc, m2, md, cfg = classify_fixture()
    d = sf.classify(scales, opac, gn, vc, m2, md, cfg, False, True, False)
    assert d["cert"].all()
    assert not d["dup"][0] and d["dup"][1] and d["keep_self"][1] and d["split"][2] and d["keep_split"][2]
    t = sf.cfg32(cfg)
    ge_grad = d["avg"].v >= t["densify_grad_thresh"]            # '>=' for '>' on the gradient threshold
    assert ge_grad[0] != (d["split"][0] or d["dup"][0])
    le_alpha = d["sig"].v <= t["cull_alpha_thresh"]             # '<=' for '<' on the alpha threshold
    assert le_alpha[1] and d["keep_self"][1]
    parent_huge = d["mx"].v > t["cull_scale_thresh"]            # the huge-child cull on the parent's scale
    assert parent_huge[2] and d["keep_split"][2]


def test_means_scales_check_rejects_wrong_conventions():
    f = np.float32
    rng = np.random.default_rng(8)
    n = 4000
    p = scene_edit_inputs(n, 4, 9)[0]
    q = p["quats"] * f(3.0)
    ar = np.arange(n, dtype=np.int64)
    rank = ar.astype(np.int32)
    src = np.concatenate([ar | (1 << 30), ar | (2 << 30)]).astype(np.uint32).view(np.int32)
    smp = rng.standard_normal((2 * n, 3)).astype(f)
    nm, ns = sf.means_scales(src, rank, n, smp, p["means"], p["scales"], q, 1.6)
    good = kernel_means_scales_fp32(src, ar, n, smp, p["means"], p["scales"], q, f(1.6))
    assert within(good[0], nm) and within(good[1], ns)
    raw = kernel_means_scales_fp32(src, ar, n, smp, p["means"], p["scales"], q, f(1.6), normalise=False)
    assert not within(raw[0], nm)
    row = kernel_means_scales_fp32(src, ar, n, smp, p["means"], p["scales"], q, f(1.6),
                                   row_of=lambda kind, r: 2 * r + kind - 1)
    assert not within(row[0], nm)


def gather_emulation(src_map, src, rf, zero_children, max_blocks=1 << 20, one_pass=False, stride=None):
    """gather_rows_kernel on the host with a grid of min(total / 256, max_blocks) blocks."""
    total = len(src_map) * rf
    out = np.full(total, np.nan, np.float32)
    step = min(-(-total // 256), max_blocks) * 256
    idx = np.arange(total, dtype=np.int64)
    if one_pass:
        idx = idx[idx < step]
    j, c = idx // rf, idx % rf
    e = src_map.view(np.uint32)[j]
    par = (e & ((1 << 30) - 1)).astype(np.int64)
    v = src.reshape(-1)[par * (rf if stride is None else stride) + c]
    out[idx] = np.where(((e >> 30) != 0) & bool(zero_children), np.float32(0), v)
    return out.reshape(-1, rf)


@pytest.mark.parametrize("rf", [9, 45])
def test_gather_check_rejects_wrong_conventions(rf):
    rng = np.random.default_rng(rf)
    n = 3000
    src = rng.standard_normal((n, rf)).astype(np.float32)
    src_map, _, _ = sf.compact(**pattern_decisions(n, 2))
    par = (src_map.view(np.uint32) & ((1 << 30) - 1)).astype(np.int64)
    want = src[par].copy()
    want[(src_map.view(np.uint32) >> 30) != 0] = 0
    assert np.array_equal(gather_emulation(src_map, src, rf, True, max_blocks=16), want)
    assert not np.array_equal(gather_emulation(src_map, src, rf, True, max_blocks=16, one_pass=True), want)
    assert not np.array_equal(gather_emulation(src_map, src, rf, True, stride=rf - 1), want)


def test_splat_checks_reject_wrong_conventions():
    f = np.float32
    p = scene_edit_inputs(5000, 4, 10)[0]
    rgb, a, q = sf.splat_bytes(p["featuresDc"], p["opacities"], p["quats"])
    alpha = np.clip((f(1) / (f(1) + np.exp(-p["opacities"][:, 0]))) * f(255), f(0), f(255))
    assert sf.byte_check(np.trunc(alpha).astype(np.uint8), a)[0].all()
    assert not sf.byte_check(np.rint(alpha).astype(np.uint8), a)[0].all()            # rounded, not truncated
    rgb8, _ = sf.splat_bytes_fp32(p["featuresDc"], p["quats"])
    assert sf.byte_check(rgb8, rgb)[0].all()
    assert not sf.byte_check(np.rint(rgb.v).astype(np.uint8), rgb)[0].all()
    key = sf.splat_key(p["scales"], p["opacities"], True, 0.37)
    no_div = sf.splat_key(p["scales"], p["opacities"])                                # keepCrs division dropped
    assert not within(no_div.v.astype(f), key)
    assert sf.order_check(np.argsort(-key.v, kind="stable"), key)[0] == 0
    assert sf.order_check(np.argsort(key.v, kind="stable"), key)[0] > 0
    ties = np.array([2.0, 2.0, 1.0], f)
    assert sf.order_check([0, 1, 2], sf.V(ties.astype(np.float64)), ties)[1] == 0
    assert sf.order_check([1, 0, 2], sf.V(ties.astype(np.float64)), ties[[1, 0, 2]])[1] == 1
