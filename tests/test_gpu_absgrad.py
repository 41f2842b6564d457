"""GPU: AbsGS's absolute screen-space gradient (DESIGN D25), from gsb_rasterize_backward_absgrad up to SplatTrainer.

1. The kernel's v_xy_abs against the float64 reference of tests/absgrad_f64.py on certified Gaussians, for all four
   SAT x DEPTH instantiations, on the case builders of test_gpu_blend_f64 (ragged images, single-tile list lengths,
   opacity regimes, the extent cull, colours above 1 with the clamp, projected scenes), with that file's bound
   C_BWD u (B + (8 + n_tiles) A).  Every other output equals gsb_rasterize_backward / _depth bit for bit, and two calls
   give the same v_xy_abs bits.
2. SplatTrainer(RefineConfig(absgrad=True)): before the first refinement the same parameters and moments as the plain
   trainer; the statistics are those of the statistics kernels on the entry's v_xy_abs, and the first refinement's
   classification is densify.classify's on them (B = 1, B = 2, a depth prior); a world-1 group run is the
   single-process run; the launch sequence swaps the backward entry and nothing else.
3. The mechanism: one large Gaussian over a stripe texture mirror-symmetric about its centre is split at the first
   refinement with absgrad and not without.
4. Quality on a fine-texture scene from a coarse start: held-out PSNR and final Gaussian count, plain at 0.0002
   against absgrad at 0.0008 (printed; run with -s)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import absgrad_f64 as af
import test_gpu_blend_f64 as tb
import test_gpu_depth_render as dr
import test_gpu_trainer as tg
from opensplat_b200 import capi, densify, ops
from opensplat_b200.scene import make_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U, C_BWD = tb.U, tb.C_BWD
CLAMP = ops.CLAMP_MAX_ONE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


# ------------------------------------------------------------------------------------------------- 1. the kernel
def _absgrad_backward(case, fwd, flags, v_depth, depth):
    """gsb_rasterize_backward_absgrad on a generic-path frame (test_gpu_depth_render._forward): returns the outputs of
    ops.rasterize_backward (v_depths last when depth) and v_xy_abs."""
    L, P = capi.lib(), capi.ptr
    _, fT, fI, _, _, rec, rd = fwd
    n, m = case.n, case.m
    rows = torch.empty(L.gsb_raster_grad_rows_bytes(m) // 4 + 4, dtype=torch.float32, device=DEV)
    outs = [torch.empty(s, dtype=torch.float32, device=DEV) for s in ((n, 2), (n, 3), (n, 3), (n, 1))]
    v_depths = torch.empty(n, dtype=torch.float32, device=DEV) if depth else None
    v_xy_abs = torch.full((n, 2), float("nan"), dtype=torch.float32, device=DEV)
    capi.check(L.gsb_rasterize_backward_absgrad(
        case.H, case.W, case.tb[0], case.tb[1], n, m, P(case.bins), None, P(case.conics), P(case.opac), P(rec),
        P(case.cum), P(case.bg), P(fT), P(fI), P(case.v_out), P(case.voa), P(rows), *(P(t) for t in outs), flags,
        P(rd) if depth else None, P(v_depth) if depth else None, P(v_depths), P(v_xy_abs), capi.stream()))
    return tuple(outs) + ((v_depths,) if depth else ()), v_xy_abs


def _check_kernel(name, case, sat, depth, v_depth=None):
    flags = CLAMP if sat else 0
    fwd = dr._forward(case, flags, depth)
    if depth and v_depth is None:
        v_depth = cu(np.random.default_rng(case.n).uniform(-1, 1, (case.H, case.W)).astype(np.float32))
    plain = dr._backward(case, fwd, flags, case.v_out, case.voa, v_depth=v_depth, depth=depth)
    got, v_abs = _absgrad_backward(case, fwd, flags, v_depth, depth)
    for x, y in zip(plain, got):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{name}: other outputs differ from the plain entry"
    _, again = _absgrad_backward(case, fwd, flags, v_depth, depth)
    assert torch.equal(v_abs.view(torch.int32), again.view(torch.int32)), f"{name}: v_xy_abs not reproducible"
    ref = af.absgrad(case.gs, case.bins, case.xys, case.conics, case.colors, case.opac, case.bg, case.H, case.W,
                     case.v_out, case.voa, clamp=sat, depths=case.depths if depth else None,
                     v_output_depth=v_depth if depth else None)
    gc = ref["gauss_cert"]
    fg = float(gc.double().mean()) if case.n else 1.0
    assert fg >= 0.95, f"{name}: certified Gaussians {fg:.4f} -- change the case"
    bound = C_BWD * U * (ref["B_v_xy_abs"] + (8 + ref["n_tiles"][:, None]) * ref["A_v_xy_abs"])
    err = (v_abs.double() - ref["v_xy_abs"]).abs()
    msk = gc[:, None].expand_as(err)
    ratio = tb._ratio(err[msk], bound[msk])
    over = (err > bound) & msk
    if bool(over.any()):
        g, j = torch.nonzero(over)[0].tolist()
        pytest.fail(f"{name}: v_xy_abs[{g}, {j}]: kernel {float(v_abs[g, j])!r} reference "
                    f"{float(ref['v_xy_abs'][g, j])!r} bound {float(bound[g, j]):.3e}")
    assert bool(torch.isfinite(v_abs).all()) and bool((v_abs >= 0).all())   # written for every Gaussian (NaN before)
    print(f"\n{name} sat={sat} depth={depth}: certified Gaussians {fg:.5f}; worst v_xy_abs err/bound {ratio:.3f}")
    return ratio


MODES = [(False, False), (True, False), (False, True), (True, True)]


def _blob_case(rng, W, H, n, s=(1.0, 6.0), opac=(0.05, 0.9), colors=(0.0, 1.0), voa=True, bg=(0.3, 0.6, 0.2)):
    xys, con, col, op = tb._blobs(rng, n, -5, W + 5, -5, H + 5, s=s, opac=opac, colors=colors)
    return tb.Case(W, H, xys, con, col, op, list(bg), seed=n, depths=dr._depths(rng, n), voa=voa)


@pytest.mark.parametrize("sat,depth", MODES)
@pytest.mark.parametrize("W,H", [(1, 1), (23, 1), (17, 17), (31, 33), (100, 72)])
def test_kernel_ragged_images(W, H, sat, depth):
    rng = np.random.default_rng(W * 1000 + H)
    _check_kernel(f"A {W}x{H}", _blob_case(rng, W, H, 40 + (W * H) // 8, s=(1.0, 8.0)), sat, depth)


@pytest.mark.parametrize("sat,depth", MODES)
@pytest.mark.parametrize("k", [1, 32, 33, 128, 129, 4097])
def test_kernel_one_tile_list_length(k, sat, depth):
    rng = np.random.default_rng(k)
    if k <= 1024:
        xys, con, col, op = tb._blobs(rng, k, -4, 20, -4, 20, s=(1.5, 6.0), opac=(0.01, 0.12))
    else:
        xys, con, col, op = tb._blobs(rng, k, 0, 16, 0, 16, s=(0.8, 2.5), opac=(0.005, 0.05))
    c = tb.Case(16, 16, xys, con, col, op, [0.4, 0.2, 0.1], seed=k, depths=dr._depths(rng, k), voa=True)
    assert c.m == k
    _check_kernel(f"B k={k}", c, sat, depth)


@pytest.mark.parametrize("sat,depth", MODES)
@pytest.mark.parametrize("regime,opac", [("faint", (0.004, 0.02)), ("mid", (0.05, 0.35)), ("opaque", (0.9, 1.0))])
def test_kernel_opacity_regimes(regime, opac, sat, depth):
    rng = np.random.default_rng(len(regime))
    n = {"faint": 1500, "mid": 600, "opaque": 300}[regime]
    _check_kernel(f"C {regime}", _blob_case(rng, 100, 72, n, opac=opac), sat, depth)


@pytest.mark.parametrize("sat,depth", MODES)
def test_kernel_extent_cull_needles(sat, depth):
    rng = np.random.default_rng(6)
    W, H, n = 100, 72, 24
    xys = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], -1).astype(np.float32)
    s_minor = rng.uniform(0.5, 2.0, n)
    con = tb._conics(s_minor * np.sqrt(10 ** rng.uniform(2, 6, n)), s_minor, rng.uniform(0, np.pi, n))
    op = rng.uniform(0.05, 0.9, n).astype(np.float32)
    xb, cb, _, ob = tb._blobs(rng, 150, 0, W, 0, H, opac=(0.05, 0.5))
    xys, con, op = np.concatenate([xys, xb]), np.concatenate([con, cb]), np.concatenate([op, ob])
    col = rng.uniform(0, 1, (xys.shape[0], 3)).astype(np.float32)
    c = tb.Case(W, H, xys, con, col, op, [0.2, 0.2, 0.5], seed=11, depths=dr._depths(rng, xys.shape[0]), voa=True)
    _check_kernel("D needles", c, sat, depth)


@pytest.mark.parametrize("sat,depth", MODES)
def test_kernel_colours_above_one(sat, depth):
    """test_gpu_blend_f64's case E (its depths too: the clamp's certificate depends on the blend order)."""
    rng = np.random.default_rng(5)
    xys, con, col, op = tb._blobs(rng, 800, -5, 105, -5, 77, s=(1.5, 5.0), opac=(0.08, 0.7), colors=(0.0, 2.0))
    c = tb.Case(100, 72, xys, con, col, op, [0.1, 0.1, 0.1], seed=5, voa=True)
    _check_kernel("E", c, sat, depth)


@pytest.mark.parametrize("sat,depth", MODES)
@pytest.mark.parametrize("n,W,H,scale", [(100_000, 320, 192, 0.17), (1_000_000, 1920, 1080, 0.02)])
def test_kernel_projected_scenes(n, W, H, scale, sat, depth):
    if n > 100_000 and (sat or depth):
        pytest.skip("the C2 scene runs once, on the plain instantiation's ABS twin")
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=(0.05, 0.95), seed=0)
    col = torch.clamp_min(ops.compute_sh_forward(3, 3, cu(sc["viewdirs"]), cu(sc["coeffs"])) + 0.5, 0.0)
    t = ops.tile_bounds(W, H)
    _, xys, depths, radii, conics, _ = ops.project_gaussians_forward(
        cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"],
        sc["fy"], sc["cx"], sc["cy"], H, W, t)
    c = tb.Case(W, H, xys, conics, col, cu(sc["opacities"]), [0.0, 0.0, 0.0], seed=0, radii=radii, depths=depths,
                voa=True)
    _check_kernel(f"F n={n}", c, sat, depth)


# ------------------------------------------------------------------------------------------------ 2. the trainer
def _params(p):
    return {k: torch.from_numpy(v) for k, v in p.items()}


def _trainer(p, cfg, B=1, **kw):
    from opensplat_b200.trainer import SplatTrainer
    torch.manual_seed(3)
    return SplatTrainer(_params(p), cfg, device=DEV, views_per_step=B, **kw)


def _views(cams, gts, B, step):
    idx = [((step - 1) * B + b) % len(cams) for b in range(B)]
    if B == 1:
        return cams[idx[0]], gts[idx[0]]
    return [cams[i] for i in idx], gts[idx]


def _snoop(tr):
    """Records a clone of (v_xy_abs, radii) after every blend backward of the trainer's pipeline."""
    pp, seen = tr.pipe, []
    for name in ("_raster_backward", "_raster_backward_depth"):
        orig = getattr(pp, name)

        def wrap(*a, _orig=orig, **kw):
            _orig(*a, **kw)
            assert kw.get("v_xy_abs") is tr.v_xy_abs
            seen.append((tr.v_xy_abs.clone(), pp.radii.clone()))
        setattr(pp, name, wrap)
    return seen


@pytest.mark.parametrize("mode", ["b1", "b2", "depth"])
def test_trainer_statistics_and_first_refinement(mode):
    from opensplat_b200.depth import DepthConfig
    B = 2 if mode == "b2" else 1
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams, gts = tg._cams(c2w, H, W, intr), torch.from_numpy(gts).to(DEV)
    kw = {}
    priors = None
    if mode == "depth":
        kw["depth"] = DepthConfig()
        import test_gpu_depth_prior as dp
        priors = dp._priors(H, W)
    cfg = tg.refine_config(densify_grad_thresh=8e-5)
    acfg = tg.refine_config(densify_grad_thresh=8e-5, absgrad=True)
    plain, tr = _trainer(p, cfg, B, **kw), _trainer(p, acfg, B, **kw)
    seen = _snoop(tr)
    R = cfg.warmup_length + (cfg.refine_every - cfg.warmup_length % cfg.refine_every)   # the first refinement step

    def step(t, s):
        cam, gt = _views(cams, gts, B, s)
        extra = {}
        if priors is not None:
            extra["depth"] = priors[(s - 1) % len(priors)]
        t.step(cam, gt, s, **extra)
    for s in range(1, R):
        step(plain, s)
        step(tr, s)
    pa, pb = plain.pipe, tr.pipe
    for x, y in ((pa.param_flat, pb.param_flat), (pa.adam_m, pb.adam_m), (pa.adam_v, pb.adam_v)):
        assert torch.equal(x, y), "the absgrad trainer's step differs from the plain one before the first refinement"
    # the statistics recomputed apart from the recorded v_xy_abs with the statistics kernels
    ref = densify.Densifier(acfg)
    for v, radii in seen:
        ref.accumulate(v, radii, H, W)
    d = tr.densifier
    assert len(seen) == (R - 1) * B
    for a, b in ((d.xys_grad_norm, ref.xys_grad_norm), (d.vis_counts, ref.vis_counts),
                 (d.max_2d_size, ref.max_2d_size)):
        assert torch.equal(a, b)
    assert not torch.equal(d.xys_grad_norm, plain.densifier.xys_grad_norm)
    # the first refinement classifies on those statistics
    got = {}
    orig = d.refine

    def refine(params, adam_m, adam_v, max_dim, chk_screen, chk_huge):
        for v, radii in seen[(R - 1) * B:]:
            ref.accumulate(v, radii, H, W)
        assert torch.equal(d.xys_grad_norm, ref.xys_grad_norm)
        _, _, counts = densify.classify(params["scales"], params["opacities"], ref.xys_grad_norm, ref.vis_counts,
                                        ref.max_2d_size, max_dim, acfg, chk_screen, chk_huge, chk_screen)
        got["counts"] = counts.cpu().tolist()
        out = orig(params, adam_m, adam_v, max_dim, chk_screen, chk_huge)
        got["info"] = out[3]
        return out
    d.refine = refine
    step(tr, R)
    step(plain, R)
    info = got["info"]
    assert got["counts"][0] == info["n_splits"] and got["counts"][5] == info["n_dups"] and got["counts"][4] == tr.n
    print(f"\n{mode}: first refinement at step {R}: absgrad splits {info['n_splits']} dups {info['n_dups']} -> n {tr.n}; "
          f"plain -> n {plain.n}")
    assert tr.n != plain.n


def test_parallel_world1_matches_single_process():
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1",
                        "--master-addr", "127.0.0.1", "--master-port", "29571",
                        os.path.join(ROOT, "tools", "check_parallel_absgrad.py")], capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "plain_trainer_bit_identical=True" in r.stdout and "check_ok=True" in r.stdout


def test_launch_sequence_swaps_only_the_backward_entry(monkeypatch):
    import test_gpu_trainer_launches as tl
    from opensplat_b200.depth import DepthConfig
    import test_gpu_depth_prior as dp
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams, gts = tg._cams(c2w, H, W, intr), torch.from_numpy(gts).to(DEV)
    prior = dp._priors(H, W)[0]

    def sequence(absgrad, B, depth):
        log = []
        monkeypatch.setattr(capi, "_lib", tl._Recorder(capi._lib or capi.lib(), log))
        tr = _trainer(p, tg.refine_config(warmup_length=10 ** 6, absgrad=absgrad), B,
                      **({"depth": DepthConfig()} if depth else {}))
        for s in range(1, 5):
            cam, gt = _views(cams, gts, B, s)
            tr.step(cam, gt, s, **({"depth": prior} if depth else {}))
        torch.cuda.synchronize()
        del log[:]
        cam, gt = _views(cams, gts, B, 5)
        tr.step(cam, gt, 5, **({"depth": prior} if depth else {}))
        torch.cuda.synchronize()
        monkeypatch.undo()
        return log
    for B, depth in ((1, False), (2, False), (1, True)):
        a, b = sequence(False, B, depth), sequence(True, B, depth)
        if not depth:
            want = tl.ONE_VIEW if B == 1 else tl.TWO_VIEWS
            assert [x for x in a if not x.startswith("gsb_densify_stats_")] == want
        entry = "gsb_rasterize_backward_depth" if depth else "gsb_rasterize_backward"
        assert "gsb_rasterize_backward_absgrad" not in a and a.count(entry) == B
        assert b == [("gsb_rasterize_backward_absgrad" if x == entry else x) for x in a], (a, b)


# --------------------------------------------------------------------------------------------- 3. the mechanism
def _one_gaussian(scale=0.3, k=4):
    f = np.float32
    p = {"means": np.zeros((1, 3), f), "scales": np.full((1, 3), np.log(scale), f),
         "quats": np.array([[1, 0, 0, 0]], f), "featuresDc": np.zeros((1, 3), f),
         "featuresRest": np.zeros((1, k - 1, 3), f), "opacities": np.full((1, 1), 1.5, f)}
    return p


def test_cancelling_gaussian_is_split_only_with_absgrad():
    """One large Gaussian on the optical axis over vertical stripes mirror-symmetric about its projected centre: the
    pixels on either side pull its mean in opposite directions, so |v_xy| stays far below the threshold; the sum of
    |per-pixel terms| does not, and AbsGS splits it at the first refinement."""
    from opensplat_b200.model import Camera
    H = W = 64
    c2w = np.eye(4, dtype=np.float32)
    c2w[2, 3] = 4.0
    cam = Camera(W, H, 0.9 * W, 0.9 * W, W / 2.0, H / 2.0, c2w)
    p = _one_gaussian()
    cfg = dict(refine_every=10, warmup_length=15, reset_alpha_every=30, densify_size_thresh=0.01,
               stop_screen_size_at=0, max_steps=200, num_cameras=1)
    probe = _trainer(p, densify.RefineConfig(**cfg))
    probe.evaluate(cam, torch.zeros((H, W, 3), device=DEV), 1)
    xc, yc = (float(v) for v in probe.pipe.xys[0])
    xs = np.arange(W)
    stripes = (np.floor(np.abs(xs - xc) / 1.5) % 2).astype(np.float32)           # period 3 px, symmetric about xc
    gt = torch.from_numpy(np.repeat(np.tile(stripes, (H, 1))[..., None], 3, -1)).to(DEV)
    res = {}
    for absgrad, thresh in ((False, 0.0002), (True, 0.0008)):
        tr = _trainer(p, densify.RefineConfig(densify_grad_thresh=thresh, absgrad=absgrad, **cfg))
        for s in range(1, 20):
            tr.step(cam, gt, s)
        d = tr.densifier
        stat = float(d.xys_grad_norm[0] / d.vis_counts[0])
        tr.step(cam, gt, 20)
        res[absgrad] = (stat, tr.last_info.get("n_splits", 0), tr.n)
    print(f"\ncentre ({xc:.3f}, {yc:.3f}); plain: mean statistic {res[False][0]:.3e} splits {res[False][1]} n "
          f"{res[False][2]}; absgrad: mean statistic {res[True][0]:.3e} splits {res[True][1]} n {res[True][2]}")
    assert res[False][0] < 0.0002 and res[False][1] == 0 and res[False][2] == 1
    assert res[True][0] > 0.0008 and res[True][1] == 1 and res[True][2] == 2


# ------------------------------------------------------------------------------------------------- 4. quality
def _texture_scene(V=9, H=96, W=128, seed=0):
    """Ground truth rendered from a teacher of small Gaussians on the plane z = 0 coloured by a fine pattern
    (stripes of 0.06 units, about 3 px, crossed by a checkerboard of 0.5 units), V + 1 cameras on an arc (the last one
    held out)."""
    from opensplat_b200.model import Camera
    from opensplat_b200.trainer import SplatTrainer
    rng = np.random.default_rng(seed)
    f = np.float32
    g = np.stack(np.meshgrid(np.arange(-1.6, 1.6, 0.02), np.arange(-1.2, 1.2, 0.02)), -1).reshape(-1, 2)
    n = g.shape[0]
    pat = ((np.floor(g[:, 0] / 0.06) % 2) * 0.7 + 0.15 + 0.15 * ((np.floor(g[:, 0] / 0.5) + np.floor(g[:, 1] / 0.5))
                                                              % 2)).astype(f)
    col = np.stack([pat, 0.6 * pat + 0.2, 1.0 - pat], -1)
    teacher = {"means": np.concatenate([g, np.zeros((n, 1))], -1).astype(f),
               "scales": np.log(np.full((n, 3), 0.012)).astype(f), "quats": np.tile(np.array([1, 0, 0, 0], f), (n, 1)),
               "featuresDc": ((col - 0.5) / 0.28209479177387814).astype(f),
               "featuresRest": np.zeros((n, 3, 3), f), "opacities": np.full((n, 1), 4.0, f)}
    cams = []
    for v in range(V + 1):
        a = 0.3 * (v / V - 0.5) + (0.017 if v == V else 0.0)
        c2w = np.eye(4, dtype=f)
        c2w[:3, :3] = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]], dtype=f)
        c2w[:3, 3] = np.array([-3.0 * np.sin(a), 0.0, 3.0 * np.cos(a)], dtype=f)
        cams.append(Camera(W, H, 0.9 * W, 0.9 * W, W / 2.0, H / 2.0, c2w))
    t = SplatTrainer({k: torch.from_numpy(x) for k, x in teacher.items()}, device=DEV)
    gts = torch.stack([t.render(c, 1)["rgb"].clone() for c in cams])
    m = 600                                           # the coarse student: large, grey, random on the plane
    student = {"means": np.concatenate([rng.uniform(-1.6, 1.6, (m, 1)), rng.uniform(-1.2, 1.2, (m, 1)),
                                        rng.normal(0, 0.02, (m, 1))], -1).astype(f),
               "scales": np.log(np.full((m, 3), 0.08)).astype(f), "quats": rng.standard_normal((m, 4)).astype(f),
               "featuresDc": np.zeros((m, 3), f), "featuresRest": np.zeros((m, 3, 3), f),
               "opacities": np.full((m, 1), 0.5, f)}
    return student, cams, gts


def _psnr(a, b):
    mse = float(((a.clamp(0, 1) - b) ** 2).mean())
    return 10 * math.log10(1.0 / mse)


def test_quality_on_fine_texture():
    """Plain refinement at 0.0002 against absgrad at 0.0008 on the same coarse start (DESIGN D25 records the numbers).
    Measured on an H100 80GB HBM3 at 700 W: plain 16.42 dB with 29 350 Gaussians, absgrad 16.00 dB with 19 841.  The
    assertions are those numbers with a margin: absgrad reaches about the same PSNR with about a third fewer
    Gaussians on this scene; it is not better here."""
    student, cams, gts = _texture_scene()
    V = len(cams) - 1
    steps = 3000
    res = {}
    for absgrad, thresh in ((False, 0.0002), (True, 0.0008)):
        cfg = densify.RefineConfig(refine_every=100, warmup_length=500, reset_alpha_every=30, max_steps=steps,
                                   num_cameras=V, densify_grad_thresh=thresh, absgrad=absgrad)
        tr = _trainer(student, cfg)
        for s in range(1, steps + 1):
            v = (s - 1) % V
            tr.step(cams[v], gts[v], s)
        out = tr.render(cams[V], steps)["rgb"]
        res[absgrad] = (_psnr(out, gts[V]), tr.n)
    print(f"\nheld-out PSNR / Gaussians after {steps} steps: plain@0.0002 {res[False][0]:.2f} dB / {res[False][1]}; "
          f"absgrad@0.0008 {res[True][0]:.2f} dB / {res[True][1]}")
    (pp, pn), (ap, an) = res[False], res[True]
    assert pp > 15.0 and ap > 15.0 and abs(ap - pp) < 1.5
    assert an < 0.85 * pn
