"""GPU: the depth and opacity maps of the blend kernels (DESIGN D18) and everything built on them.

1. The DEPTH instantiations leave colour alone: out_img, final_Ts and final_idx identical to the plain kernels, and with
   no depth cotangent the colour gradients compare equal (-0 == +0), with and without GSB_RASTER_CLAMP_MAX_ONE.
2. Against the float64 reference of tests/depth_f64.py on certified pixels and Gaussians, with the bounds and constants
   of test_gpu_blend_f64 and its case builders, depths spanning 0.02 ... 1e3: depth, alpha and every gradient,
   v_depths included, on the generic path and through the autograd operator (fast path).
3. The full chain against the reference's own numbers (tests/golden/depth_*.npz) in Python and through the C++ ops.
4. Both binning paths give the same maps bit for bit, a frame redone after outgrowing its capacity plan gives what a
   frame that fits gives, and the per-record depth gather writes nothing past M.
5. Edge cases: no Gaussians, nothing visible, a 1x1 image.
6. SplatTrainer.render: its rgb is evaluate()'s image, normalize_depth, and renders between steps change no step."""
import types

import numpy as np
import pytest
import torch

import depth_f64 as df
import test_gpu_blend_f64 as tb
from opensplat_b200 import capi, ops
from opensplat_b200.scene import make_scene
from util import image_close, load_golden, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U, C_FWD, C_BWD = tb.U, tb.C_FWD, tb.C_BWD
CLAMP = ops.CLAMP_MAX_ONE
GOLDEN = [("depth_tight_100x72", 2e-3, 1e-3), ("depth_bg_quat_128x96", 2e-3, 1e-3), ("depth_opaque_96x96", 2e-2, 1e-2)]


def cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _depths(rng, n):
    """Distinct view-space depths log-uniform in [0.02, 1e3]."""
    d = np.exp(rng.uniform(np.log(0.02), np.log(1e3), n))
    d = np.sort(d)[rng.permutation(n)]
    d = d * (1.0 + 1e-6 * np.arange(n)[rng.permutation(n)])   # ties impossible
    return cu(d.astype(np.float32))


# ---------------------------------------------------------------------------------------------- generic-path helpers
def _forward(case, flags, depth):
    """The generic path on the case's unculled lists: pack, gather, blend; returns (out, fT, fI, depth, alpha, records,
    record_depths)."""
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    H, W, m = case.H, case.W, case.m
    rec = torch.empty(L.gsb_raster_records_bytes(m), dtype=torch.uint8, device=DEV)
    capi.check(L.gsb_pack_records(m, P(case.gs), P(case.idx), P(case.xys), P(case.conics), P(case.colors),
                                  P(case.opac), P(rec), s))
    out = torch.empty((H, W, 3), device=DEV)
    fT = torch.empty((H, W), device=DEV)
    fI = torch.empty((H, W), dtype=torch.int32, device=DEV)
    if not depth:
        capi.check(L.gsb_rasterize_forward_packed(H, W, case.tb[0], case.tb[1], m, P(case.bins), None, None,
                                                  P(case.bg), P(rec), P(out), P(fT), P(fI), flags, s))
        return out, fT, fI, None, None, rec, None
    rd = torch.empty(max(m, 1), device=DEV)
    capi.check(L.gsb_gather_record_depths(m, P(case.gs), P(case.depths), None, P(rd), s))
    od, oa = torch.empty((H, W), device=DEV), torch.empty((H, W), device=DEV)
    capi.check(L.gsb_rasterize_forward_packed_depth(H, W, case.tb[0], case.tb[1], m, P(case.bins), None, None,
                                                    P(case.bg), P(rec), P(out), P(fT), P(fI), flags, P(rd), P(od),
                                                    P(oa), s))
    return out, fT, fI, od, oa, rec, rd


def _backward(case, fwd, flags, v_out, voa, v_depth=None, depth=True):
    out, fT, fI, od, oa, rec, rd = fwd
    return ops.rasterize_backward(case.H, case.W, case.n, case.m, case.bins, case.conics, case.opac, rec, case.cum,
                                  case.bg, fT, fI, v_out, voa, flags=flags, record_depths=rd if depth else None,
                                  v_output_depth=v_depth)


# ------------------------------------------------------------------------------- 1. colour untouched by the DEPTH path
def _small_case(W, H, n, seed, colors=(0.0, 1.0)):
    rng = np.random.default_rng(seed)
    xys, con, col, op = tb._blobs(rng, n, -5, W + 5, -5, H + 5, s=(1.0, 6.0), opac=(0.05, 0.95), colors=colors)
    return tb.Case(W, H, xys, con, col, op, [0.3, 0.6, 0.2], seed=seed, depths=_depths(rng, n), voa=True)


def _c2_case(n=1_000_000, W=1920, H=1080, scale=0.02, seed=0):
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=(0.05, 0.95), seed=seed)
    col = torch.clamp_min(ops.compute_sh_forward(3, 3, cu(sc["viewdirs"]), cu(sc["coeffs"])) + 0.5, 0.0)
    t = ops.tile_bounds(W, H)
    _, xys, depths, radii, conics, _ = ops.project_gaussians_forward(
        cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"],
        sc["fy"], sc["cx"], sc["cy"], H, W, t)
    return tb.Case(W, H, xys, conics, col, cu(sc["opacities"]), [0.0, 0.0, 0.0], seed=seed, radii=radii,
                   depths=depths, voa=True)


def _assert_colour_untouched(case):
    for flags in (0, CLAMP):
        a, b = _forward(case, flags, False), _forward(case, flags, True)
        for x, y in zip(a[:3], b[:3]):
            assert torch.equal(x, y)
        ga = _backward(case, a, flags, case.v_out, case.voa, depth=False)
        gb = _backward(case, b, flags, case.v_out, case.voa)
        for x, y in zip(ga, gb[:4]):
            assert torch.equal(x, y)      # == compares -0 and +0 equal
        assert float(gb[4].abs().max()) == 0.0 if case.n else True   # no depth cotangent: no depth gradient


@pytest.mark.parametrize("W,H,n", [(1, 1, 5), (17, 17, 60), (100, 72, 600)])
def test_depth_kernels_leave_colour_alone(W, H, n):
    _assert_colour_untouched(_small_case(W, H, n, W + H, colors=(0.0, 1.5)))


def test_depth_kernels_leave_colour_alone_c2():
    _assert_colour_untouched(_c2_case())


# -------------------------------------------------------------------------------- 2. against the float64 reference
def _check_depth(name, ref, od, oa, grads):
    pc, gc = ref["pix_cert"], ref["gauss_cert"]
    k = (ref["n_blend"] + 8).double()
    worst = {}
    for nm, got, want, A, B in (("depth", od, ref["out_depth"], ref["A_depth"], ref["B_depth"]),
                                # alpha = 1 - T_final: T's error plus the rounding of the subtraction
                                ("alpha", oa, ref["out_alpha"], ref["A_T"], ref["B_T"] + ref["out_alpha"])):
        bound = C_FWD * U * (k * A + B)
        err = (got.double() - want).abs()
        worst[nm] = tb._ratio(err[pc], bound[pc])
        over = (err > bound) & pc
        if bool(over.any()):
            p = torch.nonzero(over)[0].tolist()
            pytest.fail(f"{name}: {nm} at {p}: kernel {float(got[tuple(p)])!r} reference {float(want[tuple(p)])!r} "
                        f"bound {float(bound[tuple(p)]):.3e}")
    nt = ref["n_tiles"][:, None]
    for nm, got in grads.items():
        got = got.double().reshape(ref[nm].shape)
        bound = C_BWD * U * (ref["B_" + nm] + (8 + nt) * ref["A_" + nm])
        err = (got - ref[nm]).abs()
        m = gc[:, None].expand_as(err)
        worst[nm] = tb._ratio(err[m], bound[m])
        over = (err > bound) & m
        if bool(over.any()):
            g, j = torch.nonzero(over)[0].tolist()
            pytest.fail(f"{name}: {nm}[{g}, {j}]: kernel {float(got[g, j])!r} reference {float(ref[nm][g, j])!r} "
                        f"bound {float(bound[g, j]):.3e}")
    print(f"\n{name}: worst err/bound " + " ".join(f"{a}={v:.3f}" for a, v in worst.items()))


def _run(name, case, clamp_path=False):
    rng = np.random.default_rng(case.n)
    vd = cu(rng.uniform(-1, 1, (case.H, case.W)).astype(np.float32))
    voa = case.voa if case.voa is not None else cu(rng.uniform(-1, 1, (case.H, case.W)).astype(np.float32))
    args = (case.gs, case.bins, case.xys, case.conics, case.colors, case.opac, case.depths, case.bg, case.H, case.W)
    ref = df.blend_depth(*args, v_output=case.v_out, v_output_depth=vd, v_output_alpha=voa)
    fwd = _forward(case, 0, True)
    tb._check(name + "/a", case, ref, fwd[0], fwd[1], fwd[2].long() == ref["final_idx"], {})
    g = _backward(case, fwd, 0, case.v_out, voa, vd)
    _check_depth(name + "/a", ref, fwd[3], fwd[4], dict(zip(("v_xy", "v_conic", "v_colors", "v_opacity", "v_depths"), g)))
    # the autograd operator on the fast path (culled lists, tile order, planned capacities)
    for op, clamp in ((ops.RasterizeGaussiansDepth, False), (ops.RasterizeGaussiansDepthClamped, True)):
        if clamp and not clamp_path:
            continue
        r = ref if not clamp else df.blend_depth(*args, v_output=case.v_out, v_output_depth=vd, v_output_alpha=voa,
                                                 clamp=True)
        xys, depths, conics, colors, opac = (t.clone().requires_grad_() for t in (case.xys, case.depths, case.conics,
                                                                                  case.colors, case.opac))
        img, od, oa = op.apply(xys, depths, case.radii, conics, case.nth, colors, opac, case.H, case.W, case.bg)
        ((img * case.v_out).sum() + (od * vd).sum() + (oa * voa).sum()).backward()
        _check_depth(name + ("/c" if clamp else "/b"), r, od.detach(), oa.detach(),
                     dict(v_xy=xys.grad, v_conic=conics.grad, v_colors=colors.grad, v_opacity=opac.grad,
                          v_depths=depths.grad))


@pytest.mark.parametrize("W,H", [(1, 23), (15, 15), (31, 33), (100, 72)])
def test_f64_ragged_images(W, H):
    rng = np.random.default_rng(W * 1000 + H)
    n = 40 + (W * H) // 8
    xys, con, col, op = tb._blobs(rng, n, -12, W + 12, -12, H + 12, s=(1.0, 8.0))
    c = tb.Case(W, H, xys, con, col, op, [0.1, 0.3, 0.6], seed=W + H, depths=_depths(rng, n))
    _run(f"A {W}x{H}", c)


@pytest.mark.parametrize("k", [1, 32, 33, 129, 4097])
def test_f64_list_lengths(k):
    rng = np.random.default_rng(k)
    if k <= 1024:
        xys, con, col, op = tb._blobs(rng, k, -4, 20, -4, 20, s=(1.5, 6.0), opac=(0.01, 0.12))
    else:
        xys, con, col, op = tb._blobs(rng, k, 0, 16, 0, 16, s=(0.8, 2.5), opac=(0.005, 0.05))
    c = tb.Case(16, 16, xys, con, col, op, [0.4, 0.2, 0.1], seed=k, depths=_depths(rng, k))
    assert c.m == k
    _run(f"B k={k}", c)


@pytest.mark.parametrize("regime,opac", [("faint", (0.004, 0.02)), ("mid", (0.05, 0.35)), ("opaque", (0.9, 1.0))])
def test_f64_opacity_regimes(regime, opac):
    rng = np.random.default_rng(len(regime))
    W, H = 100, 72
    n = {"faint": 1500, "mid": 600, "opaque": 300}[regime]
    xys, con, col, op = tb._blobs(rng, n, -5, W + 5, -5, H + 5, s=(1.0, 6.0), opac=opac, colors=(0.0, 2.0))
    c = tb.Case(W, H, xys, con, col, op, [0.3, 0.6, 0.2], seed=7, depths=_depths(rng, n), voa=True)
    _run(f"C {regime}", c, clamp_path=True)


@pytest.mark.parametrize("variant", ["needles", "cover"])
def test_f64_needles_and_cover(variant):
    rng = np.random.default_rng(len(variant))
    W, H = 100, 72
    if variant == "needles":
        n = 24
        xys = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], -1).astype(np.float32)
        s_minor = rng.uniform(0.5, 2.0, n)
        con = tb._conics(s_minor * np.sqrt(10 ** rng.uniform(2, 6, n)), s_minor, rng.uniform(0, np.pi, n))
        op = rng.uniform(0.05, 0.9, n).astype(np.float32)
        xb, cb, _, ob = tb._blobs(rng, 150, 0, W, 0, H, opac=(0.05, 0.5))
        xys, con, op = np.concatenate([xys, xb]), np.concatenate([con, cb]), np.concatenate([op, ob])
    else:
        n = 40
        xys = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], -1).astype(np.float32)
        sm = rng.uniform(40, 120, n)
        con = tb._conics(sm, sm * rng.uniform(0.5, 1.0, n), rng.uniform(0, np.pi, n))
        op = rng.uniform(0.01, 0.08, n).astype(np.float32)
    col = rng.uniform(0, 1, (xys.shape[0], 3)).astype(np.float32)
    c = tb.Case(W, H, xys, con, col, op, [0.2, 0.2, 0.5], seed=11, depths=_depths(rng, xys.shape[0]))
    _run(f"D {variant}", c)


@pytest.mark.parametrize("n,W,H,scale", [(1_000_000, 1920, 1080, 0.02), (100_000, 320, 192, 0.17)])
def test_f64_projected_scenes(n, W, H, scale):
    _run(f"F n={n} {W}x{H}", _c2_case(n, W, H, scale))


# ------------------------------------------------------------------------------------- 3. the chain against golden
def _golden_inputs(g):
    fx, fy, cx, cy = [float(v) for v in g["intrins"]]
    H, W = [int(v) for v in g["hw"]]
    return fx, fy, cx, cy, H, W


def _check_golden(g, img, depth, alpha, grads, gtol, frac):
    scale = float(np.abs(g["ref_depth"]).max())
    for got, want, s in ((img, g["ref_img"], 1.0), (depth[..., None], g["ref_depth"][..., None], scale),
                         (alpha[..., None], g["ref_alpha"][..., None], 1.0)):
        ok, st = image_close(got.detach().cpu().numpy() / s, want / s, tol=5e-5, frac=frac)
        assert ok, st
    for got, ref in grads:
        assert rel_l2(got.cpu().numpy().reshape(g[ref].shape), g[ref]) <= gtol, (ref, rel_l2(got.cpu().numpy(),
                                                                                            g[ref]))


@pytest.mark.parametrize("name,gtol,frac", GOLDEN)
def test_chain_vs_reference_golden(name, gtol, frac):
    from opensplat_b200 import cpp_ops
    g = load_golden(name)
    fx, fy, cx, cy, H, W = _golden_inputs(g)
    vm, pm, bg = cu(g["viewmat"]), cu(g["projmat"]), cu(g["background"])
    results = []
    for impl in ("python", "cpp"):
        means, scales, quats = (cu(g[k]).requires_grad_() for k in ("means", "scales", "quats"))
        colors, opac = cu(g["colors"]).requires_grad_(), cu(g["opacities"]).requires_grad_()
        if impl == "python":
            xys, depths, radii, conics, nth, _ = ops.ProjectGaussians.apply(means, scales, 1.0, quats, vm, pm, fx, fy,
                                                                            cx, cy, H, W, ops.tile_bounds(W, H))
            img, depth, alpha = ops.RasterizeGaussiansDepth.apply(xys, depths, radii, conics, nth, colors, opac, H, W,
                                                                  bg)
        else:
            o = cpp_ops.ops()
            xys, depths, radii, conics, nth, _ = o.project_gaussians(means, scales, 1.0, quats, vm, pm, fx, fy, cx, cy,
                                                                     H, W, 0.01)
            img, depth, alpha = o.rasterize_gaussians_depth(xys, depths, radii, conics, nth, colors, opac, H, W, bg)
        xys.retain_grad(); depths.retain_grad()
        ((img * cu(g["wgt"])).sum() + (depth * cu(g["wgt_depth"])).sum() + (alpha * cu(g["wgt_alpha"])).sum()).backward()
        _check_golden(g, img, depth, alpha, [(xys.grad, "ref_v_xy"), (depths.grad, "ref_v_z"),
                                             (colors.grad, "ref_v_colors"), (opac.grad, "ref_v_opacity"),
                                             (means.grad, "ref_v_means"), (scales.grad, "ref_v_scales"),
                                             (quats.grad, "ref_v_quats")], gtol, frac)
        results.append([img, depth, alpha, means.grad, scales.grad, quats.grad])
    for a, b in zip(*results):      # the two operator layers drive the same C ABI
        assert torch.equal(a, b)


@pytest.mark.parametrize("name,gtol,frac", GOLDEN[:2])
def test_activated_chain_vs_reference_golden(name, gtol, frac):
    """ProjectGaussiansActivated (log-scales, raw quats, opacity logits) -> RasterizeGaussiansDepthClamped, Python and
    C++ (colours below 1 and a background below 1: the clamp never acts on these images)."""
    from opensplat_b200 import cpp_ops
    g = load_golden(name)
    fx, fy, cx, cy, H, W = _golden_inputs(g)
    vm, pm, bg = cu(g["viewmat"]), cu(g["projmat"]), cu(g["background"])
    out = []
    for impl in ("python", "cpp"):
        means, quats = cu(g["means"]).requires_grad_(), cu(g["quats"]).requires_grad_()
        ls = torch.log(cu(g["scales"])).requires_grad_()
        ol = torch.logit(cu(g["opacities"]).double()).float().requires_grad_()
        colors = cu(g["colors"])
        if impl == "python":
            p = ops.ProjectGaussiansActivated.apply(means, ls, 1.0, quats, ol, vm, pm, fx, fy, cx, cy, H, W,
                                                    ops.tile_bounds(W, H))
            img, depth, alpha = ops.RasterizeGaussiansDepthClamped.apply(p[0], p[1], p[2], p[3], p[4], colors, p[6],
                                                                         H, W, bg)
        else:
            o = cpp_ops.ops()
            p = o.project_gaussians_activated(means, ls, 1.0, quats, ol, vm, pm, fx, fy, cx, cy, H, W, 0.01)
            img, depth, alpha = o.rasterize_gaussians_depth_clamped(p[0], p[1], p[2], p[3], p[4], colors, p[6], H, W,
                                                                    bg)
        ((img * cu(g["wgt"])).sum() + (depth * cu(g["wgt_depth"])).sum() + (alpha * cu(g["wgt_alpha"])).sum()).backward()
        _check_golden(g, img, depth, alpha, [(means.grad, "ref_v_means"), (quats.grad, "ref_v_quats")], gtol, frac)
        assert rel_l2((ls.grad / torch.exp(ls.detach())).cpu().numpy(), g["ref_v_scales"]) <= gtol
        out.append([img, depth, alpha, means.grad, ls.grad, quats.grad, ol.grad])
    for a, b in zip(*out):
        assert torch.equal(a, b)


# --------------------------------------------------------------------------- 4. binning paths, redo, the gather
def _projected(n, W, H, scale, opacity, seed, squeeze=False):
    sc = make_scene(n, W, H, scale=scale, sh_degree=0, opacity=opacity, seed=seed)
    if squeeze:      # every Gaussian in a few tiles: lists longer than the in-shared-memory sort takes
        sc["means"][:, 0] = 0.25 + sc["means"][:, 0] * 0.05
        sc["means"][:, 1] = sc["means"][:, 1] * 0.05
    t = ops.tile_bounds(W, H)
    _, xys, depths, radii, conics, nth = ops.project_gaussians_forward(
        cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"],
        sc["fy"], sc["cx"], sc["cy"], H, W, t)
    col = cu(np.random.default_rng(seed).uniform(0, 1, (n, 3)).astype(np.float32))
    return xys, depths, radii, conics, nth, col, cu(sc["opacities"])


def _op_run(inputs, H, W, bg, w, op=ops.RasterizeGaussiansDepth):
    xys, depths, radii, conics, nth, col, opac = inputs
    x, d, c, cl, o = (t.clone().requires_grad_() for t in (xys, depths, conics, col, opac))
    img, od, oa = op.apply(x, d, radii, c, nth, cl, o, H, W, bg)
    ((img * w[0]).sum() + (od * w[1]).sum() + (oa * w[2]).sum()).backward()
    return [img.detach(), od.detach(), oa.detach(), x.grad, d.grad, c.grad, cl.grad, o.grad]


def _generic_maps(inputs, H, W, bg):
    """The depth frame on the generic path (reference-exact global sort of the unculled lists)."""
    xys, depths, radii, conics, nth, col, opac = inputs
    n = xys.shape[0]
    cum = ops.cumsum_tiles_hit(nth)
    m = int(cum[-1])
    t = ops.tile_bounds(W, H)
    _, _, _, gs, bins, idx = ops.binAndSortGaussians(n, m, xys, depths, radii, cum, t, return_index=True)
    case = types.SimpleNamespace(H=H, W=W, m=m, n=n, gs=gs, idx=idx, bins=bins, tb=t, xys=xys, conics=conics,
                                 colors=col, opac=opac, depths=depths, bg=bg)
    return _forward(case, 0, True)


def test_fast_and_generic_paths_give_the_same_maps():
    W, H = 128, 96
    inputs = _projected(3000, W, H, 0.5, (0.05, 0.9), seed=3)
    bg = torch.tensor([0.2, 0.9, 0.5], device=DEV)
    w = (torch.randn(H, W, 3, device=DEV), torch.randn(H, W, device=DEV), torch.randn(H, W, device=DEV))
    fast = _op_run(inputs, H, W, bg, w)
    gen = _generic_maps(inputs, H, W, bg)
    for a, b in ((fast[0], gen[0]), (fast[1], gen[3]), (fast[2], gen[4])):
        assert torch.equal(a, b)
    plain = ops.RasterizeGaussians.apply(*inputs[:5], inputs[5], inputs[6], H, W, bg)
    assert torch.equal(plain, fast[0])


def test_generic_fallback_inside_the_operator():
    """Tile lists longer than gsb_bucket_max_tile_len(): the operator takes the generic path for both outputs."""
    n, W, H = 24_000, 64, 48
    inputs = _projected(n, W, H, 0.5, (0.0045, 0.01), seed=n, squeeze=True)
    xys, depths, radii, conics, nth = inputs[:5]
    _, _, st, _ = ops.bucket_tile_ranges(xys, radii, conics, inputs[5], inputs[6], ops.tile_bounds(W, H), 0, 0)
    assert int(st[1]) > capi.lib().gsb_bucket_max_tile_len()
    bg = torch.tensor([0.2, 0.9, 0.5], device=DEV)
    w = (torch.randn(H, W, 3, device=DEV), torch.randn(H, W, device=DEV), torch.randn(H, W, device=DEV))
    got = _op_run(inputs, H, W, bg, w)
    gen = _generic_maps(inputs, H, W, bg)
    for a, b in ((got[0], gen[0]), (got[1], gen[3]), (got[2], gen[4])):
        assert torch.equal(a, b)
    assert float(got[2].max()) > 0.5 and float(got[4].abs().max()) > 0


def test_redone_frame_equals_a_frame_that_fits():
    W, H = 160, 128
    inputs = _projected(5000, W, H, 0.5, (0.05, 0.9), seed=4)
    bg = torch.tensor([0.6130, 0.0101, 0.3984], device=DEV)
    w = (torch.randn(H, W, 3, device=DEV), torch.randn(H, W, device=DEV), torch.randn(H, W, device=DEV))
    dev = torch.device(DEV).index or 0
    saved = ops._plans.get(dev)
    try:
        for op in (ops.RasterizeGaussiansDepth, ops.RasterizeGaussiansDepthClamped):
            ops._plans[dev] = ops.BinPlan()        # empty plan: the first frame overflows and is redone
            redone = _op_run(inputs, H, W, bg, w, op)
            m_cap = ops._plans[dev].m_cap
            assert m_cap > 0
            fits = _op_run(inputs, H, W, bg, w, op)  # the grown plan: fits at once
            assert ops._plans[dev].m_cap == m_cap
            for a, b in zip(redone, fits):
                assert torch.equal(a, b)
    finally:
        if saved is not None:
            ops._plans[dev] = saved


def test_gather_writes_only_below_m():
    L, P, s = capi.lib(), capi.ptr, capi.stream()
    n, m_cap, M = 100, 1000, 613
    depths = torch.rand(n, device=DEV) + 1.0
    ids = torch.randint(0, n, (m_cap,), dtype=torch.int32, device=DEV)   # valid ids everywhere, even past M
    stats = torch.tensor([M, 7, 0, 0], dtype=torch.int32, device=DEV)
    rd = torch.full((m_cap,), float("nan"), device=DEV)
    capi.check(L.gsb_gather_record_depths(m_cap, P(ids), P(depths), P(stats), P(rd), s))
    assert torch.equal(rd[:M], depths[ids[:M].long()])
    assert bool(torch.isnan(rd[M:]).all())
    stats[2] = 1                                                        # overflow: nothing is written
    rd.fill_(float("nan"))
    capi.check(L.gsb_gather_record_depths(m_cap, P(ids), P(depths), P(stats), P(rd), s))
    assert bool(torch.isnan(rd).all())
    capi.check(L.gsb_gather_record_depths(m_cap, P(ids), P(depths), None, P(rd), s))   # generic path: all m
    assert torch.equal(rd, depths[ids.long()])


# ----------------------------------------------------------------------------------------------------- 5. edges
def _edge(xys, depths, radii, conics, nth, col, opac, H, W, bg):
    out = []
    for op in (ops.RasterizeGaussiansDepth, ops.RasterizeGaussiansDepthClamped):
        x, d, c, cl, o = (t.clone().requires_grad_() for t in (xys, depths, conics, col, opac))
        img, od, oa = op.apply(x, d, radii, c, nth, cl, o, H, W, bg)
        ((img * 0.5).sum() + od.sum() + oa.sum()).backward()
        out.append((img, od, oa, [x.grad, d.grad, c.grad, cl.grad, o.grad]))
    return out


def test_no_gaussians():
    z = lambda *s: torch.zeros(*s, device=DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    for img, od, oa, grads in _edge(z(0, 2), z(0), torch.zeros(0, dtype=torch.int32, device=DEV), z(0, 3),
                                    torch.zeros(0, dtype=torch.int32, device=DEV), z(0, 3), z(0, 1), 24, 40, bg):
        assert torch.equal(img, bg.expand(24, 40, 3)) and float(od.abs().max()) == 0 and float(oa.abs().max()) == 0
        assert all(g.numel() == 0 for g in grads)


def test_nothing_visible_and_one_pixel():
    rng = np.random.default_rng(0)
    n, W, H = 50, 40, 24
    xys, con, col, op = tb._blobs(rng, n, 0, W, 0, H)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    zero_r = torch.zeros(n, dtype=torch.int32, device=DEV)      # radii 0: no Gaussian is binned
    for img, od, oa, grads in _edge(cu(xys), _depths(rng, n), zero_r, cu(con), zero_r, cu(col), cu(op[:, None]), H, W,
                                    bg):
        assert torch.equal(img, bg.expand(H, W, 3)) and float(od.abs().max()) == 0 and float(oa.abs().max()) == 0
        assert all(float(g.abs().max()) == 0 for g in grads)
    # a 1x1 image against the float64 reference
    c = tb.Case(1, 1, np.array([[0.3, -0.2], [0.0, 0.0]], np.float32), tb._conics(np.array([1.0, 2.0]),
                np.array([0.8, 1.5]), np.array([0.3, 1.0])), np.array([[0.2, 0.5, 0.9], [0.7, 0.1, 0.3]], np.float32),
                np.array([0.6, 0.4], np.float32), [0.3, 0.3, 0.3], seed=1, depths=cu(np.array([0.5, 40.0], np.float32)))
    _run("1x1", c, clamp_path=True)


# ------------------------------------------------------------------------------------- 6. SplatTrainer.render
def _trainer_problem():
    from test_gpu_trainer import _cams, make_problem
    p, c2w, gts, intr, H, W = make_problem(n=3000)
    return p, _cams(c2w, H, W, intr), torch.from_numpy(gts).to(DEV)


def test_render_matches_evaluate_and_normalizes():
    from opensplat_b200.trainer import SplatTrainer
    p, cams, gts = _trainer_problem()
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, device=DEV)
    for step in (1, 2):
        tr.step(cams[0], gts[0], step)
    tr.evaluate(cams[1], gts[1], 3)
    image = tr.image.clone()
    r = tr.render(cams[1], 3)
    assert torch.equal(r["rgb"], image) and torch.equal(tr.image, image)    # render() leaves `image` alone
    depth, alpha = r["depth"].clone(), r["alpha"].clone()
    assert float(alpha.max()) > 0.5 and float(alpha.min()) >= 0 and float(depth.max()) > 1.0
    rn = tr.render(cams[1], 3, normalize_depth=True)
    assert torch.equal(rn["alpha"], alpha) and torch.equal(rn["rgb"], image)
    vis = alpha > 0
    assert torch.allclose(rn["depth"][vis], depth[vis] / alpha[vis], rtol=1e-6, atol=0)
    assert float(rn["depth"][~vis].abs().max()) == 0 if bool((~vis).any()) else True
    # normalised depth lies between the nearest and farthest view-space depth of the blended Gaussians
    d = tr.pipe.depths[tr.pipe.radii > 0]
    assert float(rn["depth"][alpha > 1e-3].min()) >= float(d.min()) * (1 - 1e-5)
    assert float(rn["depth"].max()) <= float(d.max()) * (1 + 1e-5)


def test_render_between_steps_changes_no_step():
    """Renders between steps, through two refinements: Gaussian counts, parameters and Adam state stay bit-identical;
    the losses agree to the float-atomic summation order of the loss kernel."""
    from opensplat_b200.trainer import SplatTrainer
    from test_gpu_trainer import refine_config
    p, cams, gts = _trainer_problem()
    runs = []
    for with_render in (False, True):
        tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, refine_config(), device=DEV,
                          generator=torch.Generator(device=DEV).manual_seed(3))
        losses = []
        for step in range(1, 31):
            if with_render and step % 3 == 0:
                tr.render(cams[2], step, normalize_depth=step % 2 == 0)
            losses.append(tr.step(cams[(step - 1) % 2], gts[(step - 1) % 2], step).clone())
        torch.cuda.synchronize()
        runs.append((tr.n, torch.stack(losses), tr.params(), tr.adam_state()))
    (n0, l0, p0, (m0, v0)), (n1, l1, p1, (m1, v1)) = runs
    assert n0 == n1
    assert float((l0 - l1).abs().max()) <= 1e-6
    for k in p0:
        assert torch.equal(p0[k], p1[k]) and torch.equal(m0[k], m1[k]) and torch.equal(v0[k], v1[k]), k
