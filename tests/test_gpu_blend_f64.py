"""The blend kernels pixel by pixel and Gaussian by Gaussian against the float64 reference of tests/blend_f64.py.

Every case runs through
  (a) the generic path: binAndSortGaussians -> ops.rasterize_forward -> ops.rasterize_backward (unculled lists);
  (b) the fast operator path: RasterizeGaussians through autograd (culled bucket binning, longest-first tile order,
      planned capacities);
  (c) the clamped operator path: RasterizeGaussiansClamped, for the cases whose colours exceed 1.
The reference always blends the UNCULLED lists, so a cull that drops a contributing pair shows up as a wrong pixel.

On the pixels and Gaussians the reference certifies (no threshold decision within fp32 rounding of its boundary),
with no flip allowance and no aggregate norm:
  * final_idx matches exactly (paths b / c: the Gaussian of the last blended pair, and the clamp bits);
  * out_img and final_Ts within C_FWD u ((n_p + 8) A + B) per element;
  * each component of v_xy, v_conic, v_colors, v_opacity within C_BWD u (B + (8 + n_tiles) A),
with u = 2^-24, n_p the pairs blended at the pixel, n_tiles the tiles the Gaussian is binned to, and A / B the
reference's magnitude and error scale of the element (blend_f64.py).  B already carries the worst-case relative error
of every alpha (ex2.approx, the fma into the exponent, the rounding of sigma) amplified through T; the constants cover
what A and the counts leave implicit:
  C_FWD = 2: each blended pair adds at most one rounding to the colour fma and one to T (n_p A); the 8 covers the
             background term and the final additions.
  C_BWD = 4: the backward's per-pixel rcp.approx (1 ulp) and its T *= 1/(1 - alpha) per pair are in B; the 4 covers
             the order of the sums (8 pixels per lane, the 5-level lane butterfly, then the Gaussian's rows in order,
             counted by 8 + n_tiles) and the moment -> gradient map applied once per Gaussian.
Each case must certify >= 99 % of its pixels and >= 95 % of its Gaussians; the worst err / bound ratio of each case is
printed (run with -s)."""
import time

import numpy as np
import pytest
import torch

import blend_f64 as bf
from opensplat_b200 import ops
from opensplat_b200.scene import make_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = bf.U
C_FWD = 2.0
C_BWD = 4.0
SAT_MASK = 7 << 28


def cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _radii(conics):
    """ceil(3 sqrt(lambda_max)) of the covariance inverse to `conics` (the projection's radius rule)."""
    a, b, c = conics[:, 0].astype(np.float64), conics[:, 1].astype(np.float64), conics[:, 2].astype(np.float64)
    det = a * c - b * b
    ca, cc = c / det, a / det
    mid = 0.5 * (ca + cc)
    lam = mid + np.sqrt(np.maximum(0.1, mid * mid - (ca * cc - (b / det) ** 2)))
    return np.ceil(3 * np.sqrt(lam)).astype(np.int32)


def _conics(s_major, s_minor, theta):
    """Conic (inverse covariance a, b, c) of ellipses with std devs s_major / s_minor px rotated by theta."""
    ct, st = np.cos(theta), np.sin(theta)
    l1, l2 = s_major.astype(np.float64) ** 2, s_minor.astype(np.float64) ** 2
    sxx, syy, sxy = ct * ct * l1 + st * st * l2, st * st * l1 + ct * ct * l2, ct * st * (l1 - l2)
    det = sxx * syy - sxy * sxy
    return np.stack([syy / det, -sxy / det, sxx / det], -1).astype(np.float32)


class Case:
    """Synthetic 2D inputs (cases A-E) or the projection's output (case F), with per-pixel cotangents."""

    def __init__(self, W, H, xys, conics, colors, opac, bg, seed, radii=None, depths=None, voa=False):
        rng = np.random.default_rng(seed)
        n = xys.shape[0]
        self.W, self.H, self.n = W, H, n
        self.xys = xys if torch.is_tensor(xys) else cu(xys)
        self.conics = conics if torch.is_tensor(conics) else cu(conics)
        self.colors = colors if torch.is_tensor(colors) else cu(colors)
        self.opac = opac if torch.is_tensor(opac) else cu(np.asarray(opac).reshape(n, 1))
        self.bg = cu(np.asarray(bg, np.float32))
        if radii is None:
            radii = cu(_radii(self.conics.cpu().numpy()), torch.int32)
        if depths is None:
            depths = cu(rng.permutation(n).astype(np.float32) + 1.0)       # unique depths
        self.radii, self.depths = radii, depths
        self.v_out = cu(rng.uniform(-1, 1, (H, W, 3)).astype(np.float32))
        self.voa = cu(rng.uniform(-1, 1, (H, W)).astype(np.float32)) if voa else None
        self.tb = ops.tile_bounds(W, H)
        _, _, st, _ = ops.bucket_tile_ranges(self.xys, self.radii, self.conics, self.colors, self.opac, self.tb, 0, 0,
                                             cull=False)
        m, max_len = (int(v) for v in st.tolist()[:2])
        _, self.cum, _, _ = ops.bucket_tile_ranges(self.xys, self.radii, self.conics, self.colors, self.opac, self.tb,
                                                   m, max_len, cull=False)
        self.m = m
        self.nth = torch.diff(self.cum, prepend=torch.zeros(1, dtype=torch.int32, device=DEV)).to(torch.int32)
        _, _, _, self.gs, self.bins, self.idx = ops.binAndSortGaussians(n, m, self.xys, self.depths, self.radii,
                                                                        self.cum, self.tb, return_index=True)

    def reference(self, clamp=False, voa=True):
        return bf.blend(self.gs, self.bins, self.xys, self.conics, self.colors, self.opac, self.bg, self.H, self.W,
                        v_output=self.v_out, v_output_alpha=self.voa if voa else None, clamp=clamp)


def _ratio(err, bound):
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _check(name, case, ref, out, fT, fI_match, grads, sat_bits=None):
    pc, gc = ref["pix_cert"], ref["gauss_cert"]
    fp, fg = float(pc.double().mean()), float(gc.double().mean())
    assert fp >= 0.99 and fg >= 0.95, f"{name}: certified pixels {fp:.4f}, Gaussians {fg:.4f} -- change the case"
    bad = ~fI_match & pc
    assert not bool(bad.any()), f"{name}: final_idx differs at certified pixels {torch.nonzero(bad)[:8].tolist()}"
    if sat_bits is not None:
        sb = torch.stack([(ref["sat"][..., i]).long() << i for i in range(3)], -1).sum(-1)
        badc = (sat_bits != sb) & pc
        assert not bool(badc.any()), f"{name}: clamp bits differ at {torch.nonzero(badc)[:8].tolist()}"
    k = (ref["n_blend"] + 8).double()
    worst = {}
    for nm, got, want, A, B, kk in (("out_img", out, ref["out_img"], ref["A_out"], ref["B_out"], k[..., None]),
                                    ("final_Ts", fT, ref["final_Ts"], ref["A_T"], ref["B_T"], k)):
        bound = C_FWD * U * (kk * A + B)
        err = (got.double() - want).abs()
        m = pc[..., None].expand_as(err) if err.dim() == 3 else pc
        worst[nm] = _ratio(err[m], bound[m])
        over = (err > bound) & m
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
        worst[nm] = _ratio(err[m], bound[m])
        over = (err > bound) & m
        if bool(over.any()):
            g, j = torch.nonzero(over)[0].tolist()
            pytest.fail(f"{name}: {nm}[{g}, {j}]: kernel {float(got[g, j])!r} reference {float(ref[nm][g, j])!r} "
                        f"bound {float(bound[g, j]):.3e} (A {float(ref['A_' + nm][g, j]):.3e})")
    print(f"\n{name}: certified pixels {fp:.5f} Gaussians {fg:.5f}; worst err/bound "
          + " ".join(f"{k_}={v:.3f}" for k_, v in worst.items()))


def _run(name, case, paths=("a", "b")):
    ref = None
    if "a" in paths:
        ref = case.reference(voa=True)
        out, fT, fI, rec = ops.rasterize_forward(case.tb, (case.W, case.H, 1), case.gs, case.idx, case.bins, case.xys,
                                                 case.conics, case.colors, case.opac, case.bg)
        v = ops.rasterize_backward(case.H, case.W, case.n, case.m, case.bins, case.conics, case.opac, rec, case.cum,
                                   case.bg, fT, fI, case.v_out, case.voa)
        _check(name + "/a", case, ref, out, fT, fI.long() == ref["final_idx"],
               dict(zip(("v_xy", "v_conic", "v_colors", "v_opacity"), v)))
    for p, op in (("b", ops.RasterizeGaussians), ("c", ops.RasterizeGaussiansClamped)):
        if p not in paths:
            continue
        clamp = p == "c"
        # the operators take no v_output_alpha
        r = ref if (ref is not None and case.voa is None and not clamp) else case.reference(clamp=clamp, voa=False)
        xys, conics, colors, opac = (t.clone().requires_grad_() for t in (case.xys, case.conics, case.colors,
                                                                          case.opac))
        img = op.apply(xys, case.depths, case.radii, conics, case.nth, colors, opac, case.H, case.W, case.bg)
        saved = img.grad_fn.saved_tensors
        (img * case.v_out).sum().backward()
        rec, cum_c, fT, fI = saved[3], saved[4], saved[6], saved[7]
        # the fast path's sorted indices are its own (culled lists): compare the Gaussian of the last blended pair
        fi = (fI & ~SAT_MASK).long()
        q = rec.view(torch.int32)
        k = q[: q.numel() // 12 * 12].view(-1, 12)[fi, 3].long()
        g_kernel = torch.searchsorted(cum_c.long(), k, right=True)
        g_ref = case.gs.long()[r["final_idx"].clamp(max=max(case.m - 1, 0))] if case.m else torch.zeros_like(fi)
        match = torch.where(r["n_blend"] > 0, g_kernel == g_ref, fi == 0)
        _check(name + "/" + p, case, r, img.detach(), fT, match,
               dict(v_xy=xys.grad, v_conic=conics.grad, v_colors=colors.grad, v_opacity=opac.grad),
               sat_bits=(fI >> 28) & 7 if clamp else None)


# ---------------------------------------------------------------------------------------------------------- cases
def _blobs(rng, n, lo_x, hi_x, lo_y, hi_y, s=(1.0, 8.0), opac=(0.05, 0.9), colors=(0.0, 1.0)):
    xys = np.stack([rng.uniform(lo_x, hi_x, n), rng.uniform(lo_y, hi_y, n)], -1).astype(np.float32)
    sm = rng.uniform(*s, n)
    con = _conics(sm, sm * rng.uniform(0.3, 1.0, n), rng.uniform(0, np.pi, n))
    col = rng.uniform(*colors, (n, 3)).astype(np.float32)
    return xys, con, col, rng.uniform(*opac, n).astype(np.float32)


@pytest.mark.parametrize("W,H", [(1, 1), (1, 23), (23, 1), (15, 15), (16, 16), (17, 17), (31, 33), (100, 72)])
def test_A_ragged_images(W, H):
    """Lanes and slots outside the image, the partial last tile row and column; half the splats are centred outside
    the image with a footprint that enters it."""
    rng = np.random.default_rng(W * 1000 + H)
    n = 40 + (W * H) // 8
    xi, ci, coli, oi = _blobs(rng, n // 2, 0, W, 0, H)
    xo, co, colo, oo = _blobs(rng, n - n // 2, -12, W + 12, -12, H + 12, s=(3.0, 8.0))
    outside = (xo[:, 0] < 0) | (xo[:, 0] > W) | (xo[:, 1] < 0) | (xo[:, 1] > H)
    xo[~outside, 0] = np.where(rng.uniform(size=(~outside).sum()) < 0.5, -rng.uniform(1, 10, (~outside).sum()),
                               W + rng.uniform(1, 10, (~outside).sum()))
    c = Case(W, H, np.concatenate([xi, xo]), np.concatenate([ci, co]), np.concatenate([coli, colo]),
             np.concatenate([oi, oo]), [0.1, 0.3, 0.6], seed=W + H)
    _run(f"A {W}x{H}", c)


@pytest.mark.parametrize("k", [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 4097])
def test_B_one_tile_list_length(k):
    """One 16x16 tile whose list holds exactly k pairs: the 32-record chunk and 4-stage ring boundaries, and the
    zero rows behind the last contributor once the pixels saturate."""
    rng = np.random.default_rng(k)
    if k <= 1024:
        xys, con, col, op = _blobs(rng, k, -4, 20, -4, 20, s=(1.5, 6.0), opac=(0.01, 0.12))
    else:   # small splats, so that an undecided pixel is shared by few of the k Gaussians
        xys, con, col, op = _blobs(rng, k, 0, 16, 0, 16, s=(0.8, 2.5), opac=(0.005, 0.05))
    c = Case(16, 16, xys, con, col, op, [0.4, 0.2, 0.1], seed=k)
    assert c.m == k and int(c.bins[0, 1] - c.bins[0, 0]) == k
    _run(f"B k={k}", c)


@pytest.mark.parametrize("regime,opac", [("faint", (0.004, 0.02)), ("mid", (0.05, 0.35)), ("opaque", (0.9, 1.0))])
def test_C_opacity_regimes(regime, opac):
    """The alpha threshold (faint: alpha near 1/255 over much of each footprint), both alpha clamps (0.999 forward,
    0.99 backward) and early termination (opaque); non-zero background, v_output_alpha on the generic path."""
    rng = np.random.default_rng(len(regime))
    W, H = 100, 72
    n = {"faint": 1500, "mid": 600, "opaque": 300}[regime]
    xys, con, col, op = _blobs(rng, n, -5, W + 5, -5, H + 5, s=(1.0, 6.0), opac=opac)
    c = Case(W, H, xys, con, col, op, [0.3, 0.6, 0.2], seed=7, voa=True)
    _run(f"C {regime}", c)


@pytest.mark.parametrize("variant", ["needles", "centred", "cover"])
def test_D_extent_cull(variant):
    """The extent cull and slot mask, jlo/jhi dispatch and the multi-tile row reduce: needles with anisotropy
    1e2-1e6 at random angles; sub-pixel splats centred exactly on pixel centres and on tile edges (dx = 0 or dy = 0
    exactly); splats that cover every tile."""
    rng = np.random.default_rng(len(variant))
    W, H = 100, 72
    if variant == "needles":
        n = 24
        xys = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], -1).astype(np.float32)
        s_minor = rng.uniform(0.5, 2.0, n)
        aniso = 10 ** rng.uniform(2, 6, n)                      # ratio of the covariance's eigenvalues
        con = _conics(s_minor * np.sqrt(aniso), s_minor, rng.uniform(0, np.pi, n))
        op = rng.uniform(0.05, 0.9, n).astype(np.float32)
        xb, cb, _, ob = _blobs(rng, 150, 0, W, 0, H, opac=(0.05, 0.5))
        xys, con, op = np.concatenate([xys, xb]), np.concatenate([con, cb]), np.concatenate([op, ob])
    elif variant == "centred":
        n = 600
        px = rng.integers(0, W, n).astype(np.float32)
        py = rng.integers(0, H, n).astype(np.float32)
        px[: n // 4] = rng.choice([0, 15, 16, 31, 32, 47, 48, 63, 64, 79, 80, 95, 96], n // 4)
        py[n // 4: n // 2] = rng.choice([0, 15, 16, 31, 32, 47, 48, 63, 64], n // 4)
        xys = np.stack([px, py], -1)
        xys[n // 2:, 0] += rng.choice([0.0, 0.5], n - n // 2).astype(np.float32)   # dy = 0 exactly, dx = 0.5
        sm = rng.uniform(0.2, 0.7, n)
        con = _conics(sm, sm * rng.uniform(0.5, 1.0, n), rng.uniform(0, np.pi, n))
        op = rng.uniform(0.05, 1.0, n).astype(np.float32)
    else:
        n = 40
        xys = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], -1).astype(np.float32)
        sm = rng.uniform(40, 120, n)
        con = _conics(sm, sm * rng.uniform(0.5, 1.0, n), rng.uniform(0, np.pi, n))
        op = rng.uniform(0.01, 0.08, n).astype(np.float32)
    col = rng.uniform(0, 1, (xys.shape[0], 3)).astype(np.float32)
    c = Case(W, H, xys, con, col, op, [0.2, 0.2, 0.5], seed=11)
    _run(f"D {variant}", c)


def test_E_colours_above_one_clamp():
    """Colours in [0, 2]: about half of the pixels clamp -- the clamp bits in final_idx and the gradient mask."""
    rng = np.random.default_rng(5)
    W, H = 100, 72
    xys, con, col, op = _blobs(rng, 800, -5, W + 5, -5, H + 5, s=(1.5, 5.0), opac=(0.08, 0.7), colors=(0.0, 2.0))
    c = Case(W, H, xys, con, col, op, [0.1, 0.1, 0.1], seed=5)
    sat = c.reference(clamp=True, voa=False)["sat"].any(-1)
    assert 0.1 < float(sat.double().mean()) < 0.7
    _run("E", c, paths=("a", "b", "c"))


@pytest.mark.parametrize("n,W,H,scale", [(1_000_000, 1920, 1080, 0.02), (100_000, 320, 192, 0.17)])
def test_F_projected_scenes(n, W, H, scale):
    """The C2 scene of test_full_size_properties_and_oracle (SH degree 3) and a dense C5-like scene: persistent
    scheduling and tile order at full size, long lists."""
    t0 = time.time()
    sc = make_scene(n, W, H, scale=scale, sh_degree=3, opacity=(0.05, 0.95), seed=0)
    col = torch.clamp_min(ops.compute_sh_forward(3, 3, cu(sc["viewdirs"]), cu(sc["coeffs"])) + 0.5, 0.0)
    tb = ops.tile_bounds(W, H)
    _, xys, depths, radii, conics, _ = ops.project_gaussians_forward(
        cu(sc["means"]), cu(sc["scales"]), 1.0, cu(sc["quats"]), cu(sc["viewmat"]), cu(sc["projmat"]), sc["fx"],
        sc["fy"], sc["cx"], sc["cy"], H, W, tb)
    c = Case(W, H, xys, conics, col, cu(sc["opacities"]), [0.0, 0.0, 0.0], seed=0, radii=radii, depths=depths)
    _run(f"F n={n} {W}x{H}", c)
    print(f"F n={n}: {time.time() - t0:.1f} s")
