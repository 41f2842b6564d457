"""Every cell of the activated projection's mode matrix Gaussian by Gaussian against the float64 reference of
tests/project_modes_f64.py (trees pinned by tests/test_project_modes_f64_reference.py).

CELLS lists the cells: six activated modes x {write, ACC} x {CAMGRAD off, on} x {v_depth given, NULL} x {v_opacity
given, NULL}, plus the non-activated pair; between them they reach every instantiation of project_forward_kernel and
project_backward_kernel that the kernels' static_asserts allow.  Each cell runs once through its C entry point and
once through ops.project_activated_forward / project_activated_backward, which must give the same bits.  On the
certified Gaussians (every decision of the forward clear of its threshold by its bound), per element, with no
quantile:
  * radii and num_tiles_hit match exactly, and cov3d, xys, depths, conics, opacities lie within C B;
  * the four VJP outputs lie within C B, under two cotangent sets (random, and v_conic with v_opacity alone).  The
    backward is given the kernel's radii with the uncertified Gaussians' set to 0, so it is checked on every Gaussian:
    the culled ones' outputs are the opacity's terms alone (F3D's share of v_scale included);
  * ACC gives prior + write bit for bit;
  * CAMGRAD leaves the per-Gaussian outputs bit-identical, its partial rows are deterministic and each lies within
    the bound of its block's 256 Gaussians, and the reduced v_viewmat / v_projmat lie within their bound per element,
    with v_viewmat[3], v_projmat[2] and (fisheye) all of v_projmat exactly 0.
Each cell must certify >= 99 % of its Gaussians (>= 90 % on the constructed-edge scenes); with -s each scene and mode
prints its certified fraction and each cell's worst err/bound."""
import time

import numpy as np
import pytest
import torch

import project_f64 as pf
import project_modes_f64 as pm
from opensplat_b200 import capi, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = pf.U
C_FWD = C_BWD = 2.0
OUTS = ("v_mean3d", "v_scale", "v_quat", "v_opacity_logits")
FWD_OUTS = ("cov3d", "xys", "depths", "radii", "conics", "num_tiles_hit", "opacities")

# mode: the forward kernel's template flags (ACT, AA, F3D, FISH)
MODE_FLAGS = {"plain": (0, 0, 0, 0), "act": (1, 0, 0, 0), "aa": (1, 1, 0, 0), "f3d": (1, 0, 1, 0),
              "f3d_aa": (1, 1, 1, 0), "fish": (1, 0, 0, 1), "fish_aa": (1, 1, 0, 1)}
# the cells: (mode, acc, camgrad, v_depth given, v_opacity given); the non-activated pair has no ACC, CAMGRAD or opacity
CELLS = [("plain", 0, 0, vd, 0) for vd in (1, 0)] + [
    (m, acc, cg, vd, vo) for m in pm.MODES for acc in (0, 1) for cg in (0, 1) for vd in (1, 0) for vo in (1, 0)]


def _legal(act, acc, aa, camgrad, f3d, fish):
    """The kernels' static_asserts (and pj_legal in project.cu): every mode needs ACT, and FISH excludes F3D."""
    return (act or not (acc or aa or camgrad or f3d or fish)) and not (f3d and fish)


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_cell_table_covers_every_instantiation():
    fwd = {(a, aa, f, fi) for a, aa, f, fi in np.ndindex(2, 2, 2, 2) if _legal(a, 0, aa, 0, f, fi)}
    bwd = {t for t in np.ndindex(*(2,) * 6) if _legal(*t)}
    assert len(fwd) == 7 and len(bwd) == 25
    got_f = {MODE_FLAGS[m] for m, *_ in CELLS}
    got_b = set()
    for m, acc, cg, _, _ in CELLS:
        act, aa, f3d, fish = MODE_FLAGS[m]
        got_b.add((act, acc, aa, cg, f3d, fish))
    assert got_f == fwd and got_b == bwd
    assert len(CELLS) == len(set(CELLS)) == 2 + 6 * 16


# ------------------------------------------------------------------------------------------------ the calls
def cu(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype).contiguous()


class Dev:
    """A scene's device inputs and the arguments both paths share."""

    def __init__(self, mode, sc):
        self.mode, self.sc, self.n = mode, sc, sc.n
        self.aa, self.f3d, self.fish = pm.flags(mode)
        cam = sc.cam
        self.m, self.s, self.q, self.l = cu(sc.means), cu(sc.scales), cu(sc.quats), cu(sc.logits)
        self.f3 = cu(sc.f3) if self.f3d else None
        self.V = cu(cam.V.reshape(4, 4))
        self.P = None if self.fish else cu(cam.P.reshape(4, 4))
        self.fk = (*cam.k, cam.theta_lim) if self.fish else None
        self.tb = ops.tile_bounds(cam.W, cam.H)
        self.pm = ops.ProjectionMode(self.aa, self.f3, self.fk)

    def empty_fwd(self):
        n = self.n
        return [torch.empty(sh, device=DEV, dtype=dt) for sh, dt in (
            ((n, 6), torch.float32), ((n, 2), torch.float32), ((n,), torch.float32), ((n,), torch.int32),
            ((n, 3), torch.float32), ((n,), torch.int32), ((n,), torch.float32))]

    def forward_direct(self):
        L, P, st, c = capi.lib(), capi.ptr, capi.stream(), self.sc.cam
        out = self.empty_fwd()
        head = (self.n, P(self.m), P(self.s), self.sc.glob_scale, P(self.q), P(self.l))
        tail = (c.H, c.W, self.tb[0], self.tb[1], c.clip) + tuple(P(t) for t in out)
        if self.fish:
            capi.check(L.gsb_project_forward_fisheye(*head, P(self.V), c.fx, c.fy, c.cx, c.cy, *self.fk, *tail,
                                                     int(self.aa), st))
        elif self.f3d:
            capi.check(L.gsb_project_forward_activated_filter3d(*head, P(self.f3), P(self.V), P(self.P), c.fx, c.fy,
                                                                c.cx, c.cy, *tail, int(self.aa), st))
        else:
            fn = L.gsb_project_forward_activated_aa if self.aa else L.gsb_project_forward_activated
            capi.check(fn(*head, P(self.V), P(self.P), c.fx, c.fy, c.cx, c.cy, *tail, st))
        return dict(zip(FWD_OUTS, out))

    def forward_ops(self):
        c = self.sc.cam
        out = self.empty_fwd()
        ops.project_activated_forward(capi.lib(), self.pm, self.n, self.m, self.s, self.sc.glob_scale, self.q, self.l,
                                      self.V, self.P, c.fx, c.fy, c.cx, c.cy, c.H, c.W, self.tb, c.clip, out,
                                      capi.stream())
        return dict(zip(FWD_OUTS, out))

    def backward_direct(self, fw, radii, cot, grads, acc, partials):
        """The cell's C entry point; partials: the CAMGRAD rows (None: CAMGRAD off)."""
        L, P, st, c = capi.lib(), capi.ptr, capi.stream(), self.sc.cam
        plain = not (self.aa or self.f3d or self.fish)
        head = (self.n, P(self.m), P(self.s), self.sc.glob_scale, P(self.q), P(fw["opacities"] if plain else self.l))
        tail = ((c.H, c.W, P(radii), P(fw["conics"]), P(cot["v_xy"]), P(cot["v_depth"]), P(cot["v_conic"]),
                 P(cot["v_opacity"])) + tuple(P(g) for g in grads))
        if self.fish:
            capi.check(L.gsb_project_backward_fisheye(*head, P(self.V), c.fx, c.fy, *self.fk, *tail, acc, int(self.aa),
                                                      P(partials), st))
        elif self.f3d:
            capi.check(L.gsb_project_backward_activated_filter3d(*head, P(self.f3), P(self.V), P(self.P), c.fx, c.fy,
                                                                 *tail, acc, int(self.aa), int(partials is not None),
                                                                 P(partials), st))
        elif partials is not None:
            capi.check(L.gsb_project_backward_activated_camgrad(*head, P(self.V), P(self.P), c.fx, c.fy, *tail, acc,
                                                                int(self.aa), P(partials), st))
        else:
            fn = {(0, 0): L.gsb_project_backward_activated, (1, 0): L.gsb_project_backward_activated_acc,
                  (0, 1): L.gsb_project_backward_activated_aa, (1, 1): L.gsb_project_backward_activated_aa_acc}
            capi.check(fn[acc, int(self.aa)](*head, P(self.V), P(self.P), c.fx, c.fy, *tail, st))

    def reduce(self, partials):
        vv, vp = torch.full((4, 4), float("nan"), device=DEV), torch.full((4, 4), float("nan"), device=DEV)
        capi.check(capi.lib().gsb_project_camera_grad_reduce(partials.numel() // capi.CAMGRAD_TERMS,
                                                             capi.ptr(partials), capi.ptr(vv), capi.ptr(vp),
                                                             capi.stream()))
        return vv, vp

    def backward_ops(self, fw, radii, cot, grads, acc, cam_grad):
        c = self.sc.cam
        ops.project_activated_backward(capi.lib(), self.pm, self.n, self.m, self.s, self.sc.glob_scale, self.q,
                                       self.l, fw["opacities"], self.V, self.P, c.fx, c.fy, c.H, c.W, radii,
                                       fw["conics"], cot["v_xy"], cot["v_depth"], cot["v_conic"], cot["v_opacity"],
                                       grads, capi.stream(), accumulate=bool(acc), cam_grad=cam_grad)


# ------------------------------------------------------------------------------------------------ the checks
class Worst:
    def __init__(self, name):
        self.name, self.r = name, {}

    def check(self, tag, got, want, bound, mask):
        got = got.double().reshape(want.shape)
        err = (got - want).abs()
        m = mask if err.dim() == 1 else mask[:, None].expand_as(err)
        if bool(m.any()):
            self.r[tag] = max(self.r.get(tag, 0.0), float((err[m] / bound[m].clamp_min(1e-300)).max()))
        over = (err > bound) & m
        if bool(over.any()):
            i = torch.nonzero(over)[0].tolist()
            pytest.fail(f"{self.name} {tag}{i}: kernel {float(got[tuple(i)])!r} reference {float(want[tuple(i)])!r} "
                        f"bound {float(bound[tuple(i)]):.3e}")


def _bits(tag, a, b):
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"{tag}: output {k} differs"


def _bwd_reference(mode, sc, fw, cot, kept):
    bw = pm.backward_trees(mode, sc, fw, cot, kept)
    r = {}
    for nm in OUTS:
        x = bw[nm]
        r[nm], r["B_" + nm] = pf.stack_masked(x if isinstance(x, list) else [x], torch.ones_like(kept))
    r["v_opacity_logits"], r["B_v_opacity_logits"] = r["v_opacity_logits"][:, 0], r["B_v_opacity_logits"][:, 0]
    r["GV"], r["GP"], r["BV"], r["BP"] = pm.pose.camgrad_sum(bw["terms"], kept)
    # each block's partial row: its 256 Gaussians' terms summed in fp32 over the kernel's tree (depth 12), so that a
    # wrong term shows against a bound of 256 Gaussians whatever n is
    n, nb = kept.shape[0], (kept.shape[0] + 255) // 256
    t, b = pf.stack_masked(bw["terms"], kept)
    pad = lambda x: torch.cat([x, x.new_zeros((nb * 256 - n, pm.pose.CG_ROW))]).reshape(nb, 256, pm.pose.CG_ROW)
    t, b = pad(t), pad(b)
    val, bsum, asum = t.sum(1), b.sum(1), t.abs().sum(1)
    r["rows"] = val
    r["B_rows"] = pm.pose.C * (bsum + pm.pose.gamma(pm.pose.TREE_DEPTH) * (asum + bsum)) + U * val.abs()
    return r


def run_scene(name, mode, sc, min_cert=0.99):
    t0 = time.time()
    d = Dev(mode, sc)
    n = sc.n
    ref = pm.reference(mode, sc, DEV)
    cert, kept = ref["cert"], ref["kept"]
    frac = float(cert.double().mean()) if n else 1.0
    assert frac >= min_cert, f"{name} {mode}: certified {frac:.4f}"
    w = Worst(f"{name} {mode}")
    fw = d.forward_direct()
    _bits(f"{name} {mode} forward ops", list(d.forward_ops().values()), list(fw.values()))
    for k in ("radii", "num_tiles_hit"):
        bad = (fw[k].long() != ref[k]) & cert
        assert not bool(bad.any()), f"{name} {mode} {k}: differs at certified {torch.nonzero(bad)[:8].tolist()}"
    for k in pm.FWD:
        w.check("fwd." + k, fw[k], ref[k], C_FWD * ref["B_" + k], cert)

    keep = cert & kept
    radii = torch.where(keep, fw["radii"], torch.zeros_like(fw["radii"]))
    allg = torch.ones(n, dtype=torch.bool, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(n + 17)
    for ci, c in enumerate(pm.cotangent_sets(n, n + 5)):
        for vd, vo in ((1, 1), (1, 0), (0, 1), (0, 0)):
            hc = dict(c, v_depth=c["v_depth"] if vd else None, v_opacity=c["v_opacity"] if vo else None)
            dc = {k: (cu(v) if v is not None else None) for k, v in hc.items()}
            r = _bwd_reference(mode, sc, ref["fw"], hc, keep)
            cell = f"{ci}{'d' if vd else '-'}{'o' if vo else '-'}"
            shapes = ((n, 3), (n, 3), (n, 4), (n,))
            prior = [torch.randn(sh, device=DEV, generator=g) * torch.exp(
                torch.empty(sh, device=DEV).uniform_(-3, 10, generator=g)) for sh in shapes]
            results = {}
            for acc in (0, 1):
                for cg in (0, 1):
                    tag = f"{cell}{'A' if acc else 'W'}{'C' if cg else '-'}"
                    outs = [p.clone() if acc else torch.full(p.shape, float("nan"), device=DEV) for p in prior]
                    part = torch.full((capi.lib().gsb_project_camera_partials_floats(n),), float("nan"),
                                      device=DEV) if cg else None
                    d.backward_direct(fw, radii, dc, outs, acc, part)
                    outs2 = [p.clone() if acc else torch.full(p.shape, float("nan"), device=DEV) for p in prior]
                    cam2 = (torch.full((4, 4), float("nan"), device=DEV), torch.full((4, 4), float("nan"),
                                                                                     device=DEV)) if cg else None
                    d.backward_ops(fw, radii, dc, outs2, acc, cam2)
                    _bits(f"{name} {mode} {tag} ops", outs2, outs)
                    results[acc, cg] = outs
                    if acc:
                        _bits(f"{name} {mode} {tag} prior + write", outs, [p + o for p, o in zip(prior, results[0, cg])])
                    else:
                        for k, o in zip(OUTS, outs):
                            w.check(f"bwd{cell}." + k, o, r[k], C_BWD * r["B_" + k], allg)
                    if cg:
                        _bits(f"{name} {mode} {tag} camgrad", outs, results[acc, 0])
                        part2 = torch.full_like(part, float("nan"))
                        again = [p.clone() if acc else torch.empty_like(p) for p in prior]
                        d.backward_direct(fw, radii, dc, again, acc, part2)
                        assert torch.equal(part, part2), f"{name} {mode} {tag}: partial rows differ between runs"
                        w.check(f"rows{cell}.", part.reshape(-1, pm.pose.CG_ROW), r["rows"], r["B_rows"],
                                torch.ones(r["rows"].shape[0], dtype=torch.bool, device=DEV))
                        vv, vp = d.reduce(part)
                        _bits(f"{name} {mode} {tag} ops camgrad", list(cam2), [vv, vp])
                        assert not bool(vv[3].any()) and not bool(vp[2].any())
                        if d.fish:
                            assert not bool(vp.any()), f"{name} {mode}: a fisheye projmat gradient is not 0"
                        w.check(f"cg{cell}.V", vv, r["GV"], r["BV"], torch.ones(4, dtype=torch.bool, device=DEV))
                        w.check(f"cg{cell}.P", vp, r["GP"], r["BP"], torch.ones(4, dtype=torch.bool, device=DEV))
    torch.cuda.synchronize()
    worst = max(w.r.values()) if w.r else 0.0
    print(f"\n{name} {mode}: n={n} certified {frac:.5f}; worst err/bound {worst:.3f} ("
          + " ".join(f"{k}={v:.3f}" for k, v in sorted(w.r.items())) + f") {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ the scenes
@pytest.mark.parametrize("mode", pm.MODES)
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 65537])
def test_counts(mode, n):
    """Ragged counts around the 256-thread block (and the camera gradient's per-block rows) at glob_scale 1.3, through
    a general camera (rotated, translated, fx != fy, off-centre principal point)."""
    run_scene(f"n={n}", mode, pm.scene(mode, n, seed=n + 1, W=640, H=360, glob_scale=1.3))


@pytest.mark.parametrize("mode", pm.MODES)
def test_edges(mode):
    """The constructed edges of project_modes_f64.edge_scene at glob_scale 0.7: log-scales -12 .. 3, logits -30 .. 30,
    the pinhole's clip plane and fov-clamp ties, the fisheye's axis, series switch, theta_lim and the space behind the
    camera, the filter's f = 0, f << s and f >> s, and comp near 0."""
    run_scene("edges", mode, pm.edge_scene(mode, seed=21, n=20000, glob_scale=0.7), min_cert=0.9)


@pytest.mark.parametrize("mode", pm.MODES)
def test_one_million_at_1080p(mode):
    """2^20 Gaussians at 1920x1080: 4096 blocks in the camera gradient's reduction."""
    run_scene("2^20 1920x1080", mode, pm.scene(mode, 1 << 20, seed=31, W=1920, H=1080, glob_scale=1.0))


def test_non_activated_pair():
    """The non-activated pair (gsb_project_forward / gsb_project_backward) on the same footing, through
    test_gpu_project_f64's runner."""
    from test_gpu_project_f64 import run_case
    cam = pf.camera_from_setup(pf.general_camera(640, 360, 41))
    m, s, q = pf.random_gaussians(cam, 65537, seed=42)
    run_case("plain n=65537", cam, m, s, q, 0.7)
