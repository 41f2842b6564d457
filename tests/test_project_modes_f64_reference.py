"""Pins tests/project_modes_f64.py, the float64 reference of every cell of the activated projection's mode matrix
(CPU only), mode by mode on random and constructed-edge scenes:
  * the trees' values (the kernel's operation tree on value-plus-bound numbers) are those of float64 autograd of the
    mode's map, written from the definitions, so the bound is taken along the right computation;
  * the same trees evaluated on fp32 numbers -- the kernel's operations in its order, each rounded (project.cu is built
    with --fmad=false and IEEE div / sqrt) -- lie within C B of the float64 values on every certified element, per
    element, with no quantile and no aggregate norm: the bound holds an fp32 evaluation before any GPU sees it;
  * each known wrong convention (project_modes_f64.ALTS) is rejected on most of the certified Gaussians it changes."""
import numpy as np
import pytest
import torch

import project_modes_f64 as pm

C = 2.0          # as project_f64: the second-order terms B drops, and u |exact| where the fp32 result is |computed|
SCENES = ("random", "edges")


def _scene(mode, kind, n=1500):
    return pm.scene(mode, n, 3) if kind == "random" else pm.edge_scene(mode, 4, n=n)


def _ref(mode, sc, c):
    """The reference with the backward given the certified kept Gaussians as radii > 0, as the GPU test does."""
    r = pm.reference(mode, sc)
    keep = r["kept"] & r["cert"]
    return pm.reference(mode, sc, cot=c, kept=keep), keep


@pytest.mark.parametrize("kind", SCENES)
@pytest.mark.parametrize("mode", pm.MODES)
def test_trees_are_the_autograd_values(mode, kind):
    sc = _scene(mode, kind)
    for c in pm.cotangent_sets(sc.n, 5):
        r, keep = _ref(mode, sc, c)
        assert float(r["cert"].double().mean()) >= 0.95 and int(keep.sum()) > sc.n // 2
        g = pm.autograd(mode, sc, c, keep)
        for nm, gv in zip(pm.GRADS, g[:4]):
            d = (r[nm] - gv).abs()
            row = gv.abs().reshape(sc.n, -1).amax(-1).reshape((sc.n,) + (1,) * (gv.dim() - 1))
            # 1e-2 B: the fisheye series' dropped terms (in B) and float64 autograd's own cancellation near comp = 0
            ok = d <= 1e-9 * row + 1e-2 * r["B_" + nm]
            assert bool(ok.all()), (nm, float((d / r["B_" + nm].clamp_min(1e-300)).max()))
            assert float(gv.abs().max()) > 0
        for nm, G, B in (("GV", g[4], r["BV"]), ("GP", g[5], r["BP"])):
            assert bool(((r[nm] - G).abs() <= 1e-9 * G.abs().max() + 1e-2 * B).all()), nm
        assert not bool(r["GV"][3].any()) and not bool(r["GP"][2].any())
        if pm.flags(mode)[2]:
            assert not bool(r["GP"].any()) and not bool(r["BP"].any())


def _within(got, want, bound, mask, what):
    err = (got.double() - want).abs()
    m = mask if err.dim() == 1 else mask[:, None].expand_as(err)
    over = (err > C * bound) & m
    assert not bool(over.any()), (what, torch.nonzero(over)[:4].tolist(),
                                  float((err[m] / bound[m].clamp_min(1e-300)).max()))
    return float((err[m] / (C * bound[m]).clamp_min(1e-300)).max()) if bool(m.any()) else 0.0


def _stack(rs):
    return torch.stack([r.v for r in rs], -1), torch.stack([r.b for r in rs], -1)


@pytest.mark.parametrize("kind", SCENES)
@pytest.mark.parametrize("mode", pm.MODES)
def test_fp32_restatement_is_within_the_bound(mode, kind):
    aa, f3d, fish = pm.flags(mode)
    sc = _scene(mode, kind)
    worst = {}
    for ci, c in enumerate(pm.cotangent_sets(sc.n, 6)):
        r, keep = _ref(mode, sc, c)
        cert = r["cert"]
        f64, f32 = r["fw"], pm.forward_trees(mode, sc, torch.float32)
        a, b = f64["f"], f32["f"]
        sel = cert & r["kept"]
        for nm, key in (("cov3d", "cov3d"), ("conics", "conic"), ("xys", "xy")):
            v, bd = _stack(a[key])
            worst[nm] = _within(_stack(b[key])[0], v, bd, sel, nm)
        worst["depths"] = _within(b["t"][2].v, a["t"][2].v, a["t"][2].b, sel, "depths")
        op64, op32 = (fw["oe"] * fw["comp"] if aa else fw["oe"] for fw in (f64, f32))
        worst["opacities"] = _within(op32.v, op64.v, op64.b, cert & (r["kept"] | (not aa)), "opacities")
        b64 = pm.backward_trees(mode, sc, f64, c, keep)
        b32 = pm.backward_trees(mode, sc, f32, c, keep)
        for nm in pm.GRADS:
            v, bd = _stack(b64[nm]) if isinstance(b64[nm], list) else (b64[nm].v, b64[nm].b)
            g = _stack(b32[nm])[0] if isinstance(b32[nm], list) else b32[nm].v
            worst[f"{nm}.{ci}"] = _within(g, v, bd, cert, nm)
        v, bd = _stack(b64["terms"])
        worst[f"camgrad.{ci}"] = _within(_stack(b32["terms"])[0], v, bd, keep, "camgrad terms")
    print(f"\n{mode} {kind}: certified {float(r['cert'].double().mean()):.4f}; worst err/(C B) "
          + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))


# each wrong convention and the modes it is checked in
ALT_MODES = [("no_share", "f3d"), ("no_share", "f3d_aa"), ("share_cancel", "f3d"), ("no_glob_scale", "f3d"),
             ("no_glob_scale", "f3d_aa"), ("c3_twice", "f3d_aa"), ("unfiltered_camgrad", "f3d"),
             ("unfiltered_camgrad", "f3d_aa"), ("no_Jderiv", "fish"), ("no_Jderiv", "fish_aa"),
             ("series_sign", "fish"), ("series_sign", "fish_aa")]


@pytest.mark.parametrize("alt,mode", ALT_MODES)
def test_check_rejects_known_wrong_conventions(alt, mode):
    """Each alternative must fail |alt - reference| <= C B on most of the certified Gaussians whose outputs it changes
    (forward outputs, the four VJP outputs and the 24 camera-gradient terms).  The alternatives are evaluated on the
    float64 trees, except share_cancel: 1 - r^2 equals (f / sigma)^2 in exact arithmetic and differs only in fp32,
    where it cancels for f << s, so it is evaluated on fp32 numbers over Gaussians with 0 < f < s / 100, with the
    opacity's cotangent alone (the geometric part of v_scale would otherwise set its bound).
    unfiltered_camgrad runs over Gaussians with f > s / 10 (below, sigma and s agree to fp32 precision); series_sign
    on the edge scene, whose Gaussians crowd the series branch."""
    sc = pm.scene(mode, 2000, 11) if alt != "series_sign" else pm.edge_scene(mode, 12, n=2000)
    dtype = torch.float32 if alt == "share_cancel" else torch.float64
    if alt in ("share_cancel", "unfiltered_camgrad"):
        e = sc.glob_scale * np.exp(sc.scales.astype(np.float64))
        sel = ((sc.f3 > 0) & (sc.f3 < 0.01 * e.min(1))) if alt == "share_cancel" else sc.f3 > 0.1 * e.min(1)
        sc = pm.Scene(sc.cam, sc.means[sel], sc.scales[sel], sc.quats[sel], sc.logits[sel], sc.glob_scale, sc.f3[sel])
    changed = torch.zeros(sc.n, dtype=torch.bool)
    rejected = torch.zeros(sc.n, dtype=torch.bool)
    op = (lambda w: w["oe"] * w["comp"]) if pm.flags(mode)[0] else (lambda w: w["oe"])

    def outputs(fw, bw):
        """Every compared output as [N, k] (values, bounds)."""
        outs = [_stack(fw["f"][k]) for k in ("cov3d", "conic", "xy")] + [(op(fw).v[:, None], op(fw).b[:, None])]
        for nm in pm.GRADS + ("terms",):
            x = bw[nm]
            outs.append(_stack(x) if isinstance(x, list) else (x.v[:, None], x.b[:, None]))
        return outs

    cots = pm.cotangent_sets(sc.n, 13)
    if alt == "share_cancel":
        cots = [{k: (v if k == "v_opacity" else np.zeros_like(v)) for k, v in cots[0].items()}]
    for c in cots:
        r, keep = _ref(mode, sc, c)
        cert = r["cert"]
        ref = outputs(r["fw"], pm.backward_trees(mode, sc, r["fw"], c, keep))
        fa, fb = pm.forward_trees(mode, sc, dtype, alt=alt), pm.forward_trees(mode, sc, dtype)
        got = outputs(fa, pm.backward_trees(mode, sc, fa, c, keep, alt))
        base = outputs(fb, pm.backward_trees(mode, sc, fb, c, keep))
        for (g, _), (b, _), (want, bound) in zip(got, base, ref):
            g, b = g.double(), b.double()
            changed |= torch.where(cert[:, None], (g - b).abs() > 1e-12 * (want.abs() + bound / pm.pf.U), False).any(-1)
            rejected |= torch.where(cert[:, None], (g - want).abs() > C * bound, False).any(-1)
    n_changed = int(changed.sum())
    frac = float((rejected & changed).sum()) / max(n_changed, 1)
    print(f"\n{alt} in {mode}: changes {n_changed} certified Gaussians, rejected on {frac:.4f} of them")
    assert n_changed >= 50
    assert frac >= 0.6, frac
