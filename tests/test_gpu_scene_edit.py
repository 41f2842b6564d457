"""GPU parity of the "next" rows of SURVEY.md 8f: topology edits (Model::afterTrain) and scene writers
(Model::savePly / saveSplat), through the C ABI, against (a) golden vectors produced by the unmodified reference
model.cpp and (b) the CPU restatement oracle/scene_edit.py.  The float64 checks of the same kernels, at scale and
with certified decisions, are in test_gpu_scene_edit_f64.py.

Tolerances: everything that is a copy or an integer decision is bit-exact (row map, counts, copied rows, Adam
moments, visCounts, max2DSize, PLY bytes without keepCrs, u8 fields of .splat rows wherever tests/scene_edit_f64.py
certifies them);
values that pass through exp/log/sqrt on the device are within a few ulp of the reference's ATen results
(rel 4e-6): split-child means / scales, xysGradNorm, keepCrs scales, .splat scale floats."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util import PARAM_NAMES, load_golden, scene_edit_inputs  # noqa: E402
from test_scene_edit_oracle import cfg_of  # noqa: E402
import scene_edit_f64 as sf  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ULP = 4e-6


def dev(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in d.items()}


def refine_cfg(c):
    from opensplat_b200.densify import RefineConfig
    return RefineConfig(refine_every=c.refine_every, warmup_length=c.warmup_length,
                        reset_alpha_every=c.reset_alpha_every, densify_grad_thresh=c.densify_grad_thresh,
                        densify_size_thresh=c.densify_size_thresh, stop_screen_size_at=c.stop_screen_size_at,
                        split_screen_size=c.split_screen_size, max_steps=c.max_steps, num_cameras=c.num_cameras)


def close(a, b, rel=ULP):
    a, b = a.detach().cpu().double(), torch.as_tensor(b).double()
    return bool(((a - b).abs() <= rel * (1.0 + b.abs())).all())


@pytest.mark.parametrize("name", ["scene_edit_densify_screen", "scene_edit_densify_huge", "scene_edit_densify_all",
                                  "scene_edit_alpha_reset"])
def test_after_train_matches_reference_golden(name):
    from opensplat_b200.densify import Densifier
    g = load_golden(name)
    n, k, seed = int(g["n"]), int(g["k"]), int(g["seed"])
    H, W = (int(x) for x in g["hw"])
    p, m, v, draws = scene_edit_inputs(n, k, seed, max(H, W))
    p, m, v = dev(p), dev(m), dev(v)

    def sample_fn(rows, device):   # the CPU stream Model::afterTrain's torch::randn drew from
        torch.manual_seed(int(g["seed_randn"]))
        return torch.randn(rows, 3)
    dn = Densifier(refine_cfg(cfg_of(g)), sample_fn=sample_fn)
    info = None
    for si, step in enumerate(int(s) for s in g["steps"]):
        v_xy, radii = draws[si]
        p, m, v, info = dn.after_train(step, p, m, v, torch.from_numpy(v_xy).to(DEV), torch.from_numpy(radii).to(DEV),
                                       H, W)
        ref_gn = g[f"s{si}_xysGradNorm"]
        if ref_gn.size == 0:
            assert dn.xys_grad_norm is None
        else:
            assert close(dn.xys_grad_norm, ref_gn)
            assert torch.equal(dn.vis_counts.cpu(), torch.from_numpy(g[f"s{si}_visCounts"]))
            assert torch.equal(dn.max_2d_size.cpu(), torch.from_numpy(g[f"s{si}_max2DSize"]))
    assert info["refined"]
    for x in PARAM_NAMES:
        assert tuple(p[x].shape) == g["p_" + x].shape, (x, p[x].shape, g["p_" + x].shape)
    for x in ("quats", "featuresDc", "featuresRest"):
        assert torch.equal(p[x].cpu(), torch.from_numpy(g["p_" + x])), x
    if name == "scene_edit_alpha_reset":
        assert torch.equal(p["opacities"].cpu(), torch.from_numpy(g["p_opacities"]))
        assert info["alpha_reset"] and float(m["opacities"].abs().max()) == 0.0 and float(v["opacities"].abs().max()) == 0.0
        for x in PARAM_NAMES:
            if x != "opacities":    # D14: we zero the opacity moments, the reference keeps them
                assert torch.equal(m[x].cpu(), torch.from_numpy(g["m_" + x]))
        return
    assert torch.equal(p["opacities"].cpu(), torch.from_numpy(g["p_opacities"]))
    assert close(p["scales"], g["p_scales"]) and close(p["means"], g["p_means"], 1e-5)
    kinds = (info["src_map"].cpu().numpy().astype(np.uint32) >> 30)
    surv = torch.from_numpy(kinds == 0)
    assert torch.equal(p["means"].cpu()[surv], torch.from_numpy(g["p_means"])[surv])       # survivors are copies
    assert torch.equal(p["scales"].cpu()[surv], torch.from_numpy(g["p_scales"])[surv])
    for x in PARAM_NAMES:
        assert torch.equal(m[x].cpu(), torch.from_numpy(g["m_" + x])), x
        assert torch.equal(v[x].cpu(), torch.from_numpy(g["v_" + x])), x
    assert info["added"] > 0 and info["culled"] > 0


def test_classify_edge_cases():
    from opensplat_b200 import densify
    cfg = densify.RefineConfig()
    z = lambda *s: torch.zeros(*s, device=DEV)
    # nothing to do: low gradients, healthy opacity -> identity map
    n = 5000
    sc = torch.full((n, 3), -3.0, device=DEV)
    src_map, split_rank, counts = densify.classify(sc, torch.full((n, 1), 2.0, device=DEV), z(n), torch.ones(n, device=DEV),
                                                   z(n), 640, cfg, True, True, True)
    assert counts.cpu().tolist()[:6] == [0, n, 0, 0, n, 0]
    assert torch.equal(src_map[:n].cpu(), torch.arange(n, dtype=torch.int32)) and bool((split_rank == -1).all())
    # everything culled (transparent)
    _, _, counts = densify.classify(sc, torch.full((n, 1), -6.0, device=DEV), z(n), torch.ones(n, device=DEV), z(n), 640,
                                    cfg, True, True, True)
    assert counts.cpu().tolist()[4] == 0
    # vis_counts == 0 -> 0/0 = NaN never compares high (what the reference's tensor comparison does)
    _, _, counts = densify.classify(sc, torch.full((n, 1), 2.0, device=DEV), z(n), z(n), z(n), 640, cfg, True, True, True)
    assert counts.cpu().tolist()[:6] == [0, n, 0, 0, n, 0]
    # all split (big scales, high gradient): 2n children in sample-major order, parents culled
    big = torch.full((n, 3), -1.0, device=DEV)
    src_map, split_rank, counts = densify.classify(big, torch.full((n, 1), 2.0, device=DEV), torch.ones(n, device=DEV),
                                                   torch.ones(n, device=DEV), z(n), 640, cfg, False, False, False)
    assert counts.cpu().tolist()[:6] == [n, 0, n, 0, 2 * n, 0]
    ar = torch.arange(n, dtype=torch.int32)
    assert torch.equal(src_map[:2 * n].cpu(), torch.cat([ar | (1 << 30), ar | (2 << 30)]))
    assert torch.equal(split_rank.cpu(), ar)
    # n == 0
    e = torch.empty((0, 3), device=DEV)
    _, _, counts = densify.classify(e, torch.empty((0, 1), device=DEV), z(0), z(0), z(0), 640, cfg, True, True, True)
    assert counts.cpu().tolist() == [0] * 8


def test_reset_opacity():
    from opensplat_b200.densify import Densifier
    o = torch.linspace(-5, 5, 10001, device=DEV).reshape(-1, 1).contiguous()
    ref = torch.clamp_max(o.cpu(), float(torch.logit(torch.tensor(0.2))))
    m, v = torch.ones_like(o), torch.ones_like(o)
    Densifier().reset_opacity(o, m, v)
    assert torch.equal(o.cpu(), ref) and float(m.abs().max()) == 0 and float(v.abs().max()) == 0


# ---- scene writers -----------------------------------------------------------------------------------------
def merged(p):
    q = {k: v for k, v in p.items() if k not in ("featuresDc", "featuresRest")}
    q["coeffs"] = torch.cat([p["featuresDc"][:, None, :], p["featuresRest"]], 1).contiguous()
    return q


@pytest.mark.parametrize("layout", ["reference", "merged"])
def test_ply_rows_byte_exact_vs_reference(layout, tmp_path):
    from opensplat_b200 import export
    g = load_golden("scene_edit_save")
    n, k = int(g["n"]), int(g["k"])
    p = dev(scene_edit_inputs(n, k, int(g["seed"]))[0])
    if layout == "merged":
        p = merged(p)
    rows = export.pack_ply_rows(p)
    blob = export.ply_header(n, k, int(g["step"])) + rows.cpu().numpy().tobytes()
    assert blob == g["ply"].tobytes()
    fn = str(tmp_path / "scene.ply")
    export.SceneWriter(DEV).save(fn, p, step=int(g["step"])).wait()
    assert open(fn, "rb").read() == g["ply"].tobytes()


def test_ply_rows_keep_crs_vs_reference():
    from opensplat_b200 import export
    g = load_golden("scene_edit_save_crs")
    n, k = int(g["n"]), int(g["k"])
    p = dev(scene_edit_inputs(n, k, int(g["seed"]))[0])
    rows = export.pack_ply_rows(p, True, float(g["scale"]), tuple(float(x) for x in g["translation"])).cpu().numpy()
    hdr = export.ply_header(n, k, int(g["step"]))
    raw = g["ply"].tobytes()
    assert raw[:len(hdr)] == hdr
    ref = np.frombuffer(raw[len(hdr):], "<f4").reshape(n, -1)
    sc = slice(ref.shape[1] - 7, ref.shape[1] - 4)              # scale_0..2: log(exp(s)/scale) on the device
    assert np.allclose(rows[:, sc], ref[:, sc], rtol=ULP, atol=ULP)
    rows[:, sc] = ref[:, sc]
    assert rows.tobytes() == ref.tobytes()                       # every other column byte-exact (means: IEEE div + add)


@pytest.mark.parametrize("name", ["scene_edit_save", "scene_edit_save_crs"])
def test_splat_rows_vs_reference(name, tmp_path):
    from opensplat_b200 import export
    from oracle import scene_edit as se
    g = load_golden(name)
    n, k = int(g["n"]), int(g["k"])
    pn = scene_edit_inputs(n, k, int(g["seed"]))[0]
    p = dev(pn)
    keep, scale, tr = bool(g["keep_crs"]), float(g["scale"]), tuple(float(x) for x in g["translation"])
    order = export.splat_order(p, keep, scale).cpu().numpy()
    assert sorted(order.tolist()) == list(range(n))
    key = sf.splat_key(pn["scales"], pn["opacities"], keep, scale)
    assert sf.order_check(order, key)[0] == 0                              # descending wherever certified
    rows = export.pack_splat_rows(p, keep, scale, tr, order=torch.from_numpy(order).to(DEV)).cpu().numpy()
    ref_rows_unordered, _ = se.splat_rows(pn["means"], pn["featuresDc"], pn["opacities"], pn["scales"], pn["quats"],
                                          keep, scale, tr)
    ref = ref_rows_unordered[order]
    assert np.array_equal(rows[:, 0:12], ref[:, 0:12])                   # means: exact
    fs, fr = rows[:, 12:24].copy().view("<f4"), ref[:, 12:24].copy().view("<f4")
    assert np.allclose(fs, fr, rtol=ULP, atol=0)
    rgb, a, q = sf.splat_bytes(pn["featuresDc"], pn["opacities"], pn["quats"])
    for got, want, x in ((rows[:, 24:27], ref[:, 24:27], rgb[order]), (rows[:, 27], ref[:, 27], a[order]),
                         (rows[:, 28:], ref[:, 28:], q[order])):
        ok, cert = sf.byte_check(got, x)                                  # u8 fields: exact wherever certified
        assert ok.all() and np.array_equal(got[cert], want[cert])
    assert np.array_equal(rows[:, 24:27], ref[:, 24:27]) and np.array_equal(rows[:, 28:], ref[:, 28:])  # no exp involved
    fn = str(tmp_path / "scene.splat")
    export.SceneWriter(DEV).save(fn, p, keep_crs=keep, scale=scale, translation=tr).wait()
    got = np.frombuffer(open(fn, "rb").read(), np.uint8).reshape(n, 32)
    assert np.array_equal(got, export.pack_splat_rows(p, keep, scale, tr).cpu().numpy())
    # ... and against the reference's own file: each row position holds the same Gaussian (means are exact copies),
    # or two Gaussians whose keys are within their certified bounds of each other
    ref_file = g["splat"].reshape(n, 32)
    same = (got[:, 0:12] == ref_file[:, 0:12]).all(axis=1)
    means = sf.crs_means(pn["means"], scale, tr) if keep else pn["means"]
    lookup = {bytes(r): i for i, r in enumerate(means.astype("<f4").view(np.uint8).reshape(n, 12))}
    ref_order = np.array([lookup[bytes(r[:12])] for r in ref_file])
    assert np.array_equal(same, order == ref_order)
    i, j = order[~same], ref_order[~same]
    assert np.all(np.abs(key.v[i] - key.v[j]) <= sf.C * (key.b[i] + key.b[j]))
    assert sf.order_check(ref_order, key)[0] == 0


def test_export_throughput_smoke():
    """1M Gaussians: both packers run and produce the documented sizes (timing is in tools/bench_next_rows.py)."""
    from opensplat_b200 import export
    n, k = 1_000_000, 16
    p = {"means": torch.randn(n, 3, device=DEV), "scales": torch.randn(n, 3, device=DEV) - 3,
         "quats": torch.randn(n, 4, device=DEV), "opacities": torch.randn(n, 1, device=DEV),
         "coeffs": torch.randn(n, k, 3, device=DEV)}
    rows = export.pack_ply_rows(p)
    assert rows.shape == (n, 62)
    assert torch.equal(rows[:, 0:3], p["means"]) and torch.equal(rows[:, 6:9], p["coeffs"][:, 0])
    assert torch.equal(rows[:, 9:54].reshape(n, 3, 15), p["coeffs"][:, 1:].transpose(1, 2))
    s = export.pack_splat_rows(p)
    assert s.shape == (n, 32)


def test_pipeline_resize_gaussians_keeps_rendering():
    """SplatPipeline.resize_gaussians: adopt a compacted / grown Gaussian set (new flat layout, Adam moments carried
    over, n-sized intermediates re-allocated) and keep stepping."""
    from opensplat_b200.pipeline import SplatPipeline
    from opensplat_b200.scene import make_scene
    n, W, H = 20_000, 320, 240
    sc = make_scene(n, W, H, scale=0.05, sh_degree=3, seed=3)
    pipe = SplatPipeline(n, W, H, device=DEV)
    pipe.load_scene(sc)
    pipe.target.copy_(torch.rand(H, W, 3, device=DEV))
    l0 = float(pipe.train_step())
    keep = torch.arange(0, n, 2, device=DEV)                         # drop every other Gaussian, then duplicate 100
    idx = torch.cat([keep, keep[:101]])                              # odd count: the flat layout must stay aligned
    views = lambda flat: {name: flat[o:o + c].view(shp) for name, (o, c, shp) in pipe.offs.items()}
    newp = {k: v[idx].clone() for k, v in pipe.p.items()}
    newm = {k: v[idx].clone() for k, v in views(pipe.adam_m).items()}
    newv = {k: v[idx].clone() for k, v in views(pipe.adam_v).items()}
    vd = pipe.viewdirs[idx].clone()
    t = pipe.adam_t
    pipe.resize_gaussians(newp, newm, newv)
    pipe.viewdirs.copy_(vd)
    assert pipe.n == idx.numel() and pipe.n % 2 == 1 and pipe.adam_t == t
    assert pipe.param_flat.numel() >= pipe.n * 59 and all(o % 4 == 0 for o, _, _ in pipe.offs.values())
    for k in newp:
        assert torch.equal(pipe.p[k], newp[k])
    assert torch.equal(pipe.adam_m[:pipe.n * 3].view(-1, 3), newm["means"])
    l1 = float(pipe.train_step())
    l2 = float(pipe.train_step())
    assert np.isfinite([l0, l1, l2]).all() and pipe.m > 0


@pytest.mark.parametrize("name", ["scene_edit_save", "scene_edit_save_crs"])
def test_load_ply_matches_reference_loadply(name, tmp_path):
    """export.load_ply (device unpack) == Model::loadPly on the reference's own file; save -> load round trip."""
    from opensplat_b200 import export
    g = load_golden(name)
    keep, scale, tr = bool(g["keep_crs"]), float(g["scale"]), tuple(float(x) for x in g["translation"])
    fn = str(tmp_path / "ref.ply")
    open(fn, "wb").write(g["ply"].tobytes())
    p, step = export.load_ply(fn, DEV, keep, scale, tr)
    assert step == int(g["ld_step"])
    for x in PARAM_NAMES:
        a, b = p[x].cpu(), torch.from_numpy(g["ld_" + x])
        if keep and x == "scales":
            assert close(a, b)                       # log(scale * exp(s)) through device expf / logf
        else:
            assert torch.equal(a, b), x
    if not keep:                                     # round trip through our own writer is the identity
        fn2 = str(tmp_path / "ours.ply")
        export.SceneWriter(DEV).save(fn2, p, step=step).wait()
        assert open(fn2, "rb").read() == g["ply"].tobytes()
    with open(fn, "ab") as f:
        f.write(b"\0\0\0\0")
    with pytest.raises(ValueError):
        export.load_ply(fn, DEV)
