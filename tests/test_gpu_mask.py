"""GPU: per-image loss masks (DESIGN D26).

1. Ingest: gsb_resize_area_mask_u8 / gsb_undistort_mask_u8 through ImageSet(masks=) and ImageSet.mask() equal the
   numpy rule of tests/mask_ingest_np.py byte for byte, on the cameras and images of tests/golden/camera_images.npz at
   loadImage factors 1, 1.5, 2, 2.5 (distorted and undistorted) and getImage factors 2, 3, 4, 8.
2. Loss: gsb_ssim_l1_loss_masked inside the certified float64 bound of tests/loss_mask_f64.py at every element; at
   an all-ones mask its gradient is gsb_ssim_l1_loss's bit for bit, and when the ignored pixels hold junk, NaN or inf
   its gradient is unchanged bit for bit.  The scalars are sums through one float atomic per tile, whose order varies
   from run to run in both kernels, so they are compared within that reordering's bound.
3. Trainer: one step with mask= against the autograd composition through ops.MainLoss(mask=) (B = 1, B = 2 with one
   view unmasked, appearance grids); a trainer never given a mask is the plain trainer (launches and bits);
   evaluate(mask=) is the masked loss of the render.
4. It does the job: masking a transient occluder in every view keeps it out of the scene.
5. Data-parallel: replicas stay bit-identical with masks (tools/check_parallel_mask.py)."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import loss_f64  # noqa: E402
import loss_mask_f64 as lm  # noqa: E402
import mask_ingest_np as mi  # noqa: E402
import test_gpu_trainer as tg  # noqa: E402  (the training problem)
from test_gpu_trainer_launches import ONE_VIEW, _Recorder  # noqa: E402
from util import rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "camera_images.npz"))
CASES = [str(c) for c in G["cases"]]
GEOM = ("means", "scales", "quats", "opacities")


@pytest.fixture(autouse=True)
def _release_cached_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---- 1. ingest ----------------------------------------------------------------------------------------------------------
def _camera(name, distorted):
    from opensplat_b200.model import Camera
    cw, ch, fx, fy, cx, cy = G[f"{name}.camera"]
    k1, k2, p1, p2, k3 = (float(v) for v in G[f"{name}.dist"]) if distorted else (0.0,) * 5
    return Camera(int(cw), int(ch), fx, fy, cx, cy, np.eye(4, dtype=np.float32), k1=k1, k2=k2, k3=k3, p1=p1, p2=p2)


@pytest.mark.parametrize("name", CASES)
def test_ingest_equals_the_numpy_rule(name):
    from opensplat_b200.images import ImageSet
    img = G[f"{name}.image"]
    h, w = img.shape[:2]
    checked = 0
    for fi, factor in enumerate((1.0, 1.5, 2.0, 2.5)):
        for distorted in (False, True):
            kinds = ["blobs", "random"] if fi or distorted else ["blobs", "ones", "zero"]
            for ki, kind in enumerate(kinds):
                m = lm.make_mask(h, w, kind, 100 * fi + 10 * ki + int(distorted))
                cam = _camera(name, distorted)
                try:
                    s = ImageSet([cam], [img], downscale_factor=factor, device=DEV, masks=[m])
                except ValueError:      # an undistorted image with an empty valid region at this size
                    continue
                args = (cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy,
                        (cam.k1, cam.k2, cam.p1, cam.p2, cam.k3), factor)
                want = mi.load_mask(m, *args)
                got = s.mask(0)
                assert got.dtype == torch.uint8 and tuple(got.shape) == tuple(s.level(0).shape[:2])
                assert np.array_equal(got.cpu().numpy(), want), (factor, distorted, kind)
                for f in (2, 3, 4, 8):
                    if want.shape[0] // f < 1 or want.shape[1] // f < 1:
                        continue
                    lv = s.mask(0, f)
                    assert s.mask(0, f) is lv                                   # cached
                    assert tuple(lv.shape) == tuple(s.level(0, f).shape[:2])
                    assert np.array_equal(lv.cpu().numpy(), mi.get_mask(want, f)), (factor, distorted, kind, f)
                checked += 1
    assert checked >= 12


def test_image_set_masks_none_and_lists():
    from opensplat_b200.images import ImageSet
    name = CASES[0]
    img = G[f"{name}.image"]
    m = torch.from_numpy(lm.make_mask(img.shape[0], img.shape[1], "blobs", 1)).bool().to(DEV)
    s = ImageSet([_camera(name, False)] * 2, [img, img], device=DEV, masks=[None, m])
    assert s.mask(0) is None and s.mask(0, 2) is None
    both = s.mask([0, 1], 2)
    assert both[0] is None and torch.equal(both[1].cpu(), torch.from_numpy(mi.get_mask(m.cpu().numpy(), 2)))
    with pytest.raises(ValueError):
        ImageSet([_camera(name, False)], [img], device=DEV, masks=[m[:-1]])


# ---- 2. the loss --------------------------------------------------------------------------------------------------------
def _kernel(r, g, m, w=0.2, masked=True):
    from opensplat_b200 import capi
    L = capi.lib()
    H, W = r.shape[0], r.shape[1]
    ws = torch.empty(L.gsb_ssim_workspace_bytes(H, W) + 256, dtype=torch.uint8, device=DEV)
    off = (-ws.data_ptr()) % 256
    v = torch.full_like(r, 7.0)
    out = torch.full((3,), 7.0, device=DEV)
    if masked:
        capi.check(L.gsb_ssim_l1_loss_masked(H, W, capi.ptr(r), capi.ptr(g), capi.ptr(m), w, capi.ptr(v),
                                             capi.ptr(out), ws.data_ptr() + off, ws.numel() - off, capi.stream()))
    else:
        capi.check(L.gsb_ssim_l1_loss(H, W, capi.ptr(r), capi.ptr(g), w, capi.ptr(v), capi.ptr(out),
                                      ws.data_ptr() + off, ws.numel() - off, capi.stream()))
    torch.cuda.synchronize()
    return v, out


@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (97, 131), (1080, 1920)])
@pytest.mark.parametrize("kind", ["random", "blobs", "single", "zero"])
def test_masked_loss_within_the_certified_bound(H, W, kind):
    r, g = loss_f64.tie_images(H, W, H + W)
    m = lm.make_mask(H, W, kind, H * 7 + W)
    v, out = _kernel(cu(r), cu(g), cu(m))
    ref = lm.loss(cu(r), cu(g), cu(m), 0.2, device=DEV)
    err = (v.double() - ref["v_rendered"]).abs()
    worst = float((err / (ref["B_v_rendered"] + 1e-300)).max()) if int(m.sum()) else 0.0
    print(f"{H}x{W} {kind}: N={ref['n']} worst err/bound {worst:.3g}")
    assert bool((err <= ref["B_v_rendered"]).all())
    assert int(torch.count_nonzero(v[cu(m) == 0])) == 0
    o = out.cpu().double().numpy()
    for i, k in enumerate(("loss", "l1", "ssim")):
        assert abs(o[i] - ref[k]) <= ref["B_" + k], (k, o[i], ref[k], ref["B_" + k])
    if kind == "zero":
        assert o.tolist() == [0.0, 0.0, 1.0] and int(torch.count_nonzero(v)) == 0


def _same_scalars(a, b, H, W):
    """{total, L1, SSIM} equal up to the order of the per-tile atomics: the tree's depth times u, relative to sums of
    terms in [0, 1] (|S| <= 1, |y - x| <= 1 on these images) over the count, plus the finalize step's roundings."""
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    tol = 2 * (11 + tiles + 4) * 2.0 ** -24
    assert float((a - b).abs().max()) <= tol, (a, b, tol)


@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (97, 131), (1080, 1920), (2160, 3840)])
def test_all_ones_mask_is_the_unmasked_gradient_bit_for_bit(H, W):
    r, g = (cu(a) for a in loss_f64.tie_images(H, W, 4))
    ones = torch.ones((H, W), dtype=torch.uint8, device=DEV)
    v1, o1 = _kernel(r, g, ones)
    v0, o0 = _kernel(r, g, None, masked=False)
    assert torch.equal(v1, v0)
    _same_scalars(o1, o0, H, W)
    if H * W <= 256:                                   # one tile: one atomic, no reordering
        assert torch.equal(o1, o0)
    v2, o2 = _kernel(r, g, ones * 255)                 # any nonzero byte means used
    assert torch.equal(v2, v0)
    _same_scalars(o2, o0, H, W)


@pytest.mark.parametrize("H,W", [(97, 131), (1080, 1920)])
def test_ignored_content_never_reaches_the_result(H, W):
    r, g = (cu(a) for a in loss_f64.tie_images(H, W, 6))
    m = cu(lm.make_mask(H, W, "blobs", 2))
    v, o = _kernel(r, g, m)
    ign = m == 0
    gen = torch.Generator(device=DEV).manual_seed(0)
    r2, g2 = r.clone(), g.clone()
    junk = torch.rand(r.shape, generator=gen, device=DEV) * 20 - 10
    junk.view(-1)[::7] = float("nan")
    junk.view(-1)[3::11] = float("inf")
    junk.view(-1)[5::13] = -float("inf")
    r2[ign], g2[ign] = junk[ign], junk.flip(0)[ign]
    v2, o2 = _kernel(r2, g2, m)
    assert torch.equal(v, v2)
    _same_scalars(o, o2, H, W)
    assert bool(torch.isfinite(v2).all()) and bool(torch.isfinite(o2).all())


# ---- 3. the trainer -----------------------------------------------------------------------------------------------------
def _problem(n=4000, V=3):
    p, c2w, gts, intr, H, W = tg.make_problem(n=n, V=V)
    return ({k: torch.from_numpy(v) for k, v in p.items()}, tg._cams(c2w, H, W, intr), cu(gts), H, W)


def _masks(H, W, V=3):
    return [cu(lm.make_mask(H, W, "blobs", 40 + v)) for v in range(V)]


def _frozen(params, B=1, **kw):
    from opensplat_b200.trainer import SplatTrainer
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV, views_per_step=B, **kw)
    tr._adam_step = lambda: None
    return tr


def _composition(tr, params, cams, gts, masks, views, grids=None):
    """Gradients of mean_b MainLoss(render_b [sliced through grids[b]], gt, mask_b) through the autograd operators at
    the trainer's cameras and colours of its last step."""
    from opensplat_b200 import ops
    pp = tr.pipe
    H, W = pp.H, pp.W
    dev = {k: v.to(DEV).clone().requires_grad_() for k, v in params.items() if k in GEOM}
    total = 0.0
    for b, v in enumerate(views):
        c = cams[v]
        xys, depths, radii, conics, nth, _, opac = ops.ProjectGaussiansActivated.apply(
            dev["means"], dev["scales"], 1.0, dev["quats"], dev["opacities"], tr.viewmats[b].clone(),
            tr.projmats[b].clone(), c.fx, c.fy, c.cx, c.cy, H, W, ops.tile_bounds(W, H))
        img = ops.RasterizeGaussiansClamped.apply(xys, depths, radii, conics, nth, tr.rgbs_views[b].detach(), opac,
                                                  H, W, pp.background)
        if grids is not None:
            img = ops.BilateralGridSlice.apply(grids[b], img)
        total = total + ops.MainLoss.apply(img, gts[v], tr.ssim_weight, masks[b])
    (total / len(views)).backward()
    return {k: dev[k].grad for k in GEOM}


def _grads(tr):
    return {k: tr.pipe.g[k].reshape(-1).clone() for k in GEOM}


def _compare(got, want, tol=2e-4):
    for k in GEOM:
        e = rel_l2(got[k].cpu().numpy(), want[k].reshape(-1).cpu().numpy())
        print(f"  {k}: rel-L2 {e:.3g}")
        assert e <= tol, k


@pytest.mark.parametrize("mode", ["one_view", "two_views_one_mask", "appearance"])
def test_one_step_matches_the_autograd_composition(mode):
    from opensplat_b200.appearance import AppearanceConfig
    params, cams, gts, H, W = _problem()
    masks = _masks(H, W)
    grids = None
    if mode == "two_views_one_mask":
        tr = _frozen(params, 2)
        views, ms = [1, 2], [masks[1].bool(), None]
        tr.step([cams[v] for v in views], gts[views], 7, mask=ms)
    elif mode == "appearance":
        tr = _frozen(params, appearance=AppearanceConfig(num_images=3))
        tr.appearance.adam_step = lambda step: None
        views, ms = [0], [masks[0]]
        tr.step(cams[0], gts[0], 3, image=0, mask=ms[0])
        grids = [tr.appearance_grids()[0]]
    else:
        tr = _frozen(params)
        views, ms = [1], [masks[1]]
        tr.step(cams[1], gts[1], 7, mask=ms[0])
    torch.cuda.synchronize()
    got = _grads(tr)
    want = _composition(tr, params, cams, gts, ms, views, grids)
    _compare(got, want, tol=1e-3 if grids is not None else 2e-4)
    # the mask is a real part of it: without it the gradient differs
    plain = _composition(tr, params, cams, gts, [None] * len(views), views, grids)
    assert rel_l2(got["means"].cpu().numpy(), plain["means"].reshape(-1).cpu().numpy()) > 1e-2


MASK_VIEW = [x if x != "gsb_ssim_l1_loss" else "gsb_ssim_l1_loss_masked" for x in ONE_VIEW]


def test_launch_sequences_and_a_trainer_without_masks_is_the_plain_trainer(monkeypatch):
    from opensplat_b200 import capi
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem()
    masks = _masks(H, W)
    log = []
    monkeypatch.setattr(capi, "_lib", _Recorder(capi.lib(), log))
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV)
    for step in range(1, 4):
        tr.step(cams[(step - 1) % 3], gts[(step - 1) % 3], step, mask=masks[(step - 1) % 3])
    torch.cuda.synchronize()
    del log[:]
    tr.step(cams[0], gts[0], 4, mask=masks[0])
    torch.cuda.synchronize()
    assert [x for x in log if not x.startswith("gsb_densify_stats_")] == MASK_VIEW, log
    del log[:]
    tr.step(cams[1], gts[1], 5)
    torch.cuda.synchronize()
    assert [x for x in log if not x.startswith("gsb_densify_stats_")] == ONE_VIEW, log
    monkeypatch.undo()
    # with no mask ever given, the run is the plain run bit for bit (the same calls, with mask=None spelled out)
    runs = []
    for explicit in (False, True):
        torch.manual_seed(0)
        t = SplatTrainer(params, tg.refine_config(), device=DEV)
        for step in range(1, 21):
            kw = {"mask": None} if explicit else {}
            t.step(cams[(step - 1) % 3], gts[(step - 1) % 3], step, **kw)
        runs.append(t)
    torch.cuda.synchronize()
    a, b = runs
    assert a.n == b.n
    for x, y in ((a.pipe.param_flat, b.pipe.param_flat), (a.pipe.adam_m, b.pipe.adam_m)):
        assert torch.equal(x, y)


def test_all_ones_mask_trains_as_no_mask():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem()
    ones = torch.ones((H, W), dtype=torch.uint8, device=DEV)
    runs = []
    for m in (None, ones):
        torch.manual_seed(0)
        t = SplatTrainer(params, tg.refine_config(), device=DEV)
        for step in range(1, 21):
            t.step(cams[(step - 1) % 3], gts[(step - 1) % 3], step, mask=m)
        runs.append(t)
    torch.cuda.synchronize()
    assert runs[0].n == runs[1].n and torch.equal(runs[0].pipe.param_flat, runs[1].pipe.param_flat)


def test_evaluate_scores_the_used_pixels():
    from opensplat_b200 import ops
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem()
    masks = _masks(H, W)
    tr = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV)
    for step in range(1, 4):
        tr.step(cams[(step - 1) % 3], gts[(step - 1) % 3], step, mask=masks[(step - 1) % 3])
    got = tr.evaluate(cams[2], gts[2], 4, mask=masks[2].bool()).clone()
    img = tr.image.clone()
    want = ops.MainLoss.apply(img, gts[2], tr.ssim_weight, masks[2])
    assert abs(float(got[0]) - float(want)) <= 1e-6 * float(want)     # the per-tile atomics' order only
    plain = tr.evaluate(cams[2], gts[2], 4).clone()
    assert float(plain[0]) != float(got[0])
    with pytest.raises(ValueError):
        tr.evaluate(cams[2], gts[2], 4, mask=masks[2][:-1])


def test_steady_state_allocates_nothing():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts, H, W = _problem(n=1500)
    masks = _masks(H, W)
    two = SplatTrainer(params, tg.refine_config(warmup_length=10 ** 6), device=DEV, views_per_step=2)
    for step in range(1, 4):
        two.step(cams[:2], gts[:2], step, mask=[masks[0], None])
    torch.cuda.synchronize()
    before = torch.cuda.memory_stats(DEV)["allocation.all.allocated"]
    for step in range(4, 10):
        two.step(cams[:2], gts[:2], step, mask=[masks[0], None] if step % 2 else torch.stack(masks[:2]))
    torch.cuda.synchronize()
    # the stacked [2,H,W] mask of the odd steps is the test's own allocation
    assert torch.cuda.memory_stats(DEV)["allocation.all.allocated"] - before <= 3


# ---- 4. it does the job -------------------------------------------------------------------------------------------------
def _psnr(a, b):
    mse = float(((a - b) ** 2).mean())
    return 10.0 * np.log10(1.0 / max(mse, 1e-12))


def test_masking_a_transient_occluder_keeps_it_out_of_the_scene():
    """A seeded teacher scene renders clean views; every training view gets a random opaque rectangle (a transient
    occluder, placed and coloured differently per view).  Students start from the teacher with perturbed colours and
    train the same steps with and without masks over the rectangles; inside the rectangles, the masked student's
    render is closer to the clean view."""
    from opensplat_b200.trainer import SplatTrainer
    V = 4
    p, c2w, _, intr, H, W = tg.make_problem(n=4000, V=V, seed=13)
    cams = tg._cams(c2w, H, W, intr)
    cfg = tg.refine_config(warmup_length=10 ** 6, num_cameras=V, max_steps=2000)
    truth = {k: torch.from_numpy(v) for k, v in p.items()}
    teacher = SplatTrainer(truth, cfg, device=DEV)
    clean = torch.stack([teacher.render(c, 10 ** 6)["rgb"].clone() for c in cams])
    rng = np.random.default_rng(4)
    occluded, masks, boxes = clean.clone(), [], []
    for v in range(V):
        h, w = H // 3, W // 3
        y0, x0 = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        occluded[v, y0:y0 + h, x0:x0 + w] = torch.tensor(rng.uniform(0, 1, 3).astype(np.float32), device=DEV)
        m = torch.ones((H, W), dtype=torch.uint8, device=DEV)
        m[y0:y0 + h, x0:x0 + w] = 0
        masks.append(m)
        boxes.append((y0, y0 + h, x0, x0 + w))
    start = dict(truth)
    start["featuresDc"] = truth["featuresDc"] + torch.from_numpy(
        rng.normal(0, 0.4, truth["featuresDc"].shape).astype(np.float32))
    steps, res = 400, {}
    for name in ("plain", "masked"):
        tr = SplatTrainer(start, cfg, device=DEV, sh_degree_interval=1)
        for step in range(1, steps + 1):
            v = (step - 1) % V
            tr.step(cams[v], occluded[v], step, mask=masks[v] if name == "masked" else None)
        inside = []
        for v, (a, b, c, d) in enumerate(boxes):
            img = tr.render(cams[v], steps)["rgb"]
            inside.append(_psnr(img[a:b, c:d], clean[v, a:b, c:d]))
        res[name] = float(np.mean(inside))
    print(f"PSNR inside the occluders against the clean views: plain {res['plain']:.2f} dB, "
          f"masked {res['masked']:.2f} dB")
    assert res["masked"] >= res["plain"] + 3.0


# ---- 5. data-parallel ---------------------------------------------------------------------------------------------------
def _run_parallel(nproc, port):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tools", "check_parallel_mask.py")], capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-4000:])
    if r.returncode != 0:
        print(r.stderr[-6000:])
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    assert "check_ok=True" in r.stdout
    return r.stdout


def test_parallel_world1_replicas_with_masks():
    out = _run_parallel(1, 29571)
    assert "plain_trainer_bit_identical=True" in out


def test_parallel_2gpu_replicas_with_masks():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_parallel(2, 29573)
