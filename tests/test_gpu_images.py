"""images.ImageSet and SplatTrainer.evaluate on the H100: the INTER_AREA kernel byte-exact against OpenCV's golden
bytes, the undistort kernel byte-exact against the restatement (and OpenCV's bytes outside the recorded one-map-step
pixels), gt() against golden_u8 / 255 and its batched form, its steady state, and evaluate() next to step() and
model.GaussianModel."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_trainer import _cams, make_problem, refine_config  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "camera_images.npz"))
CASES = [str(c) for c in G["cases"]]


def _camera(name):
    from opensplat_b200.model import Camera
    cw, ch, fx, fy, cx, cy = G[f"{name}.camera"]
    k1, k2, p1, p2, k3 = (float(v) for v in G[f"{name}.dist"])
    return Camera(int(cw), int(ch), fx, fy, cx, cy, np.eye(4, dtype=np.float32), k1=k1, k2=k2, k3=k3, p1=p1, p2=p2)


def _u8(t):
    return t.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_image_set_load_and_levels_against_the_golden(name):
    from opensplat_b200.images import ImageSet
    cam = _camera(name)
    s = ImageSet([cam], [G[f"{name}.image"]], downscale_factor=float(G[f"{name}.factor"]), device=DEV)
    loaded = _u8(s.level(0))
    assert np.array_equal(loaded, G[f"{name}.loaded_oracle"])
    diff = np.any(loaded != G[f"{name}.loaded_cv2"], axis=-1)
    md = G[f"{name}.map_diff"]
    diff[md[:, 0], md[:, 1]] = False
    assert not diff.any()
    c = s.cameras[0]
    assert (c.width, c.height) == tuple(int(v) for v in G[f"{name}.size"])
    assert np.array_equal(np.array([c.fx, c.fy, c.cx, c.cy], np.float32), G[f"{name}.intrinsics"])
    assert tuple(s.roi[0]) == tuple(int(v) for v in G[f"{name}.roi"])
    assert cam.width == int(G[f"{name}.camera"][0])           # the input camera is left untouched
    for f in G[f"{name}.levels"]:
        f = int(f)
        # the kernel on cv2's loaded bytes: INTER_AREA byte for byte
        src = torch.from_numpy(G[f"{name}.loaded_cv2"]).to(DEV)
        out = torch.empty_like(torch.from_numpy(G[f"{name}.level{f}"])).to(DEV)
        from opensplat_b200 import capi
        capi.check(capi.lib().gsb_resize_area_u8(src.shape[0], src.shape[1], capi.ptr(src), out.shape[0],
                                                 out.shape[1], capi.ptr(out), 0.0, capi.stream()))
        assert np.array_equal(_u8(out), G[f"{name}.level{f}"]), f
        if not len(md):
            assert np.array_equal(_u8(s.level(0, f)), G[f"{name}.level{f}"]), f


@pytest.mark.parametrize("name", ["even", "odd"])
def test_gt_is_u8_over_255_and_batched_equals_singles(name):
    """'odd' (101x75) puts view 1 of a batch at a float offset that is not a multiple of 4 and leaves a tail of
    bytes, so the conversion's scalar path is checked too; 'even' runs the vector path only."""
    from opensplat_b200.images import ImageSet
    img = G[f"{name}.image"]
    imgs = [img, np.ascontiguousarray(img[::-1]), np.ascontiguousarray(255 - img)]
    s = ImageSet([_camera(name)] * 3, imgs, device=DEV)
    for f in (1, 2, 4):
        singles = []
        for i in range(3):
            g = s.gt(i, f)
            want = torch.from_numpy(_u8(s.level(i, f))).to(torch.float32) / 255.0
            assert g.shape == want.shape and torch.equal(g.cpu(), want), (i, f)
            singles.append(g.clone())
        if f"{name}.level{f}" in G.files:
            assert np.array_equal(_u8(s.level(0, f)), G[f"{name}.level{f}"])
        batch = s.gt([0, 1, 2], f)
        assert batch.shape == (3,) + singles[0].shape
        assert torch.equal(batch.cpu(), torch.stack(singles).cpu())
        assert torch.equal(s.gt([2, 0], f), torch.stack([singles[2], singles[0]]))   # not consecutive: uploaded
        # negative indices count from the end, as list indices do
        assert torch.equal(s.gt(-1, f), singles[2])
        assert torch.equal(s.gt([-2, -1], f), torch.stack([singles[1], singles[2]]))
        assert torch.equal(s.gt([-1, 0], f), torch.stack([singles[2], singles[0]]))
        assert torch.equal(s.level(-3, f), s.level(0, f))
        for bad in (3, -4, [2, 3], [-4, 0]):
            with pytest.raises(IndexError):
                s.gt(bad, f)


def test_image_set_copies_device_inputs():
    """A caller may decode every image into one reused device buffer: the set keeps its own copies."""
    from opensplat_b200.images import ImageSet
    buf = torch.from_numpy(G["even.image"]).to(DEV)
    first = buf.clone()
    s = ImageSet([_camera("even")], [buf], device=DEV)
    buf.zero_()
    assert torch.equal(s.level(0), first)


def test_gt_allocates_nothing_once_warm():
    from opensplat_b200.images import ImageSet
    s = ImageSet([_camera("odd")] * 2, [G["odd.image"]] * 2, device=DEV)
    s.gt([0, 1], 2)
    s.gt([1, 0], 1)        # the largest call sizes the shared buffer; the reversed order takes the upload path
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for k in range(50):
        s.gt(k % 2, 1)
        s.gt([0, 1], 1)
        s.gt([1, 0], 2)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before


def _trainer(p, **kw):
    from opensplat_b200.trainer import SplatTrainer
    return SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, kw.pop("cfg", refine_config()), device=DEV,
                        generator=torch.Generator(device=DEV).manual_seed(3), **kw)


def test_evaluate_then_step_renders_the_same_view():
    """evaluate() runs step()'s forward and loss: the image is bit-equal; the loss equal to the float-atomic
    summation order of the loss kernel (its per-block sums are added with atomics)."""
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts[1]).to(DEV)
    tr = _trainer(p)
    for step in range(1, 4):
        tr.step(cams[(step - 1) % 3], torch.from_numpy(gts[(step - 1) % 3]).to(DEV), step)
    ev = tr.evaluate(cams[1], gt, 4).clone()
    img = tr.image.clone()
    st = tr.step(cams[1], gt, 4).clone()
    assert torch.equal(img, tr.image)
    assert float((ev - st).abs().max()) <= 1e-6, (ev, st)


def test_evaluate_leaves_training_bit_identical():
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    g = [torch.from_numpy(x).to(DEV) for x in gts]
    runs = []
    for with_eval in (False, True):
        tr = _trainer(p)
        for step in range(1, 31):
            if with_eval and step % 3 == 0:
                tr.evaluate(cams[2], g[2], step)
            tr.step(cams[(step - 1) % 2], g[(step - 1) % 2], step)
        torch.cuda.synchronize()
        runs.append((tr.n, tr.params(), tr.adam_state()))
    (n0, p0, (m0, v0)), (n1, p1, (m1, v1)) = runs
    assert n0 == n1
    for k in p0:
        assert torch.equal(p0[k], p1[k]) and torch.equal(m0[k], m1[k]) and torch.equal(v0[k], v1[k]), k


def test_evaluate_agrees_with_gaussian_model():
    from opensplat_b200.model import GaussianModel
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts[0]).to(DEV)
    model = GaussianModel({k: torch.from_numpy(v) for k, v in p.items()}, refine_config(), device=DEV)
    tr = _trainer(p)
    for step in (1, 1000, 2000):        # SH degrees 0, 1, 2
        want = model.main_loss(model.forward(cams[0], step), gt, 0.2)
        got = tr.evaluate(cams[0], gt, step)
        assert abs(float(got[0]) - float(want)) <= 1e-6, (step, float(got[0]), float(want))


def test_downscale_schedule_through_an_image_set():
    """num_downscales=2: the gt resolution follows the trainer's factor 4 -> 2 -> 1."""
    from opensplat_b200.images import ImageSet
    from opensplat_b200.model import downscale_factor
    p, c2w, gts, intr, H, W = make_problem()
    cams = _cams(c2w, H, W, intr)
    s = ImageSet(cams, [np.clip(g * 255, 0, 255).astype(np.uint8) for g in gts], device=DEV)
    tr = _trainer(p, num_downscales=2, resolution_schedule=5)
    seen = []
    for step in range(1, 14):
        v = (step - 1) % 3
        f = downscale_factor(step, 2, 5)
        loss = tr.step(s.cameras[v], s.gt(v, f), step)
        seen.append((f, tr.resolution))
        assert bool(torch.isfinite(loss).all())
    assert sorted({sr for sr in seen}) == [(1, (W, H)), (2, (W // 2, H // 2)), (4, (W // 4, H // 4))]
    assert tr.pixel_reallocs == 2
    ev = tr.evaluate(s.cameras[0], s.gt(0, 1), 13)
    assert bool(torch.isfinite(ev).all())
