"""CPU-only host logic of trainer.SplatTrainer: the segment table of its one Adam launch, and the camera /
learning-rate helpers it shares with model.GaussianModel (checked against the code they replaced there)."""
import math

import numpy as np
import pytest
import torch

from opensplat_b200 import model, parallel, trainer
from opensplat_b200.model import LEARNING_RATES, Camera


@pytest.mark.parametrize("n", [1, 7, 333, 4097])
@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
def test_adam_segments_cover_every_slice_once_with_the_reference_rates(n, k):
    offs, numel = parallel.flat_layout(n, k)
    segs = trainer.adam_segments(offs, LEARNING_RATES)
    assert len(segs) == len(offs) <= 8
    hits = np.zeros(numel, np.int32)
    rate = np.full(numel, np.nan, np.float64)
    for o, c, row, head, lr_head, lr_rest in segs:
        assert o % 4 == 0 and row > 0 and 0 <= head <= row
        e = np.arange(c)
        hits[o:o + c] += 1
        rate[o:o + c] = np.where(e % row < head, lr_head, lr_rest)
    covered = np.zeros(numel, bool)
    for name, (o, c, shp) in offs.items():
        covered[o:o + c] = True
        r = rate[o:o + c]
        if name == "coeffs":
            rows = r.reshape(n, 3 * k)
            assert (rows[:, :3] == LEARNING_RATES["featuresDc"]).all()
            assert (rows[:, 3:] == LEARNING_RATES["featuresRest"]).all()
        else:
            assert (r == LEARNING_RATES[name]).all(), name
    assert (hits[covered] == 1).all()          # every float of every slice exactly once
    assert (hits[~covered] == 0).all()         # padding between slices: in no segment


def _old_camera_block(cam, sf, dev="cpu"):
    """GaussianModel.forward's camera code before it moved into model.camera_setup."""
    sf = float(sf)
    fx, fy, cx, cy = cam.fx / sf, cam.fy / sf, cam.cx / sf, cam.cy / sf
    height, width = int(float(cam.height) / sf), int(float(cam.width) / sf)
    c2w = cam.camToWorld
    R = c2w[:3, :3] @ torch.diag(torch.tensor([1.0, -1.0, -1.0]))
    T = c2w[:3, 3:4]
    Rinv = R.t()
    Tinv = (-Rinv) @ T
    view = torch.eye(4)
    view[:3, :3] = Rinv
    view[:3, 3:4] = Tinv
    view = view.to(dev)
    fov_x = 2.0 * math.atan(width / (2.0 * fx))
    fov_y = 2.0 * math.atan(height / (2.0 * fy))
    proj = model.projection_matrix(0.001, 1000.0, fov_x, fov_y, dev)
    cam_pos = T.reshape(3).to(dev)
    return height, width, (fx, fy, cx, cy), view, proj, cam_pos


def test_camera_setup_is_the_code_gaussian_model_used():
    rng = np.random.default_rng(3)
    for _ in range(6):
        q = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        c2w = np.eye(4, dtype=np.float32)
        c2w[:3, :3] = q
        c2w[:3, 3] = rng.uniform(-5, 5, 3)
        cam = Camera(int(rng.integers(100, 2000)), int(rng.integers(100, 1200)), rng.uniform(200, 1500),
                     rng.uniform(200, 1500), rng.uniform(50, 900), rng.uniform(50, 600), c2w)
        for sf in (1, 2, 4, 8):
            new, old = model.camera_setup(cam, sf), _old_camera_block(cam, sf)
            assert new[:3] == old[:3]
            for a, b in zip(new[3:], old[3:]):
                assert a.dtype == b.dtype and torch.equal(a, b)


def test_learning_rate_and_downscale_helpers_are_the_code_gaussian_model_used():
    lr_init = float(torch.tensor(LEARNING_RATES["means"], dtype=torch.float64).float())
    assert model.MEANS_LR_INIT == lr_init
    for max_steps in (1, 200, 30000):
        for step in (-1, 0, 1, 2, 17, max_steps // 2, max_steps - 1, max_steps, max_steps + 5):
            t = max(min(float(step) / float(max_steps), 1.0), 0.0)
            old = math.exp(math.log(lr_init) * (1.0 - t) + math.log(model.MEANS_LR_FINAL) * t)
            assert model.means_learning_rate(step, max_steps, lr_init) == old
    for nd in (0, 1, 3):
        for sched in (1, 6, 3000):
            for step in (0, 1, 5, 6, 7, 12, 3000, 9000, 10 ** 6):
                assert model.downscale_factor(step, nd, sched) == int(2 ** max(nd - step // sched, 0))


def test_trainer_refuses_a_multi_process_group(monkeypatch):
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RuntimeError, match="one process"):
        trainer.SplatTrainer({}, device="cpu")
