"""GPU: the C-ABI call sequence of one steady-state trainer.SplatTrainer step, recorded through a recorder around the
loaded library, for one and several views per step, with visible and empty views.  The sequences are literal lists, so
a change to the step body that adds, drops or swaps a launch has to change them here.  The densification statistics
kernel is checked apart: one call per visible view, after that view's rasterize-backward."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_trainer as tg  # noqa: E402  (the training problem)
from test_gpu_trainer_views import _away  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

FORWARD = ["gsb_project_forward_activated", "gsb_bucket_max_tile_len", "gsb_bucket_tile_ranges",
           "gsb_bucket_sort_pack", "gsb_rasterize_forward_packed", "gsb_ssim_l1_loss"]
ONE_VIEW = (["gsb_sh_forward_rgb_cam"] + FORWARD + ["gsb_rasterize_backward", "gsb_project_backward_activated",
                                                   "gsb_sh_backward_rgb_cam", "gsb_adam_step_segments"])
ONE_VIEW_EMPTY = ["gsb_sh_forward_rgb_cam"] + FORWARD
TWO_VIEWS = (["gsb_sh_forward_rgb_cam_multiview"]
             + FORWARD + ["gsb_rasterize_backward", "gsb_project_backward_activated"]
             + FORWARD + ["gsb_rasterize_backward", "gsb_project_backward_activated_acc"]
             + ["gsb_mask_rgb_grad", "gsb_exchange_gradients", "gsb_adam_step_segments"])
THREE_VIEWS_EMPTY = (["gsb_sh_forward_rgb_cam_multiview"]
                     + FORWARD + ["gsb_rasterize_backward", "gsb_project_backward_activated"]
                     + 2 * (FORWARD + ["gsb_rasterize_backward", "gsb_project_backward_activated_acc"]))

# (views per step, which views face away, the expected sequence without the statistics kernel)
CASES = {
    "one_view": (1, [], ONE_VIEW),
    "one_view_empty": (1, [0], ONE_VIEW_EMPTY),
    "two_views": (2, [], TWO_VIEWS),
    "two_views_first_empty": (2, [0], TWO_VIEWS),
    "three_views_empty": (3, [0, 1, 2], THREE_VIEWS_EMPTY),
}


class _Recorder:
    """Forwards every attribute of the loaded library; logs the name of every gsb_* function that is called."""

    def __init__(self, lib, log):
        self._lib, self._log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("gsb_"):
            return fn
        log = self._log

        def call(*args):
            log.append(name)
            return fn(*args)
        return call


@pytest.mark.parametrize("case", list(CASES))
def test_step_issues_the_recorded_launch_sequence(case, monkeypatch):
    from opensplat_b200 import capi
    from opensplat_b200.trainer import SplatTrainer
    B, empty, expected = CASES[case]
    p, c2w, gts, intr, H, W = tg.make_problem()
    cams = tg._cams(c2w, H, W, intr)
    gt = torch.from_numpy(gts).to(DEV)
    log = []
    # before construction: the trainer and its pipeline keep the library object they are built with
    monkeypatch.setattr(capi, "_lib", _Recorder(capi.lib(), log))
    tr = SplatTrainer({k: torch.from_numpy(v) for k, v in p.items()}, tg.refine_config(warmup_length=10 ** 6),
                      device=DEV, views_per_step=B)

    def args(views):
        return (views[0], gt[0]) if B == 1 else (views, gt[:B])
    for step in range(1, 6):                        # warm-up: plan, bins, statistics
        tr.step(*args([cams[(step - 1 + b) % 3] for b in range(B)]), step)
    torch.cuda.synchronize()
    away = _away(c2w, H, W, intr)
    views = [away if b in empty else cams[b] for b in range(B)]
    del log[:]
    tr.step(*args(views), 6)
    torch.cuda.synchronize()
    seq = [x for x in log if not x.startswith("gsb_densify_stats_")]
    assert seq == expected, log
    stats = [i for i, x in enumerate(log) if x.startswith("gsb_densify_stats_")]
    raster_bwd = [i for i, x in enumerate(log) if x == "gsb_rasterize_backward"]
    visible = [b for b in range(B) if b not in empty]
    assert len(stats) == len(visible), log
    for i, b in zip(stats, visible):
        assert i > raster_bwd[b], log
