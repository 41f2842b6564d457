"""CPU: the host side of the appearance grids -- AppearanceConfig's checks, the learning-rate schedule against the
float64 restatement, the identity start, and the C ABI's argument checks (no kernel runs)."""
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bilagrid_f64 as ref  # noqa: E402

from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.appearance import AppearanceConfig, learning_rate  # noqa: E402

P = C.c_void_p(256)      # any 256-byte aligned address: every call below is rejected before it is used
BAD = -1


def test_config_checks():
    for bad in (dict(num_images=0), dict(num_images=-3), dict(num_images=1.5), dict(num_images=True),
                dict(num_images=2, lr=0.0), dict(num_images=2, final_lr_factor=-1.0),
                dict(num_images=2, warmup_start=1.5), dict(num_images=2, warmup_steps=0),
                dict(num_images=2, max_steps=0), dict(num_images=2, tv_weight=-1.0), dict(num_images=2, grid_x=8),
                dict(num_images=2, grid_l=4)):
        with pytest.raises(ValueError):
            AppearanceConfig(**bad)
    c = AppearanceConfig(num_images=3)
    assert (c.lr, c.final_lr_factor, c.warmup_start, c.warmup_steps, c.max_steps) == (2e-3, 0.01, 0.01, 1000, 30000)
    assert (c.grid_x, c.grid_y, c.grid_l) == (16, 16, 8)


@pytest.mark.parametrize("step", [1, 2, 500, 1000, 1001, 29999, 30000])
def test_learning_rate(step):
    c = AppearanceConfig(num_images=1)
    assert learning_rate(c, step) == pytest.approx(ref.learning_rate(step), rel=1e-14)
    if step == 1:
        assert learning_rate(c, step) == pytest.approx(2e-3 * 0.01, rel=1e-14)       # warm-up starts at w0
    if step == 1001:
        assert learning_rate(c, step) == pytest.approx(2e-3 * 0.01 ** (1000 / 30000), rel=1e-14)   # warmed up


def test_capi_bilagrid_argument_checks():
    L = capi.lib()
    assert L.gsb_bilagrid_workspace_bytes(0, 5) == 0 and L.gsb_bilagrid_workspace_bytes(5, -1) == 0
    assert L.gsb_bilagrid_workspace_bytes(1 << 15, 1 << 15) > 0 and L.gsb_bilagrid_workspace_bytes(1 << 16, 4) == 0
    sizes = [L.gsb_bilagrid_workspace_bytes(h, w) for h, w in ((1, 1), (48, 64), (1080, 1920), (4000, 6000))]
    assert sizes == sorted(sizes) and sizes[0] > 0
    assert sizes[2] == 225 * ref.chunks(1080, 1920) * 384 * 4
    ws = L.gsb_bilagrid_workspace_bytes(48, 64)
    # forward: sizes, NULLs, a misaligned grid
    assert L.gsb_bilagrid_slice_forward(0, 64, P, P, P, None) == BAD
    assert L.gsb_bilagrid_slice_forward(48, (1 << 15) + 1, P, P, P, None) == BAD
    assert L.gsb_bilagrid_slice_forward(48, 64, None, P, P, None) == BAD
    assert L.gsb_bilagrid_slice_forward(48, 64, P, P, None, None) == BAD
    assert L.gsb_bilagrid_slice_forward(48, 64, C.c_void_p(260), P, P, None) == BAD
    # backward: sizes, NULLs, a short or misaligned workspace
    args = lambda **kw: [kw.get(k, d) for k, d in (("H", 48), ("W", 64), ("grid", P), ("rgb", P), ("v_out", P),
                                                   ("scale", 1.0), ("v_rgb", P), ("v_grid", P), ("ws", P),
                                                   ("ws_bytes", ws), ("stream", None))]
    assert L.gsb_bilagrid_slice_backward(*args(H=-1)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(v_rgb=None)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(v_grid=None)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(v_out=None)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(ws=None)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(ws_bytes=ws - 1)) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(ws=C.c_void_p(272))) == BAD
    assert L.gsb_bilagrid_slice_backward(*args(grid=C.c_void_p(260))) == BAD
    # tv: the grid count, NULLs
    assert L.gsb_bilagrid_tv(0, P, 1.0, P, None, None) == BAD
    assert L.gsb_bilagrid_tv(3, None, 1.0, P, None, None) == BAD
    assert L.gsb_bilagrid_tv(3, P, 1.0, None, P, None) == BAD
    assert capi.BILAGRID_FLOATS == 8 * 16 * 16 * 12


def test_identity_grids_in_both_orders():
    import torch
    from opensplat_b200.appearance import from_gsplat_order, identity_grids, to_gsplat_order
    g = identity_grids(2, "cpu")
    gs = to_gsplat_order(g)
    assert tuple(gs.shape) == (2, 12, 8, 16, 16)
    eye = torch.tensor([1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])
    assert torch.equal(gs[1, :, 3, 4, 5], eye)
    assert torch.equal(from_gsplat_order(gs), g)
    import numpy as np
    assert np.array_equal(g[0].numpy(), ref.identity())


def test_trainer_refuses_appearance_with_a_group():
    from opensplat_b200.trainer import SplatTrainer
    with pytest.raises(ValueError):
        SplatTrainer({}, appearance=AppearanceConfig(num_images=2), group=object(), device="cpu")
