"""CPU: the host side of the 3-D smoothing filter (DESIGN D24) -- Filter3DConfig's checks, the recompute schedule for
both refinement strategies, the C ABI's argument checks (no kernel runs) and the trainer's refusals."""
import ctypes as C

import pytest
import torch

from opensplat_b200 import capi
from opensplat_b200.densify import RefineConfig
from opensplat_b200.filter3d import Filter3DConfig, recompute_due
from opensplat_b200.mcmc import MCMCConfig
from opensplat_b200.model import Camera

P = C.c_void_p(256)      # any 256-byte aligned address: every call below is rejected before it is used
BAD = -1


def cam(**kw):
    a = dict(width=64, height=48, fx=50.0, fy=50.0, cx=32.0, cy=24.0, cam_to_world=torch.eye(4))
    a.update(kw)
    return Camera(**a)


def test_config_checks():
    c = Filter3DConfig(cameras=[cam(), cam()])
    assert (c.variance, c.near, c.margin, c.recompute_every) == (0.2, 0.2, 0.15, 100)
    assert isinstance(c.cameras, tuple) and len(c.cameras) == 2
    with pytest.raises(Exception):
        c.variance = 1.0                                     # frozen
    for bad in (dict(cameras=[]), dict(cameras=cam()), dict(cameras=[object()]), dict(cameras=[cam(fx=0.0)]),
                dict(cameras=[cam(width=0)]), dict(cameras=[cam()], variance=-1.0),
                dict(cameras=[cam()], near=float("nan")), dict(cameras=[cam()], margin=float("inf")),
                dict(cameras=[cam()], variance=True), dict(cameras=[cam()], recompute_every=0),
                dict(cameras=[cam()], recompute_every=2.0)):
        with pytest.raises(ValueError):
            Filter3DConfig(**bad)
    assert Filter3DConfig(cameras=[cam()], variance=0, near=0, margin=0).near == 0


def test_schedule_refine_config():
    rc, fc = RefineConfig(max_steps=1000), Filter3DConfig(cameras=[cam()], recompute_every=100)
    assert rc.stop_split_at == 500
    due = [s for s in range(1, 1001) if recompute_due(rc, fc, s, False)]
    assert due == [600, 700, 800]                     # > 500, and not within the last 100 steps before 1000
    assert recompute_due(rc, fc, 7, True) and recompute_due(rc, fc, 1000, True)
    assert not recompute_due(rc, fc, 500, False) and not recompute_due(rc, fc, 900, False)


def test_schedule_mcmc():
    mc, fc = MCMCConfig(refine_stop=500, max_steps=1000), Filter3DConfig(cameras=[cam()], recompute_every=50)
    due = [s for s in range(1, 1001) if recompute_due(mc, fc, s, False)]
    assert due == list(range(500, 950, 50))           # >= refine_stop, and step < max_steps - 50
    assert recompute_due(mc, fc, 300, True)


def test_capi_argument_checks():
    L = capi.lib()
    assert capi.FILTER3D_CAM_FLOATS == 18 and L.gsb_filter3d_workspace_bytes() == 8
    fc = L.gsb_filter3d_compute
    ok = dict(n=10, means=P, k=3, cams=P, near=0.2, margin=0.15, var=0.2, ws=P, wsb=8, out=P)

    def call(**kw):
        a = dict(ok)
        a.update(kw)
        return fc(a["n"], a["means"], a["k"], a["cams"], a["near"], a["margin"], a["var"], a["ws"], a["wsb"],
                  a["out"], None)
    for bad in (dict(n=-1), dict(k=0), dict(near=-0.1), dict(near=float("inf")), dict(margin=-1.0),
                dict(var=float("nan")), dict(means=None), dict(cams=None), dict(out=None), dict(ws=None), dict(wsb=4),
                dict(ws=C.c_void_p(258))):
        assert call(**bad) == BAD, bad
    assert call(n=0, means=None, out=None, ws=None) == 0      # nothing to do: no launch
    assert L.gsb_filter3d_bake(-1, P, P, P, P, P, None) == BAD
    for k in range(5):
        a = [P] * 5
        a[k] = None
        assert L.gsb_filter3d_bake(4, *a, None) == BAD
        b = [P] * 3
        if k < 3:
            b[k] = None
            assert L.gsb_reset_opacity_filter3d(4, 0.0, 0.2, *b, P, P, None) == BAD
    assert L.gsb_filter3d_bake(0, None, None, None, None, None, None) == 0
    assert L.gsb_reset_opacity_filter3d(-1, 0.0, 0.2, P, P, P, None, None, None) == BAD


def test_capi_projection_argument_checks():
    L = capi.lib()
    fwd = lambda **kw: [kw.get(k, d) for k, d in (
        ("n", 10), ("means", P), ("scales", P), ("glob", 1.0), ("quats", P), ("logits", P), ("f", P), ("view", P),
        ("proj", P), ("fx", 100.0), ("fy", 100.0), ("cx", 32.0), ("cy", 24.0), ("H", 48), ("W", 64), ("tx", 4),
        ("ty", 3), ("clip", 0.01), ("cov3d", P), ("xys", P), ("depths", P), ("radii", P), ("conics", P),
        ("nth", P), ("opac", P), ("aa", 0), ("stream", None))]
    f = L.gsb_project_forward_activated_filter3d
    for bad in (dict(aa=2), dict(aa=-1), dict(f=None), dict(n=-1), dict(H=0), dict(logits=None), dict(opac=None),
                dict(quats=C.c_void_p(260)), dict(xys=C.c_void_p(260))):
        assert f(*fwd(**bad)) == BAD, bad
    assert f(*fwd(n=0, f=None)) == 0
    bwd = lambda **kw: [kw.get(k, d) for k, d in (
        ("n", 10), ("means", P), ("scales", P), ("glob", 1.0), ("quats", P), ("logits", P), ("f", P), ("view", P),
        ("proj", P), ("fx", 100.0), ("fy", 100.0), ("H", 48), ("W", 64), ("radii", P), ("conics", P), ("v_xy", P),
        ("v_depth", None), ("v_conic", P), ("v_opacity", P), ("v_means", P), ("v_scales", P), ("v_quats", P),
        ("v_logits", P), ("acc", 0), ("aa", 0), ("cg", 0), ("partials", None), ("stream", None))]
    b = L.gsb_project_backward_activated_filter3d
    for bad in (dict(acc=2), dict(aa=-1), dict(cg=2), dict(cg=1), dict(f=None), dict(n=-1), dict(W=0),
                dict(logits=None), dict(v_logits=None), dict(means=None), dict(v_quats=C.c_void_p(264))):
        assert b(*bwd(**bad)) == BAD, bad
    assert b(*bwd(n=0, f=None, cg=1)) == 0


def test_trainer_refusals():
    from opensplat_b200.trainer import SplatTrainer
    with pytest.raises(ValueError, match="filter3d"):
        SplatTrainer({}, filter3d=object(), device="cpu")
    with pytest.raises(ValueError, match="filter3d"):
        SplatTrainer({}, filter3d={"cameras": [cam()]}, device="cpu")
