"""Host-side checks of fisheye cameras (DESIGN D27): Camera validation, what carries the model, and the refusals."""
import numpy as np
import pytest

from opensplat_b200.model import Camera


def _fish(**kw):
    a = dict(width=64, height=48, fx=30.0, fy=31.0, cx=32.0, cy=24.0, cam_to_world=np.eye(4, dtype=np.float32),
             k1=0.05, k2=-0.01, k3=0.002, k4=-0.0003, model="fisheye")
    a.update(kw)
    return Camera(**a)


def test_camera_validation():
    c = _fish()
    assert c.model == "fisheye" and c.k4 == pytest.approx(-0.0003)
    p = Camera(64, 48, 30.0, 31.0, 32.0, 24.0, np.eye(4), 0.1, 0.01, 0.0, 0.001, 0.002)   # positional use unchanged
    assert p.model == "pinhole" and p.k4 == 0.0 and p.p2 == pytest.approx(0.002)
    with pytest.raises(ValueError):
        _fish(p1=0.01)
    with pytest.raises(ValueError):
        _fish(p2=-0.01)
    with pytest.raises(ValueError):
        Camera(64, 48, 30.0, 31.0, 32.0, 24.0, np.eye(4), k4=0.1)
    with pytest.raises(ValueError):
        _fish(model="equirect")


def test_adjusted_camera_and_replace_keep_the_model():
    from opensplat_b200.pose import adjusted_camera
    c = _fish()
    d = adjusted_camera(c, np.array([0.1, 0.0, 0.0, 1, 0, 0, 0, 1, 0], np.float32))
    assert (d.model, d.k1, d.k2, d.k3, d.k4) == (c.model, c.k1, c.k2, c.k3, c.k4)
    assert float(d.camToWorld[0, 3]) == pytest.approx(0.1)
    r = c.replace(width=32, fx=15.0)
    assert (r.model, r.k4, r.width, r.fx, r.height) == ("fisheye", c.k4, 32, 15.0, 48)


def test_filter3d_and_model_refuse_fisheye_cameras():
    from opensplat_b200.filter3d import Filter3DConfig
    from opensplat_b200.model import GaussianModel
    pin = Camera(64, 48, 30.0, 31.0, 32.0, 24.0, np.eye(4, dtype=np.float32))
    Filter3DConfig(cameras=[pin])
    with pytest.raises(ValueError):
        Filter3DConfig(cameras=[pin, _fish()])
    with pytest.raises(ValueError):
        GaussianModel.forward(object(), _fish(), 1)


def test_capi_fisheye_argument_checks():
    from opensplat_b200 import capi
    L = capi.lib()
    z = (0, None, None, 1.0, None, None, None)
    tail = (16, 16, 1, 1, 0.01) + (None,) * 7

    def fwd(fx=30.0, k=(0.0, 0.0, 0.0, 0.0), th=1.5, aa=0):
        return L.gsb_project_forward_fisheye(*z, fx, 30.0, 8.0, 8.0, *k, th, *tail, aa, None)

    def bwd(fx=30.0, k=(0.0, 0.0, 0.0, 0.0), th=1.5, acc=0, aa=0):
        return L.gsb_project_backward_fisheye(*z, fx, 30.0, *k, th, 16, 16, *(None,) * 10, acc, aa, None, None)

    assert fwd() == 0 and bwd() == 0
    for bad in (dict(fx=0.0), dict(k=(float("nan"), 0.0, 0.0, 0.0)), dict(k=(0.0, 0.0, 0.0, float("inf"))),
                dict(th=0.0), dict(th=1.6), dict(aa=2)):
        assert fwd(**bad) != 0, bad
        assert bwd(**bad) != 0, bad
    assert bwd(acc=-1) != 0


def test_trainer_refuses_fisheye_views_under_the_3d_filter():
    """SplatTrainer._fisheye is where a step's views are checked before any launch: the 3-D filter refuses a fisheye
    view, and a fisheye view's projection arguments carry theta_lim."""
    from types import SimpleNamespace

    from opensplat_b200.model import fisheye_theta_limit
    from opensplat_b200.trainer import SplatTrainer
    c = _fish()
    plain = SimpleNamespace(filter3d_cfg=None, _theta_lims={})
    assert SplatTrainer._fisheye(plain, Camera(64, 48, 30.0, 31.0, 32.0, 24.0, np.eye(4))) is None
    assert SplatTrainer._fisheye(plain, c) == (c.k1, c.k2, c.k3, c.k4, fisheye_theta_limit(c.k1, c.k2, c.k3, c.k4))
    with pytest.raises(ValueError):
        SplatTrainer._fisheye(SimpleNamespace(filter3d_cfg=object(), _theta_lims={}), c)


def test_image_set_argument_errors_with_fisheye_cameras():
    from opensplat_b200.images import ImageSet
    c = _fish()
    img = np.zeros((48, 64, 3), np.uint8)
    with pytest.raises(ValueError):
        ImageSet([c, c], [img])
    with pytest.raises(ValueError):
        ImageSet([c], [img], masks=[None, None])
    with pytest.raises(ValueError):
        ImageSet([c], [img.astype(np.float32)])
    with pytest.raises(ValueError):
        ImageSet([c], [img], downscale_factor=0.0)
