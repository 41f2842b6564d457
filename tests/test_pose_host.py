"""CPU: the host side of the pose corrections (DESIGN D22) -- PoseConfig's checks, the learning-rate schedule, the
shared image-index check, the trainer's refusals, and the C ABI's argument checks (no kernel runs)."""
import ctypes as C

import pytest

from opensplat_b200 import capi
from opensplat_b200.pose import PoseConfig, learning_rate

P = C.c_void_p(256)      # any 256-byte aligned address: every call below is rejected before it is used
BAD = -1


def test_config_checks():
    for bad in (dict(num_images=0), dict(num_images=-3), dict(num_images=1.5), dict(num_images=True),
                dict(num_images=2, lr=-1e-5), dict(num_images=2, reg=-1.0), dict(num_images=2, final_lr_factor=0.0),
                dict(num_images=2, max_steps=0), dict(num_images=2, max_steps=2.5), dict(num_images=2, lr=float("nan"))):
        with pytest.raises(ValueError):
            PoseConfig(**bad)
    c = PoseConfig(num_images=3)
    assert (c.lr, c.reg, c.final_lr_factor, c.max_steps) == (1e-5, 1e-6, 0.01, 30000)
    assert PoseConfig(num_images=1, lr=0.0).lr == 0.0        # a frozen correction is allowed


@pytest.mark.parametrize("step", [1, 2, 15000, 30000, 30001])
def test_learning_rate(step):
    c = PoseConfig(num_images=1)
    assert learning_rate(c, step) == pytest.approx(1e-5 * 0.01 ** ((step - 1) / 30000), rel=1e-14)
    assert learning_rate(c, 1) == 1e-5
    assert learning_rate(PoseConfig(num_images=1, lr=2e-4, final_lr_factor=0.5, max_steps=10), 11) == \
        pytest.approx(1e-4, rel=1e-14)


def test_image_index_check():
    from opensplat_b200.trainer import check_images
    assert check_images(2, 1, 3) == [2] and check_images([0, 2], 2, 3) == [0, 2] and check_images((1,), 1, 3) == [1]
    for image, views in ((None, 1), (-1, 1), (3, 1), (1.0, 1), (True, 1), ([0, 1], 1), (0, 2), ([0], 2),
                         ([0, 3], 2)):
        with pytest.raises(ValueError):
            check_images(image, views, 3)


def test_trainer_refusals():
    from opensplat_b200.appearance import AppearanceConfig
    from opensplat_b200.trainer import SplatTrainer
    with pytest.raises(ValueError, match="group"):
        SplatTrainer({}, pose=PoseConfig(num_images=2), group=object(), device="cpu")
    with pytest.raises(ValueError, match="num_images"):
        SplatTrainer({}, pose=PoseConfig(num_images=2), appearance=AppearanceConfig(num_images=3), device="cpu")


def test_capi_pose_argument_checks():
    L = capi.lib()
    assert capi.POSE_FLOATS == 9 and capi.CAMGRAD_TERMS == 24
    assert L.gsb_project_camera_partials_floats(0) == 0 and L.gsb_project_camera_partials_floats(-5) == 0
    assert L.gsb_project_camera_partials_floats(1) == 24 and L.gsb_project_camera_partials_floats(256) == 24
    assert L.gsb_project_camera_partials_floats(257) == 48 and L.gsb_project_camera_partials_floats(65537) == 24 * 257
    # the camgrad projection backward: the flags, the partials, and the checks of the plain entry point
    args = lambda **kw: [kw.get(k, d) for k, d in (
        ("n", 10), ("means", P), ("scales", P), ("glob", 1.0), ("quats", P), ("opac", P), ("view", P), ("proj", P),
        ("fx", 100.0), ("fy", 100.0), ("H", 48), ("W", 64), ("radii", P), ("conics", P), ("v_xy", P),
        ("v_depth", None), ("v_conic", P), ("v_opacity", P), ("v_means", P), ("v_scales", P), ("v_quats", P),
        ("v_logits", P), ("acc", 0), ("aa", 0), ("partials", P), ("stream", None))]
    fn = L.gsb_project_backward_activated_camgrad
    assert fn(*args(acc=2)) == BAD and fn(*args(aa=-1)) == BAD
    assert fn(*args(partials=None)) == BAD
    assert fn(*args(n=-1)) == BAD and fn(*args(H=0)) == BAD
    assert fn(*args(means=None)) == BAD and fn(*args(v_logits=None)) == BAD and fn(*args(opac=None)) == BAD
    assert fn(*args(quats=C.c_void_p(260))) == BAD and fn(*args(v_quats=C.c_void_p(264))) == BAD
    assert fn(*args(n=0, partials=None)) == 0                # nothing to do: no launch
    # the reduce
    assert L.gsb_project_camera_grad_reduce(-1, P, P, P, None) == BAD
    assert L.gsb_project_camera_grad_reduce(3, None, P, P, None) == BAD
    assert L.gsb_project_camera_grad_reduce(3, P, None, P, None) == BAD
    assert L.gsb_project_camera_grad_reduce(3, P, P, None, None) == BAD
    # apply and backward
    for k in range(5):
        a = [P] * 5
        a[k] = None
        assert L.gsb_pose_apply(*a, None) == BAD
    for k in range(5):
        a = [P] * 5
        a[k] = None
        assert L.gsb_pose_backward(*a, 1.0, P, None) == BAD
    assert L.gsb_pose_backward(P, P, P, P, P, 1.0, None, None) == BAD
