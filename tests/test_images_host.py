"""CPU-only: the image preparation of Camera::loadImage / getImage without a GPU -- the numpy restatement
(oracle/camera_images.py) against the OpenCV golden (tests/golden/camera_images.npz), the host
get_optimal_new_camera_matrix, the validation split against stored glibc values, model.Camera's distortion fields
and the argument checks of the three C entry points (which return before any launch)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import camera_images as ci  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "camera_images.npz"))
CASES = [str(c) for c in G["cases"]]


def _args(name):
    cw, ch, fx, fy, cx, cy = G[f"{name}.camera"]
    return int(cw), int(ch), fx, fy, cx, cy, tuple(float(v) for v in G[f"{name}.dist"]), float(G[f"{name}.factor"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_load_image_matches_the_golden(name):
    cw, ch, fx, fy, cx, cy, dist, factor = _args(name)
    img, intr, new_k, roi = ci.load_image(G[f"{name}.image"], cw, ch, fx, fy, cx, cy, dist, factor)
    assert np.array_equal(img, G[f"{name}.loaded_oracle"])
    assert tuple(roi) == tuple(G[f"{name}.roi"])
    assert np.array_equal(np.array(intr[2:], np.float32), G[f"{name}.intrinsics"])
    assert tuple(intr[:2]) == tuple(G[f"{name}.size"])
    # equal to cv2 outside the recorded one-map-step pixels
    diff = np.any(img != G[f"{name}.loaded_cv2"], axis=-1)
    recorded = np.zeros_like(diff)
    md = G[f"{name}.map_diff"]
    recorded[md[:, 0], md[:, 1]] = True
    assert not (diff & ~recorded).any()


@pytest.mark.parametrize("name", CASES)
def test_oracle_get_image_is_cv2_byte_for_byte(name):
    ref = G[f"{name}.loaded_cv2"]
    for f in G[f"{name}.levels"]:
        assert np.array_equal(ci.get_image(ref, int(f)), G[f"{name}.level{int(f)}"]), f


@pytest.mark.parametrize("name", [c for c in CASES if f"{c}.new_k" in G.files])
def test_optimal_new_camera_matrix_is_cv2s(name):
    """newK bit-equal to cv2's CV_32F matrix, the ROI exact."""
    from opensplat_b200.images import get_optimal_new_camera_matrix
    cw, ch, fx, fy, cx, cy, dist, factor = _args(name)
    f32 = np.float32
    img = G[f"{name}.image"]
    rescale = f32(img.shape[0]) / f32(ch) if img.shape[:2] != (ch, cw) else f32(1.0)
    K = [f32(v) * rescale for v in (fx, fy, cx, cy)]
    if f32(factor) > 1:
        K = [k * (f32(1.0) / f32(factor)) for k in K]
    h, w = ci.load_image(img, cw, ch, fx, fy, cx, cy, (0, 0, 0, 0, 0), factor)[0].shape[:2]
    new_k, roi = get_optimal_new_camera_matrix(K, dist, (w, h))
    assert np.array_equal(np.array(new_k, np.float32), G[f"{name}.new_k"])
    assert tuple(roi) == tuple(G[f"{name}.roi"])


def test_split_matches_glibc():
    from opensplat_b200.images import split_cameras
    for n, val in zip(G["split.n"], G["split.val"]):
        train, v = split_cameras(int(n), True)
        assert v == int(val) and train == [k for k in range(int(n)) if k != v]
    assert split_cameras(4, False) == ([0, 1, 2, 3], None)
    assert split_cameras(3, True, "b.jpg", ["x/a.jpg", "y/b.jpg", "c.jpg"]) == ([0, 2], 1)
    with pytest.raises(ValueError):
        split_cameras(3, True, "d.jpg", ["a.jpg", "b.jpg", "c.jpg"])


def test_camera_distortion_fields_default_to_zero():
    from opensplat_b200.model import Camera
    c = Camera(4, 3, 1.0, 2.0, 3.0, 4.0, np.eye(4))
    assert (c.k1, c.k2, c.k3, c.p1, c.p2) == (0.0, 0.0, 0.0, 0.0, 0.0)
    d = Camera(4, 3, 1.0, 2.0, 3.0, 4.0, np.eye(4), k1=-0.1, p2=0.01)
    assert (d.k1, d.p2, d.width, d.fx) == (-0.1, 0.01, 4, 1.0)


def test_capi_image_argument_checks():
    """Bad arguments return GSB_ERR_INVALID_ARG before anything is launched (no GPU needed)."""
    from opensplat_b200 import capi
    L = capi.lib()
    a, b = C.c_void_p(256), C.c_void_p(512)
    bad_resize = [(0, 8, a, 4, 4, b, 0.0), (8, 8, a, 9, 4, b, 0.0), (8, 8, None, 4, 4, b, 0.0),
                  (8, 8, a, 4, 4, a, 0.0), (8, 8, a, 4, 4, b, 1.5), (8, 8, a, 4, 4, b, -0.5),
                  (8, 8, a, 3, 4, b, 0.5)]
    for args in bad_resize:
        assert L.gsb_resize_area_u8(*args, None) == -1, args
    K = (10.0, 10.0, 4.0, 4.0)
    D = (-0.1, 0.0, 0.0, 0.0, 0.0)
    bad_und = [((0, 8), (0, 0, 8, 8)), ((8, 8), (1, 0, 8, 8)), ((8, 8), (0, 0, 8, 9)), ((8, 8), (-1, 0, 4, 4))]
    for (h, w), roi in bad_und:
        assert L.gsb_undistort_u8(h, w, a, *K, *D, *K, *roi, b, None) == -1, (h, w, roi)
    assert L.gsb_undistort_u8(8, 8, a, 0.0, 10.0, 4.0, 4.0, *D, *K, 0, 0, 8, 8, b, None) == -1
    assert L.gsb_undistort_u8(8, 8, a, *K, float("nan"), 0.0, 0.0, 0.0, 0.0, *K, 0, 0, 8, 8, b, None) == -1
    assert L.gsb_undistort_u8(8, 8, None, *K, *D, *K, 0, 0, 8, 8, b, None) == -1
    assert L.gsb_undistort_u8(8, 8, a, *K, *D, *K, 0, 0, 0, 8, None, None) == 0      # empty ROI: a no-op
    assert L.gsb_u8_to_f32_views(0, None, 4, 4, None, None) == 0
    assert L.gsb_u8_to_f32_views(-1, a, 4, 4, b, None) == -1
    assert L.gsb_u8_to_f32_views(1, a, 0, 4, b, None) == -1
    assert L.gsb_u8_to_f32_views(1, None, 4, 4, b, None) == -1
    assert L.gsb_version() >= 800


def test_u8_level_is_the_references_float_level():
    """tensorToImage(imageToTensor(u)) == u for every byte: (float(u) / 255 * 255) truncated to u8 is u, so the u8
    level the set stores is the reference's float level."""
    import torch
    u = torch.arange(256, dtype=torch.uint8)
    assert torch.equal((u.to(torch.float32) / 255.0 * 255.0).to(torch.uint8), u)
