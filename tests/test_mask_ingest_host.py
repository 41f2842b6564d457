"""CPU: the loss-mask ingest rules of DESIGN D26 (tests/mask_ingest_np.py) against the footprints read off the colour
restatement's weights (oracle/camera_images.py), the rules' purpose (a used output pixel's colour does not depend on
any ignored source pixel), and the argument checks of ImageSet(masks=), SplatTrainer.step(mask=) and
ops.MainLoss(mask=)."""
import types

import numpy as np
import pytest
import torch

import mask_ingest_np as mi
from oracle import camera_images as ci


def _mask(h, w, seed, p=0.08):
    rng = np.random.default_rng(seed)
    m = (rng.uniform(size=(h, w)) >= p).astype(np.uint8)
    m[rng.integers(0, h), :] = 0 if h > 2 else m[0, 0]
    return m


def _resize_footprints(H, W, dh, dw, inv_scale):
    """[dh,dw] lists of source pixels with a nonzero weight, from area_tab's float weights (the general path) or, on
    the integer-scale path, from the same table (whose entries there are the clipped cell)."""
    sx, sy = ci.resize_scales(H, W, dh, dw, inv_scale)
    tx = [[s for s, a in e if np.float32(a) != 0] for e in ci.area_tab(W, dw, sx)]
    ty = [[s for s, a in e if np.float32(a) != 0] for e in ci.area_tab(H, dh, sy)]
    return tx, ty


@pytest.mark.parametrize("H,W,dh,dw,inv", [(12, 17, 6, 8, None), (13, 19, 6, 9, None), (25, 33, 8, 11, None),
                                           (21, 30, 14, 20, np.float32(1 / 1.5)), (27, 31, 11, 12, np.float32(0.4)),
                                           (19, 26, 10, 13, np.float32(0.5)), (16, 24, 4, 6, None),
                                           (17, 23, 2, 2, None)])
def test_resize_mask_is_the_weight_footprint(H, W, dh, dw, inv):
    m = _mask(H, W, H * W)
    got = mi.resize_area_mask(m, dh, dw, inv_scale=inv)
    tx, ty = _resize_footprints(H, W, dh, dw, inv)
    want = np.array([[m[np.ix_(ty[y], tx[x])].all() for x in range(dw)] for y in range(dh)], np.uint8)
    assert np.array_equal(got, want)
    assert got.sum() < got.size and (got.sum() > 0 or dh * dw <= 4)


@pytest.mark.parametrize("H,W,dh,dw,inv", [(13, 19, 6, 9, None), (21, 30, 14, 20, np.float32(1 / 1.5)),
                                           (27, 31, 11, 12, np.float32(0.4)), (19, 26, 10, 13, np.float32(0.5))])
def test_a_used_resized_pixel_never_reads_an_ignored_one(H, W, dh, dw, inv):
    rng = np.random.default_rng(3)
    m = _mask(H, W, 5, p=0.1)
    img = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    img2 = img.copy()
    img2[m == 0] = rng.integers(0, 256, (int((m == 0).sum()), 3))
    used = mi.resize_area_mask(m, dh, dw, inv_scale=inv) != 0
    a, b = ci.resize_area(img, dh, dw, inv), ci.resize_area(img2, dh, dw, inv)
    assert np.array_equal(a[used], b[used])


def _tap_footprint(iu, iv, H, W):
    """Per output pixel: (taps with a nonzero fixed-point weight, whether all of them lie inside the image)."""
    sx, sy = ((iu >> 5) + 32768) % 65536 - 32768, ((iv >> 5) + 32768) % 65536 - 32768
    ax, ay = iu & 31, iv & 31
    out = np.empty(iu.shape, object)
    for idx in np.ndindex(iu.shape):
        w = {(0, 0): (32 - ay[idx]) * (32 - ax[idx]), (0, 1): (32 - ay[idx]) * ax[idx],
             (1, 0): ay[idx] * (32 - ax[idx]), (1, 1): ay[idx] * ax[idx]}
        taps = [(sy[idx] + dy, sx[idx] + dx) for (dy, dx), wt in w.items() if wt * 32 != 0]
        out[idx] = (taps, all(0 <= y < H and 0 <= x < W for y, x in taps))
    return out


@pytest.mark.parametrize("dist", [(-0.12, 0.03, 0.0, 0.0, 0.0), (0.08, -0.02, 0.002, -0.003, 0.01)])
@pytest.mark.parametrize("H,W", [(30, 41), (37, 52)])
def test_undistort_mask_is_the_tap_footprint(dist, H, W):
    from opensplat_b200.images import get_optimal_new_camera_matrix
    K = (np.float32(0.9 * W), np.float32(0.9 * W), np.float32(W / 2 - 0.3), np.float32(H / 2 + 0.2))
    newK, roi = get_optimal_new_camera_matrix(K, dist, (W, H))
    m = _mask(H, W, 11)
    iu, iv = ci.undistort_map(H, W, K, dist, newK)
    x, y, rw, rh = roi
    iu, iv = iu[y:y + rh, x:x + rw], iv[y:y + rh, x:x + rw]
    fp = _tap_footprint(iu, iv, H, W)
    want = np.array([[fp[i, j][1] and all(m[a, b] for a, b in fp[i, j][0]) for j in range(rw)] for i in range(rh)],
                    np.uint8)
    got = mi.undistort_mask(m, K, dist, newK, roi)
    assert np.array_equal(got, want)
    assert 0 < got.sum() < got.size
    # the purpose: a used pixel's colour does not depend on any ignored source pixel
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    img2 = img.copy()
    img2[m == 0] = rng.integers(0, 256, (int((m == 0).sum()), 3))
    a, b = ci.undistort(img, K, dist, newK, roi), ci.undistort(img2, K, dist, newK, roi)
    assert np.array_equal(a[got != 0], b[got != 0])


def test_remap_mask_edges():
    m = np.ones((4, 5), np.uint8)
    iu = np.array([[0, 31, 4 * 32, 4 * 32 + 1, -1, -32]])       # x = 0, 0 + 31/32, 4, 4 + 1/32, -1/32, -1
    iv = np.zeros_like(iu)
    assert mi.remap_mask(m, iu, iv).tolist() == [[1, 1, 1, 0, 0, 0]]
    iv = np.array([[3 * 32, 3 * 32 + 5, 0, 0, 0, 0]])
    iu = np.zeros_like(iv)
    assert mi.remap_mask(m, iu, iv)[0, :2].tolist() == [1, 0]


def test_load_and_get_mask_sizes_follow_the_image():
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (45, 61, 3)).astype(np.uint8)
    m = _mask(45, 61, 2)
    for f in (1.0, 1.5, 2.0, 2.5):
        for dist in ((0, 0, 0, 0, 0), (-0.1, 0.02, 0, 0, 0)):
            im, *_ = ci.load_image(img, 61, 45, 50.0, 50.0, 30.0, 22.0, dist, f)
            mm = mi.load_mask(m, 61, 45, 50.0, 50.0, 30.0, 22.0, dist, f)
            assert mm.shape == im.shape[:2] and mm.dtype == np.uint8
            for k in (2, 3, 4):
                assert mi.get_mask(mm, k).shape == ci.get_image(im, k).shape[:2]


# ---- argument checks ---------------------------------------------------------------------------------------------
def test_image_set_mask_arguments():
    from opensplat_b200 import images
    d = torch.device("cpu")
    ok = images._device_mask(np.array([[0, 3], [1, 0]], np.uint8), (2, 2), d, "m")
    assert ok.dtype == torch.uint8 and ok.tolist() == [[0, 1], [1, 0]]
    assert images._device_mask(torch.tensor([[True, False]]), (1, 2), d, "m").tolist() == [[1, 0]]
    for bad in (np.zeros((2, 3), np.uint8), np.zeros((2, 2, 1), np.uint8), np.zeros((2, 2), np.float32),
                torch.zeros(2, 2, dtype=torch.int32), [[1, 0], [0, 1]]):
        with pytest.raises(ValueError):
            images._device_mask(bad, (2, 2), d, "m")
    from opensplat_b200.model import Camera
    cam = Camera(4, 2, 3.0, 3.0, 2.0, 1.0, np.eye(4, dtype=np.float32))
    with pytest.raises(ValueError, match="masks for"):
        images.ImageSet([cam], [np.zeros((2, 4, 3), np.uint8)], masks=[None, None], device="cpu")


def test_step_mask_arguments():
    from opensplat_b200.trainer import SplatTrainer
    fake = types.SimpleNamespace(device=torch.device("cpu"))
    H, W = 3, 4
    u8, bl = torch.ones(H, W, dtype=torch.uint8), torch.ones(H, W, dtype=torch.bool)
    assert SplatTrainer._masks(fake, None, 2, H, W) == [None, None]
    got = SplatTrainer._masks(fake, bl, 1, H, W)
    assert got[0].dtype == torch.uint8 and got[0].data_ptr() == bl.data_ptr()
    got = SplatTrainer._masks(fake, [u8, None], 2, H, W)
    assert got[0] is u8 and got[1] is None
    assert len(SplatTrainer._masks(fake, torch.ones(2, H, W, dtype=torch.uint8), 2, H, W)) == 2
    bad = [torch.ones(H, W + 1, dtype=torch.uint8),                 # wrong size
           torch.ones(H, W, dtype=torch.float32),                   # wrong dtype
           torch.ones(1, H, W, dtype=torch.uint8),                  # wrong rank at B = 1
           torch.ones(W, H, dtype=torch.uint8).t(),                 # not contiguous
           np.ones((H, W), np.uint8)]                               # not a tensor
    for b in bad:
        with pytest.raises(ValueError):
            SplatTrainer._masks(fake, b, 1, H, W)
    with pytest.raises(ValueError):
        SplatTrainer._masks(fake, [u8], 2, H, W)                    # wrong count
    with pytest.raises(ValueError):
        SplatTrainer._masks(fake, u8, 2, H, W)                      # [H,W] at B = 2
    on_gpu = types.SimpleNamespace(device=torch.device("cuda:0"))
    with pytest.raises(ValueError):
        SplatTrainer._masks(on_gpu, u8, 1, H, W)                    # wrong device


def test_main_loss_mask_arguments():
    from opensplat_b200 import ops
    r = torch.zeros(3, 4, 3)
    for bad in (torch.ones(4, 3, dtype=torch.uint8), torch.ones(3, 4), torch.ones(3, 4, 1, dtype=torch.uint8)):
        with pytest.raises(ValueError):
            ops.MainLoss.apply(r, r, 0.2, bad)
