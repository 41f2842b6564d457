"""Writes tests/golden/camera_images.npz: Camera::loadImage / Camera::getImage (input_data.cpp:40-117) of OpenCV 4
(the Python cv2, the library the reference links) on seeded images, next to the restatement in
oracle/camera_images.py.  Needs cv2; the GPU tests only read the .npz.

    python tests/golden/make_golden_images.py

It refuses to write unless
  - every INTER_AREA resize of the restatement (loadImage's downscale and every getImage level) equals cv2's bytes;
  - the newK of images.get_optimal_new_camera_matrix equals cv2's float32 matrix and the ROI is equal;
  - every pixel where the restated undistortion differs from cv2.undistort has a quantised map coordinate exactly
    one 1/32 step from cv2's (cv2.initUndistortRectifyMap with CV_16SC2, stripe by stripe as cv::undistort calls it).
Those pixels are recorded per case (`<case>.map_diff`, [k,2] (y, x) in the cropped image)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "camera_images.npz")

# name: (image h, w, camera width, height, fx, fy, cx, cy, (k1, k2, p1, p2, k3), loadImage factor, getImage factors)
CASES = {
    "even": (96, 128, 128, 96, 110.0, 112.0, 64.5, 47.25, (0, 0, 0, 0, 0), 1.0, (2, 4, 8)),
    "odd": (75, 101, 101, 75, 90.0, 90.5, 50.3, 37.1, (0, 0, 0, 0, 0), 1.0, (2, 3, 4, 8)),
    "load_1_5": (90, 121, 121, 90, 100.0, 101.0, 60.2, 44.9, (0, 0, 0, 0, 0), 1.5, (2, 3)),
    "load_2_odd": (77, 103, 103, 77, 95.0, 95.0, 51.7, 38.2, (0, 0, 0, 0, 0), 2.0, (2, 4)),
    "load_2_5": (101, 151, 151, 101, 130.0, 129.0, 75.1, 50.6, (0, 0, 0, 0, 0), 2.5, (2, 3)),
    "radial": (120, 160, 160, 120, 150.0, 148.0, 81.3, 59.7, (-0.12, 0.03, 0, 0, 0.001), 1.0, (2, 4)),
    "radial_tangential": (121, 161, 161, 121, 140.0, 141.5, 79.9, 61.2, (-0.08, 0.02, 0.0015, -0.002, 0.0), 1.0,
                          (2, 3, 4)),
    "barrel": (144, 192, 192, 144, 120.0, 120.0, 96.4, 71.8, (-0.3, 0.09, 0, 0, -0.01), 2.0, (2,)),
    "rescaled": (75, 100, 200, 150, 180.0, 182.0, 99.6, 75.3, (-0.1, 0.02, 0.001, 0.0005, 0.0), 1.0, (2, 4)),
}
SPLIT_SIZES = (1, 2, 3, 5, 7, 10, 64, 1000)


def make_image(h, w, seed):
    """Smooth colour ramps plus noise: every byte value occurs, and the file stays small."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([127 + 120 * np.sin(0.11 * xx + 0.07 * yy), 127 + 120 * np.cos(0.05 * xx - 0.13 * yy),
                     255 * (xx + yy) / (h + w)], -1)
    return np.clip(base + rng.normal(0, 25, (h, w, 3)), 0, 255).astype(np.uint8)


def cv2_load(cv2, img, width, height, fx, fy, cx, cy, dist, factor):
    f32 = np.float32
    fx, fy, cx, cy = f32(fx), f32(fy), f32(cx), f32(cy)
    rescale = f32(1.0)
    if img.shape[0] != height or img.shape[1] != width:
        rescale = f32(img.shape[0]) / f32(height)
    fx, fy, cx, cy = fx * rescale, fy * rescale, cx * rescale, cy * rescale
    if f32(factor) > 1:
        s = f32(1.0) / f32(factor)
        img = cv2.resize(img, None, fx=float(s), fy=float(s), interpolation=cv2.INTER_AREA)
        fx, fy, cx, cy = fx * s, fy * s, cx * s, cy * s
    h, w = img.shape[:2]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    d8 = np.array(list(dist) + [0, 0, 0], np.float32)
    if np.any(d8 != 0):
        newK, roi = cv2.getOptimalNewCameraMatrix(K, d8, (w, h), 0)
        und = cv2.undistort(img, K, d8, None, newK)
        x, y, rw, rh = roi
        return und[y:y + rh, x:x + rw].copy(), K, d8, newK, tuple(int(v) for v in roi), img
    return img.copy(), K, d8, None, (0, 0, w, h), img


def cv2_map(cv2, h, w, K, d8, newK):
    """The (iu, iv) 1/32-pixel map cv::undistort uses, stripe by stripe."""
    from oracle.camera_images import stripe_rows
    st = stripe_rows(h, w)
    iu, iv = np.zeros((h, w), np.int64), np.zeros((h, w), np.int64)
    Ar = newK.astype(np.float64)
    v0 = Ar[1, 2]
    for y in range(0, h, st):
        n = min(st, h - y)
        Ar[1, 2] = v0 - y
        m1, m2 = cv2.initUndistortRectifyMap(K.astype(np.float64), d8.astype(np.float64), np.eye(3), Ar, (w, n),
                                             cv2.CV_16SC2)
        iu[y:y + n] = (m1[..., 0].astype(np.int64) << 5) | (m2.astype(np.int64) & 31)
        iv[y:y + n] = (m1[..., 1].astype(np.int64) << 5) | (m2.astype(np.int64) >> 5)
    return iu, iv


def main():
    import ctypes

    import cv2
    from oracle import camera_images as ci

    out = {}
    for ci_idx, (name, (h, w, cw, ch, fx, fy, cx, cy, dist, factor, levels)) in enumerate(CASES.items()):
        img = make_image(h, w, 100 + ci_idx)
        ref, K, d8, newK, roi, pre = cv2_load(cv2, img, cw, ch, fx, fy, cx, cy, dist, factor)
        mine, intr, my_newK, my_roi = ci.load_image(img, cw, ch, fx, fy, cx, cy, dist, factor)[:4]
        if not np.array_equal(ci.load_image(img, cw, ch, fx, fy, cx, cy, (0, 0, 0, 0, 0), factor)[0], pre):
            raise SystemExit(f"{name}: the loadImage resize differs from cv2")
        map_diff = np.zeros((0, 2), np.int32)
        if newK is not None:
            nk = (newK[0, 0], newK[1, 1], newK[0, 2], newK[1, 2])
            if tuple(np.float32(v) for v in my_newK) != tuple(np.float32(v) for v in nk) or my_roi != roi:
                raise SystemExit(f"{name}: newK / ROI differ from cv2: {my_newK} {my_roi} vs {nk} {roi}")
            diff = np.any(mine != ref, axis=-1)
            if diff.any():
                ph, pw = pre.shape[:2]
                iu_c, iv_c = cv2_map(cv2, ph, pw, K, d8, newK)
                iu_o, iv_o = ci.undistort_map(ph, pw, (K[0, 0], K[1, 1], K[0, 2], K[1, 2]), dist, my_newK)
                x, y = roi[0], roi[1]
                ys, xs = np.nonzero(diff)
                step = np.abs(iu_o[ys + y, xs + x] - iu_c[ys + y, xs + x]) + np.abs(iv_o[ys + y, xs + x] -
                                                                                    iv_c[ys + y, xs + x])
                if not np.all(step == 1):
                    raise SystemExit(f"{name}: {int(diff.sum())} undistorted pixels differ, not all by one map step")
                map_diff = np.stack([ys, xs], -1).astype(np.int32)
            out[f"{name}.new_k"] = np.array(nk, np.float32)
        elif not np.array_equal(mine, ref):
            raise SystemExit(f"{name}: the loaded image differs from cv2")
        out[f"{name}.image"] = img
        out[f"{name}.camera"] = np.array([cw, ch, fx, fy, cx, cy], np.float64)
        out[f"{name}.dist"] = np.array(dist, np.float32)
        out[f"{name}.factor"] = np.float32(factor)
        out[f"{name}.intrinsics"] = np.array(intr[2:], np.float32)      # fx, fy, cx, cy after loadImage
        out[f"{name}.size"] = np.array(intr[:2], np.int32)              # width, height after loadImage
        out[f"{name}.roi"] = np.array(roi, np.int32)
        out[f"{name}.loaded_cv2"] = ref
        out[f"{name}.loaded_oracle"] = mine
        out[f"{name}.map_diff"] = map_diff
        out[f"{name}.levels"] = np.array(levels, np.int32)
        for f in levels:
            lv = cv2.resize(ref, (ref.shape[1] // f, ref.shape[0] // f), interpolation=cv2.INTER_AREA)
            if not np.array_equal(ci.get_image(ref, f), lv):
                raise SystemExit(f"{name}: getImage({f}) differs from cv2")
            out[f"{name}.level{f}"] = lv
        print(f"{name}: loaded {mine.shape[1]}x{mine.shape[0]} roi {roi} newK "
              f"{None if newK is None else out[f'{name}.new_k'].tolist()} map-step pixels {len(map_diff)}")
    libc = ctypes.CDLL(None)
    vals = []
    for n in SPLIT_SIZES:
        libc.srand(ctypes.c_uint(42))
        vals.append(libc.rand() % n)
    out["split.n"] = np.array(SPLIT_SIZES, np.int64)
    out["split.val"] = np.array(vals, np.int64)
    out["cases"] = np.array(list(CASES))
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
