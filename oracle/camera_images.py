"""numpy restatement of the reference's image preparation (Camera::loadImage / Camera::getImage,
input_data.cpp:40-117) at the level of the OpenCV 4 calls it makes, for tests/golden/make_golden_images.py and the
host tests.  Every float operation is a separate numpy ufunc in the precision OpenCV uses (nothing contracted), so
the results are the bytes csrc/image.cu writes.

  - resize_area: cv::resize(INTER_AREA) on 3-channel u8 (hal::resize): the integer-scale fast path
    (resizeAreaFast_Invoker: (s+2)>>2 at scale 2, rint(float(s) * (1.f/area)) otherwise, rint(float(s)/count) on
    partial border cells) and the general path (computeResizeAreaTab weights from double cell edges, a float
    horizontal accumulation per source row, sum += beta*buf per source row, saturating rint);
  - undistort: cv::undistort with newK, stripe by stripe as OpenCV computes it (rows of
    min(max(1, 4096 / cols), rows), the new principal point shifted by the stripe's first row), the fp64
    initUndistortRectifyMap quantised to 1/32 pixel (CV_16SC2) and the fixed-point bilinear remap (15-bit weights,
    BORDER_CONSTANT 0);
  - load_image / get_image: the two Camera methods on a decoded RGB u8 image.
The optimal new camera matrix is opensplat_b200.images.get_optimal_new_camera_matrix (a host fp64 function, tested
against cv2 directly)."""
import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps


def cv_round(x):
    """cvRound / saturate_cast<int>(double): round half to even."""
    return int(np.rint(np.float64(x)))


def resize_scales(src_h, src_w, dst_h, dst_w, inv_scale=None):
    """(scale_x, scale_y) of hal::resize: from the sizes (dsize given), or 1/inv_scale (dsize empty, inv_scale the
    float factor cv::resize received)."""
    if inv_scale is None:
        ix, iy = np.float64(dst_w) / np.float64(src_w), np.float64(dst_h) / np.float64(src_h)
    else:
        ix = iy = np.float64(np.float32(inv_scale))
    return np.float64(1.0) / ix, np.float64(1.0) / iy


def area_tab(ssize, dsize, scale):
    """computeResizeAreaTab: per destination index the list [(source index, float32 weight)] in OpenCV's order."""
    out = []
    for d in range(dsize):
        fs1 = np.float64(d) * scale
        fs2 = fs1 + scale
        cell = min(scale, np.float64(ssize) - fs1)
        s1, s2 = int(np.ceil(fs1)), int(np.floor(fs2))
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        e = []
        if s1 - fs1 > 1e-3:
            e.append((s1 - 1, np.float32((s1 - fs1) / cell)))
        for s in range(s1, s2):
            e.append((s, np.float32(1.0 / cell)))
        if fs2 - s2 > 1e-3:
            e.append((s2, np.float32(min(min(fs2 - s2, 1.0), cell) / cell)))
        out.append(e)
    return out


def _padded(tab):
    """[d, E] index / weight arrays; padding entries have weight 0 (adding 0*x to a non-negative sum is exact)."""
    E = max(len(e) for e in tab)
    idx = np.zeros((len(tab), E), np.int64)
    w = np.zeros((len(tab), E), np.float32)
    for d, e in enumerate(tab):
        for k, (s, a) in enumerate(e):
            idx[d, k], w[d, k] = s, a
    return idx, w


def resize_area(img, dst_h, dst_w, inv_scale=None):
    """cv::resize(img, Size(dst_w, dst_h), INTER_AREA) of a u8 [h,w,3] image; inv_scale: the float factor when
    cv::resize was called with an empty dsize (dst then = cvRound(src * inv_scale))."""
    img = np.ascontiguousarray(img, np.uint8)
    H, W, _ = img.shape
    if (dst_h, dst_w) == (H, W):
        return img.copy()
    sx, sy = resize_scales(H, W, dst_h, dst_w, inv_scale)
    assert sx >= 1 and sy >= 1
    isx, isy = cv_round(sx), cv_round(sy)
    if abs(sx - isx) < DBL_EPSILON and abs(sy - isy) < DBL_EPSILON:
        return _resize_area_fast(img, dst_h, dst_w, isx, isy)
    xi, xw = _padded(area_tab(W, dst_w, sx))
    yi, yw = _padded(area_tab(H, dst_h, sy))
    f = img.astype(np.float32)
    acc = np.zeros((dst_h, dst_w, 3), np.float32)
    for ey in range(yi.shape[1]):
        rows = f[yi[:, ey]]                                   # [dh, W, 3]
        buf = np.zeros((dst_h, dst_w, 3), np.float32)
        for ex in range(xi.shape[1]):
            buf = buf + rows[:, xi[:, ex], :] * xw[None, :, ex, None]
        acc = acc + yw[:, ey, None, None] * buf
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def _resize_area_fast(img, dh, dw, isx, isy):
    H, W, _ = img.shape
    out = np.zeros((dh, dw, 3), np.uint8)
    full_w = W // isx
    scale = np.float32(1.0) / np.float32(isx * isy)
    for dy in range(dh):
        y0 = dy * isy
        if y0 >= H:
            continue
        full_row = y0 + isy <= H
        for dx in range(dw):
            x0 = dx * isx
            cell = img[y0:min(y0 + isy, H), x0:min(x0 + isx, W)].astype(np.int64)
            s = cell.sum(axis=(0, 1))
            if full_row and dx < full_w:
                if isx == 2 and isy == 2:
                    out[dy, dx] = (s + 2) >> 2
                else:
                    out[dy, dx] = np.clip(np.rint(s.astype(np.float32) * scale), 0, 255)
            else:
                cnt = np.float32(cell.shape[0] * cell.shape[1])
                out[dy, dx] = np.clip(np.rint(s.astype(np.float32) / cnt), 0, 255)
    return out


def stripe_rows(h, w):
    """The stripe height of cv::undistort."""
    return min(max(1, 4096 // max(w, 1)), h)


def undistort_map(h, w, K, dist, newK):
    """The CV_16SC2 map cv::undistort uses, as (iu, iv) int64 [h,w] in 1/32 pixel: K / newK (fx, fy, cx, cy) and
    dist (k1, k2, p1, p2, k3), each value a float32 widened to double."""
    fx, fy, u0, v0 = (np.float64(np.float32(v)) for v in K)
    a, b, c, e0 = (np.float64(np.float32(v)) for v in newK)
    k1, k2, p1, p2, k3 = (np.float64(np.float32(v)) for v in dist)
    r = np.arange(h)
    ys = (r // stripe_rows(h, w)) * stripe_rows(h, w)
    i = (r - ys).astype(np.float64)[:, None]
    e = (e0 - ys.astype(np.float64))[:, None]           # Ar(1,2) = v0 - y of the stripe
    dinv = np.float64(1.0) / (a * b)                      # cv::invert's 3x3 closed form: d = 1/det
    ir0, ir2, ir4 = b * dinv, -(c * b) * dinv, a * dinv
    ir5, ir8 = -(a * e) * dinv, (a * b) * dinv
    j = np.arange(w, dtype=np.float64)[None, :]
    inv_w = np.float64(1.0) / ir8
    x = (j * ir0 + ir2) * inv_w
    y = (i * ir4 + ir5) * inv_w
    x, y = np.broadcast_arrays(x, y)
    x2, y2 = x * x, y * y
    r2 = x2 + y2
    xy2 = 2.0 * x * y
    kr = 1.0 + ((k3 * r2 + k2) * r2 + k1) * r2
    xd = x * kr + p1 * xy2 + p2 * (r2 + 2.0 * x2)
    yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * xy2
    u = fx * xd + u0
    v = fy * yd + v0
    lim = np.float64(2 ** 31 - 1)
    iu = np.rint(np.clip(u * 32.0, -lim - 1, lim)).astype(np.int64)
    iv = np.rint(np.clip(v * 32.0, -lim - 1, lim)).astype(np.int64)
    return iu, iv


def remap_bilinear(img, iu, iv):
    """cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a u8 [h,w,3] image with the quantised map (iu, iv)."""
    H, W, _ = img.shape
    sx = ((iu >> 5) + 32768) % 65536 - 32768           # (short)(iu >> INTER_BITS)
    sy = ((iv >> 5) + 32768) % 65536 - 32768
    ax, ay = iu & 31, iv & 31
    wts = [(32 - ay) * (32 - ax) * 32, (32 - ay) * ax * 32, ay * (32 - ax) * 32, ay * ax * 32]
    src = img.astype(np.int64)

    def px(yy, xx):
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        return np.where(ok[..., None], src[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0)

    acc = (px(sy, sx) * wts[0][..., None] + px(sy, sx + 1) * wts[1][..., None]
           + px(sy + 1, sx) * wts[2][..., None] + px(sy + 1, sx + 1) * wts[3][..., None])
    out = np.clip((acc + (1 << 14)) >> 15, 0, 255)
    outside = (sx >= W) | (sx + 1 < 0) | (sy >= H) | (sy + 1 < 0)
    out[outside] = 0
    return out.astype(np.uint8)


def undistort(img, K, dist, newK, roi=None):
    """cv::undistort(img, K, dist, newK), cropped to roi (x, y, w, h) if given."""
    h, w, _ = img.shape
    iu, iv = undistort_map(h, w, K, dist, newK)
    if roi is not None:
        x, y, rw, rh = roi
        iu, iv = iu[y:y + rh, x:x + rw], iv[y:y + rh, x:x + rw]
    return remap_bilinear(img, iu, iv)


def load_image(img, width, height, fx, fy, cx, cy, dist=(0, 0, 0, 0, 0), downscale_factor=1.0):
    """Camera::loadImage on a decoded RGB u8 image: returns (u8 image, (width, height, fx, fy, cx, cy), newK, roi).
    dist = (k1, k2, p1, p2, k3).  newK is the float32 (fx, fy, cx, cy) of getOptimalNewCameraMatrix (or None without
    distortion); roi the crop (x, y, w, h)."""
    from opensplat_b200.images import get_optimal_new_camera_matrix
    f32 = np.float32
    img = np.ascontiguousarray(img, np.uint8)
    fx, fy, cx, cy = f32(fx), f32(fy), f32(cx), f32(cy)
    rescale = f32(1.0)
    if img.shape[0] != height or img.shape[1] != width:
        rescale = f32(img.shape[0]) / f32(height)
    fx, fy, cx, cy = fx * rescale, fy * rescale, cx * rescale, cy * rescale
    if f32(downscale_factor) > f32(1.0):
        s = f32(1.0) / f32(downscale_factor)
        dh, dw = cv_round(img.shape[0] * np.float64(s)), cv_round(img.shape[1] * np.float64(s))
        img = resize_area(img, dh, dw, inv_scale=s)
        fx, fy, cx, cy = fx * s, fy * s, cx * s, cy * s
    h, w, _ = img.shape
    newK, roi = None, (0, 0, w, h)
    if any(f32(d) != 0 for d in dist):
        newK, roi = get_optimal_new_camera_matrix((fx, fy, cx, cy), dist, (w, h))
        img = undistort(img, (fx, fy, cx, cy), dist, newK, roi)
        fx, fy, cx, cy = (f32(v) for v in newK)
    else:
        img = img.copy()
    return img, (img.shape[1], img.shape[0], float(fx), float(fy), float(cx), float(cy)), newK, roi


def get_image(img, factor):
    """Camera::getImage(factor) on the stored u8 level (tensorToImage(imageToTensor(u)) == u for every byte)."""
    if factor <= 1:
        return img
    return resize_area(img, img.shape[0] // factor, img.shape[1] // factor)
