"""numpy restatement of the loss-mask ingest of DESIGN D26 (csrc/image.cu: gsb_resize_area_mask_u8,
gsb_undistort_mask_u8), next to oracle/camera_images.py's restatement of the colour path it follows.

A mask is u8 [h,w], nonzero = used; the outputs are 0 / 1.  An output pixel is used iff every source pixel with a
nonzero weight in the colour's output pixel is used:
  - resize_area_mask: on OpenCV's integer-scale fast path the cell clipped to the image (a cell wholly outside it is
    0); on the general path the entries of computeResizeAreaTab (oracle.camera_images.area_tab, its 1e-3 cut-offs
    included) on both axes; equal sizes normalise the mask;
  - remap_mask: the bilinear taps of the quantised map -- (sx, sy) always, the right taps iff ax > 0, the bottom taps
    iff ay > 0 -- all inside the image and used;
  - load_mask / get_mask: Camera::loadImage / Camera::getImage's steps, as oracle.camera_images.load_image /
    get_image take them."""
import numpy as np

from oracle.camera_images import (DBL_EPSILON, area_tab, cv_round, resize_scales, stripe_rows,  # noqa: F401
                                  undistort_map)


def resize_area_mask(mask, dst_h, dst_w, inv_scale=None):
    m = np.ascontiguousarray(mask) != 0
    H, W = m.shape
    if (dst_h, dst_w) == (H, W):
        return m.astype(np.uint8)
    sx, sy = resize_scales(H, W, dst_h, dst_w, inv_scale)
    isx, isy = cv_round(sx), cv_round(sy)
    out = np.zeros((dst_h, dst_w), np.uint8)
    if abs(sx - isx) < DBL_EPSILON and abs(sy - isy) < DBL_EPSILON:
        for dy in range(dst_h):
            for dx in range(dst_w):
                y0, x0 = dy * isy, dx * isx
                if y0 < H and x0 < W:
                    out[dy, dx] = m[y0:min(y0 + isy, H), x0:min(x0 + isx, W)].all()
        return out
    xs = [[s for s, _ in e] for e in area_tab(W, dst_w, sx)]
    ys = [[s for s, _ in e] for e in area_tab(H, dst_h, sy)]
    for dy in range(dst_h):
        rows = m[ys[dy]]
        for dx in range(dst_w):
            out[dy, dx] = rows[:, xs[dx]].all()
    return out


def remap_mask(mask, iu, iv):
    m = np.ascontiguousarray(mask) != 0
    H, W = m.shape
    sx = ((iu >> 5) + 32768) % 65536 - 32768
    sy = ((iv >> 5) + 32768) % 65536 - 32768
    xe = np.where((iu & 31) > 0, sx + 1, sx)
    ye = np.where((iv & 31) > 0, sy + 1, sy)
    inside = (sx >= 0) & (sy >= 0) & (xe < W) & (ye < H)
    c = lambda a, n: np.clip(a, 0, n - 1)
    used = inside & m[c(sy, H), c(sx, W)] & m[c(sy, H), c(xe, W)] & m[c(ye, H), c(sx, W)] & m[c(ye, H), c(xe, W)]
    return used.astype(np.uint8)


def undistort_mask(mask, K, dist, newK, roi=None):
    h, w = mask.shape
    iu, iv = undistort_map(h, w, K, dist, newK)
    if roi is not None:
        x, y, rw, rh = roi
        iu, iv = iu[y:y + rh, x:x + rw], iv[y:y + rh, x:x + rw]
    return remap_mask(mask, iu, iv)


def load_mask(mask, width, height, fx, fy, cx, cy, dist=(0, 0, 0, 0, 0), downscale_factor=1.0):
    """The mask of oracle.camera_images.load_image's image (same arguments, mask [h,w] at the decoded image's size)."""
    from opensplat_b200.images import get_optimal_new_camera_matrix
    f32 = np.float32
    m = (np.ascontiguousarray(mask) != 0).astype(np.uint8)
    fx, fy, cx, cy = f32(fx), f32(fy), f32(cx), f32(cy)
    rescale = f32(1.0)
    if m.shape[0] != height or m.shape[1] != width:
        rescale = f32(m.shape[0]) / f32(height)
    fx, fy, cx, cy = fx * rescale, fy * rescale, cx * rescale, cy * rescale
    if f32(downscale_factor) > f32(1.0):
        s = f32(1.0) / f32(downscale_factor)
        dh, dw = cv_round(m.shape[0] * np.float64(s)), cv_round(m.shape[1] * np.float64(s))
        m = resize_area_mask(m, dh, dw, inv_scale=s)
        fx, fy, cx, cy = fx * s, fy * s, cx * s, cy * s
    h, w = m.shape
    if any(f32(d) != 0 for d in dist):
        newK, roi = get_optimal_new_camera_matrix((fx, fy, cx, cy), dist, (w, h))
        m = undistort_mask(m, (fx, fy, cx, cy), dist, newK, roi)
    return m


def get_mask(mask, factor):
    if factor <= 1:
        return mask
    return resize_area_mask(mask, mask.shape[0] // factor, mask.shape[1] // factor)
