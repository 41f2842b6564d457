"""The training images prepared on the device as the reference's Camera prepares them (input_data.cpp:40-117).

    imgs = ImageSet(cams, images, downscale_factor=1.0)    # Camera::loadImage for every camera
    train, val = imgs.split(validate=True)                  # InputData::getCameras (--val)
    gt = imgs.gt(i, trainer_factor)                         # Camera::getImage: float32 [H,W,3] on the device

`images` are decoded RGB u8 [h,w,3] images (host or device), which is where the reference's imreadRGB hands over.
Everything after that runs on the device (csrc/image.cu):

  - loadImage: the intrinsics are rescaled to the decoded image (rescaleF), the image is downsized by
    `downscale_factor` with INTER_AREA (gsb_resize_area_u8, OpenCV 4's bytes), and a camera with k1/k2/k3/p1/p2 is
    undistorted with getOptimalNewCameraMatrix(alpha=0) and cropped to its ROI (gsb_undistort_u8, one launch that
    writes only the ROI).  As in the reference, cx/cy are newK's and are not shifted by the ROI origin.
  - getImage(f): the level f is INTER_AREA to (cols/f, rows/f) of the stored image, built on first use and kept as
    u8 on the device.  The reference converts its float image back to u8 with a truncating (t*255) first; that gives
    back the stored bytes for all 256 values, so the u8 level is the reference's level exactly, at a quarter of the
    memory of a float copy.
  - loss masks (DESIGN D26): `ImageSet(cams, images, masks=[...])` takes one u8 / bool [h,w] mask per image (nonzero =
    used) or None; each goes through its image's resize, undistortion and ROI crop (gsb_resize_area_mask_u8,
    gsb_undistort_mask_u8: a pixel stays used iff every source pixel its colour reads is used), and mask(i, f) serves
    the level f as a device u8 [H,W] 0 / 1 tensor, built on first use and cached as level() is (1 byte per pixel).
  - gt(): one gsb_u8_to_f32_views launch turns one or B stored levels into float32 u/255 (IEEE division, as
    imageToTensor) in a buffer the set owns; the next call overwrites it, so a training step allocates nothing.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import capi

UNDISTORT_GRID = 9          # getUndistortRectangles: a 9x9 grid over the image
UNDISTORT_ITERS = 5         # undistortPoints' default criteria: 5 iterations


def _undistort_points(pts, K, dist, P=None):
    """cv::undistortPoints of double points [m,2] with camera K = (fx, fy, cx, cy) (doubles), dist = (k1, k2, p1, p2,
    k3) (doubles) and the projection P = (fx, fy, cx, cy) (None: normalised coordinates)."""
    fx, fy, cx, cy = K
    k1, k2, p1, p2, k3 = dist
    ifx, ify = 1.0 / fx, 1.0 / fy
    out = []
    for u, v in pts:
        x = (u - cx) * ifx
        y = (v - cy) * ify
        x0, y0 = x, y
        for _ in range(UNDISTORT_ITERS):
            r2 = x * x + y * y
            icdist = 1.0 / (1.0 + ((k3 * r2 + k2) * r2 + k1) * r2)
            if icdist < 0:
                x = (u - cx) * ifx
                y = (v - cy) * ify
                break
            dx = 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
            dy = p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
            x = (x0 - dx) * icdist
            y = (y0 - dy) * icdist
        if P is not None:
            x, y = P[0] * x + P[2], P[1] * y + P[3]
        out.append((x, y))
    return out


def _rectangles(K, dist, size, P=None):
    """getUndistortRectangles: (inner, outer) as (x, y, w, h) doubles, from the 9x9 grid over [0, w-1] x [0, h-1]."""
    w, h = size
    N = UNDISTORT_GRID
    pts = [(float(x) * (w - 1) / (N - 1), float(y) * (h - 1) / (N - 1)) for y in range(N) for x in range(N)]
    und = _undistort_points(pts, K, dist, P)
    big = float(np.finfo(np.float32).max)
    iX0, iX1, iY0, iY1 = -big, big, -big, big
    oX0, oX1, oY0, oY1 = big, -big, big, -big
    k = 0
    for y in range(N):
        for x in range(N):
            px, py = und[k]
            k += 1
            oX0, oX1, oY0, oY1 = min(oX0, px), max(oX1, px), min(oY0, py), max(oY1, py)
            if x == 0:
                iX0 = max(iX0, px)
            if x == N - 1:
                iX1 = min(iX1, px)
            if y == 0:
                iY0 = max(iY0, py)
            if y == N - 1:
                iY1 = min(iY1, py)
    return (iX0, iY0, iX1 - iX0, iY1 - iY0), (oX0, oY0, oX1 - oX0, oY1 - oY0)


def get_optimal_new_camera_matrix(K, dist, size):
    """cv::getOptimalNewCameraMatrix(K, dist, size, alpha=0, size, &roi) with a CV_32F K, restated in fp64: the
    iterative undistortPoints of a 9x9 grid over the image, its inscribed rectangle mapped to the image, and the
    valid ROI: the inscribed rectangle of the same grid undistorted with K and projected with the new matrix.
    K = (fx, fy, cx, cy), dist = (k1, k2, p1, p2, k3) (float32 values), size = (width, height).
    Returns (newK, roi): newK the float32 (fx, fy, cx, cy), roi the int (x, y, w, h)."""
    K = tuple(float(np.float32(v)) for v in K)
    dist = tuple(float(np.float32(v)) for v in dist)
    w, h = int(size[0]), int(size[1])
    inner, _ = _rectangles(K, dist, (w, h))
    fx0 = (w - 1) / inner[2]
    fy0 = (h - 1) / inner[3]
    cx0 = -fx0 * inner[0]
    cy0 = -fy0 * inner[1]
    M = (fx0, fy0, cx0, cy0)
    inner, _ = _rectangles(K, dist, (w, h), P=M)
    x, y, rw, rh = (int(np.rint(v)) for v in inner)     # Rect_<double> -> Rect: saturate_cast<int> each
    x0, y0 = max(x, 0), max(y, 0)                       # r &= Rect(0, 0, w, h)
    x1, y1 = min(x + rw, w), min(y + rh, h)
    roi = (x0, y0, x1 - x0, y1 - y0) if x1 > x0 and y1 > y0 else (0, 0, 0, 0)
    return tuple(float(np.float32(v)) for v in M), roi


def _round_half_even(x):
    return int(np.rint(np.float64(x)))


def _device_image(img, device, what):
    """A contiguous copy of img on `device` that the set owns: a caller may reuse its own buffer for the next image
    (as the reference's imageToTensor copies)."""
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 \
            or t.shape[0] < 1 or t.shape[1] < 1:
        raise ValueError(f"{what} must be an RGB uint8 [h,w,3] image (torch tensor or numpy array), got "
                         f"{getattr(t, 'dtype', type(t).__name__)} {list(getattr(t, 'shape', []))}")
    return t.to(device, copy=True, memory_format=torch.contiguous_format)


def _device_mask(m, shape, device, what):
    """A 0 / 1 u8 copy of a u8 or bool [h,w] mask on `device` (nonzero = used); ValueError unless its size is the
    decoded image's `shape` (h, w)."""
    t = torch.from_numpy(np.ascontiguousarray(m)) if isinstance(m, np.ndarray) else m
    if not isinstance(t, torch.Tensor) or t.dtype not in (torch.uint8, torch.bool) or t.dim() != 2:
        raise ValueError(f"{what} must be a uint8 or bool [h,w] mask (torch tensor or numpy array), got "
                         f"{getattr(t, 'dtype', type(t).__name__)} {list(getattr(t, 'shape', []))}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what} is {list(t.shape)}, its image is {list(shape)}")
    return (t.to(device) != 0).to(torch.uint8).contiguous()


class ImageSet:
    """The ground-truth images of a set of cameras, prepared as Camera::loadImage and served as Camera::getImage
    (see the module docstring).  `.cameras` are the updated cameras (new model.Camera objects: size and intrinsics
    of the prepared image; the inputs are left untouched), `.new_k` / `.roi` what getOptimalNewCameraMatrix gave per
    camera (None / the whole image without distortion)."""

    def __init__(self, cams, images, downscale_factor=1.0, names=None, device="cuda:0", masks=None):
        """masks (DESIGN D26): None, or one loss mask per image -- a u8 or bool [h,w] array or tensor at the decoded
        image's size, nonzero where the pixel is used -- or None for an image without one."""
        cams, images = list(cams), list(images)
        if len(cams) != len(images) or not cams:
            raise ValueError(f"an ImageSet takes one image per camera, got {len(cams)} cameras and {len(images)} images")
        masks = [None] * len(cams) if masks is None else list(masks)
        if len(masks) != len(cams):
            raise ValueError(f"{len(masks)} masks for {len(cams)} images (None for an image without one)")
        if names is not None:
            names = [str(n) for n in names]
            if len(names) != len(cams):
                raise ValueError(f"{len(names)} names for {len(cams)} cameras")
        if not float(downscale_factor) > 0:
            raise ValueError(f"downscale_factor must be > 0, got {downscale_factor!r}")
        self.device = torch.device(device)
        self.names = names
        self.L = capi.lib()
        self.cameras, self.new_k, self.roi, self._levels, self._mask_levels = [], [], [], [], []
        for i, (cam, img, m) in enumerate(zip(cams, images, masks)):
            img = _device_image(img, self.device, f"image {i}")
            if m is not None:
                m = _device_mask(m, img.shape[:2], self.device, f"mask {i}")
            self._load(cam, img, float(downscale_factor), m)
        self._out = torch.empty(0, dtype=torch.float32, device=self.device)
        # per factor, the device addresses of every camera's level (0 until built): gt() of one camera or of a
        # run of consecutive cameras points the conversion at a slice of it, with no upload
        self._tables = {1: torch.tensor([lv[1].data_ptr() for lv in self._levels], dtype=torch.int64,
                                        device=self.device)}
        # a list of other indices uploads its addresses through these
        self._ptr_host = torch.empty(0, dtype=torch.int64).pin_memory()
        self._ptr_dev = torch.empty(0, dtype=torch.int64, device=self.device)
        self._ptr_copied = None

    def __len__(self):
        return len(self.cameras)

    def _load(self, cam, img, downscale_factor, mask=None):
        """Camera::loadImage (input_data.cpp:40-97) of one camera on its device image, and its mask (0 / 1 u8 [h,w]
        or None) through the same steps."""
        f32, L, s = np.float32, self.L, capi.stream()
        h, w = img.shape[0], img.shape[1]
        rescale = f32(1.0)
        if h != cam.height or w != cam.width:
            rescale = f32(h) / f32(cam.height)
        fx, fy, cx, cy = (f32(v) * rescale for v in (cam.fx, cam.fy, cam.cx, cam.cy))
        if f32(downscale_factor) > f32(1.0):
            sf = f32(1.0) / f32(downscale_factor)
            dh, dw = _round_half_even(h * np.float64(sf)), _round_half_even(w * np.float64(sf))
            if dh < 1 or dw < 1:
                raise ValueError(f"downscale_factor {downscale_factor} leaves nothing of a {w}x{h} image")
            out = torch.empty((dh, dw, 3), dtype=torch.uint8, device=self.device)
            capi.check(L.gsb_resize_area_u8(h, w, capi.ptr(img), dh, dw, capi.ptr(out), float(sf), s))
            if mask is not None:
                m = torch.empty((dh, dw), dtype=torch.uint8, device=self.device)
                capi.check(L.gsb_resize_area_mask_u8(h, w, capi.ptr(mask), dh, dw, capi.ptr(m), float(sf), s))
                mask = m
            img, h, w = out, dh, dw
            fx, fy, cx, cy = fx * sf, fy * sf, cx * sf, cy * sf
        dist = tuple(f32(v) for v in (cam.k1, cam.k2, cam.p1, cam.p2, cam.k3))
        new_k, roi = None, (0, 0, w, h)
        # a fisheye camera (DESIGN D27) is rendered through its distortion, so its image is not resampled
        if cam.model == "pinhole" and any(d != 0 for d in dist):
            new_k, roi = get_optimal_new_camera_matrix((fx, fy, cx, cy), dist, (w, h))
            if roi[2] < 1 or roi[3] < 1:
                raise ValueError(f"the undistorted image of camera {len(self.cameras)} has an empty valid region")
            out = torch.empty((roi[3], roi[2], 3), dtype=torch.uint8, device=self.device)
            capi.check(L.gsb_undistort_u8(h, w, capi.ptr(img), float(fx), float(fy), float(cx), float(cy),
                                          *(float(d) for d in dist), *new_k, *roi, capi.ptr(out), s))
            if mask is not None:
                m = torch.empty((roi[3], roi[2]), dtype=torch.uint8, device=self.device)
                capi.check(L.gsb_undistort_mask_u8(h, w, capi.ptr(mask), float(fx), float(fy), float(cx), float(cy),
                                                   *(float(d) for d in dist), *new_k, *roi, capi.ptr(m), s))
                mask = m
            img = out
            fx, fy, cx, cy = (f32(v) for v in new_k)
        self.cameras.append(cam.replace(width=img.shape[1], height=img.shape[0], fx=fx, fy=fy, cx=cx, cy=cy))
        self.new_k.append(new_k)
        self.roi.append(roi)
        self._levels.append({1: img})
        self._mask_levels.append(None if mask is None else {1: mask})

    def level(self, i, factor=1):
        """Camera::getImage(factor) of camera i as the stored u8 [H,W,3] device image, built on first use and cached:
        INTER_AREA to (cols/factor, rows/factor) of the prepared image.  i may be negative, as a list index;
        IndexError outside [-len, len)."""
        factor = int(factor)
        i = self._index(i)
        levels = self._levels[i]
        if factor <= 1:
            return levels[1]
        if factor not in levels:
            if factor not in self._tables:
                self._tables[factor] = torch.zeros(len(self._levels), dtype=torch.int64, device=self.device)
            src = levels[1]
            h, w = src.shape[0], src.shape[1]
            dh, dw = h // factor, w // factor
            if dh < 1 or dw < 1:
                raise ValueError(f"factor {factor} leaves nothing of the {w}x{h} image of camera {i}")
            out = torch.empty((dh, dw, 3), dtype=torch.uint8, device=self.device)
            capi.check(self.L.gsb_resize_area_u8(h, w, capi.ptr(src), dh, dw, capi.ptr(out), 0.0, capi.stream()))
            levels[factor] = out
            self._tables[factor][i].fill_(out.data_ptr())
        return levels[factor]

    def mask(self, i, factor=1):
        """The loss mask of camera i at Camera::getImage(factor)'s size (DESIGN D26): a device u8 [H,W] tensor of 0 /
        1 (1 = used), or None for an image without a mask; for a list of indices, a list of those.  A level is built
        on first use with gsb_resize_area_mask_u8 (a pixel is used iff every pixel INTER_AREA averages into it is)
        and cached."""
        if not isinstance(i, (int, np.integer)):
            return [self.mask(k, factor) for k in i]
        factor = int(factor)
        i = self._index(i)
        levels = self._mask_levels[i]
        if levels is None:
            return None
        if factor <= 1:
            return levels[1]
        if factor not in levels:
            src = levels[1]
            h, w = src.shape[0], src.shape[1]
            dh, dw = h // factor, w // factor
            if dh < 1 or dw < 1:
                raise ValueError(f"factor {factor} leaves nothing of the {w}x{h} mask of camera {i}")
            out = torch.empty((dh, dw), dtype=torch.uint8, device=self.device)
            capi.check(self.L.gsb_resize_area_mask_u8(h, w, capi.ptr(src), dh, dw, capi.ptr(out), 0.0,
                                                      capi.stream()))
            levels[factor] = out
        return levels[factor]

    def gt(self, i, factor=1):
        """Camera::getImage(factor) as float32 u/255 on the device: [H,W,3] for one index, [B,H,W,3] for a list of B
        indices (one resolution).  One launch, and no upload for one index or consecutive indices.  The result is a
        view of a buffer the set owns and the next call overwrites it (as SplatTrainer.step's loss), so a training
        loop allocates nothing here once every level it uses is built and the buffer has its largest size."""
        single = isinstance(i, (int, np.integer))
        # normalised to [0, len) before anything indexes the address tables (negative indices count from the end)
        idx = [self._index(i)] if single else [self._index(k) for k in i]
        if not idx:
            raise ValueError("gt() needs at least one index")
        levels = [self.level(k, factor) for k in idx]
        H, W = levels[0].shape[0], levels[0].shape[1]
        if any(lv.shape[:2] != (H, W) for lv in levels):
            raise ValueError(f"the images of {idx} differ in size at factor {factor}")
        B, numel = len(idx), len(idx) * H * W * 3
        if self._out.numel() < numel:
            self._out = torch.empty(numel, dtype=torch.float32, device=self.device)
        if idx == list(range(idx[0], idx[0] + B)):
            views = self._tables[max(int(factor), 1)].data_ptr() + 8 * idx[0]
        else:
            views = self._upload_addresses(levels)
        capi.check(self.L.gsb_u8_to_f32_views(B, views, H, W, capi.ptr(self._out), capi.stream()))
        out = self._out[:numel].view(B, H, W, 3)
        return out[0] if single else out

    def _index(self, i):
        """Camera index i in [0, len): a negative i counts from the end; IndexError outside [-len, len)."""
        return range(len(self._levels))[int(i)]

    def _upload_addresses(self, levels):
        """The device address table of `levels` (any order), through a pinned staging table."""
        B = len(levels)
        if self._ptr_dev.numel() < B:
            self._ptr_host = torch.empty(B, dtype=torch.int64).pin_memory()
            self._ptr_dev = torch.empty(B, dtype=torch.int64, device=self.device)
            self._ptr_copied = None
        if self._ptr_copied is not None:
            self._ptr_copied.synchronize()      # the previous upload has left the pinned table
        for b, lv in enumerate(levels):
            self._ptr_host[b] = lv.data_ptr()
        self._ptr_dev[:B].copy_(self._ptr_host[:B], non_blocking=True)
        if self._ptr_copied is None:
            self._ptr_copied = torch.cuda.Event()
        self._ptr_copied.record()
        return self._ptr_dev.data_ptr()

    def split(self, validate, val_image="random"):
        """InputData::getCameras (input_data.cpp:128-156) over this set: (train_indices, val_index); see
        split_cameras."""
        return split_cameras(len(self.cameras), validate, val_image, self.names)


def split_cameras(n, validate, val_image="random", names=None):
    """InputData::getCameras for n cameras: (train_indices, val_index).  Without validation every camera trains and
    val_index is None.  With it the held-out camera is libc's srand(42); rand() % n, or the camera whose name's file
    name equals val_image (ValueError if none does)."""
    if not validate:
        return list(range(n)), None
    if val_image == "random":
        libc = C.CDLL(None)
        libc.srand(C.c_uint(42))
        libc.rand.restype = C.c_int
        val = libc.rand() % n
    else:
        val = next((k for k, nm in enumerate(names or []) if os.path.basename(nm) == val_image), None)
        if val is None:
            raise ValueError(f"{val_image} not in the list of cameras")
    return [k for k in range(n) if k != val], val
