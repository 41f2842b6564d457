"""Gaussians from a point cloud, as the reference's Model constructor makes them (model.hpp:23-57).

`params_from_points(xyz, rgb)` turns a cloud (xyz [n,3] float32, rgb [n,3] uint8) into the six parameter tensors that
`model.GaussianModel` and `trainer.SplatTrainer` take:

    means        = xyz
    scales       = log(mean distance to the 3 nearest neighbours), repeated x3   (PointsTensor::scales)
    quats        = randomQuatTensor(n) after torch::manual_seed(42)             (model.cpp:23-33)
    featuresDc   = rgb2sh(rgb.double() / 255).float()                            (spherical_harmonics.cpp:20-23)
    featuresRest = 0
    opacities    = logit(0.1f)

The nearest-neighbour distances run on the device (csrc/knn.cu, exact: bit-identical to a brute force with the
reference's roundings).  Quaternions, colours and opacities are computed on the CPU with the reference's torch ops and
uploaded once, so they are bit-identical to the reference's: the quaternions come from a private generator seeded
with 42 (the same mt19937 stream torch::manual_seed(42) gives; the caller's global RNG is left alone), and the colour
division is torch's CPU double division (torch CUDA's `tensor / scalar` multiplies by the reciprocal instead).
Scene normalisation (InputData's scale / translation) is the loaders' job, as in the reference."""
import math

import numpy as np
import torch

from . import capi

SH_C0 = 0.28209479177387814   # spherical_harmonics.cpp:18
QUAT_SEED = 42                # model.hpp:36


def _as_cpu_tensor(a, name):
    if isinstance(a, np.ndarray):
        return torch.from_numpy(a)
    if isinstance(a, torch.Tensor):
        return a
    raise ValueError(f"{name} must be a torch tensor or a numpy array, got {type(a).__name__}")


def _check_xyz(xyz):
    if xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError(f"xyz must be a float32 [n,3] tensor, got {xyz.dtype} {list(xyz.shape)}")
    n = xyz.shape[0]
    if 1 <= n < 4:
        raise ValueError(f"at least 4 points are needed for the 3 nearest neighbours of every point, got {n}")
    if n and not bool(torch.isfinite(xyz).all()):
        raise ValueError("xyz has non-finite coordinates")
    return n


def _knn_mean_dist(xyz_dev):
    """mean_dist [n] of a validated contiguous fp32 [n,3] CUDA tensor with n == 0 or n >= 4."""
    n = xyz_dev.shape[0]
    out = torch.empty(n, dtype=torch.float32, device=xyz_dev.device)
    if n == 0:
        return out
    L = capi.lib()
    ws = torch.empty(L.gsb_knn_workspace_bytes(n) + 256, dtype=torch.uint8, device=xyz_dev.device)
    off = (-ws.data_ptr()) % 256
    capi.check(L.gsb_knn_mean_dist(n, capi.ptr(xyz_dev), capi.ptr(out), ws.data_ptr() + off, ws.numel() - off,
                                   capi.stream()))
    return out


def knn_mean_dist(xyz, device=None):
    """PointsTensor::scales before the log: [n] fp32 device tensor, the mean distance from every point to its 3
    nearest neighbours.  xyz: float32 [n,3] (CPU or CUDA tensor, or numpy array); device: where to compute (default:
    xyz's CUDA device, else cuda:0).  Raises ValueError for a wrong shape / dtype, 1 <= n < 4 or non-finite
    coordinates."""
    xyz = _as_cpu_tensor(xyz, "xyz")
    _check_xyz(xyz)
    if device is None:
        device = xyz.device if xyz.is_cuda else "cuda:0"
    return _knn_mean_dist(xyz.to(device).contiguous())


def random_quats(n):
    """randomQuatTensor(n) (model.cpp:23-33) drawn right after torch::manual_seed(42), on the CPU, from a private
    generator: [n,4] fp32."""
    g = torch.Generator().manual_seed(QUAT_SEED)
    u = torch.rand(n, generator=g)
    v = torch.rand(n, generator=g)
    w = torch.rand(n, generator=g)
    return torch.stack([torch.sqrt(1 - u) * torch.sin(2 * math.pi * v),
                        torch.sqrt(1 - u) * torch.cos(2 * math.pi * v),
                        torch.sqrt(u) * torch.sin(2 * math.pi * w),
                        torch.sqrt(u) * torch.cos(2 * math.pi * w)], -1)


def rgb_to_features_dc(rgb):
    """rgb2sh(rgb.double() / 255).float() (model.hpp:46) on the CPU: [n,3] fp32."""
    return ((rgb.cpu().to(torch.float64) / 255.0 - 0.5) / SH_C0).to(torch.float32)


def opacity_logit():
    """logit(0.1f) as torch computes it on the CPU (model.hpp:50)."""
    return float(torch.logit(torch.ones(1, 1) * float(np.float32(0.1)))[0, 0])


def params_from_points(xyz, rgb, sh_degree=3, device="cuda:0"):
    """The six parameter tensors of Model's constructor for the cloud xyz [n,3] float32 / rgb [n,3] uint8 (torch
    tensors or numpy arrays): {means, scales, quats, featuresDc, featuresRest [n,(sh_degree+1)^2-1,3], opacities [n,1]},
    contiguous fp32 on `device`, as GaussianModel and SplatTrainer take them.  Every argument is checked before
    anything runs on the device: ValueError for a wrong shape or dtype, 1 <= n < 4, non-finite coordinates or
    sh_degree outside 0..4.  n = 0 gives empty tensors."""
    xyz = _as_cpu_tensor(xyz, "xyz")
    rgb = _as_cpu_tensor(rgb, "rgb")
    if isinstance(sh_degree, bool) or not isinstance(sh_degree, (int, np.integer)) or not 0 <= sh_degree <= 4:
        raise ValueError(f"sh_degree must be an integer in 0..4, got {sh_degree!r}")
    if rgb.dtype != torch.uint8 or rgb.dim() != 2 or rgb.shape[1] != 3:
        raise ValueError(f"rgb must be a uint8 [n,3] tensor, got {rgb.dtype} {list(rgb.shape)}")
    n = _check_xyz(xyz)
    if rgb.shape[0] != n:
        raise ValueError(f"xyz has {n} points but rgb has {rgb.shape[0]}")
    dev = torch.device(device)
    k = (int(sh_degree) + 1) ** 2
    f32 = dict(dtype=torch.float32, device=dev)
    means = xyz.to(**f32).contiguous().clone() if xyz.device == dev else xyz.to(**f32).contiguous()
    scales = torch.log(_knn_mean_dist(means))[:, None].repeat(1, 3)
    return {
        "means": means,
        "scales": scales,
        "quats": random_quats(n).to(**f32),
        "featuresDc": rgb_to_features_dc(rgb).to(**f32),
        "featuresRest": torch.zeros((n, k - 1, 3), **f32),
        "opacities": torch.full((n, 1), opacity_logit(), **f32),
    }
