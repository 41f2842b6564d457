"""ctypes binding of libgsplat_b200.so (C ABI in include/gsplat_b200.h).

torch is used only for device memory and streams; every call passes raw device pointers and the
current CUDA stream.  There is NO CPU fallback: if the library is missing or a call fails, this
module raises."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# GSB_LIB overrides the library path (tools/bench_blend.py uses it to A/B kernel variants)
LIB_PATH = os.environ.get("GSB_LIB") or os.path.join(_HERE, "lib", "libgsplat_b200.so")
_lib = None

_vp, _i, _f, _sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t

_SIGS = {
    "gsb_version": (C.c_int, []),
    "gsb_last_error": (C.c_char_p, []),
    "gsb_sh_forward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_sh_backward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_sh_forward_rgb": (_i, [_i, _i, _i, _vp, _vp, _f, _vp, _vp]),
    "gsb_sh_backward_rgb": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "gsb_sh_forward_split": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    "gsb_sh_backward_split": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_mask_rgb_grad": (_i, [_i, _vp, _vp, _vp]),
    "gsb_sh_backward_multiview": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _vp]),
    "gsb_exchange_gradients": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _i, _i, C.c_longlong, _vp, _vp, _vp]),
    "gsb_project_forward": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i, _i, _i, _f,
                                 _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_project_backward": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i,
                                  _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    # n, means, log_scales, glob, raw_quats, logits, view, proj, fx, fy, cx, cy, H, W, tx, ty, clip, 6 outputs, opac, stream
    "gsb_project_forward_activated": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i, _i, _i, _f,
                                           _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    # n, means, log_scales, glob, raw_quats, opac, view, proj, fx, fy, H, W, radii, conics, v_xy, v_depth, v_conic,
    # v_opacity, v_means, v_log_scales, v_raw_quats, v_logits, stream
    "gsb_project_backward_activated": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                            _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_cumsum_workspace_bytes": (_sz, [_i]),
    "gsb_cumsum_tiles_hit": (_i, [_i, _vp, _vp, _vp, _sz, _vp, _vp]),
    "gsb_map_gaussian_to_intersects": (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "gsb_sort_workspace_bytes": (_sz, [_i]),
    "gsb_sort_intersects": (_i, [_i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "gsb_gather_bin_edges": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_raster_records_bytes": (_sz, [_i]),
    "gsb_raster_grad_rows_bytes": (_sz, [_i]),
    "gsb_pack_records": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_rasterize_forward_packed": (_i, [_i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint, _vp]),
    "gsb_rasterize_forward_count": (_i, [_i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_rasterize_backward": (_i, [_i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint, _vp]),
    "gsb_bucket_max_tile_len": (_i, []),
    "gsb_bucket_workspace_bytes": (_sz, [_i, _i, _i]),
    "gsb_bucket_tile_ranges": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _vp]),
    "gsb_bucket_sort_pack": (_i, [_i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "gsb_activate_forward": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_activate_backward": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_densify_stats_update": (_i, [_i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_densify_stats_init": (_i, [_i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_densify_workspace_bytes": (_sz, [_i]),
    "gsb_densify_classify": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _i, _f, _f, _i, _f, _i, _f, _f, _vp, _sz,
                                  _vp, _vp, _vp, _vp]),
    "gsb_densify_means_scales": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp]),
    "gsb_densify_gather_rows": (_i, [_i, _i, _vp, _vp, _vp, _i, _vp]),
    "gsb_reset_opacity": (_i, [_i, _f, _vp, _vp, _vp, _vp]),
    "gsb_ply_row_floats": (_i, [_i]),
    "gsb_pack_ply_rows": (_i, [_i, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp]),
    "gsb_unpack_ply_rows": (_i, [_i, _i, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "gsb_splat_order_keys": (_i, [_i, _vp, _vp, _i, _f, _vp, _vp]),
    "gsb_pack_splat_rows": (_i, [_i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp]),
    "gsb_ssim_workspace_bytes": (_sz, [_i, _i]),
    "gsb_ssim_l1_loss": (_i, [_i, _i, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    "gsb_adam_step": (_i, [C.c_longlong, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _vp]),
    "gsb_mse_loss_grad": (_i, [C.c_longlong, _vp, _vp, _vp, _vp, _f, _vp]),
}
# optional symbols (experimental entry points) are bound when present
_OPT_SIGS = {}


class GsbError(RuntimeError):
    pass


def lib():
    """Loads the library (must have been built: `python -m opensplat_b200.build`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GsbError(f"{LIB_PATH} not built -- run `python -m opensplat_b200.build` "
                           "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        for name, (res, args) in _OPT_SIGS.items():
            if hasattr(L, name):
                fn = getattr(L, name)
                fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def exported_symbols():
    return list(_SIGS.keys())


def check(code):
    if code != 0:
        raise GsbError(lib().gsb_last_error().decode() or f"gsplat_b200 error {code}")


def ptr(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise GsbError("gsplat_b200 kernels need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise GsbError("tensor must be contiguous")
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def f32(t):
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()
