"""ctypes binding of libgsplat_b200.so (C ABI in include/gsplat_b200.h).

torch is used only for device memory and streams; every call passes raw device pointers and the
current CUDA stream.  There is NO CPU fallback: if the library is missing or a call fails, this
module raises."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# GSB_LIB overrides the library path (tools/bench_blend.py uses it to compare the builds of two commits)
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
    "gsb_sh_forward_rgb_cam": (_i, [_i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp]),
    "gsb_sh_backward_rgb_cam": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_sh_forward_rgb_cam_multiview": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _vp]),
    "gsb_mask_rgb_grad": (_i, [_i, _vp, _vp, _vp]),
    "gsb_sh_backward_multiview": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _vp]),
    "gsb_exchange_gradients": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _i, _i, C.c_longlong, _vp, _vp, _vp]),
    "gsb_sh_backward_multiview_cams": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _vp]),
    "gsb_exchange_gradients_cams": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _i, _i, C.c_longlong, _vp, _vp,
                                         _vp]),
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
    "gsb_project_backward_activated_acc": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                                _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    # the anti-aliased opacity (DESIGN D19): the arguments of the three above; the backward takes logits for opac
    "gsb_project_forward_activated_aa": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i, _i, _i,
                                              _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_project_backward_activated_aa": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                               _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_project_backward_activated_aa_acc": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                                   _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_cumsum_workspace_bytes": (_sz, [_i]),
    "gsb_cumsum_tiles_hit": (_i, [_i, _vp, _vp, _vp, _sz, _vp]),
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
    "gsb_gather_record_depths": (_i, [_i, _vp, _vp, _vp, _vp, _vp]),
    "gsb_rasterize_forward_packed_depth": (_i, [_i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint,
                                                _vp, _vp, _vp, _vp]),
    "gsb_rasterize_backward_depth": (_i, [_i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                          _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint, _vp, _vp, _vp, _vp]),
    # D25: the arguments of gsb_rasterize_backward_depth with v_xy_abs before the stream
    "gsb_rasterize_backward_absgrad": (_i, [_i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                            _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint, _vp, _vp, _vp, _vp, _vp]),
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
    "gsb_mcmc_workspace_bytes": (_sz, [_i]),
    # n, logits, min_opacity, mask_dead, workspace, workspace_bytes, cdf, dead, result, stream
    "gsb_mcmc_plan": (_i, [_i, _vp, _f, _i, _vp, _sz, _vp, _vp, _vp, _vp]),
    # num_samples, n, cdf, key0, key1, step, tag, samples, counts, stream
    "gsb_mcmc_sample": (_i, [_i, _i, _vp, C.c_uint, C.c_uint, _i, _i, _vp, _vp, _vp]),
    # n, counts, min_opacity, logits, log_scales, zero_moments, num_segments, segments (host), exp_avg, exp_avg_sq, stream
    "gsb_mcmc_relocate": (_i, [_i, _vp, _f, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_mcmc_copy_rows": (_i, [_i, _vp, _vp, _i, _vp, _vp, _vp]),
    "gsb_mcmc_regularize": (_i, [_i, _vp, _vp, _f, _f, _vp, _vp, _vp]),
    # n, logits, log_scales, raw_quats, key0, key1, step, noise_scale, means, stream
    "gsb_mcmc_add_noise": (_i, [_i, _vp, _vp, _vp, C.c_uint, C.c_uint, _i, _f, _vp, _vp]),
    "gsb_mcmc_draws": (_i, [_i, C.c_uint, C.c_uint, _i, _i, _vp, _vp, _vp]),
    "gsb_bilagrid_slice_forward": (_i, [_i, _i, _vp, _vp, _vp, _vp]),
    "gsb_bilagrid_workspace_bytes": (_sz, [_i, _i]),
    # H, W, grid, rgb, v_out, scale, v_rgb, v_grid, workspace, workspace_bytes, stream
    "gsb_bilagrid_slice_backward": (_i, [_i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    "gsb_bilagrid_tv": (_i, [_i, _vp, _f, _vp, _vp, _vp]),
    "gsb_project_camera_partials_floats": (_sz, [_i]),
    # the arguments of gsb_project_backward_activated, then accumulate, antialiased, cam_partials, stream
    "gsb_project_backward_activated_camgrad": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                                    _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp,
                                                    _vp]),
    # nblocks, partials, v_viewmat, v_projmat, stream
    "gsb_project_camera_grad_reduce": (_i, [_i, _vp, _vp, _vp, _vp]),
    # pose, view, centre, view_out, centre_out, stream
    "gsb_pose_apply": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    # pose, view, proj, v_viewmat, v_projmat, scale, grad, stream
    "gsb_pose_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    # n, depths, radii, inv, stream / n, depths, radii, v_inv, v_z, stream
    "gsb_inverse_depths": (_i, [_i, _vp, _vp, _vp, _vp]),
    "gsb_inverse_depths_backward": (_i, [_i, _vp, _vp, _vp, _vp, _vp]),
    "gsb_inverse_depth_l1_workspace_bytes": (_sz, [_i, _i]),
    # H, W, rendered, prior, scale_g, v_rendered, loss_out, workspace, workspace_bytes, stream
    "gsb_inverse_depth_l1": (_i, [_i, _i, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    # h, w, factor, src, dst, stream
    "gsb_depth_downscale_mean": (_i, [_i, _i, _i, _vp, _vp, _vp]),
    # D24: the arguments of gsb_project_forward_activated with filter3d after the logits, then antialiased, stream
    "gsb_project_forward_activated_filter3d": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i,
                                                    _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    # the arguments of gsb_project_backward_activated (logits for opac) with filter3d after the logits, then
    # accumulate, antialiased, camgrad, cam_partials, stream
    "gsb_project_backward_activated_filter3d": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                                     _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i,
                                                     _vp, _vp]),
    # D27: n, means, log_scales, glob_scale, raw_quats, logits, viewmat, fx, fy, cx, cy, k1..k4, theta_lim, img_h,
    # img_w, tiles_x, tiles_y, clip_thresh, 7 outputs, antialiased, stream
    "gsb_project_forward_fisheye": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _f, _f, _i, _i,
                                         _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    # n, means, log_scales, glob_scale, raw_quats, logits, viewmat, fx, fy, k1..k4, theta_lim, img_h, img_w, radii,
    # conics, v_xy, v_depth, v_conic, v_opacity, 4 gradients, accumulate, antialiased, cam_partials, stream
    "gsb_project_backward_fisheye": (_i, [_i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _i, _i, _vp,
                                          _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "gsb_filter3d_workspace_bytes": (_sz, []),
    # n, means, num_cameras, cameras, near, margin, variance, workspace, workspace_bytes, filter3d, stream
    "gsb_filter3d_compute": (_i, [_i, _vp, _i, _vp, _f, _f, _f, _vp, _sz, _vp, _vp]),
    # n, log_scales, logits, filter3d, out_log_scales, out_logits, stream
    "gsb_filter3d_bake": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp]),
    # n, max_logit, reset_value, log_scales, filter3d, logits, exp_avg, exp_avg_sq, stream
    "gsb_reset_opacity_filter3d": (_i, [_i, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_ply_row_floats": (_i, [_i]),
    "gsb_pack_ply_rows": (_i, [_i, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp]),
    "gsb_unpack_ply_rows": (_i, [_i, _i, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "gsb_splat_order_keys": (_i, [_i, _vp, _vp, _i, _f, _vp, _vp]),
    "gsb_pack_splat_rows": (_i, [_i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _f, C.POINTER(C.c_float), _vp, _vp]),
    "gsb_ssim_workspace_bytes": (_sz, [_i, _i]),
    "gsb_ssim_l1_loss": (_i, [_i, _i, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    # D26: H, W, rendered, gt, mask, w, v_rendered, loss_out, workspace, workspace_bytes, stream
    "gsb_ssim_l1_loss_masked": (_i, [_i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    "gsb_adam_step": (_i, [C.c_longlong, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _vp]),
    # num_segments, segments (host AdamSegment array), param, grad, exp_avg, exp_avg_sq, b1, b2, eps, bc1, bc2, stream
    "gsb_adam_step_segments": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _vp]),
    "gsb_mse_loss_grad": (_i, [C.c_longlong, _vp, _vp, _vp, _vp, _f, _vp]),
    "gsb_knn_workspace_bytes": (_sz, [_i]),
    "gsb_knn_mean_dist": (_i, [_i, _vp, _vp, _vp, _sz, _vp]),
    "gsb_resize_area_u8": (_i, [_i, _i, _vp, _i, _i, _vp, _f, _vp]),
    # h, w, src, fx, fy, cx, cy, k1, k2, p1, p2, k3, new fx, fy, cx, cy, roi x, y, w, h, dst, stream
    "gsb_undistort_u8": (_i, [_i, _i, _vp, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _i, _i, _i, _i, _vp,
                              _vp]),
    "gsb_u8_to_f32_views": (_i, [_i, _vp, _i, _i, _vp, _vp]),
    # D26: the loss masks, with the arguments of the two above
    "gsb_resize_area_mask_u8": (_i, [_i, _i, _vp, _i, _i, _vp, _f, _vp]),
    "gsb_undistort_mask_u8": (_i, [_i, _i, _vp, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _f, _i, _i, _i, _i,
                                   _vp, _vp]),
}

ADAM_MAX_SEGMENTS = 8   # GSB_ADAM_MAX_SEGMENTS


class AdamSegment(C.Structure):
    """gsb_adam_segment (include/gsplat_b200.h)."""
    _fields_ = [("offset", C.c_longlong), ("count", C.c_longlong), ("row_floats", C.c_int),
                ("head_floats", C.c_int), ("lr_head", C.c_float), ("lr_rest", C.c_float)]


MCMC_MAX_SEGMENTS = 8   # GSB_MCMC_MAX_SEGMENTS


class RowSegment(C.Structure):
    """gsb_row_segment (include/gsplat_b200.h)."""
    _fields_ = [("offset", C.c_longlong), ("row_floats", C.c_int), ("reserved", C.c_int)]


BILAGRID_X, BILAGRID_Y, BILAGRID_L, BILAGRID_COEFFS = 16, 16, 8, 12   # GSB_BILAGRID_*
BILAGRID_FLOATS = BILAGRID_L * BILAGRID_Y * BILAGRID_X * BILAGRID_COEFFS
POSE_FLOATS = 9   # GSB_POSE_FLOATS
CAMGRAD_TERMS = 24   # floats per block row of gsb_project_backward_activated_camgrad's partials
FILTER3D_CAM_FLOATS = 18   # GSB_FILTER3D_CAM_FLOATS


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
