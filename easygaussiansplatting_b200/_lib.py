"""ctypes loader for libgsplat_b200.so (include/gsplat_b200.h).  There is NO fallback:
if the library is missing or an entry point fails, the operators raise."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GSB_LIB") or os.path.join(_HERE, "libgsplat_b200.so")  # GSB_LIB: A/B builds

_vp, _i, _f, _i64, _sz = C.c_void_p, C.c_int, C.c_float, C.c_int64, C.c_size_t

GAUSSIAN_TENSORS = ("pws", "low_shs", "high_shs", "alphas_raw", "scales_raw", "rots_raw")
GAUSSIAN_WIDTHS = (3, 3, 45, 1, 3, 4)


class Gaussians(C.Structure):
    """gsb_gaussians: device pointers of the reference's six training tensors"""
    _fields_ = [(k, _vp) for k in GAUSSIAN_TENSORS]


_gp = C.POINTER(Gaussians)


class AdamTensor(C.Structure):
    """gsb_adam_tensor: one row of gsb_adam_step's table"""
    _fields_ = [("param", _vp), ("grad", _vp), ("exp_avg", _vp), ("exp_avg_sq", _vp), ("numel", _i64),
                ("D", C.c_int32), ("step_size", _f), ("bc2_sqrt", _f)]

# name -> (restype, argtypes); mirrors include/gsplat_b200.h one to one
SIGNATURES = {
    "gsb_abi_version": (_i, []),
    "gsb_last_error": (C.c_char_p, []),
    "gsb_project": (_i, [_i, _vp, _vp, _vp, _f, _f, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "gsb_compute_cov3d": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_compute_cov2d": (_i, [_i, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _vp, _vp, _vp, _vp]),
    "gsb_sh2color": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_inverse_cov2d": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_preprocess_forward": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 8),
    "gsb_preprocess_backward": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 12),
    "gsb_splat_bin_workspace_bytes": (_sz, [_i]),
    "gsb_splat_bin": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _sz, C.POINTER(_i64), C.POINTER(C.c_uint32), _vp]),
    "gsb_splat_workspace_bytes": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_records_offset": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_render": (_i, [_i, _i, _i, _i64, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp,
                              _vp, _vp, _vp, _vp]),
    "gsb_splat_backward_workspace_bytes": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_forward": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_uint32, _vp, _sz, _vp, _sz,
                               _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_splat_forward_enqueue": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_uint32, _vp, _sz, _vp,
                                       _sz, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_splat_backward": (_i, [_i, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                _sz, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_preprocess_backward_rgbd": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 13),
    "gsb_splat_render_rgbd": (_i, [_i, _i, _i, _i64, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp,
                                   _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_splat_forward_rgbd": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_uint32, _vp, _sz, _vp,
                                    _sz, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_splat_backward_rgbd": (_i, [_i, _i, _i, _i64] + [_vp] * 14 + [_sz] + [_vp] * 7),
    "gsb_splat_backward_abs": (_i, [_i, _i, _i, _i64] + [_vp] * 11 + [_sz] + [_vp] * 7),
    "gsb_splat_backward_rgbd_abs": (_i, [_i, _i, _i, _i64] + [_vp] * 14 + [_sz] + [_vp] * 8),
    "gsb_preprocess_backward_pose_workspace_bytes": (_sz, [_i]),
    "gsb_preprocess_backward_pose": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 14 + [_sz, _vp]),
    "gsb_preprocess_forward_aa": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 9),
    "gsb_preprocess_backward_aa": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 15 + [_sz, _vp]),
    "gsb_preprocess_forward_model": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 10),
    "gsb_preprocess_backward_model": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 15 + [_sz, _vp, _vp]),
    "gsb_preprocess_forward_batch": (_i, [_i, _i, _i] + [_vp] * 6 + [_i, _f, _f] + [_vp] * 9),
    "gsb_preprocess_backward_batch": (_i, [_i, _i, _i] + [_vp] * 6 + [_i, _f, _f] + [_vp] * 11),
    "gsb_preprocess_backward_batch_pose_workspace_bytes": (_sz, [_i, _i]),
    "gsb_preprocess_backward_batch_pose": (_i, [_i, _i, _i] + [_vp] * 6 + [_i, _f, _f] + [_vp] * 12 + [_sz, _vp]),
    "gsb_preprocess_backward_intrinsics_workspace_bytes": (_sz, [_i]),
    "gsb_preprocess_backward_intrinsics": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 16 + [_sz, _vp, _vp]),
    "gsb_preprocess_backward_batch_intrinsics_workspace_bytes": (_sz, [_i, _i]),
    "gsb_preprocess_backward_batch_intrinsics": (_i, [_i, _i, _i] + [_vp] * 6 + [_i, _f, _f] + [_vp] * 13 +
                                                 [_sz, _vp]),
    "gsb_splat_bin_batch_workspace_bytes": (_sz, [_i, _i]),
    "gsb_splat_bin_batch": (_i, [_i, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, C.POINTER(_i64), C.POINTER(C.c_uint32),
                                 _vp]),
    "gsb_splat_batch_workspace_bytes": (_sz, [_i, _i, _i, _i, _i64]),
    "gsb_splat_batch_records_offset": (_sz, [_i, _i, _i, _i, _i64]),
    "gsb_splat_render_batch": (_i, [_i, _i, _i, _i, _i64, C.c_uint32] + [_vp] * 8 + [_sz] + [_vp] * 6),
    "gsb_splat_render_batch_rgbd": (_i, [_i, _i, _i, _i, _i64, C.c_uint32] + [_vp] * 8 + [_sz] + [_vp] * 8),
    "gsb_splat_forward_batch": (_i, [_i, _i, _i, _i] + [_vp] * 7 + [_i64, C.c_uint32, _vp, _sz, _vp, _sz] +
                                [_vp] * 7),
    "gsb_splat_forward_batch_rgbd": (_i, [_i, _i, _i, _i] + [_vp] * 7 + [_i64, C.c_uint32, _vp, _sz, _vp, _sz] +
                                     [_vp] * 9),
    "gsb_splat_backward_batch_workspace_bytes": (_sz, [_i, _i, _i, _i, _i64]),
    "gsb_splat_backward_batch": (_i, [_i, _i, _i, _i, _i64] + [_vp] * 11 + [_sz, _vp, _vp]),
    "gsb_splat_backward_batch_rgbd": (_i, [_i, _i, _i, _i, _i64] + [_vp] * 14 + [_sz, _vp, _vp, _vp]),
    "gsb_sh_grad_expand": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "gsb_filter3d_workspace_bytes": (_sz, [_i, _i]),
    "gsb_filter3d": (_i, [_i, _vp, _i, _vp, _f, _vp, _vp, _sz, _vp]),
    "gsb_filter3d_apply": (_i, [_i] + [_vp] * 6),
    "gsb_filter3d_backward": (_i, [_i] + [_vp] * 8),
    "gsb_splat_features_workspace_bytes": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_features": (_i, [_i, _i, _i, _i64, _i] + [_vp] * 9 + [_vp, _sz, _vp, _vp]),
    "gsb_splat_features_backward": (_i, [_i, _i, _i, _i64, _i] + [_vp] * 11 + [_vp, _sz, _vp, _vp, _vp]),
    "gsb_density_apply_rows": (_i, [_i64, _vp, _vp, _i64, _i64, _i64, _i] + [_vp] * 7),
    "gsb_splat_stats_workspace_bytes": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_stats": (_i, [_i, _i, _i, _i64] + [_vp] * 8 + [_vp, _sz, _vp, _vp, _vp, _vp]),
    "gsb_splat_stats_2dgs": (_i, [_i, _i, _i, _i64] + [_vp] * 8),
    "gsb_density_plan_keep": (_i, [_i64, _vp, _vp, _sz, _vp, _vp, C.POINTER(_i64), _vp]),
    "gsb_small_bmm": (_i, [C.c_longlong, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "gsb_gau_loss_workspace_bytes": (_sz, [_i, _i]),
    "gsb_gau_loss": (_i, [_i, _i, _vp, _vp, _f, _vp, _vp, _vp, _sz, _vp]),
    "gsb_density_accumulate": (_i, [_i64, _vp, _vp, _vp, _vp, _i, _vp]),
    "gsb_density_workspace_bytes": (_sz, [_i64]),
    "gsb_density_plan": (_i, [_i64, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _vp, _sz, _vp, _vp, C.POINTER(_i64), _vp]),
    "gsb_density_apply": (_i, [_i64, _vp, _vp, _i64, _i64, _i64, _gp, _gp, _gp, _vp, _gp, _gp, _gp, _vp]),
    "gsb_reset_alpha": (_i, [_i64, _vp, _vp, _vp, _f, _vp]),
    "gsb_mcmc_workspace_bytes": (_sz, [_i64, _i64]),
    "gsb_mcmc_plan": (_i, [_i64, _vp, _f, _i, _vp, _sz, C.POINTER(_i64), _vp]),
    "gsb_mcmc_sample": (_i, [_i64, _i64, _vp, _vp, _sz, _vp, _vp]),
    "gsb_mcmc_relocate": (_i, [_i64, _i64, _vp, _vp, _sz, C.c_double, _i, _gp, _gp, _gp, _vp]),
    "gsb_mcmc_relocate_rows": (_i, [_i64, _i64, _vp, _vp, _sz, _i, _vp, _vp, _vp, _vp]),
    "gsb_mcmc_grow": (_i, [_i64, _i64, _vp, _vp, _sz, C.c_double, _i, _gp, _gp, _gp, _gp, _gp, _gp, _vp]),
    "gsb_mcmc_grow_rows": (_i, [_i64, _i64, _vp, _vp, _sz, _i] + [_vp] * 7),
    "gsb_mcmc_noise": (_i, [_i64] + [_vp] * 5 + [_f, _f, _f, _vp]),
    "gsb_adam_step": (_i, [_i, C.POINTER(AdamTensor), _i64, _vp, C.c_double, C.c_double, C.c_double, _vp]),
    "gsb_ply_rows_to_gs": (_i, [_i64, _i, _i, _vp, _vp, _vp, _vp]),
    "gsb_gs_to_params": (_i, [_i64, _i, _vp, _gp, _vp]),
    "gsb_params_to_gs": (_i, [_i64, _gp, _vp, _vp]),
    "gsb_exchange_region_bytes": (_sz, [_i, _i, _i]),
    "gsb_exchange_result_offset": (_sz, [_i, _i, _i, _i]),
    "gsb_comm_alloc": (_i, [_sz, C.POINTER(_vp), _vp]),
    "gsb_comm_open": (_i, [_vp, C.POINTER(_vp)]),
    "gsb_comm_close": (_i, [_vp]),
    "gsb_comm_free": (_i, [_vp]),
    "gsb_exchange_status": (_i, [_vp, C.POINTER(_i)]),
    "gsb_preprocess_backward_push": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 7 + [_i, _i, C.POINTER(_vp),
                                                                                          C.c_uint32, _vp]),
    "gsb_grad_reduce_broadcast": (_i, [_i, _i, _i, _i, C.POINTER(_vp), C.c_uint32, _vp]),
    "gsb_surfel_preprocess_forward": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 7),
    "gsb_surfel_preprocess_backward": (_i, [_i, _i] + [_vp] * 7 + [_f] * 6 + [_vp] * 8),
    "gsb_splat_surfel_workspace_bytes": (_sz, [_i, _i, _i, _i64]),
    "gsb_splat_surfel_render": (_i, [_i, _i, _i, _i64, C.c_uint32] + [_vp] * 5 + [_sz] + [_vp] * 9),
    "gsb_splat_surfel_forward": (_i, [_i, _i, _i] + [_vp] * 4 + [_i64, C.c_uint32, _vp, _sz, _vp, _sz] + [_vp] * 10),
    "gsb_splat_surfel_backward": (_i, [_i, _i, _i, _i64] + [_vp] * 10 + [_sz] + [_vp] * 2),
    "gsb_splat_2dgs_render": (_i, [_i, _i, _i, _i64, C.c_uint32] + [_vp] * 3 + [_f, _f] + [_vp] * 2 + [_sz]
                              + [_vp] * 13),
    "gsb_splat_2dgs_forward": (_i, [_i, _i, _i] + [_vp] * 4 + [_f, _f, _i64, C.c_uint32, _vp, _sz, _vp, _sz]
                               + [_vp] * 14),
    "gsb_splat_2dgs_backward": (_i, [_i, _i, _i, _i64] + [_vp] * 10 + [_sz, _vp, _f, _f] + [_vp] * 6),
    "gsb_2dgs_batch_workspace_bytes": (_sz, [_i, _i, _i, _i, _i64]),
    "gsb_2dgs_batch_preprocess_forward": (_i, [_i] * 3 + [_vp] * 6 + [_i, _f, _f] + [_vp] * 7),
    "gsb_2dgs_batch_preprocess_backward": (_i, [_i] * 3 + [_vp] * 6 + [_i, _f, _f] + [_vp] * 8),
    "gsb_2dgs_batch_render": (_i, [_i] * 4 + [_i64, C.c_uint32] + [_vp] * 5 + [_sz] + [_vp] * 9),
    "gsb_2dgs_batch_forward": (_i, [_i] * 4 + [_vp] * 4 + [_i64, C.c_uint32, _vp, _sz, _vp, _sz] + [_vp] * 10),
    "gsb_2dgs_batch_backward": (_i, [_i] * 4 + [_i64] + [_vp] * 10 + [_sz] + [_vp] * 2),
    "gsb_2dgs_batch_render_geometry": (_i, [_i] * 4 + [_i64, C.c_uint32] + [_vp] * 3 + [_f, _f] + [_vp] * 2 + [_sz]
                                       + [_vp] * 13),
    "gsb_2dgs_batch_forward_geometry": (_i, [_i] * 4 + [_vp] * 4 + [_f, _f, _i64, C.c_uint32, _vp, _sz, _vp, _sz]
                                        + [_vp] * 14),
    "gsb_2dgs_batch_backward_geometry": (_i, [_i] * 4 + [_i64] + [_vp] * 10 + [_sz, _vp, _f, _f] + [_vp] * 6),
    "gsb_tsdf_integrate": (_i, [_i, _i, _i] + [_f] * 6 + [_i, _i, _i] + [_vp] * 7),
    "gsb_tsdf_extract_workspace_bytes": (_sz, [_i, _i, _i]),
    "gsb_tsdf_extract_plan": (_i, [_i, _i, _i, _vp, _vp, _vp, _sz, C.POINTER(_i64), _vp]),
    "gsb_tsdf_extract_emit": (_i, [_i, _i, _i] + [_f] * 4 + [_vp] * 4 + [_sz, _i64, _i64] + [_vp] * 4),
    "gsb_bilagrid_slice": (_i, [_i] * 4 + [_vp, _i, C.POINTER(C.c_int32), _i, _i, _vp, _vp, _vp]),
    "gsb_bilagrid_slice_backward": (_i, [_i] * 4 + [_vp, _i, C.POINTER(C.c_int32), _i, _i] + [_vp] * 5),
    "gsb_bilagrid_tv_workspace_bytes": (_sz, [_i] * 4),
    "gsb_bilagrid_tv": (_i, [_i] * 4 + [_vp] * 4 + [_sz, _vp]),
    "gsb_kmeans_assign_workspace_bytes": (_sz, [_i, _i]),
    "gsb_kmeans_assign": (_i, [_i, _i, _i, _vp, _i64] + [_vp] * 4 + [_sz, _vp]),
    "gsb_kmeans_update": (_i, [_i, _i, _i, _vp, _i64] + [_vp] * 6),
    "gsb_quantize": (_i, [_i, _i, _vp, _i64, _i, _i, _i, _vp, _vp, _vp]),
    "gsb_dequantize": (_i, [_i, _i, _vp, _i, _vp, _i, _vp, _vp]),
    "gsb_profile_enable": (None, [_i]),
    "gsb_profile_kernels": (_i, []),
    "gsb_profile_kernel_name": (C.c_char_p, [_i]),
    "gsb_profile_launches": (C.c_longlong, [_i]),
    "gsb_profile_read": (_i, [_i, C.POINTER(C.c_double), C.POINTER(C.c_longlong)]),
}

_lib = None


def load():
    """Returns the CDLL with every entry point typed; raises if the library is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "libgsplat_b200.so is not built (%s). Run `python -m easygaussiansplatting_b200.build` "
                "or __graft_entry__.build(); there is no CPU / PyTorch fallback." % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the ABI drifted
            fn.restype, fn.argtypes = res, args
        if lib.gsb_abi_version() != 1:
            raise ImportError("libgsplat_b200.so ABI version mismatch")
        _lib = lib
    return _lib


def check(rc, lib):
    if rc != 0:
        raise RuntimeError("gsplat_b200: %s (rc=%d)" % (lib.gsb_last_error().decode(), rc))
