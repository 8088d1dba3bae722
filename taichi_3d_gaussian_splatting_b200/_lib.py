"""ctypes binding of ``libgsb200.so`` (the C ABI declared in ``include/gsb200.h``).

The product path has NO fallback: if the shared library is missing or fails to load this module
raises, and every wrapper raises ``RuntimeError`` with ``gsb200_last_error()`` on a non-zero return.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GSB200_LIB_PATH", os.path.join(_HERE, "libgsb200.so"))  # override: tuning experiments only

GSB_FLAG_EXACT_EXP = 1
GSB_FLAG_FORCE_KEY64 = 2
GSB_FLAG_Q_ALREADY_NORMALISED = 4
GSB_FLAG_KEEP_ALL_TILE_PAIRS = 8
GSB_FLAG_BACKWARD_TRANSPOSED = 16  # experimental, csrc/blend_bwd_transposed.cu
GSB_FLAG_NO_HOOK_STATS = 32
GSB_FLAG_COMPACT_GRADS = 64

c_i64, c_i32, c_u32, c_f32, c_vp = (ctypes.c_int64, ctypes.c_int32, ctypes.c_uint32, ctypes.c_float,
                                    ctypes.c_void_p)


class GsbWorkspaceLayout(ctypes.Structure):
    _fields_ = [
        ("total_bytes", c_i64), ("zero_bytes", c_i64), ("counters", c_i64), ("tickets", c_i64),
        ("scan_state", c_i64), ("sort_hist", c_i64), ("sort_state", c_i64), ("tile_start", c_i64),
        ("tile_end", c_i64), ("poses", c_i64), ("point_id", c_i64), ("point_offset", c_i64), ("num_tiles", c_i64),
        ("records", c_i64), ("point_in_camera", c_i64), ("keys_a", c_i64), ("keys_b", c_i64),
        ("vals_a", c_i64), ("vals_b", c_i64), ("keys_c", c_i64), ("vals_c", c_i64), ("key_bytes", c_i32), ("tile_bits", c_i32),
        ("depth_bits", c_i32), ("sort_passes", c_i32), ("key_capacity_padded", c_i64),
        ("sort_blocks", c_i32), ("scan_blocks", c_i32), ("radix_bits", c_i32), ("reserved", c_i32),
    ]


class GsbForwardArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("pointcloud", c_vp), ("pointcloud_features", c_vp),
        ("point_invalid_mask", c_vp), ("point_object_id", c_vp), ("num_objects", c_i32),
        ("q_pointcloud_camera", c_vp), ("t_pointcloud_camera", c_vp), ("camera_intrinsics", c_vp),
        ("camera_height", c_i32), ("camera_width", c_i32), ("near_plane", c_f32), ("far_plane", c_f32),
        ("depth_to_sort_key_scale", c_f32), ("rgb_only", c_i32), ("flags", c_u32), ("workspace", c_vp),
        ("workspace_bytes", c_i64), ("key_capacity", c_i64), ("rasterized_image", c_vp),
        ("rasterized_depth", c_vp), ("pixel_accumulated_alpha", c_vp),
        ("pixel_offset_of_last_effective_point", c_vp), ("pixel_valid_point_count", c_vp),
        ("stream", c_vp), ("host_counters", c_vp), ("host_counters_event", c_vp),
    ]


class GsbBackwardArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("pointcloud", c_vp), ("pointcloud_features", c_vp),
        ("point_object_id", c_vp), ("num_objects", c_i32), ("t_pointcloud_camera", c_vp),
        ("camera_intrinsics", c_vp), ("camera_height", c_i32), ("camera_width", c_i32),
        ("far_plane", c_f32), ("depth_to_sort_key_scale", c_f32), ("color_max_sh_band", c_i32),
        ("grad_q_factor", c_f32), ("grad_s_factor", c_f32), ("grad_alpha_factor", c_f32),
        ("grad_color_factor", c_f32), ("grad_high_order_color_factor", c_f32), ("flags", c_u32),
        ("workspace", c_vp), ("workspace_bytes", c_i64), ("key_capacity", c_i64),
        ("grad_rasterized_image", c_vp), ("pixel_accumulated_alpha", c_vp),
        ("pixel_offset_of_last_effective_point", c_vp), ("accum", c_vp), ("accum_rows", c_i64),
        ("grad_pointcloud", c_vp), ("grad_pointcloud_features", c_vp),
        ("magnitude_grad_viewspace_on_image", c_vp), ("stream", c_vp),
        ("grad_sum_compact", c_vp), ("grad_color_compact", c_vp),
        ("ctl_accumulated_num_in_camera", c_vp), ("ctl_accumulated_num_pixels", c_vp),
        ("ctl_accumulated_view_space_position_gradients", c_vp), ("ctl_accumulated_view_space_position_gradients_avg", c_vp),
        ("ctl_accumulated_position_gradients", c_vp), ("ctl_accumulated_position_gradients_norm", c_vp),
    ]


class GsbMultimemExchangeArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("num_objects", c_i32), ("rank", c_i32), ("world_size", c_i32), ("num_blocks", c_i32),
        ("phases", c_i32), ("reserved", c_i32), ("multicast_grad_sum", c_vp), ("multicast_blocks", c_vp), ("local_block", c_vp), ("block_stride", c_i64), ("stream", c_vp),
    ]


class GsbTrainStepArgs(ctypes.Structure):
    _fields_ = [
        ("forward", GsbForwardArgs), ("backward", GsbBackwardArgs), ("ground_truth_image", c_vp), ("lambda_value", c_f32),
        ("loss_out3", c_vp), ("loss_temp", c_vp), ("loss_temp_bytes", c_i64), ("feature_exp_avg", c_vp),
        ("feature_exp_avg_sq", c_vp), ("position_exp_avg", c_vp), ("position_exp_avg_sq", c_vp),
        ("feature_learning_rate", ctypes.c_double), ("position_learning_rate", ctypes.c_double), ("beta1", ctypes.c_double),
        ("beta2", ctypes.c_double), ("eps", ctypes.c_double), ("step", c_i32),
    ]


class GsbSupervisionArgs(ctypes.Structure):
    _fields_ = [
        ("depth_target", c_vp), ("mask_target", c_vp), ("background", c_vp), ("depth_weight", c_f32), ("mask_weight", c_f32),
        ("grad_depth", c_vp), ("grad_pixel_accumulated_alpha", c_vp), ("loss_out3", c_vp), ("temp", c_vp), ("temp_bytes", c_i64),
    ]


class GsbExtraFeatureArgs(ctypes.Structure):
    _fields_ = [
        ("channels", c_i32), ("features", c_vp), ("rasterized", c_vp), ("grad_rasterized", c_vp), ("grad_features", c_vp),
    ]


class GsbFeatureTrainArgs(ctypes.Structure):
    _fields_ = [
        ("features", GsbExtraFeatureArgs), ("loss_kind", c_i32), ("weight", c_f32), ("labels", c_vp), ("target", c_vp),
        ("loss_out2", c_vp), ("temp", c_vp), ("temp_bytes", c_i64), ("exp_avg", c_vp), ("exp_avg_sq", c_vp),
        ("learning_rate", ctypes.c_double),
    ]


class GsbPoseGradArgs(ctypes.Structure):
    _fields_ = [
        ("q_pointcloud_camera", c_vp), ("grad_q_pointcloud_camera", c_vp), ("grad_t_pointcloud_camera", c_vp), ("temp", c_vp),
    ]


GSB_POSE_MAX_OBJECTS = 64


class GsbIntrinsicsGradArgs(ctypes.Structure):
    _fields_ = [("grad_camera_intrinsics", c_vp), ("temp", c_vp)]


class GsbLensArgs(ctypes.Structure):
    _fields_ = [("model", c_i32), ("coefficients", c_f32 * 5)]


GSB_LENS_PINHOLE = 0
GSB_LENS_OPENCV = 1
GSB_LENS_FISHEYE = 2


class GsbLensGradArgs(ctypes.Structure):
    _fields_ = [("grad_coefficients", c_vp), ("temp", c_vp)]


class GsbRollingShutterArgs(ctypes.Structure):
    _fields_ = [("motion", c_f32 * 6), ("row_time", c_vp)]


class GsbRollingShutterGradArgs(ctypes.Structure):
    _fields_ = [("grad_motion", c_vp), ("temp", c_vp)]


class GsbMotionBlurArgs(ctypes.Structure):
    _fields_ = [("motion", c_f32 * 6)]


class GsbMotionBlurGradArgs(ctypes.Structure):
    _fields_ = [("grad_motion", c_vp), ("temp", c_vp)]


class GsbDefocusArgs(ctypes.Structure):
    _fields_ = [("aperture", c_f32), ("inverse_focus", c_f32)]


class GsbDefocusGradArgs(ctypes.Structure):
    _fields_ = [("grad", c_vp), ("temp", c_vp)]


class GsbAppearanceArgs(ctypes.Structure):
    _fields_ = [
        ("grid", c_vp), ("grad_grid", c_vp), ("grid_x", c_i32), ("grid_y", c_i32), ("grid_z", c_i32), ("tv_weight", c_f32),
        ("exp_avg", c_vp), ("exp_avg_sq", c_vp), ("learning_rate", ctypes.c_double), ("step", c_i32), ("image", c_vp),
        ("temp", c_vp), ("temp_bytes", c_i64), ("loss_out1", c_vp),
    ]


class GsbMcmcRelocateArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("num_sources", c_i64), ("source_ids", c_vp), ("source_counts", c_vp),
        ("num_destinations", c_i64), ("destination_ids", c_vp), ("destination_sources", c_vp), ("pointcloud", c_vp),
        ("pointcloud_features", c_vp), ("point_invalid_mask", c_vp), ("point_object_id", c_vp), ("extra_features", c_vp),
        ("channels", c_i32), ("min_opacity", c_f32), ("feature_exp_avg", c_vp), ("feature_exp_avg_sq", c_vp),
        ("position_exp_avg", c_vp), ("position_exp_avg_sq", c_vp), ("extra_exp_avg", c_vp), ("extra_exp_avg_sq", c_vp),
        ("stream", c_vp),
    ]


class GsbMcmcStepArgs(ctypes.Structure):
    _fields_ = [
        ("num_valid", c_i64), ("lambda_opacity", c_f32), ("lambda_scale", c_f32), ("noise_scale", c_f32), ("gate_k", c_f32),
        ("min_opacity", c_f32), ("seed", ctypes.c_uint64), ("step", c_i64), ("terms_out2", c_vp), ("temp", c_vp),
    ]


class GsbFilter3dArgs(ctypes.Structure):
    _fields_ = [("filter3d", c_vp)]


class GsbRobustLossArgs(ctypes.Structure):
    _fields_ = [
        ("static_weight", c_vp), ("robust", c_i32), ("inlier_quantile", c_f32), ("box_threshold", c_f32),
        ("patch_threshold", c_f32), ("weight_out", c_vp), ("composite", c_vp), ("temp", c_vp), ("temp_bytes", c_i64),
        ("stats_out2", c_vp),
    ]


class GsbFilter3dViewsArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("pointcloud", c_vp), ("point_invalid_mask", c_vp), ("point_object_id", c_vp),
        ("num_objects", c_i32), ("num_views", c_i32), ("q_pointcloud_camera", c_vp), ("t_pointcloud_camera", c_vp),
        ("camera_intrinsics", c_vp), ("camera_size", c_vp), ("near_plane", c_f32), ("variance", c_f32), ("filter3d", c_vp),
        ("temp", c_vp), ("temp_bytes", c_i64), ("stream", c_vp),
    ]


def lens_args(distortion) -> GsbLensArgs:
    """The C argument of a ``Camera.LensDistortion`` (host floats; unused coefficients 0).  The equirectangular model has
    none: it goes through ``gsb200_forward_equirect`` / ``gsb200_backward_equirect``."""
    model = {"opencv": GSB_LENS_OPENCV, "fisheye": GSB_LENS_FISHEYE}[distortion.model]
    co = list(distortion.coefficients) + [0.0] * (5 - len(distortion.coefficients))
    return GsbLensArgs(model=model, coefficients=(c_f32 * 5)(*co))


GSB_FEATURE_LOSS_CROSS_ENTROPY = 1
GSB_FEATURE_LOSS_L2 = 2


class GsbExpandArgs(ctypes.Structure):
    _fields_ = [
        ("num_points", c_i64), ("num_views", c_i32), ("num_objects", c_i32), ("grad_sum", c_vp),
        ("grad_color_views", c_vp), ("view_stride", c_i64), ("pointcloud", c_vp), ("point_object_id", c_vp),
        ("color_max_sh_band", c_i32), ("grad_color_factor", c_f32), ("grad_high_order_color_factor", c_f32),
        ("part", c_i32), ("grad_pointcloud", c_vp), ("grad_pointcloud_features", c_vp), ("stream", c_vp),
    ]


EXPORTS = (
    "gsb200_version", "gsb200_last_error", "gsb200_workspace_layout", "gsb200_forward",
    "gsb200_backward", "gsb200_stage_preprocess", "gsb200_stage_sort", "gsb200_stage_tile_ranges",
    "gsb200_stage_blend", "gsb200_sort_temp_bytes", "gsb200_sort_pairs", "gsb200_render_host", "gsb200_find_tile_start_and_end",
    "gsb200_forward_timed", "gsb200_backward_timed", "gsb200_abi_sizes", "gsb200_l1_loss_temp_bytes", "gsb200_l1_loss",
    "gsb200_image_loss_temp_bytes", "gsb200_image_loss", "gsb200_adam_step", "gsb200_controller_update",
    "gsb200_forward_blend_work", "gsb200_backward_blend_work", "gsb200_device_selftest", "gsb200_expand_view_gradients",
    "gsb200_train_step", "gsb200_abi_sizes_ext", "gsb200_exchange_multimem", "gsb200_backward_with_depth",
    "gsb200_backward_aux", "gsb200_supervision_temp_bytes", "gsb200_train_step_aux", "gsb200_forward_ext",
    "gsb200_backward_ext", "gsb200_feature_loss_temp_bytes", "gsb200_train_step_ext", "gsb200_backward_pose",
    "gsb200_pose_grad_temp_bytes", "gsb200_backward_calib", "gsb200_intrinsics_grad_temp_bytes", "gsb200_forward_lens",
    "gsb200_backward_lens", "gsb200_backward_lens_grad", "gsb200_lens_grad_temp_bytes", "gsb200_backward_lens_calib",
    "gsb200_forward_rolling_shutter",
    "gsb200_backward_rolling_shutter", "gsb200_rolling_shutter_grad_temp_bytes", "gsb200_bilateral_grid_temp_bytes",
    "gsb200_bilateral_grid_forward", "gsb200_bilateral_grid_backward", "gsb200_train_step_appearance",
    "gsb200_mcmc_temp_bytes", "gsb200_mcmc_regulariser", "gsb200_mcmc_noise", "gsb200_mcmc_relocate", "gsb200_train_step_mcmc",
    "gsb200_abi_sizes_mcmc", "gsb200_forward_filter3d", "gsb200_backward_filter3d", "gsb200_train_step_filter3d",
    "gsb200_filter3d_temp_bytes", "gsb200_filter3d_from_views", "gsb200_abi_sizes_filter3d", "gsb200_robust_temp_bytes",
    "gsb200_robust_image_loss", "gsb200_train_step_robust", "gsb200_abi_sizes_robust", "gsb200_forward_motion_blur",
    "gsb200_backward_motion_blur", "gsb200_motion_blur_grad_temp_bytes", "gsb200_abi_sizes_motion_blur",
    "gsb200_forward_defocus", "gsb200_backward_defocus", "gsb200_defocus_grad_temp_bytes", "gsb200_abi_sizes_defocus",
    "gsb200_forward_equirect", "gsb200_backward_equirect", "gsb200_forward_ortho", "gsb200_backward_ortho",
)

_lib = None


def load() -> ctypes.CDLL:
    """Load the shared library (building it is ``__graft_entry__.build()``'s job, never implicit)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m taichi_3d_gaussian_splatting_b200.build` "
            "(there is no CPU / PyTorch fallback for the rasteriser)")
    lib = ctypes.CDLL(LIB_PATH)
    lib.gsb200_version.restype = ctypes.c_int
    lib.gsb200_last_error.restype = ctypes.c_char_p
    lib.gsb200_workspace_layout.argtypes = [c_i64, c_i32, c_i64, c_i32, c_i32, c_f32, c_f32, c_u32,
                                            ctypes.POINTER(GsbWorkspaceLayout)]
    for name in ("gsb200_forward", "gsb200_stage_preprocess", "gsb200_stage_sort",
                 "gsb200_stage_tile_ranges", "gsb200_stage_blend"):
        getattr(lib, name).argtypes = [ctypes.POINTER(GsbForwardArgs)]
        getattr(lib, name).restype = ctypes.c_int
    lib.gsb200_backward.argtypes = [ctypes.POINTER(GsbBackwardArgs)]
    lib.gsb200_backward.restype = ctypes.c_int
    lib.gsb200_backward_with_depth.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp]
    lib.gsb200_backward_with_depth.restype = ctypes.c_int
    lib.gsb200_backward_aux.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp]
    lib.gsb200_backward_aux.restype = ctypes.c_int
    lib.gsb200_forward_ext.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs)]
    lib.gsb200_forward_ext.restype = ctypes.c_int
    lib.gsb200_backward_ext.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs)]
    lib.gsb200_backward_ext.restype = ctypes.c_int
    lib.gsb200_backward_pose.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs),
                                         ctypes.POINTER(GsbPoseGradArgs)]
    lib.gsb200_backward_pose.restype = ctypes.c_int
    lib.gsb200_pose_grad_temp_bytes.argtypes = [c_i32]
    lib.gsb200_pose_grad_temp_bytes.restype = c_i64
    lib.gsb200_backward_calib.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs),
                                          ctypes.POINTER(GsbPoseGradArgs), ctypes.POINTER(GsbIntrinsicsGradArgs)]
    lib.gsb200_backward_calib.restype = ctypes.c_int
    lib.gsb200_forward_lens.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                        ctypes.POINTER(GsbLensArgs)]
    lib.gsb200_forward_lens.restype = ctypes.c_int
    lib.gsb200_backward_lens.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs),
                                         ctypes.POINTER(GsbLensArgs)]
    lib.gsb200_backward_lens.restype = ctypes.c_int
    lib.gsb200_forward_equirect.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs)]
    lib.gsb200_forward_equirect.restype = ctypes.c_int
    lib.gsb200_backward_equirect.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                             ctypes.POINTER(GsbExtraFeatureArgs)]
    lib.gsb200_backward_equirect.restype = ctypes.c_int
    lib.gsb200_backward_lens_grad.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                              ctypes.POINTER(GsbExtraFeatureArgs), ctypes.POINTER(GsbLensArgs),
                                              ctypes.POINTER(GsbLensGradArgs)]
    lib.gsb200_backward_lens_grad.restype = ctypes.c_int
    lib.gsb200_lens_grad_temp_bytes.argtypes = []
    lib.gsb200_lens_grad_temp_bytes.restype = c_i64
    lib.gsb200_backward_lens_calib.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                               ctypes.POINTER(GsbExtraFeatureArgs), ctypes.POINTER(GsbLensArgs),
                                               ctypes.POINTER(GsbLensGradArgs), ctypes.POINTER(GsbPoseGradArgs),
                                               ctypes.POINTER(GsbIntrinsicsGradArgs)]
    lib.gsb200_backward_lens_calib.restype = ctypes.c_int
    lib.gsb200_forward_rolling_shutter.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                                   ctypes.POINTER(GsbLensArgs), ctypes.POINTER(GsbRollingShutterArgs)]
    lib.gsb200_forward_rolling_shutter.restype = ctypes.c_int
    lib.gsb200_backward_rolling_shutter.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                                    ctypes.POINTER(GsbExtraFeatureArgs), ctypes.POINTER(GsbLensArgs),
                                                    ctypes.POINTER(GsbRollingShutterArgs),
                                                    ctypes.POINTER(GsbRollingShutterGradArgs)]
    lib.gsb200_backward_rolling_shutter.restype = ctypes.c_int
    lib.gsb200_rolling_shutter_grad_temp_bytes.argtypes = []
    lib.gsb200_rolling_shutter_grad_temp_bytes.restype = c_i64
    lib.gsb200_forward_motion_blur.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                               ctypes.POINTER(GsbLensArgs), ctypes.POINTER(GsbRollingShutterArgs),
                                               ctypes.POINTER(GsbMotionBlurArgs)]
    lib.gsb200_forward_motion_blur.restype = ctypes.c_int
    lib.gsb200_backward_motion_blur.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                                ctypes.POINTER(GsbExtraFeatureArgs), ctypes.POINTER(GsbLensArgs),
                                                ctypes.POINTER(GsbRollingShutterArgs), ctypes.POINTER(GsbMotionBlurArgs),
                                                ctypes.POINTER(GsbMotionBlurGradArgs)]
    lib.gsb200_backward_motion_blur.restype = ctypes.c_int
    lib.gsb200_motion_blur_grad_temp_bytes.argtypes = []
    lib.gsb200_motion_blur_grad_temp_bytes.restype = c_i64
    lib.gsb200_forward_defocus.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                           ctypes.POINTER(GsbLensArgs), ctypes.POINTER(GsbRollingShutterArgs),
                                           ctypes.POINTER(GsbMotionBlurArgs), ctypes.POINTER(GsbDefocusArgs)]
    lib.gsb200_forward_defocus.restype = ctypes.c_int
    lib.gsb200_backward_defocus.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp,
                                            ctypes.POINTER(GsbExtraFeatureArgs), ctypes.POINTER(GsbLensArgs),
                                            ctypes.POINTER(GsbRollingShutterArgs), ctypes.POINTER(GsbMotionBlurArgs),
                                            ctypes.POINTER(GsbDefocusArgs), ctypes.POINTER(GsbDefocusGradArgs)]
    lib.gsb200_backward_defocus.restype = ctypes.c_int
    lib.gsb200_defocus_grad_temp_bytes.argtypes = []
    lib.gsb200_defocus_grad_temp_bytes.restype = c_i64
    lib.gsb200_intrinsics_grad_temp_bytes.argtypes = []
    lib.gsb200_intrinsics_grad_temp_bytes.restype = c_i64
    lib.gsb200_sort_temp_bytes.argtypes = [c_i64, c_i32]
    lib.gsb200_sort_temp_bytes.restype = c_i64
    lib.gsb200_sort_pairs.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_vp, c_i64, c_vp]
    lib.gsb200_sort_pairs.restype = ctypes.c_int
    lib.gsb200_render_host.argtypes = [ctypes.POINTER(GsbForwardArgs), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.gsb200_render_host.restype = ctypes.c_int
    lib.gsb200_l1_loss_temp_bytes.argtypes = []
    lib.gsb200_l1_loss_temp_bytes.restype = c_i64
    lib.gsb200_l1_loss.argtypes = [c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.gsb200_l1_loss.restype = ctypes.c_int
    lib.gsb200_image_loss_temp_bytes.argtypes = [c_i32, c_i32]
    lib.gsb200_image_loss_temp_bytes.restype = c_i64
    lib.gsb200_image_loss.argtypes = [c_vp, c_vp, c_i32, c_i32, c_f32, c_f32, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.gsb200_image_loss.restype = ctypes.c_int
    lib.gsb200_adam_step.argtypes = [c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                     ctypes.c_double, c_i32, c_vp]
    lib.gsb200_adam_step.restype = ctypes.c_int
    lib.gsb200_controller_update.argtypes = [c_vp, c_i64] + [c_vp] * 10
    lib.gsb200_controller_update.restype = ctypes.c_int
    lib.gsb200_forward_blend_work.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(ctypes.c_uint64)]
    lib.gsb200_forward_blend_work.restype = ctypes.c_int
    lib.gsb200_backward_blend_work.argtypes = [ctypes.POINTER(GsbBackwardArgs), ctypes.POINTER(ctypes.c_uint64)]
    lib.gsb200_backward_blend_work.restype = ctypes.c_int
    lib.gsb200_expand_view_gradients.argtypes = [ctypes.POINTER(GsbExpandArgs)]
    lib.gsb200_expand_view_gradients.restype = ctypes.c_int
    lib.gsb200_exchange_multimem.argtypes = [ctypes.POINTER(GsbMultimemExchangeArgs)]
    lib.gsb200_exchange_multimem.restype = ctypes.c_int
    lib.gsb200_train_step.argtypes = [ctypes.POINTER(GsbTrainStepArgs)]
    lib.gsb200_train_step.restype = ctypes.c_int
    lib.gsb200_train_step_aux.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs)]
    lib.gsb200_train_step_aux.restype = ctypes.c_int
    lib.gsb200_train_step_ext.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs),
                                          ctypes.POINTER(GsbFeatureTrainArgs)]
    lib.gsb200_train_step_ext.restype = ctypes.c_int
    lib.gsb200_train_step_appearance.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs),
                                                 ctypes.POINTER(GsbFeatureTrainArgs), ctypes.POINTER(GsbAppearanceArgs)]
    lib.gsb200_train_step_appearance.restype = ctypes.c_int
    lib.gsb200_train_step_mcmc.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs),
                                           ctypes.POINTER(GsbFeatureTrainArgs), ctypes.POINTER(GsbAppearanceArgs),
                                           ctypes.POINTER(GsbMcmcStepArgs)]
    lib.gsb200_train_step_mcmc.restype = ctypes.c_int
    lib.gsb200_forward_filter3d.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                            ctypes.POINTER(GsbLensArgs), ctypes.POINTER(GsbRollingShutterArgs),
                                            ctypes.POINTER(GsbFilter3dArgs)]
    lib.gsb200_forward_filter3d.restype = ctypes.c_int
    lib.gsb200_backward_filter3d.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs),
                                             ctypes.POINTER(GsbLensArgs), ctypes.POINTER(GsbRollingShutterArgs),
                                             ctypes.POINTER(GsbFilter3dArgs)]
    lib.gsb200_backward_filter3d.restype = ctypes.c_int
    lib.gsb200_forward_ortho.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(GsbExtraFeatureArgs),
                                         ctypes.POINTER(GsbFilter3dArgs)]
    lib.gsb200_forward_ortho.restype = ctypes.c_int
    lib.gsb200_backward_ortho.argtypes = [ctypes.POINTER(GsbBackwardArgs), c_vp, c_vp, c_vp, ctypes.POINTER(GsbExtraFeatureArgs),
                                          ctypes.POINTER(GsbFilter3dArgs), ctypes.POINTER(GsbPoseGradArgs),
                                          ctypes.POINTER(GsbIntrinsicsGradArgs)]
    lib.gsb200_backward_ortho.restype = ctypes.c_int
    lib.gsb200_train_step_filter3d.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs),
                                               ctypes.POINTER(GsbFeatureTrainArgs), ctypes.POINTER(GsbAppearanceArgs),
                                               ctypes.POINTER(GsbMcmcStepArgs), ctypes.POINTER(GsbFilter3dArgs)]
    lib.gsb200_train_step_filter3d.restype = ctypes.c_int
    lib.gsb200_train_step_robust.argtypes = [ctypes.POINTER(GsbTrainStepArgs), ctypes.POINTER(GsbSupervisionArgs),
                                             ctypes.POINTER(GsbFeatureTrainArgs), ctypes.POINTER(GsbAppearanceArgs),
                                             ctypes.POINTER(GsbMcmcStepArgs), ctypes.POINTER(GsbFilter3dArgs),
                                             ctypes.POINTER(GsbRobustLossArgs)]
    lib.gsb200_train_step_robust.restype = ctypes.c_int
    lib.gsb200_robust_temp_bytes.argtypes = [c_i32, c_i32]
    lib.gsb200_robust_temp_bytes.restype = c_i64
    lib.gsb200_robust_image_loss.argtypes = [c_vp, c_vp, c_i32, c_i32, c_f32, ctypes.POINTER(GsbRobustLossArgs), c_vp, c_vp,
                                             c_vp, c_i64, c_vp]
    lib.gsb200_robust_image_loss.restype = ctypes.c_int
    lib.gsb200_filter3d_temp_bytes.argtypes = [c_i32, c_i32]
    lib.gsb200_filter3d_temp_bytes.restype = c_i64
    lib.gsb200_filter3d_from_views.argtypes = [ctypes.POINTER(GsbFilter3dViewsArgs)]
    lib.gsb200_filter3d_from_views.restype = ctypes.c_int
    lib.gsb200_mcmc_temp_bytes.argtypes = []
    lib.gsb200_mcmc_temp_bytes.restype = c_i64
    lib.gsb200_mcmc_regulariser.argtypes = [c_vp, c_vp, c_vp, c_i64, c_i64, c_f32, c_f32, c_vp, c_vp, c_vp]
    lib.gsb200_mcmc_regulariser.restype = ctypes.c_int
    lib.gsb200_mcmc_noise.argtypes = [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, ctypes.c_uint64, c_i64, c_vp]
    lib.gsb200_mcmc_noise.restype = ctypes.c_int
    lib.gsb200_mcmc_relocate.argtypes = [ctypes.POINTER(GsbMcmcRelocateArgs)]
    lib.gsb200_mcmc_relocate.restype = ctypes.c_int
    lib.gsb200_bilateral_grid_temp_bytes.argtypes = [c_i32] * 5
    lib.gsb200_bilateral_grid_temp_bytes.restype = c_i64
    lib.gsb200_bilateral_grid_forward.argtypes = [c_vp, c_vp] + [c_i32] * 5 + [c_vp, c_vp]
    lib.gsb200_bilateral_grid_forward.restype = ctypes.c_int
    lib.gsb200_bilateral_grid_backward.argtypes = [c_vp, c_vp] + [c_i32] * 5 + [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.gsb200_bilateral_grid_backward.restype = ctypes.c_int
    lib.gsb200_feature_loss_temp_bytes.argtypes = [c_i32, c_i32]
    lib.gsb200_feature_loss_temp_bytes.restype = c_i64
    lib.gsb200_supervision_temp_bytes.argtypes = [c_i32, c_i32]
    lib.gsb200_supervision_temp_bytes.restype = c_i64
    lib.gsb200_device_selftest.argtypes = [c_vp]
    lib.gsb200_device_selftest.restype = ctypes.c_int
    # Every export gets its signature here: without argtypes ctypes passes a Python int as a 32-bit C int, which silently
    # truncates device pointers and 64-bit sizes.
    lib.gsb200_find_tile_start_and_end.argtypes = [c_vp, c_i64, c_vp, c_vp, c_i32, c_vp]
    lib.gsb200_find_tile_start_and_end.restype = ctypes.c_int
    lib.gsb200_forward_timed.argtypes = [ctypes.POINTER(GsbForwardArgs), ctypes.POINTER(c_f32)]
    lib.gsb200_forward_timed.restype = ctypes.c_int
    lib.gsb200_backward_timed.argtypes = [ctypes.POINTER(GsbBackwardArgs), ctypes.POINTER(c_f32)]
    lib.gsb200_backward_timed.restype = ctypes.c_int
    lib.gsb200_version.argtypes = []
    lib.gsb200_last_error.argtypes = []
    lib.gsb200_abi_sizes.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes.restype = None
    lib.gsb200_abi_sizes_ext.argtypes = [ctypes.POINTER(c_i64), c_i32]
    lib.gsb200_abi_sizes_ext.restype = None
    sizes = (c_i64 * 3)()
    lib.gsb200_abi_sizes(sizes)
    mine = (ctypes.sizeof(GsbWorkspaceLayout), ctypes.sizeof(GsbForwardArgs), ctypes.sizeof(GsbBackwardArgs))
    if tuple(sizes) != mine:
        raise RuntimeError(f"libgsb200.so ABI mismatch: C struct sizes {tuple(sizes)} != ctypes mirrors {mine}; "
                           "rebuild with `python -m taichi_3d_gaussian_splatting_b200.build --force`")
    sizes5 = (c_i64 * 5)()
    lib.gsb200_abi_sizes_ext(sizes5, 5)
    mine5 = mine + (ctypes.sizeof(GsbExpandArgs), ctypes.sizeof(GsbTrainStepArgs))
    if tuple(sizes5) != mine5:
        raise RuntimeError(f"libgsb200.so ABI mismatch: C struct sizes {tuple(sizes5)} != ctypes mirrors {mine5}")
    sizes6 = (c_i64 * 6)()
    lib.gsb200_abi_sizes_ext(sizes6, 6)
    if sizes6[5] != ctypes.sizeof(GsbSupervisionArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbSupervisionArgs) {sizes6[5]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbSupervisionArgs)}")
    sizes7 = (c_i64 * 7)()
    lib.gsb200_abi_sizes_ext(sizes7, 7)
    if sizes7[6] != ctypes.sizeof(GsbExtraFeatureArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbExtraFeatureArgs) {sizes7[6]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbExtraFeatureArgs)}")
    sizes8 = (c_i64 * 8)()
    lib.gsb200_abi_sizes_ext(sizes8, 8)
    if sizes8[7] != ctypes.sizeof(GsbFeatureTrainArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbFeatureTrainArgs) {sizes8[7]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbFeatureTrainArgs)}")
    sizes9 = (c_i64 * 9)()
    lib.gsb200_abi_sizes_ext(sizes9, 9)
    if sizes9[8] != ctypes.sizeof(GsbPoseGradArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbPoseGradArgs) {sizes9[8]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbPoseGradArgs)}")
    sizes10 = (c_i64 * 10)()
    lib.gsb200_abi_sizes_ext(sizes10, 10)
    if sizes10[9] != ctypes.sizeof(GsbIntrinsicsGradArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbIntrinsicsGradArgs) {sizes10[9]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbIntrinsicsGradArgs)}")
    sizes11 = (c_i64 * 11)()
    lib.gsb200_abi_sizes_ext(sizes11, 11)
    if sizes11[10] != ctypes.sizeof(GsbLensArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbLensArgs) {sizes11[10]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbLensArgs)}")
    sizes12 = (c_i64 * 12)()
    lib.gsb200_abi_sizes_ext(sizes12, 12)
    if sizes12[11] != ctypes.sizeof(GsbLensGradArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbLensGradArgs) {sizes12[11]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbLensGradArgs)}")
    sizes14 = (c_i64 * 14)()
    lib.gsb200_abi_sizes_ext(sizes14, 14)
    for i, mirror in ((12, GsbRollingShutterArgs), (13, GsbRollingShutterGradArgs)):
        if sizes14[i] != ctypes.sizeof(mirror):
            raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof({mirror.__name__}) {sizes14[i]} != ctypes mirror "
                               f"{ctypes.sizeof(mirror)}")
    sizes15 = (c_i64 * 15)()
    lib.gsb200_abi_sizes_ext(sizes15, 15)
    if sizes15[14] != ctypes.sizeof(GsbAppearanceArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbAppearanceArgs) {sizes15[14]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbAppearanceArgs)}")
    lib.gsb200_abi_sizes_motion_blur.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes_motion_blur.restype = None
    sizes_blur = (c_i64 * 2)()
    lib.gsb200_abi_sizes_motion_blur(sizes_blur)
    for i, mirror in ((0, GsbMotionBlurArgs), (1, GsbMotionBlurGradArgs)):
        if sizes_blur[i] != ctypes.sizeof(mirror):
            raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof({mirror.__name__}) {sizes_blur[i]} != ctypes mirror "
                               f"{ctypes.sizeof(mirror)}")
    lib.gsb200_abi_sizes_defocus.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes_defocus.restype = None
    sizes_defocus = (c_i64 * 2)()
    lib.gsb200_abi_sizes_defocus(sizes_defocus)
    for i, mirror in ((0, GsbDefocusArgs), (1, GsbDefocusGradArgs)):
        if sizes_defocus[i] != ctypes.sizeof(mirror):
            raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof({mirror.__name__}) {sizes_defocus[i]} != ctypes mirror "
                               f"{ctypes.sizeof(mirror)}")
    lib.gsb200_abi_sizes_mcmc.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes_mcmc.restype = None
    sizes_mcmc = (c_i64 * 2)()
    lib.gsb200_abi_sizes_mcmc(sizes_mcmc)
    for i, mirror in ((0, GsbMcmcRelocateArgs), (1, GsbMcmcStepArgs)):
        if sizes_mcmc[i] != ctypes.sizeof(mirror):
            raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof({mirror.__name__}) {sizes_mcmc[i]} != ctypes mirror "
                               f"{ctypes.sizeof(mirror)}")
    lib.gsb200_abi_sizes_filter3d.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes_filter3d.restype = None
    sizes_filter = (c_i64 * 2)()
    lib.gsb200_abi_sizes_filter3d(sizes_filter)
    for i, mirror in ((0, GsbFilter3dArgs), (1, GsbFilter3dViewsArgs)):
        if sizes_filter[i] != ctypes.sizeof(mirror):
            raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof({mirror.__name__}) {sizes_filter[i]} != ctypes mirror "
                               f"{ctypes.sizeof(mirror)}")
    lib.gsb200_abi_sizes_robust.argtypes = [ctypes.POINTER(c_i64)]
    lib.gsb200_abi_sizes_robust.restype = None
    sizes_robust = (c_i64 * 1)()
    lib.gsb200_abi_sizes_robust(sizes_robust)
    if sizes_robust[0] != ctypes.sizeof(GsbRobustLossArgs):
        raise RuntimeError(f"libgsb200.so ABI mismatch: sizeof(GsbRobustLossArgs) {sizes_robust[0]} != ctypes mirror "
                           f"{ctypes.sizeof(GsbRobustLossArgs)}")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().gsb200_last_error()
        raise RuntimeError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


def workspace_layout(num_points: int, num_objects: int, key_capacity: int, height: int, width: int,
                     far_plane: float, depth_scale: float, flags: int = 0) -> GsbWorkspaceLayout:
    out = GsbWorkspaceLayout()
    check(load().gsb200_workspace_layout(num_points, num_objects, key_capacity, height, width,
                                         far_plane, depth_scale, flags, ctypes.byref(out)),
          "gsb200_workspace_layout")
    return out
