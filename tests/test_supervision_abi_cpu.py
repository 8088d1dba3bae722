"""CPU checks of ``gsb200_train_step_aux``'s argument rules (every one is checked before any CUDA call, so the calls below
return without touching a device: the pointers are placeholders that are never dereferenced) and of the
``GsbSupervisionArgs`` mirror."""
import ctypes
import math

import pytest

from taichi_3d_gaussian_splatting_b200 import _lib

H, W = 64, 96
GSB_EINVAL, GSB_EUNSUPPORTED = -1, -4


def _fake(k):
    return 0x10000 * (k + 1)  # 16-byte aligned, never dereferenced


def _train_step_args():
    """A train step whose own blocks pass every check of gsb200_train_step (so the supervision checks decide)."""
    fwd = _lib.GsbForwardArgs(num_points=10, pointcloud=_fake(1), pointcloud_features=_fake(2), point_invalid_mask=_fake(3),
                              point_object_id=_fake(4), num_objects=1, q_pointcloud_camera=_fake(5),
                              t_pointcloud_camera=_fake(6), camera_intrinsics=_fake(7), camera_height=H, camera_width=W,
                              near_plane=0.8, far_plane=1000.0, depth_to_sort_key_scale=100.0, workspace=_fake(8),
                              workspace_bytes=1 << 30, key_capacity=1 << 20, rasterized_image=_fake(9),
                              rasterized_depth=_fake(10), pixel_accumulated_alpha=_fake(11),
                              pixel_offset_of_last_effective_point=_fake(12), pixel_valid_point_count=_fake(13))
    bwd = _lib.GsbBackwardArgs(num_points=10, pointcloud=_fake(1), pointcloud_features=_fake(2), point_object_id=_fake(4),
                               num_objects=1, t_pointcloud_camera=_fake(6), camera_intrinsics=_fake(7), camera_height=H,
                               camera_width=W, far_plane=1000.0, depth_to_sort_key_scale=100.0, color_max_sh_band=3,
                               flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, workspace=_fake(8), workspace_bytes=1 << 30,
                               key_capacity=1 << 20, grad_rasterized_image=_fake(14), pixel_accumulated_alpha=_fake(11),
                               pixel_offset_of_last_effective_point=_fake(12), accum=_fake(15), accum_rows=10,
                               grad_pointcloud=_fake(16), grad_pointcloud_features=_fake(17),
                               magnitude_grad_viewspace_on_image=_fake(18))
    return _lib.GsbTrainStepArgs(forward=fwd, backward=bwd, ground_truth_image=_fake(19), lambda_value=0.2,
                                 loss_out3=_fake(20), loss_temp=_fake(21), loss_temp_bytes=1 << 24,
                                 feature_exp_avg=_fake(22), feature_exp_avg_sq=_fake(23), position_exp_avg=_fake(24),
                                 position_exp_avg_sq=_fake(25), feature_learning_rate=1e-3, position_learning_rate=1e-5,
                                 beta1=0.9, beta2=0.999, eps=1e-8, step=1)


def _supervision(**kw):
    lib = _lib.load()
    s = dict(depth_target=_fake(30), mask_target=_fake(31), background=_fake(32), depth_weight=0.5, mask_weight=0.5,
             grad_depth=_fake(33), grad_pixel_accumulated_alpha=_fake(34), loss_out3=_fake(35), temp=_fake(36),
             temp_bytes=int(lib.gsb200_supervision_temp_bytes(H, W)))
    s.update(kw)
    return _lib.GsbSupervisionArgs(**s)


def _call(s, t=None):
    lib = _lib.load()
    t = t or _train_step_args()
    rc = lib.gsb200_train_step_aux(ctypes.byref(t), ctypes.byref(s))
    return rc, (lib.gsb200_last_error() or b"").decode()


@pytest.mark.parametrize("field,value", [("depth_weight", -1.0), ("depth_weight", math.nan), ("depth_weight", math.inf),
                                         ("mask_weight", -0.5), ("mask_weight", math.nan), ("mask_weight", -math.inf)])
def test_negative_or_non_finite_weights_are_refused(field, value):
    rc, msg = _call(_supervision(**{field: value}))
    assert rc == GSB_EINVAL and "weights" in msg


@pytest.mark.parametrize("missing", ["depth_target", "grad_depth"])
def test_depth_weight_needs_its_target_and_gradient(missing):
    rc, msg = _call(_supervision(mask_weight=0.0, background=None, **{missing: None}))
    assert rc == GSB_EINVAL and "depth" in msg
    # with the weight at zero the same arguments are not an error of the depth term (the mask term's temp check decides)
    rc, msg = _call(_supervision(depth_weight=0.0, background=None, temp=None, **{missing: None}))
    assert rc == GSB_EINVAL and "temp" in msg and "depth" not in msg


def test_mask_weight_needs_its_target_and_the_alpha_gradient():
    rc, msg = _call(_supervision(depth_weight=0.0, background=None, mask_target=None))
    assert rc == GSB_EINVAL and "mask_target" in msg
    rc, msg = _call(_supervision(depth_weight=0.0, background=None, grad_pixel_accumulated_alpha=None))
    assert rc == GSB_EINVAL and "grad_pixel_accumulated_alpha" in msg


def test_background_needs_the_alpha_gradient():
    rc, msg = _call(_supervision(depth_weight=0.0, mask_weight=0.0, mask_target=None, grad_pixel_accumulated_alpha=None))
    assert rc == GSB_EINVAL and "grad_pixel_accumulated_alpha" in msg


@pytest.mark.parametrize("temp,delta", [(None, 0), (_fake(36) + 8, 0), (_fake(36) + 4, 0), (_fake(36), -1)])
def test_temp_must_be_large_enough_and_aligned(temp, delta):
    lib = _lib.load()
    need = int(lib.gsb200_supervision_temp_bytes(H, W))
    rc, msg = _call(_supervision(temp=temp, temp_bytes=need + delta))
    assert rc == GSB_EINVAL and "temp" in msg


def test_terms_need_the_transposed_backward():
    t = _train_step_args()
    t.backward.flags = 0
    rc, msg = _call(_supervision(), t)
    assert rc == GSB_EUNSUPPORTED and "TRANSPOSED" in msg


def test_train_step_checks_still_come_first():
    t = _train_step_args()
    t.step = 0
    rc, msg = _call(_supervision(depth_weight=-1.0), t)
    assert rc == GSB_EINVAL and "step" in msg
    lib = _lib.load()
    assert lib.gsb200_train_step_aux(ctypes.byref(t), None) == GSB_EINVAL
    assert lib.gsb200_train_step(ctypes.byref(t)) == GSB_EINVAL


def test_supervision_temp_bytes_and_struct_mirror():
    lib = _lib.load()
    need = int(lib.gsb200_supervision_temp_bytes(1072, 1920))
    assert need >= 24 * 1072 * 1920 and need % 16 == 0
    assert lib.gsb200_supervision_temp_bytes(0, 16) == 0 and lib.gsb200_supervision_temp_bytes(16, -1) == 0
    sizes = (ctypes.c_int64 * 7)(*([-7] * 7))
    lib.gsb200_abi_sizes_ext(sizes, 6)
    assert sizes[5] == ctypes.sizeof(_lib.GsbSupervisionArgs) == 72 and sizes[6] == -7
    five = (ctypes.c_int64 * 6)(*([-7] * 6))
    lib.gsb200_abi_sizes_ext(five, 5)  # n <= 5: as before, the sixth slot untouched
    assert list(five[:5]) == list(sizes[:5]) and five[5] == -7
    assert sizes[4] == ctypes.sizeof(_lib.GsbTrainStepArgs)
    assert "gsb200_train_step_aux" in _lib.EXPORTS and lib.gsb200_train_step_aux.argtypes is not None
