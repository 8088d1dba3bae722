"""CPU checks of the loss weights' entry points (``gsb200_train_step_robust``, ``gsb200_robust_image_loss``): every argument
rule is checked before any CUDA call, so the calls below return without touching a device (the pointers are placeholders
that are never dereferenced), and of the ``GsbRobustLossArgs`` mirror."""
import ctypes
import math

import pytest

from taichi_3d_gaussian_splatting_b200 import _lib

from test_supervision_abi_cpu import H, W, _fake, _train_step_args

GSB_EINVAL = -1


def _robust(**kw):
    lib = _lib.load()
    a = dict(static_weight=_fake(60), robust=1, inlier_quantile=0.5, box_threshold=0.5, patch_threshold=0.6,
             weight_out=_fake(61), composite=_fake(62), temp=_fake(63), temp_bytes=int(lib.gsb200_robust_temp_bytes(H, W)),
             stats_out2=_fake(64))
    a.update(kw)
    return _lib.GsbRobustLossArgs(**a)


def _call(r, t=None):
    lib = _lib.load()
    t = t or _train_step_args()
    rc = lib.gsb200_train_step_robust(ctypes.byref(t), None, None, None, None, None, ctypes.byref(r))
    return rc, (lib.gsb200_last_error() or b"").decode()


@pytest.mark.parametrize("value", [-1, 2, 7])
def test_robust_flag_must_be_0_or_1(value):
    rc, msg = _call(_robust(robust=value))
    assert rc == GSB_EINVAL and "robust must be 0 or 1" in msg


@pytest.mark.parametrize("field,value", [("inlier_quantile", 0.0), ("inlier_quantile", -0.1), ("inlier_quantile", 1.0001),
                                         ("inlier_quantile", math.nan), ("box_threshold", -0.01), ("box_threshold", 1.01),
                                         ("box_threshold", math.nan), ("patch_threshold", -0.01),
                                         ("patch_threshold", 1.01), ("patch_threshold", math.inf)])
def test_quantile_and_thresholds_outside_their_ranges_are_refused(field, value):
    rc, msg = _call(_robust(**{field: value}))
    assert rc == GSB_EINVAL and "quantile" in msg


@pytest.mark.parametrize("field,value", [("inlier_quantile", 0.0), ("box_threshold", 2.0), ("patch_threshold", math.nan)])
def test_without_the_robust_mask_the_quantile_and_thresholds_are_not_read(field, value):
    rc, msg = _call(_robust(robust=0, **{field: value}, temp=None))
    assert rc == GSB_EINVAL and "temp" in msg  # the next rule decides


@pytest.mark.parametrize("h,w", [(40, 96), (64, 88), (8, 8)])
def test_sizes_must_be_multiples_of_16(h, w):
    t = _train_step_args()
    t.forward.camera_height = t.backward.camera_height = h
    t.forward.camera_width = t.backward.camera_width = w
    rc, msg = _call(_robust(), t)
    assert rc == GSB_EINVAL and "multiples of 16" in msg


@pytest.mark.parametrize("field,value", [("weight_out", None), ("composite", None), ("stats_out2", None),
                                         ("static_weight", _fake(60) + 2), ("weight_out", _fake(61) + 1),
                                         ("composite", _fake(62) + 2)])
def test_null_or_misaligned_outputs_are_refused(field, value):
    rc, msg = _call(_robust(**{field: value}))
    assert rc == GSB_EINVAL and "aligned" in msg


@pytest.mark.parametrize("temp,delta", [(None, 0), (_fake(63) + 8, 0), (_fake(63), -1)])
def test_temp_must_be_large_enough_and_aligned(temp, delta):
    need = int(_lib.load().gsb200_robust_temp_bytes(H, W))
    rc, msg = _call(_robust(temp=temp, temp_bytes=need + delta))
    assert rc == GSB_EINVAL and "temp" in msg


@pytest.mark.parametrize("temp,delta", [(_fake(21) + 8, 0), (_fake(21), -1)])
def test_the_image_loss_temp_is_checked_before_any_launch(temp, delta):
    t = _train_step_args()
    t.loss_temp = temp
    t.loss_temp_bytes = int(_lib.load().gsb200_image_loss_temp_bytes(H, W)) + delta
    rc, msg = _call(_robust(), t)
    assert rc == GSB_EINVAL and "image loss's temp" in msg


def test_train_step_checks_still_come_first():
    t = _train_step_args()
    t.step = 0
    rc, msg = _call(_robust(robust=5), t)
    assert rc == GSB_EINVAL and "step" in msg


def test_filter_checks_come_before_the_weights():
    lib = _lib.load()
    bad_filter = _lib.GsbFilter3dArgs(filter3d=None)
    r = _robust(robust=5)
    rc = lib.gsb200_train_step_robust(ctypes.byref(_train_step_args()), None, None, None, None, ctypes.byref(bad_filter),
                                      ctypes.byref(r))
    assert rc == GSB_EINVAL and "filter" in (lib.gsb200_last_error() or b"").decode()


def test_standalone_entry_point_checks_its_arguments():
    lib = _lib.load()
    f = _fake
    il = int(lib.gsb200_image_loss_temp_bytes(H, W))
    r = _robust()
    ok = lambda **kw: lib.gsb200_robust_image_loss(  # noqa: E731
        kw.get("x", f(1)), kw.get("g", f(2)), kw.get("h", H), W, 0.2, ctypes.byref(kw.get("r", r)) if kw.get("r", r) else None,
        kw.get("out", f(3)), kw.get("grad", f(4)), kw.get("temp", f(5)), kw.get("bytes", il), None)
    assert ok(x=None) == GSB_EINVAL
    assert ok(g=None) == GSB_EINVAL
    assert ok(grad=None) == GSB_EINVAL
    assert ok(r=None) == GSB_EINVAL
    assert ok(r=_robust(inlier_quantile=0.0)) == GSB_EINVAL
    assert ok(h=40) == GSB_EINVAL
    assert ok(out=None) == GSB_EINVAL
    assert ok(temp=None) == GSB_EINVAL
    assert ok(temp=f(5) + 8) == GSB_EINVAL
    assert ok(bytes=il - 1) == GSB_EINVAL
    assert "robust_image_loss" in (lib.gsb200_last_error() or b"").decode()


def test_temp_bytes_and_struct_mirror():
    lib = _lib.load()
    assert lib.gsb200_robust_temp_bytes(1072, 1920) == lib.gsb200_robust_temp_bytes(16, 16) > 0
    assert lib.gsb200_robust_temp_bytes(1072, 1920) % 16 == 0
    for bad in ((0, 16), (16, 0), (8, 16), (24, 16), (16, 40), (-16, 16)):
        assert lib.gsb200_robust_temp_bytes(*bad) == 0
    size = (ctypes.c_int64 * 2)(-7, -7)
    lib.gsb200_abi_sizes_robust(size)
    assert size[0] == ctypes.sizeof(_lib.GsbRobustLossArgs) == 64 and size[1] == -7
    assert lib.gsb200_version() == 102
    for name in ("gsb200_train_step_robust", "gsb200_robust_image_loss", "gsb200_robust_temp_bytes",
                 "gsb200_abi_sizes_robust"):
        assert name in _lib.EXPORTS and getattr(lib, name).argtypes is not None
