"""CPU checks of the appearance entry points' argument rules (every one is checked before any CUDA call, so the calls below
return without touching a device: the pointers are placeholders that are never dereferenced) and of the
``GsbAppearanceArgs`` mirror."""
import ctypes
import math

import pytest

from taichi_3d_gaussian_splatting_b200 import _lib

from test_supervision_abi_cpu import H, W, _fake, _train_step_args

GSB_EINVAL = -1


def _appearance(**kw):
    lib = _lib.load()
    a = dict(grid=_fake(40), grad_grid=_fake(41), grid_x=16, grid_y=16, grid_z=8, tv_weight=10.0, exp_avg=_fake(42),
             exp_avg_sq=_fake(43), learning_rate=2e-3, step=1, image=_fake(44), temp=_fake(45),
             temp_bytes=int(lib.gsb200_bilateral_grid_temp_bytes(H, W, 16, 16, 8)), loss_out1=_fake(46))
    a.update(kw)
    return _lib.GsbAppearanceArgs(**a)


def _call(a, t=None):
    lib = _lib.load()
    t = t or _train_step_args()
    rc = lib.gsb200_train_step_appearance(ctypes.byref(t), None, None, ctypes.byref(a))
    return rc, (lib.gsb200_last_error() or b"").decode()


@pytest.mark.parametrize("field,value", [("grid_x", 0), ("grid_x", 65), ("grid_y", 0), ("grid_y", 65), ("grid_z", 0),
                                         ("grid_z", 17)])
def test_shape_outside_the_limits_is_refused(field, value):
    rc, msg = _call(_appearance(**{field: value}))
    assert rc == GSB_EINVAL and "nodes" in msg


@pytest.mark.parametrize("field,value", [("tv_weight", -1.0), ("tv_weight", math.nan), ("tv_weight", math.inf),
                                         ("learning_rate", -1e-3), ("learning_rate", math.nan), ("learning_rate", math.inf)])
def test_negative_or_non_finite_weight_and_rate_are_refused(field, value):
    rc, msg = _call(_appearance(**{field: value}))
    assert rc == GSB_EINVAL and "finite" in msg


def test_step_must_be_positive():
    rc, msg = _call(_appearance(step=0))
    assert rc == GSB_EINVAL and "step" in msg


@pytest.mark.parametrize("field", ["grid", "grad_grid", "exp_avg", "exp_avg_sq", "image", "loss_out1"])
@pytest.mark.parametrize("bad", ["null", "misaligned"])
def test_null_or_misaligned_pointers_are_refused(field, bad):
    if bad == "misaligned" and field == "loss_out1":
        return  # one float, any 4-byte alignment
    value = None if bad == "null" else _fake(50) + 4
    rc, msg = _call(_appearance(**{field: value}))
    assert rc == GSB_EINVAL and "aligned" in msg


@pytest.mark.parametrize("temp,delta", [(None, 0), (_fake(45) + 8, 0), (_fake(45), -1)])
def test_temp_must_be_large_enough_and_aligned(temp, delta):
    need = int(_lib.load().gsb200_bilateral_grid_temp_bytes(H, W, 16, 16, 8))
    rc, msg = _call(_appearance(temp=temp, temp_bytes=need + delta))
    assert rc == GSB_EINVAL and "temp" in msg


def test_train_step_checks_still_come_first():
    t = _train_step_args()
    t.step = 0
    rc, msg = _call(_appearance(grid_x=0), t)
    assert rc == GSB_EINVAL and "step" in msg


def test_standalone_entry_points_check_their_arguments():
    lib = _lib.load()
    f = _fake
    assert lib.gsb200_bilateral_grid_forward(f(1), f(2), H, W, 0, 1, 1, f(3), None) == GSB_EINVAL
    assert lib.gsb200_bilateral_grid_forward(None, f(2), H, W, 1, 1, 1, f(3), None) == GSB_EINVAL
    assert lib.gsb200_bilateral_grid_forward(f(1), f(2), 0, W, 1, 1, 1, f(3), None) == GSB_EINVAL
    need = int(lib.gsb200_bilateral_grid_temp_bytes(H, W, 4, 4, 4))
    assert lib.gsb200_bilateral_grid_backward(f(1), f(2), H, W, 4, 4, 17, f(3), f(4), f(5), f(6), need, None) == GSB_EINVAL
    assert lib.gsb200_bilateral_grid_backward(f(1), f(2), H, W, 4, 4, 4, f(3), f(4), None, f(6), need, None) == GSB_EINVAL
    assert lib.gsb200_bilateral_grid_backward(f(1), f(2), H, W, 4, 4, 4, f(3), f(4), f(5), f(6), need - 1, None) == GSB_EINVAL
    assert lib.gsb200_bilateral_grid_backward(f(1), f(2), H, W, 4, 4, 4, f(3), f(4), f(5), f(6) + 8, need, None) == GSB_EINVAL


def test_temp_bytes_and_struct_mirror():
    lib = _lib.load()
    assert lib.gsb200_bilateral_grid_temp_bytes(1072, 1920, 16, 16, 8) % 16 == 0
    assert lib.gsb200_bilateral_grid_temp_bytes(1072, 1920, 16, 16, 8) > 0
    for bad in ((0, 16, 1, 1, 1), (16, 16, 65, 1, 1), (16, 16, 1, 1, 17), (16, 16, 1, 0, 1)):
        assert lib.gsb200_bilateral_grid_temp_bytes(*bad) == 0
    sizes = (ctypes.c_int64 * 16)(*([-7] * 16))
    lib.gsb200_abi_sizes_ext(sizes, 16)
    assert sizes[14] == ctypes.sizeof(_lib.GsbAppearanceArgs) == 96 and sizes[15] == -7
    fourteen = (ctypes.c_int64 * 15)(*([-7] * 15))
    lib.gsb200_abi_sizes_ext(fourteen, 14)  # n <= 14: as before, the fifteenth slot untouched
    assert list(fourteen[:14]) == list(sizes[:14]) and fourteen[14] == -7
    for name in ("gsb200_train_step_appearance", "gsb200_bilateral_grid_forward", "gsb200_bilateral_grid_backward",
                 "gsb200_bilateral_grid_temp_bytes"):
        assert name in _lib.EXPORTS and getattr(lib, name).argtypes is not None
