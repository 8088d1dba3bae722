"""CPU checks of ``gsb200_train_step_ext``'s feature rules (every one is checked before any CUDA call, so the calls below
return without touching a device: the pointers are placeholders that are never dereferenced) and of the
``GsbFeatureTrainArgs`` mirror."""
import ctypes
import math

import pytest

from taichi_3d_gaussian_splatting_b200 import _lib
from test_supervision_abi_cpu import H, W, _fake, _supervision, _train_step_args

GSB_EINVAL, GSB_EUNSUPPORTED = -1, -4
CE, L2 = _lib.GSB_FEATURE_LOSS_CROSS_ENTROPY, _lib.GSB_FEATURE_LOSS_L2


def _features(channels=8, **kw):
    lib = _lib.load()
    ext = dict(channels=channels, features=_fake(40), rasterized=_fake(41), grad_rasterized=_fake(42), grad_features=_fake(43))
    for k in list(kw):
        if k in ext:
            ext[k] = kw.pop(k)
    x = dict(features=_lib.GsbExtraFeatureArgs(**ext), loss_kind=CE, weight=0.5, labels=_fake(44), target=_fake(45),
             loss_out2=_fake(46), temp=_fake(47), temp_bytes=int(lib.gsb200_feature_loss_temp_bytes(H, W)),
             exp_avg=_fake(48), exp_avg_sq=_fake(49), learning_rate=1e-2)
    x.update(kw)
    return _lib.GsbFeatureTrainArgs(**x)


def _call(x, t=None, s=None):
    lib = _lib.load()
    t = t or _train_step_args()
    rc = lib.gsb200_train_step_ext(ctypes.byref(t), None if s is None else ctypes.byref(s), ctypes.byref(x))
    return rc, (lib.gsb200_last_error() or b"").decode()


@pytest.mark.parametrize("channels", [0, -1, 17, 64])
def test_channels_outside_1_to_16_are_refused(channels):
    rc, msg = _call(_features(channels))
    assert rc == GSB_EINVAL and "channels must be in 1..16" in msg


@pytest.mark.parametrize("kind", [0, 3, -1])
def test_an_unknown_kind_is_refused(kind):
    rc, msg = _call(_features(loss_kind=kind))
    assert rc == GSB_EINVAL and "unknown feature loss kind" in msg


def test_cross_entropy_needs_two_channels():
    rc, msg = _call(_features(1, loss_kind=CE))
    assert rc == GSB_EINVAL and "C >= 2" in msg
    rc, msg = _call(_features(1, loss_kind=L2, exp_avg=None))  # l2 with C = 1 passes this rule (the next one decides)
    assert rc == GSB_EINVAL and "exp_avg" in msg


@pytest.mark.parametrize("weight", [0.0, -1.0, math.nan, math.inf, -math.inf])
def test_a_weight_that_is_not_finite_and_positive_is_refused(weight):
    rc, msg = _call(_features(weight=weight))
    assert rc == GSB_EINVAL and "weight" in msg


def test_each_kind_needs_its_own_target():
    rc, msg = _call(_features(loss_kind=CE, labels=None))
    assert rc == GSB_EINVAL and "labels" in msg
    rc, msg = _call(_features(loss_kind=L2, target=None))
    assert rc == GSB_EINVAL and "target" in msg
    # the other kind's pointer is not read: NULL is fine there (the transposed-flag rule decides below)
    t = _train_step_args()
    t.backward.flags = 0
    assert _call(_features(loss_kind=CE, target=None), t)[0] == GSB_EUNSUPPORTED
    assert _call(_features(loss_kind=L2, labels=None), t)[0] == GSB_EUNSUPPORTED


@pytest.mark.parametrize("missing", ["features", "rasterized", "grad_rasterized", "grad_features", "exp_avg", "exp_avg_sq",
                                     "loss_out2"])
def test_null_maps_gradients_moments_and_outputs_are_refused(missing):
    rc, msg = _call(_features(**{missing: None}))
    assert rc == GSB_EINVAL and "null" in msg


@pytest.mark.parametrize("temp,delta", [(None, 0), (_fake(47) + 8, 0), (_fake(47) + 4, 0), (_fake(47), -1)])
def test_temp_must_be_large_enough_and_aligned(temp, delta):
    need = int(_lib.load().gsb200_feature_loss_temp_bytes(H, W))
    rc, msg = _call(_features(temp=temp, temp_bytes=need + delta))
    assert rc == GSB_EINVAL and "temp" in msg


@pytest.mark.parametrize("field", ["exp_avg", "exp_avg_sq", "features", "grad_features"])
def test_moments_and_rows_must_be_16_byte_aligned(field):
    rc, msg = _call(_features(**{field: _fake(50) + 4}))
    assert rc == GSB_EINVAL and "16-byte aligned" in msg


def test_the_transposed_backward_is_required_and_compact_gradients_are_not_supported():
    t = _train_step_args()
    t.backward.flags = 0
    rc, msg = _call(_features(), t)
    assert rc == GSB_EUNSUPPORTED and "TRANSPOSED" in msg
    t = _train_step_args()
    t.backward.flags = _lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS
    rc, msg = _call(_features(), t)
    assert rc == GSB_EUNSUPPORTED and "COMPACT" in msg


def test_train_step_and_supervision_checks_still_apply():
    t = _train_step_args()
    t.step = 0
    rc, msg = _call(_features(channels=0), t)
    assert rc == GSB_EINVAL and "step" in msg
    rc, msg = _call(_features(channels=0), s=_supervision(depth_weight=-1.0))
    assert rc == GSB_EINVAL and "weights" in msg
    lib = _lib.load()
    assert lib.gsb200_train_step_ext(ctypes.byref(t), None, None) == lib.gsb200_train_step_aux(ctypes.byref(t), None) == GSB_EINVAL
    assert lib.gsb200_train_step_ext(None, None, ctypes.byref(_features())) == GSB_EINVAL


def test_feature_temp_bytes_and_struct_mirror():
    lib = _lib.load()
    need = int(lib.gsb200_feature_loss_temp_bytes(1072, 1920))
    assert need >= 64 + 16 * 1024 and need % 16 == 0
    assert lib.gsb200_feature_loss_temp_bytes(0, 16) == 0 and lib.gsb200_feature_loss_temp_bytes(16, -1) == 0
    sizes = (ctypes.c_int64 * 9)(*([-7] * 9))
    lib.gsb200_abi_sizes_ext(sizes, 8)
    assert sizes[7] == ctypes.sizeof(_lib.GsbFeatureTrainArgs) == 112 and sizes[8] == -7
    seven = (ctypes.c_int64 * 8)(*([-7] * 8))
    lib.gsb200_abi_sizes_ext(seven, 7)  # n <= 7: as before, the eighth slot untouched
    assert list(seven[:7]) == list(sizes[:7]) and seven[7] == -7
    assert sizes[6] == ctypes.sizeof(_lib.GsbExtraFeatureArgs) == 40 and sizes[5] == ctypes.sizeof(_lib.GsbSupervisionArgs) == 72
    for name in ("gsb200_train_step_ext", "gsb200_feature_loss_temp_bytes"):
        assert name in _lib.EXPORTS and getattr(lib, name).argtypes is not None
    assert lib.gsb200_version() == 102
