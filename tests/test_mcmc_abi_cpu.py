"""CPU checks of the MCMC entry points' argument rules (every one is checked before any CUDA call, so the calls below return
without touching a device: the pointers are placeholders that are never dereferenced) and of the struct mirrors."""
import ctypes
import math

import pytest

from taichi_3d_gaussian_splatting_b200 import _lib

from test_supervision_abi_cpu import _fake, _train_step_args

GSB_EINVAL = -1
N = 10  # num_points of _train_step_args


def _mcmc(**kw):
    a = dict(num_valid=N, lambda_opacity=0.01, lambda_scale=0.01, noise_scale=5.0, gate_k=100.0, min_opacity=0.005, seed=1,
             step=0, terms_out2=_fake(60), temp=_fake(61))
    a.update(kw)
    return _lib.GsbMcmcStepArgs(**a)


def _call(m, t=None):
    lib = _lib.load()
    t = t or _train_step_args()
    rc = lib.gsb200_train_step_mcmc(ctypes.byref(t), None, None, None, ctypes.byref(m) if m is not None else None)
    return rc, (lib.gsb200_last_error() or b"").decode()


@pytest.mark.parametrize("field,value,word", [
    ("num_valid", -1, "num_valid"), ("num_valid", N + 1, "num_valid"), ("step", -1, "step"),
    ("lambda_opacity", -1.0, "weights"), ("lambda_opacity", math.nan, "weights"), ("lambda_scale", math.inf, "weights"),
    ("lambda_scale", -0.01, "weights"), ("noise_scale", -1.0, "noise_scale"), ("noise_scale", math.nan, "noise_scale"),
    ("gate_k", math.inf, "noise_scale"), ("min_opacity", -0.1, "noise_scale"), ("terms_out2", None, "terms_out2"),
    ("temp", None, "temp"), ("temp", _fake(61) + 8, "temp")])
def test_train_step_mcmc_refuses(field, value, word):
    rc, msg = _call(_mcmc(**{field: value}))
    assert rc == GSB_EINVAL and word in msg and "train_step_mcmc" in msg


def test_train_step_mcmc_needs_aligned_rows_and_a_mask():
    for block, field, value in (("forward", "point_invalid_mask", None), ("both", "pointcloud_features", _fake(2) + 4),
                                ("backward", "grad_pointcloud_features", _fake(17) + 8)):
        t = _train_step_args()
        for b in ("forward", "backward") if block == "both" else (block,):
            setattr(getattr(t, b), field, value)
        rc, msg = _call(_mcmc(), t)
        assert rc == GSB_EINVAL and "train_step_mcmc" in msg, (field, msg)


def test_train_step_checks_still_come_first_and_null_forwards():
    """With mcmc == NULL the call is gsb200_train_step_appearance: the same refusals, with the same messages."""
    lib = _lib.load()
    t = _train_step_args()
    t.step = 0
    rc, msg = _call(_mcmc(num_valid=-1), t)
    assert rc == GSB_EINVAL and "step" in msg and "mcmc" not in msg
    for make in (lambda t: setattr(t, "step", 0), lambda t: setattr(t.backward, "accum_rows", 1),
                 lambda t: setattr(t, "loss_temp", None)):
        t = _train_step_args()
        make(t)
        rc_a = lib.gsb200_train_step_appearance(ctypes.byref(t), None, None, None)
        msg_a = lib.gsb200_last_error()
        rc_m, msg_m = _call(None, t)
        assert rc_a == rc_m == GSB_EINVAL and msg_a.decode() == msg_m


def test_standalone_entry_points_check_their_arguments():
    lib = _lib.load()
    f = _fake
    reg = lambda *a: lib.gsb200_mcmc_regulariser(*a)  # noqa: E731
    assert reg(f(1), f(2), f(3), 10, 11, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert "num_valid" in lib.gsb200_last_error().decode()
    assert reg(f(1), f(2), f(3), 10, -1, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3), -1, 0, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3), 10, 10, -0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3), 10, 10, 0.01, math.nan, f(4), f(5), None) == GSB_EINVAL
    assert reg(None, f(2), f(3), 10, 10, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), None, f(3), 10, 10, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1) + 4, f(2), f(3), 10, 10, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3) + 8, 10, 10, 0.01, 0.01, f(4), f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3), 10, 10, 0.01, 0.01, None, f(5), None) == GSB_EINVAL
    assert reg(f(1), f(2), f(3), 10, 10, 0.01, 0.01, f(4), f(5) + 4, None) == GSB_EINVAL
    noise = lambda *a: lib.gsb200_mcmc_noise(*a)  # noqa: E731
    assert noise(f(1), f(2), f(3), -1, 1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1), f(2), f(3), 10, 1.0, 100.0, 0.005, 0, -1, None) == GSB_EINVAL
    assert noise(f(1), f(2), f(3), 10, -1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1), f(2), f(3), 10, 1.0, math.nan, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1), f(2), f(3), 10, 1.0, 100.0, math.inf, 0, 0, None) == GSB_EINVAL
    assert noise(None, f(2), f(3), 10, 1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1) + 2, f(2), f(3), 10, 1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1), f(2) + 4, f(3), 10, 1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL
    assert noise(f(1), f(2), None, 10, 1.0, 100.0, 0.005, 0, 0, None) == GSB_EINVAL


def _relocate(**kw):
    f = _fake
    a = dict(num_points=100, num_sources=3, source_ids=f(1), source_counts=f(2), num_destinations=4, destination_ids=f(3),
             destination_sources=f(4), pointcloud=f(5), pointcloud_features=f(6), point_invalid_mask=f(7),
             point_object_id=f(8), extra_features=f(9), channels=4, min_opacity=0.005, feature_exp_avg=f(10),
             feature_exp_avg_sq=f(11), position_exp_avg=f(12), position_exp_avg_sq=f(13), extra_exp_avg=f(14),
             extra_exp_avg_sq=f(15))
    a.update(kw)
    return _lib.GsbMcmcRelocateArgs(**a)


@pytest.mark.parametrize("kw", [
    dict(num_points=-1), dict(num_sources=-1), dict(num_sources=101), dict(num_destinations=-1), dict(num_destinations=101),
    dict(source_ids=None), dict(source_counts=None), dict(destination_ids=None), dict(destination_sources=None),
    dict(pointcloud=None), dict(pointcloud_features=None), dict(point_invalid_mask=None), dict(point_object_id=None),
    dict(pointcloud_features=_fake(6) + 4), dict(channels=0), dict(channels=17), dict(feature_exp_avg=None),
    dict(feature_exp_avg_sq=_fake(11) + 8), dict(position_exp_avg_sq=None), dict(extra_exp_avg=None),
    dict(extra_features=None), dict(min_opacity=0.0), dict(min_opacity=1.0), dict(min_opacity=math.nan)])
def test_relocate_refuses(kw):
    lib = _lib.load()
    assert lib.gsb200_mcmc_relocate(ctypes.byref(_relocate(**kw))) == GSB_EINVAL
    assert "mcmc_relocate" in lib.gsb200_last_error().decode()
    assert lib.gsb200_mcmc_relocate(None) == GSB_EINVAL


def test_empty_relocation_is_accepted_without_a_launch():
    lib = _lib.load()
    a = _relocate(num_sources=0, num_destinations=0, source_ids=None, source_counts=None, destination_ids=None,
                  destination_sources=None)
    assert lib.gsb200_mcmc_relocate(ctypes.byref(a)) == 0


def test_temp_bytes_struct_mirrors_and_exports():
    lib = _lib.load()
    assert lib.gsb200_mcmc_temp_bytes() >= 16 + 2 * 8 and lib.gsb200_mcmc_temp_bytes() % 16 == 0
    sizes = (ctypes.c_int64 * 3)(*([-7] * 3))
    lib.gsb200_abi_sizes_mcmc(sizes)
    assert sizes[0] == ctypes.sizeof(_lib.GsbMcmcRelocateArgs) == 160
    assert sizes[1] == ctypes.sizeof(_lib.GsbMcmcStepArgs) == 64 and sizes[2] == -7
    for name in ("gsb200_train_step_mcmc", "gsb200_mcmc_regulariser", "gsb200_mcmc_noise", "gsb200_mcmc_relocate",
                 "gsb200_mcmc_temp_bytes", "gsb200_abi_sizes_mcmc"):
        assert name in _lib.EXPORTS and getattr(lib, name).argtypes is not None
