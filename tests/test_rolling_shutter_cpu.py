"""Rolling-shutter cameras (``gsb200_forward_rolling_shutter`` / ``gsb200_backward_rolling_shutter``,
``CameraInfo.rolling_shutter``, ``differentiable_rolling_shutter``, ``TrainConfig.rolling_shutter_learning_rate``) without a
GPU.

* A known answer without the reference: a pinhole with a pure vertical translation makes the row time affine in tau, so
  tau_3 = a (1 + b + b^2) in closed form (and its clamped variant).
* An independent cross-check: the rolling-shutter record of an isolated small Gaussian is the pinhole kernel's record of the
  same Gaussian with the object pose moved to its row time (composed on the host in float64).
* The emulated rolling-shutter kernels (the unmodified CUDA sources under the SIMT emulator of ``tests/simt``) against the
  float64 evaluator ``torch_reference_rolling_shutter``: the forward (row times, records, image) and the per-point backward
  (point gradients and dL/dm) for image, depth, alpha and feature-map losses, pinhole, opencv and fisheye, three objects
  sharing warps and both loop-A kernels.  Zero motion is bit-identical to the global-shutter kernels; MGRAD on and off give
  bit-identical other outputs; two runs are deterministic.
* The C entry points' argument rules and ABI sizes, the operator's, trainer's and dataset's configuration, and
  ``RollingShutter.from_camera_velocity`` against a render at the moved pose."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth, emulated_points
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator, emulated_forward
from simt_lens_helpers import build_lens_emulator, emulated_forward_lens, emulated_points_lens
from simt_rolling_shutter_helpers import (build_rolling_shutter_emulator, emulated_forward_rs, emulated_points_rs,
                                          rotation, run_preprocess_rs)
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference import postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_rolling_shutter import dense_render_rs, rodrigues

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "pinhole": ("pinhole", ()),
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
MOTION = (0.06, -0.09, 0.04, 0.05, -0.08, 0.06)  # v (scene units), w (rad) over one readout


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator(), remu=build_rolling_shutter_emulator())


def _single(xyz, feats_row, K, H, W, q=(0.0, 0.0, 0.0, 1.0), t=(0.0, 0.0, 0.0)):
    """A one-Gaussian scene with the camera at pose (q, t)."""
    from types import SimpleNamespace
    return SimpleNamespace(
        point_cloud=torch.tensor([xyz], dtype=torch.float32), point_cloud_features=torch.tensor([feats_row], dtype=torch.float32),
        point_invalid_mask=torch.zeros(1, dtype=torch.int8), point_object_id=torch.zeros(1, dtype=torch.int32),
        q_pointcloud_camera=torch.tensor([q], dtype=torch.float32), t_pointcloud_camera=torch.tensor([t], dtype=torch.float32),
        camera_info=CameraInfo(torch.tensor(K, dtype=torch.float32), H, W, 0))


def _feats_row(log_scale=-3.0):
    row = [0.0] * 56
    row[3] = 1.0
    row[4] = row[5] = row[6] = log_scale
    row[7] = 2.0
    row[8] = row[24] = row[40] = 0.5
    return row


# ------------------------------------------------------------------ known answers
@pytest.mark.parametrize("clamped", [False, True])
def test_row_time_of_a_vertical_translation_is_the_affine_fixed_point(emus, clamped):
    """Pinhole, w = 0, v = (0, vy, 0): row(pc(tau)) = a + b tau with a = v0/H - 1/2 and b = fy vy / (z H), so three steps from 0
    give tau_3 = a (1 + b + b^2) when nothing clamps."""
    H, W, fy, cy = 64, 64, 50.0, 32.0
    K = [[50.0, 0, 32.0], [0, fy, cy], [0, 0, 1]]
    z, y0 = 4.0, (0.6 if not clamped else 1.9)
    vy = 0.8 if not clamped else 2.0
    sc = _single((0.1, y0, z), _feats_row(), K, H, W)
    pre = run_preprocess_rs(emus["remu"], sc, "pinhole", (), (0.0, vy, 0.0, 0.0, 0.0, 0.0))
    a = (fy * y0 / z + cy) / H - 0.5
    b = fy * vy / (z * H)
    if not clamped:
        assert abs(a * (1 + b + b * b)) < 0.5
        want = a * (1 + b + b * b)
    else:
        tau = 0.0
        for _ in range(3):
            tau = min(max(a + b * tau, -0.5), 0.5)
        assert a + b * a > 0.5  # the second step clamps
        want = tau
    assert pre.point_offset[0] == 0
    assert abs(float(pre.row_time[0]) - want) <= 2e-6
    # the point is rendered at pc(tau_3): the record's v and depth
    assert abs(pre.pic[0, 1] - (y0 + want * vy)) <= 1e-5 and pre.pic[0, 2] == np.float32(z)


def test_rotation_helper_is_rodrigues_and_exact_at_zero(emus):
    w = np.array([0.3, -0.2, 0.5], np.float32)
    taus = np.array([-0.5, -0.1, 0.0, 1e-4, 0.05, 0.5], np.float32)
    R = rotation(emus["remu"], taus, w)
    want = rodrigues(torch.from_numpy(taus).double()[:, None] * torch.from_numpy(w).double()[None, :]).numpy()
    assert np.abs(R - want).max() <= 2e-7
    assert np.array_equal(rotation(emus["remu"], taus, np.zeros(3, np.float32)), np.broadcast_to(np.eye(3, dtype=np.float32),
                                                                                                   (6, 3, 3)))


def _pose_inverse64(R, t):
    """(q xyzw, t) of the camera -> pointcloud pose whose inverse is x -> R x + t (float64)."""
    Ri = R.T
    return Rotation.from_matrix(Ri).as_quat(), -Ri @ t


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_record_equals_the_global_shutter_record_at_the_moved_pose(emus, lens):
    """Independent of the fixed point: take tau_3 from the kernel, compose the pose at tau_3 on the host in float64, and render
    the isolated Gaussian with the global-shutter kernel at that pose: position, conic, rescale, opacity, depth and radius
    agree to float32 rounding (the colour differs: the SH direction keeps the mid-readout camera centre)."""
    model, k = LENSES[lens]
    H, W = 64, 64
    K = [[48.0, 0, 31.0], [0, 52.0, 30.0], [0, 0, 1]]
    a = math.radians(4.0) / 2
    q0 = np.array([math.sin(a) * 0.6, math.sin(a) * 0.8, 0.0, math.cos(a)])
    t0 = np.array([0.2, -0.1, -0.3])
    sc = _single((0.3, 0.5, 3.5), _feats_row(-2.5), K, H, W, tuple(q0), tuple(t0))
    pre = run_preprocess_rs(emus["remu"], sc, model, k, MOTION)
    tau = float(pre.row_time[0])
    assert pre.point_offset[0] == 0 and 0.05 < abs(tau) < 0.5
    W0 = Rotation.from_quat(q0 / np.linalg.norm(q0)).as_matrix().T
    tw = -W0 @ t0
    m = np.array(MOTION, np.float64)
    Rd = rodrigues(torch.tensor(tau * m[3:])[None, :]).numpy()[0]
    q1, t1 = _pose_inverse64(Rd @ W0, Rd @ tw + tau * m[:3])
    moved = _single((0.3, 0.5, 3.5), _feats_row(-2.5), K, H, W, tuple(q1), tuple(t1))
    if lens == "pinhole":
        ref = run_preprocess_rs(emus["remu"], moved, model, k, (0.0,) * 6)
    else:
        from simt_lens_helpers import run_preprocess_lens
        ref = run_preprocess_lens(emus["lemu"], moved, model, k)
    r, e = pre.records[0], ref.records[0]
    cols = [0, 1, 2, 3, 4, 5, 6, 7, 11]  # u v a b | c rescale opacity depth | radius
    assert np.allclose(r[cols], e[cols], rtol=2e-5, atol=2e-5 * np.abs(e[cols]).max()), (r, e)
    assert np.allclose(pre.pic[0], ref.pic[0], rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------ forward against the float64 evaluator
def _dense(sc, feats_n, model, k, motion, requires_grad=False):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = torch.from_numpy(feats_n).double().requires_grad_(requires_grad)
    m = torch.tensor(motion, dtype=torch.float64, requires_grad=requires_grad)
    image, aux = dense_render_rs(xyz, feats, sc.point_invalid_mask, sc.point_object_id, sc.camera_info.camera_intrinsics,
                                 sc.q_pointcloud_camera, sc.t_pointcloud_camera, H, W, model, k, m)
    return xyz, feats, m, image, aux


@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_forward_matches_dense_evaluator(emus, lens):
    model, k = LENSES[lens]
    sc = _scene(61, objects=2)
    st = emulated_forward_rs(emus["emu"], emus["remu"], sc, model, k, MOTION, exact=True)
    _, _, _, image, aux = _dense(sc, st.pre.feats, model, k, MOTION)
    H, W = st.pre.H, st.pre.W
    assert np.abs(aux["tau"].numpy() - st.pre.row_time).max() <= 1e-5
    assert (np.abs(st.pre.row_time) > 0.2).any()
    ids = st.pre.point_id[:st.M]
    assert np.array_equal(np.sort(ids), np.sort(aux["ids"].numpy()))
    order = np.argsort(ids)
    rec = st.pre.records[:st.M][order]
    assert np.allclose(rec[:, 0:2], aux["uv"].detach().numpy(), rtol=1e-5, atol=1e-4)
    conic = aux["conic"].detach().numpy()
    assert np.allclose(rec[:, 2:5], conic[:, 0:3], rtol=1e-4, atol=1e-5 * np.abs(conic[:, 0:3]).max())
    assert np.allclose(rec[:, 7], aux["pc"].detach().numpy()[:, 2], rtol=1e-6)
    assert np.array_equal(aux["count"].numpy(), st.count)
    assert np.abs(image.detach().numpy() - st.image).max() < 1e-4
    depth, _ = differentiable_depth(aux, H, W)
    assert np.abs(depth.detach().numpy() - st.depth).max() < 1e-3
    # the motion moved the splats: the global-shutter forward renders a different image
    base = emulated_forward(emus["emu"], sc) if lens == "pinhole" else emulated_forward_lens(emus["emu"], emus["lemu"], sc, model, k)
    assert np.abs(base.image - st.image).max() > 0.05


def test_zero_motion_is_bit_identical_to_the_global_shutter_kernels(emus):
    g_img = torch.randn((32, 48, 3), generator=torch.Generator().manual_seed(3)).numpy()
    for lens in ("pinhole", "opencv", "fisheye"):
        model, k = LENSES[lens]
        sc = _scene(63, objects=3)
        st = emulated_forward_rs(emus["emu"], emus["remu"], sc, model, k, (0.0,) * 6)
        ref = emulated_forward(emus["emu"], sc) if lens == "pinhole" else \
            emulated_forward_lens(emus["emu"], emus["lemu"], sc, model, k)
        assert st.M == ref.M and np.array_equal(st.pre.point_offset, ref.pre.point_offset)
        assert np.array_equal(st.pre.records, ref.pre.records) and np.array_equal(st.pre.pic, ref.pre.pic)
        assert np.array_equal(st.sorted_vals, ref.sorted_vals) and np.array_equal(st.image, ref.image)
        assert (st.pre.row_time[st.pre.point_offset < 0] == 0).all()
        for depth in (False, True):
            if depth:
                g_dep = torch.randn((32, 48), generator=torch.Generator().manual_seed(4)).numpy()
                _, _, accum, _ = emulated_backward_depth(emus["emu"], emus["demu"], st, g_img, g_dep)
            else:
                accum = _loop_a_image(emus["emu"], st, g_img, True)
            res = emulated_points_rs(emus["emu"], emus["remu"], st, accum, depth=depth, mgrad=True)
            if lens == "pinhole":
                gx0, gf0 = emulated_points(emus["emu"], emus["demu"], ref, accum, depth=depth)
            else:
                gx0, gf0 = emulated_points_lens(emus["emu"], emus["lemu"], ref, accum, depth=depth)
            assert np.array_equal(res.gx, gx0) and np.array_equal(res.gf, gf0), (lens, depth)
            assert np.isfinite(res.gm).all() and (res.gm != 0).any()  # refining from zero has a gradient


# ------------------------------------------------------------------ backward against float64 autograd
def _case(emus, lens, kind, seed, objects=1, transposed=True, band=3, motion=MOTION):
    model, k = LENSES[lens]
    emu, demu = emus["emu"], emus["demu"]
    sc = _scene(seed, objects=objects)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward_rs(emu, emus["remu"], sc, model, k, motion, exact=False)
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g, dtype=torch.float32)
    g_dep = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "depth" else None
    g_alpha = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "alpha" else None
    extra = g_map = None
    if kind == "image":
        accum = _loop_a_image(emu, st, g_img.numpy(), transposed)
    elif kind == "depth":
        _, _, accum, _ = emulated_backward_depth(emu, demu, st, g_img.numpy(), g_dep.numpy(), band)
    elif kind == "alpha":
        _, _, accum, _ = emulated_backward_alpha(emu, demu, emus["aemu"], st, g_img.numpy(), g_alpha.numpy(), band=band)
    else:
        N = sc.point_cloud.shape[0]
        extra = torch.randn((N, 5), generator=g, dtype=torch.float32).numpy()
        g_map = torch.randn((H, W, 5), generator=g, dtype=torch.float32)
        _, _, _, accum, _ = emulated_backward_features(emu, demu, emus["femu"], st, extra, g_map.numpy(), g_img.numpy(),
                                                       band=band)
    res = emulated_points_rs(emu, emus["remu"], st, accum, band, depth=kind == "depth")
    xyz, feats, m, image, aux = _dense(sc, st.pre.feats, model, k, motion, requires_grad=True)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)
    return st, accum, res, xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), m.grad.numpy()


def _check(res, ex, ef, em, groups=GROUPS):
    ok = grad_close(res.gx, ex)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], ok
    for sl in groups:
        ok = grad_close(res.gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    scale = np.abs(em).max()
    assert scale > 0
    assert (np.abs(res.gm - em) <= 2e-3 * np.abs(em) + 2e-4 * scale).all(), (res.gm, em)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_gradients_match_dense_autograd(emus, lens, kind):
    _, _, res, ex, ef, em = _case(emus, lens, kind, 71)
    _check(res, ex, ef, em)


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_emulated_gradients_with_three_objects_sharing_warps(emus, lens):
    st, _, res, ex, ef, em = _case(emus, lens, "image", 73, objects=3)
    obj = st.scene.point_object_id.numpy()
    kept = st.pre.point_offset >= 0
    assert len(set(obj[:32][kept[:32]].tolist())) == 3  # one warp holds in-camera points of all three objects
    # not the SH columns: the SH view direction of the per-point backward takes t_pc as the camera centre, which is the
    # evaluator's only for a unit q (these scenes give the other objects non-unit ones); the motion does not reach them
    _check(res, ex, ef, em, groups=GROUPS[:3])


@pytest.mark.parametrize("lens", ["pinhole", "opencv"])
def test_emulated_gradients_under_the_butterfly_loop_a(emus, lens):
    _, _, res, ex, ef, em = _case(emus, lens, "image", 75, transposed=False, band=1)
    _check(res, ex, ef, em)


@pytest.mark.parametrize("kind", ["image", "depth"])
def test_motion_gradient_is_deterministic_and_leaves_every_other_output_unchanged(emus, kind):
    st, accum, res, _, _, _ = _case(emus, "opencv", kind, 77)
    again = emulated_points_rs(emus["emu"], emus["remu"], st, accum, depth=kind == "depth")
    assert np.array_equal(res.gm, again.gm) and np.array_equal(res.partials, again.partials)
    assert res.blocks == min(math.ceil(st.pre.point_offset.shape[0] / 128), 2048)
    assert np.allclose(res.partials.astype(np.float64).sum(0), res.gm, rtol=1e-5, atol=1e-6 * np.abs(res.gm).max())
    off = emulated_points_rs(emus["emu"], emus["remu"], st, accum, depth=kind == "depth", mgrad=False)
    assert off.gm is None and np.array_equal(res.gx, off.gx) and np.array_equal(res.gf, off.gf)


# ------------------------------------------------------------------ C ABI
def _rs(*motion, row_time=256):
    m = list(motion) + [0.0] * (6 - len(motion))
    return _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(*m), row_time=ctypes.c_void_p(row_time))


def test_abi_sizes_of_the_rolling_shutter_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 14)()
    lib.gsb200_abi_sizes_ext(sizes, 14)
    assert sizes[12] == ctypes.sizeof(_lib.GsbRollingShutterArgs) == 32
    assert sizes[13] == ctypes.sizeof(_lib.GsbRollingShutterGradArgs) == 16
    first12 = (ctypes.c_int64 * 12)()
    lib.gsb200_abi_sizes_ext(first12, 12)
    assert list(first12) == list(sizes)[:12]
    assert lib.gsb200_rolling_shutter_grad_temp_bytes() == 2048 * 6 * 4
    for name in ("gsb200_forward_rolling_shutter", "gsb200_backward_rolling_shutter", "gsb200_rolling_shutter_grad_temp_bytes"):
        assert hasattr(lib, name) and name in _lib.EXPORTS


def test_c_entry_points_check_their_arguments_before_any_cuda_call():
    lib = _lib.load()
    fargs = _lib.GsbForwardArgs()
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    ok = ctypes.c_void_p(256)
    good = _lib.GsbRollingShutterGradArgs(grad_motion=ok, temp=ok)
    bad_rs = [(_rs(0.1, math.nan), b"not finite"), (_rs(0, 0, 0, 0, 0, math.inf), b"not finite"),
              (_rs(0.1, row_time=0), b"null row_time"), (_rs(0.1, row_time=258), b"4-byte aligned")]
    for rs, msg in bad_rs:  # args point at nothing the call could use: these checks come first
        assert lib.gsb200_forward_rolling_shutter(ctypes.byref(fargs), None, None, ctypes.byref(rs)) == -1
        assert msg in lib.gsb200_last_error()
        assert lib.gsb200_backward_rolling_shutter(ctypes.byref(bargs), None, None, None, None, None, ctypes.byref(rs),
                                                   ctypes.byref(good)) == -1
        assert msg in lib.gsb200_last_error()
    lens = _lib.GsbLensArgs(model=7)
    assert lib.gsb200_forward_rolling_shutter(ctypes.byref(fargs), None, ctypes.byref(lens), ctypes.byref(_rs(0.1))) == -1
    assert b"unknown lens model" in lib.gsb200_last_error()
    bad_grad = [(_lib.GsbRollingShutterGradArgs(grad_motion=None, temp=ok), b"null grad_motion"),
                (_lib.GsbRollingShutterGradArgs(grad_motion=ok, temp=None), b"null grad_motion"),
                (_lib.GsbRollingShutterGradArgs(grad_motion=ctypes.c_void_p(258), temp=ok), b"4-byte aligned"),
                (_lib.GsbRollingShutterGradArgs(grad_motion=ok, temp=ctypes.c_void_p(260)), b"16-byte aligned")]
    for g, msg in bad_grad:
        assert lib.gsb200_backward_rolling_shutter(ctypes.byref(bargs), None, None, None, None, None, ctypes.byref(_rs(0.1)),
                                                   ctypes.byref(g)) == -1
        assert msg in lib.gsb200_last_error()
    assert lib.gsb200_backward_rolling_shutter(ctypes.byref(bargs), None, None, None, None, None, None, ctypes.byref(good)) == -1
    assert b"needs a rolling shutter" in lib.gsb200_last_error()
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for g in (None, ctypes.byref(good)):
        assert lib.gsb200_backward_rolling_shutter(ctypes.byref(compact), None, None, None, None, None,
                                                   ctypes.byref(_rs(0.1)), g) == -4
        assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # valid arguments reach the usual argument checks
    assert lib.gsb200_forward_rolling_shutter(ctypes.byref(fargs), None, None, ctypes.byref(_rs(0.1))) == -1
    assert b"forward: null camera_intrinsics" in lib.gsb200_last_error()
    assert lib.gsb200_backward_rolling_shutter(ctypes.byref(bargs), None, None, None, None, None, ctypes.byref(_rs(0.1)),
                                               ctypes.byref(good)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_rolling_shutter_is_exactly_the_lens_calls():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    for lens in (None, ctypes.byref(_lib.GsbLensArgs(model=0)), ctypes.byref(_lib.GsbLensArgs(model=3))):
        fargs = _lib.GsbForwardArgs()
        want = lib.gsb200_forward_lens(ctypes.byref(fargs), None, lens)
        want_msg = lib.gsb200_last_error()
        assert lib.gsb200_forward_rolling_shutter(ctypes.byref(fargs), None, lens, None) == want != 0
        assert lib.gsb200_last_error() == want_msg
        for args, extra in ((_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                            (_lib.GsbBackwardArgs(), (fake, fake, None, None))):
            want = lib.gsb200_backward_lens(ctypes.byref(args), *extra, lens)
            want_msg = lib.gsb200_last_error()
            assert lib.gsb200_backward_rolling_shutter(ctypes.byref(args), *extra, lens, None, None) == want != 0
            assert lib.gsb200_last_error() == want_msg


# ------------------------------------------------------------------ Python surface
def test_rolling_shutter_record_and_camera_velocity():
    rs = RollingShutter((0.1, 0, 0), [0, 0.2, 0])
    assert rs.linear == (0.1, 0.0, 0.0) and rs.angular == (0.0, 0.2, 0.0) and rs.motion == (0.1, 0, 0, 0, 0.2, 0)
    for bad in (((0, 0), (0, 0, 0)), ((0, 0, math.nan), (0, 0, 0)), ((0, 0, 0), (math.inf, 0, 0))):
        with pytest.raises(ValueError):
            RollingShutter(*bad)
    m = RollingShutter.from_camera_velocity((1.0, -2.0, 0.5), (0.1, 0.0, -0.3), 0.02)
    assert m.linear == pytest.approx((-0.02, 0.04, -0.01)) and m.angular == pytest.approx((-0.002, 0.0, 0.006))
    with pytest.raises(ValueError, match="readout_time"):
        RollingShutter.from_camera_velocity((0, 0, 0), (0, 0, 0), -1.0)
    assert CameraInfo(torch.eye(3), 16, 16, 0).rolling_shutter is None


def test_camera_velocity_matches_a_render_at_the_moved_pose(emus):
    """A camera translating at u (camera frame) for readout T: the row at time tau is seen from the centre moved by tau T u,
    which is the global-shutter render with the camera translated by tau T u."""
    H, W = 64, 64
    K = [[50.0, 0, 32.0], [0, 50.0, 32.0], [0, 0, 1]]
    u, T = np.array([0.5, 1.5, -0.8]), 0.03
    rs = RollingShutter.from_camera_velocity(tuple(u), (0.0, 0.0, 0.0), T)
    sc = _single((-0.2, 0.4, 3.0), _feats_row(-2.5), K, H, W)
    pre = run_preprocess_rs(emus["remu"], sc, "pinhole", (), rs.motion)
    tau = float(pre.row_time[0])
    # camera -> pointcloud pose: identity rotation, centre at tau T u
    moved = _single((-0.2, 0.4, 3.0), _feats_row(-2.5), K, H, W, t=tuple(tau * T * u))
    ref = run_preprocess_rs(emus["remu"], moved, "pinhole", (), (0.0,) * 6)
    cols = [0, 1, 2, 3, 4, 5, 6, 7, 11]
    assert np.allclose(pre.records[0][cols], ref.records[0][cols], rtol=2e-5, atol=1e-5)


def _input(rolling=True, lens=None):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, lens,
                    RollingShutter((0.1, 0, 0), (0, 0.02, 0)) if rolling else None)
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_configuration_of_the_rolling_shutter():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_rolling_shutter=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_rolling_shutter=True, gradient_exchange=object())
    inp = _input()
    for option in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion"):
        with pytest.raises(ValueError, match=option):
            G(Config(), **{option: True})._rolling_shutter_args(inp.camera_info)
    op = G(Config(), differentiable_rolling_shutter=True)
    op.gradient_exchange = object()
    with pytest.raises(ValueError, match="gradient_exchange"):
        op._rolling_shutter_args(inp.camera_info)
    op = G(Config(), differentiable_rolling_shutter=True)
    for m, msg in ((torch.zeros(5), r"\(6,\)"), (torch.zeros(6, dtype=torch.float64), "float32"), (torch.zeros(2, 3), r"\(6,\)"),
                   ([0.0] * 6, "torch.Tensor"), (torch.tensor([math.nan] + [0.0] * 5), "finite")):
        with pytest.raises(ValueError, match=msg):
            op(inp, rolling_shutter_motion=m)
    with pytest.raises(ValueError, match="without a rolling shutter"):
        op(_input(rolling=False), rolling_shutter_motion=torch.zeros(6))
    with pytest.raises(ValueError, match="differentiable_rolling_shutter"):
        G(Config())(inp, rolling_shutter_motion=torch.zeros(6))
    # the values rendered are the tensor's
    rs = op._rolling_shutter_args(inp.camera_info, torch.tensor([0.2, -0.01, 0.0, 0.0, 0.03, 0.0]))
    assert list(rs.motion) == pytest.approx([0.2, -0.01, 0, 0, 0.03, 0])
    assert list(G(Config())._rolling_shutter_args(inp.camera_info).motion) == pytest.approx([0.1, 0, 0, 0, 0.02, 0])
    assert G(Config())._rolling_shutter_args(_input(rolling=False).camera_info) is None
    # with a lens as well
    assert G(Config())._rolling_shutter_args(_input(lens=LensDistortion("fisheye", (0.1, 0, 0, 0))).camera_info) is not None


def _trainer(cams, fused_step=False, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, cam, lens, rs))
             for cam, lens, rs in cams]
    seen = {}
    factory = lambda **kwargs: seen.update(kwargs) or (lambda *a, **k: None)  # noqa: E731
    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=factory, fused_step=fused_step), seen


def test_trainer_configuration_of_the_rolling_shutter():
    a = RollingShutter((0.1, 0, 0), (0, 0.02, 0))
    b = RollingShutter((0, -0.05, 0), (0.01, 0, 0))
    for rate in (-1e-3, math.nan, math.inf):
        with pytest.raises(ValueError, match="rolling_shutter_learning_rate"):
            _trainer([(0, None, a)], rolling_shutter_learning_rate=rate)
    with pytest.raises(ValueError, match="rolling-shutter"):
        _trainer([(0, None, None)], rolling_shutter_learning_rate=1e-3)
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(pose_learning_rate=1e-3), "pose"),
                    (dict(intrinsics_learning_rate=1e-3), "intrinsics"), (dict(distortion_learning_rate=1e-3), "distortion")):
        lens = LensDistortion("opencv", (-0.1, 0, 0, 0, 0)) if "distortion" in kw else None
        with pytest.raises(ValueError, match=msg):
            _trainer([(0, lens, a)], **kw)
    trainer, seen = _trainer([(0, None, a), (1, None, b), (0, None, None)], rolling_shutter_learning_rate=1e-3)
    assert seen.get("differentiable_rolling_shutter") is True
    assert sorted(trainer._rolling_shutter) == [0, 1]
    leaf = trainer._rolling_shutter[0]
    assert leaf.is_leaf and leaf.requires_grad and leaf.device.type == "cpu" and leaf.dtype == torch.float32
    f32 = lambda r: RollingShutter(*(tuple(float(np.float32(v)) for v in x) for x in (r.linear, r.angular)))  # noqa: E731
    assert trainer.refined_rolling_shutter() == [f32(a), f32(b), None]
    with torch.no_grad():
        leaf[0] = 0.25
    assert trainer.refined_rolling_shutter()[0] == f32(RollingShutter((0.25, 0, 0), (0, 0.02, 0)))
    # off: the views' own motions and no extra operator option; rolling-shutter views train through the autograd loop
    trainer, seen = _trainer([(0, None, a)])
    assert "differentiable_rolling_shutter" not in seen and trainer.refined_rolling_shutter() == [a]


def test_dataset_reads_the_rolling_shutter_record_key(tmp_path):
    from PIL import Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    img = tmp_path / "a.png"
    Image.fromarray(np.zeros((32, 48, 3), np.uint8)).save(img)
    base = {"image_path": str(img), "T_pointcloud_camera": np.eye(4).tolist(),
            "camera_intrinsics": [[40.0, 0, 24.0], [0, 40.0, 16.0], [0, 0, 1]], "camera_height": 32, "camera_width": 48,
            "camera_id": 0}
    records = [dict(base), dict(base, rolling_shutter={"linear_velocity": [1.0, 0, 0], "angular_velocity": [0, 0.5, 0],
                                                       "readout_time": 0.02})]
    path = tmp_path / "poses.json"
    path.write_text(json.dumps(records))
    ds = ImagePoseDataset(str(path))
    assert ds[0][3].rolling_shutter is None
    rs = ds[1][3].rolling_shutter
    assert rs == RollingShutter.from_camera_velocity((1.0, 0, 0), (0, 0.5, 0), 0.02)
    bad = tmp_path / "bad.json"
    bad.write_text(json.dumps([dict(base, rolling_shutter={"linear_velocity": [1.0, 0], "angular_velocity": [0, 0, 0],
                                                           "readout_time": 0.02})]))
    with pytest.raises(ValueError):
        ImagePoseDataset(str(bad))[0]
    from taichi_3d_gaussian_splatting_b200.trainer import downsample_image_and_camera_info
    _, ci = downsample_image_and_camera_info(torch.zeros((3, 32, 48)), ds[1][3], 2)
    assert ci.rolling_shutter == rs
