"""Motion blur (``gsb200_forward_motion_blur`` / ``gsb200_backward_motion_blur``) on the CPU: the unmodified BLUR kernels under
the SIMT emulator against the float64 dense evaluator (``torch_reference_motion_blur``) and autograd on it, zero exposure
motion against the rolling-shutter and lens kernels bit for bit, the determinism of the motion gradient, the C ABI's argument
checks, and the Python surface (``Camera.MotionBlur``, the dataset key, the operator's and the trainer's refusals)."""
import ctypes
import json
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion, MotionBlur, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator
from simt_lens_helpers import build_lens_emulator
from simt_motion_blur_helpers import build_motion_blur_emulator, emulated_forward_blur, emulated_points_blur
from simt_rolling_shutter_helpers import build_rolling_shutter_emulator, emulated_forward_rs, emulated_points_rs
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference import postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_motion_blur import dense_render_blur
from torch_reference_rolling_shutter import rodrigues

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "pinhole": ("pinhole", ()),
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
RS_MOTION = (0.06, -0.09, 0.04, 0.05, -0.08, 0.06)  # v, w over one readout
BLUR = (0.05, 0.03, -0.02, -0.02, 0.03, 0.01)  # v, w over the exposure: streaks of a few pixels in the 48 x 32 scenes


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator(), remu=build_rolling_shutter_emulator(), bemu=build_motion_blur_emulator())


def _dense(sc, feats_n, model, k, motion, blur, requires_grad=False):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = torch.from_numpy(feats_n).double().requires_grad_(requires_grad)
    mb = torch.tensor(blur, dtype=torch.float64, requires_grad=requires_grad)
    image, aux = dense_render_blur(xyz, feats, sc.point_invalid_mask, sc.point_object_id, sc.camera_info.camera_intrinsics,
                                   sc.q_pointcloud_camera, sc.t_pointcloud_camera, H, W, model, k, motion, mb)
    return xyz, feats, mb, image, aux


# ------------------------------------------------------------------ forward against the float64 evaluator
@pytest.mark.parametrize("rolling", [False, True])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_forward_matches_dense_evaluator(emus, lens, rolling):
    model, k = LENSES[lens]
    motion = RS_MOTION if rolling else (0.0,) * 6
    sc = _scene(61, objects=2)
    st = emulated_forward_blur(emus["emu"], emus["bemu"], sc, model, k, motion, BLUR, rolling, exact=True)
    _, _, _, image, aux = _dense(sc, st.pre.feats, model, k, motion, BLUR)
    ids = st.pre.point_id[:st.M]
    assert np.array_equal(np.sort(ids), np.sort(aux["ids"].numpy()))
    assert aux["streak"].max() > 2.0  # the blur is visible
    order = np.argsort(ids)
    rec = st.pre.records[:st.M][order]
    assert np.allclose(rec[:, 0:2], aux["uv"].detach().numpy(), rtol=1e-5, atol=1e-4)
    conic = aux["conic"].detach().numpy()
    assert np.allclose(rec[:, 2:5], conic[:, 0:3], rtol=1e-4, atol=1e-5 * np.abs(conic[:, 0:3]).max())
    slot = (aux["conic"][:, 3] * aux["comp"]).detach().numpy()  # rescale c_b
    assert np.allclose(rec[:, 5], slot, rtol=1e-4, atol=1e-6)
    assert (aux["comp"].detach().numpy() < 0.9).any()
    assert np.allclose(rec[:, 11], aux["radius"].numpy(), rtol=1e-4, atol=1e-4)  # from Sigma' + B
    assert np.array_equal(aux["count"].numpy(), st.count)
    assert np.abs(image.detach().numpy() - st.image).max() < 1e-4
    H, W = st.pre.H, st.pre.W
    depth, _ = differentiable_depth(aux, H, W)
    assert np.abs(depth.detach().numpy() - st.depth).max() < 1e-3
    # the keys: every (tile, splat) pair the blurred square reaches, sorted as the sort wants them
    assert st.K >= int(st.pre.num_tiles[:st.M].sum()) // 4
    # the blur changed the render
    sharp = emulated_forward_rs(emus["emu"], emus["remu"], sc, model, k, motion)
    assert np.abs(sharp.image - st.image).max() > 0.02


def test_blurred_radius_covers_the_streak(emus):
    """A small isotropic splat moved sideways: the radius is 3 sqrt(lambda_max(Sigma' + B)), so the tile square reaches the
    ends of a long streak (|d| / 2 = 3 sqrt(|d|^2 / 12) * 0.29), and the conic is the inverse of Sigma_d + B."""
    H, W = 64, 96
    K = [[50.0, 0, 48.0], [0, 50.0, 32.0], [0, 0, 1]]
    from types import SimpleNamespace
    row = [0.0] * 56
    row[3] = 1.0
    row[4] = row[5] = row[6] = -4.0
    row[7] = 2.0
    sc = SimpleNamespace(point_cloud=torch.tensor([[0.0, 0.0, 2.0]]), point_cloud_features=torch.tensor([row]),
                         point_invalid_mask=torch.zeros(1, dtype=torch.int8), point_object_id=torch.zeros(1, dtype=torch.int32),
                         q_pointcloud_camera=torch.tensor([[0.0, 0.0, 0.0, 1.0]]), t_pointcloud_camera=torch.zeros(1, 3),
                         camera_info=CameraInfo(torch.tensor(K), H, W, 0))
    from simt_motion_blur_helpers import run_preprocess_blur
    vx = 0.8  # d = fx vx / z = 20 px
    pre = run_preprocess_blur(emus["bemu"], sc, "pinhole", (), (0.0,) * 6, (vx, 0, 0, 0, 0, 0), False)
    base = run_preprocess_blur(emus["bemu"], sc, "pinhole", (), (0.0,) * 6, (0.0,) * 6, False)
    d = 50.0 * vx / 2.0
    r0 = base.records[0]
    s = np.exp(-4.0) * 50.0 / 2.0  # the splat's screen std
    sig = np.array([[s * s + 0.3 + d * d / 12, 0.0], [0.0, s * s + 0.3]])
    inv = np.linalg.inv(sig)
    r = pre.records[0]
    assert np.allclose([r[2], r[3], r[4]], [inv[0, 0], inv[0, 1], inv[1, 1]], rtol=1e-5)
    assert r[11] == pytest.approx(3 * math.sqrt(s * s + d * d / 12), rel=1e-5) and r[11] > 3 * r0[11]
    cb = math.sqrt((s * s + 0.3) / (s * s + 0.3 + d * d / 12))
    assert r[5] == pytest.approx(r0[5] * cb, rel=1e-5)
    assert pre.num_tiles[0] > base.num_tiles[0]


def test_zero_exposure_motion_is_bit_identical_to_the_kernels_without_blur(emus):
    g_img = torch.randn((32, 48, 3), generator=torch.Generator().manual_seed(3)).numpy()
    for lens in ("pinhole", "opencv", "fisheye"):
        model, k = LENSES[lens]
        for rolling in (False, True):
            motion = RS_MOTION if rolling else (0.0,) * 6
            sc = _scene(63, objects=3)
            st = emulated_forward_blur(emus["emu"], emus["bemu"], sc, model, k, motion, (0.0,) * 6, rolling)
            # the rolling-shutter kernel with zero motion is the global-shutter (lens) kernel bit for bit (its own test)
            ref = emulated_forward_rs(emus["emu"], emus["remu"], sc, model, k, motion)
            assert st.M == ref.M and st.K == ref.K and np.array_equal(st.pre.point_offset, ref.pre.point_offset)
            assert np.array_equal(st.pre.records, ref.pre.records) and np.array_equal(st.pre.pic, ref.pre.pic)
            assert np.array_equal(st.pre.keys[:st.K], ref.pre.keys[:ref.K])
            assert np.array_equal(st.sorted_vals, ref.sorted_vals) and np.array_equal(st.image, ref.image)
            if rolling:
                assert np.array_equal(st.pre.row_time, ref.pre.row_time)
            for depth in (False, True):
                if depth:
                    g_dep = torch.randn((32, 48), generator=torch.Generator().manual_seed(4)).numpy()
                    _, _, accum, _ = emulated_backward_depth(emus["emu"], emus["demu"], st, g_img, g_dep)
                else:
                    accum = _loop_a_image(emus["emu"], st, g_img, True)
                res = emulated_points_blur(emus["emu"], emus["bemu"], st, accum, depth=depth, bgrad=True)
                want = emulated_points_rs(emus["emu"], emus["remu"], ref, accum, depth=depth, mgrad=False)
                assert np.array_equal(res.gx, want.gx) and np.array_equal(res.gf, want.gf), (lens, rolling, depth)
                assert (res.gm == 0).all()  # dB/dm_b = 0 at m_b = 0: refinement cannot start from zero


# ------------------------------------------------------------------ backward against float64 autograd
def _case(emus, lens, kind, seed, objects=1, transposed=True, band=3, rolling=False, blur=BLUR):
    model, k = LENSES[lens]
    motion = RS_MOTION if rolling else (0.0,) * 6
    emu, demu = emus["emu"], emus["demu"]
    sc = _scene(seed, objects=objects)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward_blur(emu, emus["bemu"], sc, model, k, motion, blur, rolling, exact=False)
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
    res = emulated_points_blur(emu, emus["bemu"], st, accum, band, depth=kind == "depth")
    xyz, feats, mb, image, aux = _dense(sc, st.pre.feats, model, k, motion, blur, requires_grad=True)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)
    return st, accum, res, xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), mb.grad.numpy()


def _check(res, ex, ef, em, groups=GROUPS):
    ok = grad_close(res.gx, ex)
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


@pytest.mark.parametrize("kind", ["image", "depth"])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_gradients_through_a_rolling_shutter(emus, lens, kind):
    _, _, res, ex, ef, em = _case(emus, lens, kind, 72, rolling=True)
    _check(res, ex, ef, em)


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_emulated_gradients_with_three_objects_sharing_warps(emus, lens):
    st, _, res, ex, ef, em = _case(emus, lens, "image", 73, objects=3)
    obj = st.scene.point_object_id.numpy()
    kept = st.pre.point_offset >= 0
    assert len(set(obj[:32][kept[:32]].tolist())) == 3
    _check(res, ex, ef, em, groups=GROUPS[:3])  # SH columns: see the rolling-shutter test of the same name


def test_emulated_gradients_under_the_butterfly_loop_a(emus):
    _, _, res, ex, ef, em = _case(emus, "opencv", "image", 75, transposed=False, band=1)
    _check(res, ex, ef, em)


def test_reference_motion_gradient_matches_finite_differences():
    """The evaluator's dL/dm_b by autograd against central differences (tile membership and the blend order are piecewise
    constant in m_b; the step is small enough to keep them)."""
    sc = _scene(79)
    feats = sc.point_cloud_features.numpy().astype(np.float32)
    g = torch.randn((32, 48, 3), generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    _, _, mb, image, _ = _dense(sc, feats, "opencv", LENSES["opencv"][1], (0.0,) * 6, BLUR, requires_grad=True)
    (image * g).sum().backward()
    want = mb.grad.numpy()
    h = 1e-6
    for i in range(6):
        e = np.zeros(6)
        e[i] = h
        lp = float((_dense(sc, feats, "opencv", LENSES["opencv"][1], (0.0,) * 6, tuple(np.add(BLUR, e)))[3] * g).sum())
        lm = float((_dense(sc, feats, "opencv", LENSES["opencv"][1], (0.0,) * 6, tuple(np.subtract(BLUR, e)))[3] * g).sum())
        assert (lp - lm) / (2 * h) == pytest.approx(want[i], rel=1e-4, abs=1e-6 * np.abs(want).max())


def test_sign_of_the_exposure_motion_is_not_observable(emus):
    sc = _scene(81)
    a = emulated_forward_blur(emus["emu"], emus["bemu"], sc, "pinhole", (), (0.0,) * 6, BLUR, False)
    b = emulated_forward_blur(emus["emu"], emus["bemu"], sc, "pinhole", (), (0.0,) * 6, tuple(-x for x in BLUR), False)
    assert np.array_equal(a.pre.records, b.pre.records) and np.array_equal(a.image, b.image)


@pytest.mark.parametrize("kind", ["image", "depth"])
def test_motion_gradient_is_deterministic_and_leaves_every_other_output_unchanged(emus, kind):
    st, accum, res, _, _, _ = _case(emus, "opencv", kind, 77)
    again = emulated_points_blur(emus["emu"], emus["bemu"], st, accum, depth=kind == "depth")
    assert np.array_equal(res.gm, again.gm) and np.array_equal(res.partials, again.partials)
    assert res.blocks == min(math.ceil(st.pre.point_offset.shape[0] / 128), 2048)
    assert np.allclose(res.partials.astype(np.float64).sum(0), res.gm, rtol=1e-5, atol=1e-6 * np.abs(res.gm).max())
    off = emulated_points_blur(emus["emu"], emus["bemu"], st, accum, depth=kind == "depth", bgrad=False)
    assert off.gm is None and np.array_equal(res.gx, off.gx) and np.array_equal(res.gf, off.gf)


# ------------------------------------------------------------------ C ABI
def _blur(*motion):
    m = list(motion) + [0.0] * (6 - len(motion))
    return _lib.GsbMotionBlurArgs(motion=(ctypes.c_float * 6)(*m))


def test_abi_sizes_of_the_motion_blur_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 3)(*([-7] * 3))
    lib.gsb200_abi_sizes_motion_blur(sizes)
    assert sizes[0] == ctypes.sizeof(_lib.GsbMotionBlurArgs) == 24
    assert sizes[1] == ctypes.sizeof(_lib.GsbMotionBlurGradArgs) == 16
    assert sizes[2] == -7
    ext = (ctypes.c_int64 * 17)(*([-7] * 17))
    lib.gsb200_abi_sizes_ext(ext, 17)  # the extension table still ends at GsbAppearanceArgs
    assert ext[15] == ext[16] == -7
    assert lib.gsb200_motion_blur_grad_temp_bytes() == 2048 * 6 * 4
    for name in ("gsb200_forward_motion_blur", "gsb200_backward_motion_blur", "gsb200_motion_blur_grad_temp_bytes",
                 "gsb200_abi_sizes_motion_blur"):
        assert hasattr(lib, name) and name in _lib.EXPORTS


def test_c_entry_points_check_their_arguments_before_any_cuda_call():
    lib = _lib.load()
    fargs = _lib.GsbForwardArgs()
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    ok = ctypes.c_void_p(256)
    good = _lib.GsbMotionBlurGradArgs(grad_motion=ok, temp=ok)
    for blur in (_blur(0.1, math.nan), _blur(0, 0, 0, 0, 0, math.inf)):
        assert lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, None, None, ctypes.byref(blur)) == -1
        assert b"not finite" in lib.gsb200_last_error()
        assert lib.gsb200_backward_motion_blur(ctypes.byref(bargs), None, None, None, None, None, None, ctypes.byref(blur),
                                               ctypes.byref(good)) == -1
        assert b"not finite" in lib.gsb200_last_error()
    lens = _lib.GsbLensArgs(model=7)
    assert lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, ctypes.byref(lens), None, ctypes.byref(_blur(0.1))) == -1
    assert b"unknown lens model" in lib.gsb200_last_error()
    rs = _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(0.1, 0, 0, 0, 0, 0), row_time=None)
    assert lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, None, ctypes.byref(rs), ctypes.byref(_blur(0.1))) == -1
    assert b"null row_time" in lib.gsb200_last_error()
    bad_grad = [(_lib.GsbMotionBlurGradArgs(grad_motion=None, temp=ok), b"null grad_motion"),
                (_lib.GsbMotionBlurGradArgs(grad_motion=ok, temp=None), b"null grad_motion"),
                (_lib.GsbMotionBlurGradArgs(grad_motion=ctypes.c_void_p(258), temp=ok), b"4-byte aligned"),
                (_lib.GsbMotionBlurGradArgs(grad_motion=ok, temp=ctypes.c_void_p(260)), b"16-byte aligned")]
    for g, msg in bad_grad:
        assert lib.gsb200_backward_motion_blur(ctypes.byref(bargs), None, None, None, None, None, None,
                                               ctypes.byref(_blur(0.1)), ctypes.byref(g)) == -1
        assert msg in lib.gsb200_last_error()
    assert lib.gsb200_backward_motion_blur(ctypes.byref(bargs), None, None, None, None, None, None, None,
                                           ctypes.byref(good)) == -1
    assert b"needs a motion blur" in lib.gsb200_last_error()
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for g in (None, ctypes.byref(good)):
        assert lib.gsb200_backward_motion_blur(ctypes.byref(compact), None, None, None, None, None, None,
                                               ctypes.byref(_blur(0.1)), g) == -4
        assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # valid arguments reach the usual argument checks
    assert lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, None, None, ctypes.byref(_blur(0.1))) == -1
    assert b"forward: null camera_intrinsics" in lib.gsb200_last_error()
    assert lib.gsb200_backward_motion_blur(ctypes.byref(bargs), None, None, None, None, None, None, ctypes.byref(_blur(0.1)),
                                           ctypes.byref(good)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_blur_is_exactly_the_rolling_shutter_calls():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    rs = _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(0.1, 0, 0, 0, 0, 0), row_time=fake)
    for lens in (None, ctypes.byref(_lib.GsbLensArgs(model=0)), ctypes.byref(_lib.GsbLensArgs(model=3))):
        for r in (None, ctypes.byref(rs)):
            fargs = _lib.GsbForwardArgs()
            want = lib.gsb200_forward_rolling_shutter(ctypes.byref(fargs), None, lens, r)
            want_msg = lib.gsb200_last_error()
            assert lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, lens, r, None) == want != 0
            assert lib.gsb200_last_error() == want_msg
            for args, extra in ((_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                                (_lib.GsbBackwardArgs(), (fake, fake, None, None))):
                want = lib.gsb200_backward_rolling_shutter(ctypes.byref(args), *extra, lens, r, None)
                want_msg = lib.gsb200_last_error()
                assert lib.gsb200_backward_motion_blur(ctypes.byref(args), *extra, lens, r, None, None) == want != 0
                assert lib.gsb200_last_error() == want_msg


# ------------------------------------------------------------------ Python surface
def test_motion_blur_record_and_camera_velocity():
    mb = MotionBlur((0.1, 0, 0), [0, 0.2, 0])
    assert mb.linear == (0.1, 0.0, 0.0) and mb.angular == (0.0, 0.2, 0.0) and mb.motion == (0.1, 0, 0, 0, 0.2, 0)
    for bad in (((0, 0), (0, 0, 0)), ((0, 0, math.nan), (0, 0, 0)), ((0, 0, 0), (math.inf, 0, 0))):
        with pytest.raises(ValueError):
            MotionBlur(*bad)
    m = MotionBlur.from_camera_velocity((1.0, -2.0, 0.5), (0.1, 0.0, -0.3), 1 / 50)
    assert m.linear == pytest.approx((-0.02, 0.04, -0.01)) and m.angular == pytest.approx((-0.002, 0.0, 0.006))
    with pytest.raises(ValueError, match="exposure_time"):
        MotionBlur.from_camera_velocity((0, 0, 0), (0, 0, 0), -1.0)
    assert CameraInfo(torch.eye(3), 16, 16, 0).motion_blur is None


@pytest.mark.parametrize("angle", [0.0, 0.3, 3.0])
def test_between_poses_moves_the_earlier_frame_onto_the_later_one(angle):
    """pc(tau) = exp(tau [w]x) pc0 + tau v at tau = 1 / fraction is the later frame's camera-frame point."""
    rng = np.random.default_rng(int(angle * 10))
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    T_before = np.eye(4)
    T_before[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * 0.5).as_matrix()
    T_before[:3, 3] = rng.normal(size=3)
    A = np.eye(4)
    A[:3, :3] = Rotation.from_rotvec(axis * angle).as_matrix()
    A[:3, 3] = rng.normal(size=3) * 0.3
    T_after = T_before @ np.linalg.inv(A)  # A = T_after^-1 T_before
    fraction = 0.25
    mb = MotionBlur.between_poses(torch.tensor(T_before), torch.tensor(T_after), fraction)
    m = np.array(mb.motion)
    tau = 1 / fraction
    x = rng.normal(size=(5, 3)) + np.array([0, 0, 4.0])  # scene points
    pc0 = (np.linalg.inv(T_before) @ np.c_[x, np.ones(5)].T).T[:, :3]
    R = rodrigues(torch.tensor(tau * m[3:])[None, :]).numpy()[0]
    moved = pc0 @ R.T + tau * m[:3]
    want = (np.linalg.inv(T_after) @ np.c_[x, np.ones(5)].T).T[:, :3]
    assert np.allclose(moved, want, atol=1e-9)
    with pytest.raises(ValueError, match="fraction"):
        MotionBlur.between_poses(torch.eye(4), torch.eye(4), -0.5)
    assert MotionBlur.between_poses(torch.eye(4), torch.eye(4), 0.5).motion == (0.0,) * 6


def _input(blur=True, lens=None, rolling=False):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, lens,
                    RollingShutter((0.1, 0, 0), (0, 0.02, 0)) if rolling else None,
                    MotionBlur((0.1, 0, 0), (0, 0.02, 0)) if blur else None)
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_configuration_of_the_motion_blur():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_motion_blur=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_motion_blur=True, gradient_exchange=object())
    inp = _input()
    for option in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion"):
        with pytest.raises(ValueError, match=option):
            G(Config(), **{option: True})(inp)
    op = G(Config(), differentiable_motion_blur=True)
    op.gradient_exchange = object()
    with pytest.raises(ValueError, match="gradient_exchange"):
        op(inp)
    op = G(Config(), differentiable_motion_blur=True, differentiable_rolling_shutter=True)
    with pytest.raises(ValueError, match="point_filter_3d"):
        op(inp, point_filter_3d=torch.zeros(64))
    with pytest.raises(ValueError, match="rolling_shutter_motion"):
        op(_input(rolling=True), rolling_shutter_motion=torch.zeros(6), exposure_motion=torch.zeros(6))
    for m, msg in ((torch.zeros(5), r"\(6,\)"), (torch.zeros(6, dtype=torch.float64), "float32"),
                   ([0.0] * 6, "torch.Tensor"), (torch.tensor([math.nan] + [0.0] * 5), "finite")):
        with pytest.raises(ValueError, match=msg):
            op(inp, exposure_motion=m)
    with pytest.raises(ValueError, match="without motion blur"):
        op(_input(blur=False), exposure_motion=torch.zeros(6))
    with pytest.raises(ValueError, match="differentiable_motion_blur"):
        G(Config())(inp, exposure_motion=torch.zeros(6))
    blur = op._motion_blur_args(inp.camera_info, torch.tensor([0.2, -0.01, 0.0, 0.0, 0.03, 0.0]))
    assert list(blur.motion) == pytest.approx([0.2, -0.01, 0, 0, 0.03, 0])
    assert list(G(Config())._motion_blur_args(inp.camera_info).motion) == pytest.approx([0.1, 0, 0, 0, 0.02, 0])
    assert G(Config())._motion_blur_args(_input(blur=False).camera_info) is None
    assert G(Config())._motion_blur_args(_input(lens=LensDistortion("fisheye", (0.1, 0, 0, 0)), rolling=True).camera_info) \
        is not None


def _trainer(cams, fused_step=False, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, cam, lens, rs, mb))
             for cam, lens, rs, mb in cams]
    seen = {}

    class Factory:
        gradient_exchange = kw.pop("_exchange", None)

        def __init__(self, **kwargs):
            seen.update(kwargs)

    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=Factory, fused_step=fused_step), seen


def test_trainer_configuration_of_the_motion_blur():
    a = MotionBlur((0.1, 0, 0), (0, 0.02, 0))
    b = MotionBlur((0, -0.05, 0), (0.01, 0, 0))
    rs = RollingShutter((0.05, 0, 0), (0, 0, 0))
    for rate in (-1e-3, math.nan, math.inf):
        with pytest.raises(ValueError, match="motion_blur_learning_rate"):
            _trainer([(0, None, None, a)], motion_blur_learning_rate=rate)
    with pytest.raises(ValueError, match="motion-blurred"):
        _trainer([(0, None, None, None)], motion_blur_learning_rate=1e-3)
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(pose_learning_rate=1e-3), "pose"),
                    (dict(intrinsics_learning_rate=1e-3), "intrinsics"), (dict(distortion_learning_rate=1e-3), "distortion"),
                    (dict(rolling_shutter_learning_rate=1e-3), "rolling_shutter_learning_rate"),
                    (dict(mip_filter_3d=True), "mip_filter_3d"), (dict(_exchange=object()), "gradient exchange")):
        lens = LensDistortion("opencv", (-0.1, 0, 0, 0, 0)) if "distortion" in kw else None
        with pytest.raises(ValueError, match=msg):
            _trainer([(0, lens, rs, a)], **kw)
    trainer, seen = _trainer([(0, None, None, a), (1, None, rs, b), (0, None, None, None)], motion_blur_learning_rate=1e-3)
    assert seen.get("differentiable_motion_blur") is True
    assert sorted(trainer._motion_blur) == [0, 1]
    leaf = trainer._motion_blur[0]
    assert leaf.is_leaf and leaf.requires_grad and leaf.device.type == "cpu" and leaf.dtype == torch.float32
    f32 = lambda r: MotionBlur(*(tuple(float(np.float32(v)) for v in x) for x in (r.linear, r.angular)))  # noqa: E731
    assert trainer.refined_motion_blur() == [f32(a), f32(b), None]
    with torch.no_grad():
        leaf[0] = 0.25
    assert trainer.refined_motion_blur()[0] == f32(MotionBlur((0.25, 0, 0), (0, 0.02, 0)))
    trainer, seen = _trainer([(0, None, None, a)])
    assert "differentiable_motion_blur" not in seen and trainer.refined_motion_blur() == [a]


def test_dataset_reads_the_motion_blur_record_key_and_downsampling_keeps_it(tmp_path):
    from PIL import Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    from taichi_3d_gaussian_splatting_b200.trainer import downsample_image_and_camera_info
    img = tmp_path / "a.png"
    Image.fromarray(np.zeros((32, 48, 3), np.uint8)).save(img)
    base = {"image_path": str(img), "T_pointcloud_camera": np.eye(4).tolist(),
            "camera_intrinsics": [[40.0, 0, 24.0], [0, 40.0, 16.0], [0, 0, 1]], "camera_height": 32, "camera_width": 48,
            "camera_id": 0}
    records = [dict(base), dict(base, motion_blur={"linear_velocity": [1.0, 0, 0], "angular_velocity": [0, 0.5, 0],
                                                   "exposure_time": 1 / 30},
                                rolling_shutter={"linear_velocity": [1.0, 0, 0], "angular_velocity": [0, 0.5, 0],
                                                 "readout_time": 0.02})]
    path = tmp_path / "poses.json"
    path.write_text(json.dumps(records))
    ds = ImagePoseDataset(str(path))
    assert ds[0][3].motion_blur is None
    mb = ds[1][3].motion_blur
    assert mb == MotionBlur.from_camera_velocity((1.0, 0, 0), (0, 0.5, 0), 1 / 30) and ds[1][3].rolling_shutter is not None
    for broken in ({"linear_velocity": [1.0, 0], "angular_velocity": [0, 0, 0], "exposure_time": 0.02},
                   {"linear_velocity": [1.0, 0, 0], "angular_velocity": [0, 0, 0]}):
        bad = tmp_path / "bad.json"
        bad.write_text(json.dumps([dict(base, motion_blur=broken)]))
        with pytest.raises(ValueError, match="motion_blur"):
            ImagePoseDataset(str(bad))[0]
    _, ci = downsample_image_and_camera_info(torch.zeros((3, 32, 48)), ds[1][3], 2)
    assert ci.motion_blur == mb and ci.rolling_shutter == ds[1][3].rolling_shutter
    from taichi_3d_gaussian_splatting_b200.synthetic import SyntheticScene
    sc = make_scene(16, 32, 48, 0.12, 3)
    sc.camera_info.motion_blur = mb
    assert SyntheticScene.to(sc, "cpu").camera_info.motion_blur == mb
