"""Pose and intrinsics gradients through a lens (``gsb200_backward_lens_calib``; ``differentiable_pose`` and
``differentiable_intrinsics`` on an OpenCV or fisheye view, with or without ``differentiable_distortion``) without a GPU.

* The emulated per-point kernel (the unmodified CUDA sources under the SIMT emulator of ``tests/simt``) on emulated loop-A rows
  against torch autograd of the dense float64 lens evaluator with q_pc, t_pc, K and k as leaves, for image, depth, alpha and
  feature-map losses, both lenses and every combination of the camera gradients; three objects sharing warps; the butterfly
  loop A; the pinhole limit against ``gsb200_backward_calib``'s kernel; determinism; every other output bit-identical to the
  LENS kernel's, and the coefficient sums to the LGRAD kernel's.
* The C entry point's argument rules, and the operator's and trainer's configuration."""
import ctypes
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator
from simt_intrinsics_helpers import build_intrinsics_emulator, emulated_points_calib
from simt_lens_calib_helpers import build_lens_calib_emulator, emulated_points_lens_calib
from simt_lens_grad_helpers import build_lens_grad_emulator, emulated_points_lens_grad
from simt_lens_helpers import build_lens_emulator, emulated_forward_lens, emulated_points_lens
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_lens_grad import dense_render_lens_k

LENSES = {
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
CAMERA_GRADS = {  # (pose, intrinsics, coefficients)
    "pose": (True, False, False),
    "intrinsics": (False, True, False),
    "pose+intrinsics": (True, True, False),
    "pose+intrinsics+coefficients": (True, True, True),
}


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator(), gemu=build_lens_grad_emulator(), cemu=build_lens_calib_emulator(),
                iemu=build_intrinsics_emulator())


def _accum(emus, st, kind, seed, band=3, transposed=True):
    """Emulated loop A for the loss `kind` on the lens state `st`; returns (rows, the loss's upstream tensors)."""
    emu, demu = emus["emu"], emus["demu"]
    sc = st.scene
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
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
    return accum, (g_img, g_dep, g_alpha, extra, g_map)


def _dense_grads(st, upstream):
    """dL/dq_pc, dL/dt_pc, dL/dK, dL/dk of the loss by float64 autograd of the dense lens evaluator."""
    sc = st.scene
    model, k = st.lens
    g_img, g_dep, g_alpha, extra, g_map = upstream
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    q = sc.q_pointcloud_camera.clone().double().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().double().requires_grad_(True)
    K = sc.camera_info.camera_intrinsics.clone().double().requires_grad_(True)
    kk = torch.tensor(k, dtype=torch.float64, requires_grad=True)
    image, aux = dense_render_lens_k(sc.point_cloud.double(), torch.from_numpy(st.pre.feats).double(), sc.point_invalid_mask,
                                     sc.point_object_id, K, q, t, H, W, model, kk)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)  # the evaluator composites the same pairs
    return q.grad.numpy(), t.grad.numpy(), K.grad.numpy(), kk.grad.numpy()


def _close(got, want):
    ok = grad_close(got, want)  # the camera gradients' criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], (got, want, ok)


def _check(res, grads, expected, model, lens_only, lgrad_only):
    pose, intr, lgrad = grads
    eq, et, eK, ek = expected
    if pose:
        _close(res.gq, eq)
        _close(res.gt, et)
    if intr:
        _close(res.gK, eK)
        assert (res.gK[2] == 0).all() and (eK[2] == 0).all()
    if lgrad:
        n = 5 if model == "opencv" else 4
        scale = np.abs(ek).max()
        assert (np.abs(res.gk[:n] - ek) <= 2e-3 * np.abs(ek) + 2e-4 * scale).all(), (res.gk, ek)
        assert (res.gk[n:] == 0).all()
        # the coefficient sums of the joint kernel are the LGRAD kernel's
        assert np.array_equal(res.gk, lgrad_only.gk) and np.array_equal(res.lens_partials, lgrad_only.partials)
    # every other output is the LENS kernel's, bit for bit
    assert np.array_equal(res.gx, lens_only[0]) and np.array_equal(res.gf, lens_only[1])


def _run(emus, lens, kind, seed, grads, objects=1, transposed=True, band=3):
    model, k = LENSES[lens]
    sc = _scene(seed, objects=objects)
    st = emulated_forward_lens(emus["emu"], emus["lemu"], sc, model, k, exact=False)
    accum, upstream = _accum(emus, st, kind, seed, band, transposed)
    pose, intr, lgrad = grads
    depth = kind == "depth"
    res = emulated_points_lens_calib(emus["emu"], emus["cemu"], st, accum, band, depth=depth, pose=pose, intr=intr,
                                     lgrad=lgrad)
    lens_only = emulated_points_lens(emus["emu"], emus["lemu"], st, accum, band, depth=depth)
    lgrad_only = emulated_points_lens_grad(emus["emu"], emus["gemu"], st, accum, band, depth=depth) if lgrad else None
    return st, accum, res, lens_only, lgrad_only, _dense_grads(st, upstream)


@pytest.mark.parametrize("grads", list(CAMERA_GRADS))
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_camera_gradients_through_a_lens_match_dense_autograd(emus, lens, kind, grads):
    _, _, res, lens_only, lgrad_only, expected = _run(emus, lens, kind, 51, CAMERA_GRADS[grads])
    _check(res, CAMERA_GRADS[grads], expected, LENSES[lens][0], lens_only, lgrad_only)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_camera_gradients_with_three_objects_sharing_warps(emus, lens):
    grads = CAMERA_GRADS["pose+intrinsics+coefficients"]
    st, _, res, lens_only, lgrad_only, expected = _run(emus, lens, "image", 53, grads, objects=3)
    obj = st.scene.point_object_id.numpy()
    kept = st.pre.point_offset >= 0
    assert len(set(obj[:32][kept[:32]].tolist())) == 3  # one warp holds in-camera points of all three objects
    assert res.gq.shape == (3, 4) and (np.abs(res.gq).sum(1) > 0).all()
    _check(res, grads, expected, LENSES[lens][0], lens_only, lgrad_only)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_camera_gradients_under_the_butterfly_loop_a(emus, lens):
    grads = CAMERA_GRADS["pose+intrinsics+coefficients"]
    _, _, res, lens_only, lgrad_only, expected = _run(emus, lens, "image", 55, grads, transposed=False, band=1)
    _check(res, grads, expected, LENSES[lens][0], lens_only, lgrad_only)


@pytest.mark.parametrize("kind", ["image", "depth"])
def test_pinhole_limit_matches_the_calib_kernel(emus, kind):
    """An opencv lens with all coefficients 0 is the pinhole: the pose and intrinsics gradients are gsb200_backward_calib's to
    float rounding, and every other output is bit-identical."""
    sc = _scene(57)
    st = emulated_forward_lens(emus["emu"], emus["lemu"], sc, "opencv", (0.0,) * 5, exact=False)
    accum, _ = _accum(emus, st, kind, 57)
    depth = kind == "depth"
    res = emulated_points_lens_calib(emus["emu"], emus["cemu"], st, accum, depth=depth, pose=True, intr=True)
    calib = emulated_points_calib(emus["emu"], emus["iemu"], st, accum, depth=depth, pose=True)
    for got, want in ((res.gq, calib.gq), (res.gt, calib.gt), (res.gK, calib.gK)):
        assert np.allclose(got, want, rtol=1e-5, atol=1e-6 * np.abs(want).max()), (got, want)
    assert np.array_equal(res.gx, calib.gx) and np.array_equal(res.gf, calib.gf)


@pytest.mark.parametrize("grads", list(CAMERA_GRADS))
def test_camera_gradients_are_deterministic(emus, grads):
    pose, intr, lgrad = CAMERA_GRADS[grads]
    st, accum, res, _, _, _ = _run(emus, "fisheye", "depth", 59, CAMERA_GRADS[grads])
    again = emulated_points_lens_calib(emus["emu"], emus["cemu"], st, accum, depth=True, pose=pose, intr=intr, lgrad=lgrad)
    assert res.blocks == again.blocks == min(math.ceil(st.pre.point_offset.shape[0] / 128), 2048)
    for name in ("gx", "gf", "gq", "gt", "gK", "gk", "pose_partials", "intr_partials", "lens_partials"):
        a, b = getattr(res, name), getattr(again, name)
        assert (a is None and b is None) or np.array_equal(a, b), name
    if intr:  # the finishing kernel's sum of the per-CTA rows
        got = res.gK[:2].reshape(-1)
        assert np.allclose(res.intr_partials.astype(np.float64).sum(0), got, rtol=1e-5, atol=1e-6 * np.abs(got).max())


# ------------------------------------------------------------------ C ABI
def _lens(model, *co):
    return _lib.GsbLensArgs(model=model, coefficients=(ctypes.c_float * 5)(*(list(co) + [0.0] * (5 - len(co)))))


def test_c_entry_point_checks_its_arguments_before_any_cuda_call():
    lib = _lib.load()
    assert hasattr(lib, "gsb200_backward_lens_calib") and "gsb200_backward_lens_calib" in _lib.EXPORTS
    assert lib.gsb200_backward_lens_calib.argtypes is not None
    ok = ctypes.c_void_p(256)
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    pose = _lib.GsbPoseGradArgs(q_pointcloud_camera=ok, grad_q_pointcloud_camera=ok, grad_t_pointcloud_camera=ok, temp=ok)
    intr = _lib.GsbIntrinsicsGradArgs(grad_camera_intrinsics=ok, temp=ok)
    lg = _lib.GsbLensGradArgs(grad_coefficients=ok, temp=ok)
    call = lambda args, lens, lgrad, p, i: lib.gsb200_backward_lens_calib(  # noqa: E731
        ctypes.byref(args), None, None, None, None, ctypes.byref(lens) if lens is not None else None,
        ctypes.byref(lgrad) if lgrad is not None else None, ctypes.byref(p) if p is not None else None,
        ctypes.byref(i) if i is not None else None)
    # args point at nothing the call could use: these checks come first
    bad = [(bargs, None, None, pose, None, -1, b"need an opencv or fisheye lens"),
           (bargs, _lens(0), None, None, intr, -1, b"need an opencv or fisheye lens"),
           (bargs, _lens(1, float("nan")), None, pose, None, -1, b"not finite"),
           (bargs, _lens(7), None, pose, None, -1, b"unknown lens model"),
           (bargs, _lens(1, 0.1), _lib.GsbLensGradArgs(grad_coefficients=None, temp=ok), pose, None, -1,
            b"null grad_coefficients"),
           (bargs, _lens(2, 0.1), _lib.GsbLensGradArgs(grad_coefficients=ok, temp=ctypes.c_void_p(260)), None, intr, -1,
            b"16-byte aligned"),
           (bargs, _lens(1, 0.1), None, _lib.GsbPoseGradArgs(q_pointcloud_camera=None, grad_q_pointcloud_camera=ok,
                                                             grad_t_pointcloud_camera=ok, temp=ok), None, -1, b"null q"),
           (bargs, _lens(1, 0.1), None, None, _lib.GsbIntrinsicsGradArgs(grad_camera_intrinsics=ok, temp=None), -1,
            b"null grad_camera_intrinsics"),
           (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=65), _lens(1, 0.1), None, pose, None,
            -4, b"GSB_POSE_MAX_OBJECTS"),
           (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=0), _lens(2, 0.1), lg, pose, intr,
            -1, b"num_objects >= 1")]
    for args, lens, lgrad, p, i, rc, msg in bad:
        assert call(args, lens, lgrad, p, i) == rc, msg
        assert msg in lib.gsb200_last_error(), (msg, lib.gsb200_last_error())
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for model in (1, 2):
        for lgrad, p, i in ((None, pose, None), (None, None, intr), (lg, pose, intr)):
            assert call(compact, _lens(model, 0.1), lgrad, p, i) == -4
            assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # valid arguments reach the usual argument checks
    for lgrad, p, i in ((None, pose, None), (None, None, intr), (lg, pose, intr)):
        assert call(bargs, _lens(1, 0.1), lgrad, p, i) == -1
        assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_pose_and_intrinsics_is_exactly_backward_lens_grad():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ext = _lib.GsbExtraFeatureArgs(channels=0, features=fake, grad_rasterized=fake, grad_features=fake)
    lgs = (None, _lib.GsbLensGradArgs(grad_coefficients=fake, temp=fake), _lib.GsbLensGradArgs(grad_coefficients=None, temp=fake))
    for lens in (None, _lens(0), _lens(1, 0.1), _lens(2, 0.1), _lens(3)):
        for lg in lgs:
            for args, extra in ((_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                                (_lib.GsbBackwardArgs(), (fake, fake, None, None)),
                                (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_COMPACT_GRADS), (None, None, None, ctypes.byref(ext)))):
                lens_p = ctypes.byref(lens) if lens is not None else None
                lg_p = ctypes.byref(lg) if lg is not None else None
                want = lib.gsb200_backward_lens_grad(ctypes.byref(args), *extra, lens_p, lg_p)
                want_msg = lib.gsb200_last_error()
                assert lib.gsb200_backward_lens_calib(ctypes.byref(args), *extra, lens_p, lg_p, None, None) == want != 0
                assert lib.gsb200_last_error() == want_msg


# ------------------------------------------------------------------ Python surface
def _input(distortion=LensDistortion("fisheye", (0.1, 0, 0, 0)), **camera):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, distortion, **camera)
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


LENS_GRAD_OPTIONS = (dict(differentiable_pose=True), dict(differentiable_intrinsics=True),
                     dict(differentiable_pose=True, differentiable_intrinsics=True),
                     dict(differentiable_pose=True, differentiable_intrinsics=True, differentiable_distortion=True))


def test_operator_takes_pose_and_intrinsics_through_a_lens_only_when_opted_in():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    for distortion in (LensDistortion("fisheye", (0.1, 0, 0, 0)), LensDistortion("opencv", (-0.2, 0.01, 0, 0, 0))):
        ci = _input(distortion).camera_info
        for kw in LENS_GRAD_OPTIONS:
            # off (the default): a lens keeps refusing the camera gradients, before any device work
            with pytest.raises(ValueError, match="camera_gradients_through_lens"):
                G(Config(), **kw)._lens_args(ci)
            # on: the checks pass and the lens is the camera's
            lens = G(Config(), camera_gradients_through_lens=True, **kw)._lens_args(ci)
            assert lens.model == (_lib.GSB_LENS_FISHEYE if distortion.model == "fisheye" else _lib.GSB_LENS_OPENCV)
            want = list(distortion.coefficients) + [0] * (5 - len(distortion.coefficients))
            assert list(lens.coefficients) == pytest.approx(want)
    # the option alone changes nothing: a lens without camera gradients, a pinhole view
    assert G(Config(), camera_gradients_through_lens=True)._lens_args(_input().camera_info).model == _lib.GSB_LENS_FISHEYE
    assert G(Config(), camera_gradients_through_lens=True)._lens_args(make_scene(64, 32, 48, 0.12, 3).camera_info) is None
    # with the coefficients as an input, K fills its slot only under differentiable_intrinsics
    import inspect
    assert "camera_info.camera_intrinsics if self.differentiable_intrinsics else None, lens_coefficients" in \
        inspect.getsource(G.forward)


def test_operator_keeps_the_other_refusals_with_camera_gradients_through_a_lens():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    from taichi_3d_gaussian_splatting_b200.Camera import Defocus, MotionBlur, RollingShutter
    Config = G.GaussianPointCloudRasterisationConfig
    for kw in (dict(differentiable_pose=True), dict(differentiable_intrinsics=True)):
        op = G(Config(), camera_gradients_through_lens=True, **kw)
        for camera in (dict(rolling_shutter=RollingShutter((0.01, 0, 0), (0, 0.01, 0))),
                       dict(motion_blur=MotionBlur((0.01, 0, 0), (0, 0.01, 0))), dict(defocus=Defocus(0.01, 0.5))):
            with pytest.raises(ValueError, match="differentiable_"):
                op(_input(**camera))
        with pytest.raises(ValueError, match="point_filter_3d"):
            op(_input(), point_filter_3d=torch.zeros(64))
        with pytest.raises(ValueError, match="equirectangular|differentiable_"):
            op(_input(LensDistortion("equirectangular", ())))
        with pytest.raises(ValueError, match="gradient_exchange"):
            G(Config(), gradient_exchange=object(), camera_gradients_through_lens=True, **kw)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), gradient_exchange=object(), camera_gradients_through_lens=True)(_input())
    # the coefficients' own checks come first with the joint options too
    joint = G(Config(), camera_gradients_through_lens=True, **LENS_GRAD_OPTIONS[-1])
    with pytest.raises(ValueError, match="4"):
        joint(_input(), lens_coefficients=torch.zeros(5))
    lens = joint._lens_args(_input().camera_info, torch.tensor([0.2, -0.01, 0.0, 0.0]))
    assert list(lens.coefficients) == pytest.approx([0.2, -0.01, 0, 0, 0])


def _lens_trainer(lenses, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, cam, lens))
             for cam, lens in lenses]
    seen = {}
    factory = lambda **kwargs: seen.update(kwargs) or (lambda *a, **k: None)  # noqa: E731
    fused = kw.pop("fused_step", False)
    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=factory, fused_step=fused), seen


def test_trainer_refines_cameras_through_a_lens_only_when_opted_in():
    lens = LensDistortion("opencv", (-0.1, 0.01, 0, 0, 0))
    for kw, flag in ((dict(pose_learning_rate=1e-3), "differentiable_pose"),
                     (dict(intrinsics_learning_rate=1e-3), "differentiable_intrinsics")):
        with pytest.raises(ValueError, match="camera_refinement_through_lens"):  # off: the refusal stays
            _lens_trainer([(0, lens)], **kw)
        with pytest.raises(ValueError, match="camera_refinement_through_lens"):
            _lens_trainer([(0, lens)], distortion_learning_rate=1e-3, **kw)
        _, seen = _lens_trainer([(0, lens)], camera_refinement_through_lens=True, **kw)
        assert seen.get(flag) is True and seen.get("camera_gradients_through_lens") is True
        # a pinhole training set needs no option, and the operator gets none
        _, seen = _lens_trainer([(0, None)], camera_refinement_through_lens=True, **kw)
        assert seen.get(flag) is True and "camera_gradients_through_lens" not in seen
    # the option without pose or intrinsics refinement changes nothing
    _, seen = _lens_trainer([(0, lens)], camera_refinement_through_lens=True, distortion_learning_rate=1e-3)
    assert seen.get("differentiable_distortion") is True and "camera_gradients_through_lens" not in seen
    # fused_step and the 3D filter with camera refinement keep raising
    with pytest.raises(ValueError, match="fused_step"):
        _lens_trainer([(0, lens)], fused_step=True, camera_refinement_through_lens=True)
    with pytest.raises(ValueError, match="mip_filter_3d"):
        _lens_trainer([(0, lens)], mip_filter_3d=True, camera_refinement_through_lens=True, pose_learning_rate=1e-3)


def test_trainer_joint_self_calibration_configuration():
    """Pose, intrinsics and lens refinement together: per-view poses (view 0 the gauge), K per camera_id, the lens per
    camera_id; the camera rebuilt each step keeps the lens."""
    import dataclasses
    a = LensDistortion("opencv", (-0.1, 0.01, 0, 0, 0))
    fisheye = LensDistortion("fisheye", (0.05, 0, 0, 0))
    kw = dict(pose_learning_rate=1e-3, intrinsics_learning_rate=1e-3, distortion_learning_rate=1e-3,
              camera_refinement_through_lens=True)
    trainer, seen = _lens_trainer([(0, a), (1, fisheye), (0, a)], **kw)
    assert all(seen.get(f) is True for f in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion",
                                             "camera_gradients_through_lens"))
    assert sorted(trainer._intrinsics) == [0, 1] and sorted(trainer._distortion) == [0, 1]
    assert trainer._poses[0][0] is trainer.train_views[0][1]  # view 0 is the gauge
    assert all(q.is_leaf and q.requires_grad for q, _ in trainer._poses[1:])
    with torch.no_grad():
        trainer._intrinsics[1][0] = math.log(1.02)
        trainer._distortion[1][0] = 0.07
    K1 = trainer.refined_intrinsics()[1]
    assert float(K1[0, 0]) == pytest.approx(1.02 * float(trainer.train_views[1][3].camera_intrinsics[0, 0]), rel=1e-6)
    assert trainer.refined_distortion()[1].coefficients[0] == pytest.approx(0.07)
    # the per-step camera: the refined K with the view's lens
    _, _, _, ci, _ = trainer._view(1, 1)
    ci = dataclasses.replace(ci, camera_intrinsics=trainer._intrinsics_of(1, 1))
    assert ci.distortion == fisheye and torch.allclose(ci.camera_intrinsics, K1)
