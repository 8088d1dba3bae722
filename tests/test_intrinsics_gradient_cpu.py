"""The camera-intrinsics gradient (``differentiable_intrinsics=True``, ``gsb200_backward_calib``) without a GPU.

The INTR instantiations of the per-point kernel (intrinsics alone, and with the pose sums in the same pass) and the
finishing kernels run under the SIMT emulator of ``tests/simt`` (the unmodified CUDA sources), on the accumulator rows of
the emulated loop A (both kernels for an image loss; the transposed one with the depth, alpha and feature terms), chained
with the emulated preprocess, sort, tile ranges and forward blend.  They are compared with torch autograd of the
multi-object float64 dense evaluator (``torch_reference_pose``) with respect to K.  Also: the combined kernel's pose
gradient, determinism, every other output bit-identical to the pose-only and default kernels', the C entry point's argument
rules, and the operator's and trainer's configuration."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth, emulated_points
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator, emulated_forward
from simt_intrinsics_helpers import build_intrinsics_emulator, emulated_points_calib
from simt_pose_helpers import build_pose_emulator, emulated_points_pose
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_pose import dense_render_objects


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                pemu=build_pose_emulator(), iemu=build_intrinsics_emulator())


def _general_K(sc):
    """The scene's K with skew, a non-zero K[1,0] and an off-centre principal point (the forward reads all six entries)."""
    K = sc.camera_info.camera_intrinsics.clone()
    K[0, 1], K[1, 0] = 2.5, -1.5
    K[0, 2] += 5.0
    K[1, 2] -= 4.0
    sc.camera_info.camera_intrinsics = K.contiguous()
    return sc


def _dense_grads(sc, feats_n, g_img, g_dep=None, g_alpha=None, extra=None, g_map=None):
    """dL/dK (3,3), dL/dq_pc, dL/dt_pc of L = <image, g_img> (+ <depth, g_dep>) (+ <alpha, g_alpha>) (+ <F, g_map>) by
    float64 autograd."""
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    K = sc.camera_info.camera_intrinsics.clone().double().requires_grad_(True)
    q = sc.q_pointcloud_camera.clone().double().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().double().requires_grad_(True)
    image, aux = dense_render_objects(sc.point_cloud.double(), torch.from_numpy(feats_n).double(), sc.point_invalid_mask,
                                      sc.point_object_id, K, q, t, H, W)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        depth, _ = differentiable_depth(aux, H, W)
        loss = loss + (depth * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    return K.grad.numpy(), q.grad.numpy(), t.grad.numpy(), aux


def _case(emus, sc, exact, band, kind, seed, transposed=True, pose=False):
    """Emulated loop A for the loss `kind`, the default, POSE and INTR per-point kernels on its rows, and the dense
    gradients.  Returns (default dense gradients, pose-only result or None, INTR result, expected dL/dK, dL/dq, dL/dt)."""
    emu, demu = emus["emu"], emus["demu"]
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g, dtype=torch.float32)
    g_dep = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "depth" else None
    g_alpha = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "alpha" else None
    extra = g_map = None
    depth = kind == "depth"
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
    default = emulated_points(emu, demu, st, accum, band, depth=depth)
    pose_only = emulated_points_pose(emu, emus["pemu"], st, accum, band, depth=depth) if pose else None
    calib = emulated_points_calib(emu, emus["iemu"], st, accum, band, depth=depth, pose=pose)
    eK, eq, et, aux = _dense_grads(sc, st.pre.feats, g_img, g_dep, g_alpha, extra, g_map)
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()  # multi-splat blending and saturated pixels
    assert np.array_equal(aux["count"].numpy(), st.count)  # the evaluator composites the same pairs
    return default, pose_only, calib, eK, eq, et


def _check(default, pose_only, calib, eK, eq, et):
    ok = grad_close(calib.gK, eK)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], (calib.gK, eK, ok)
    assert (calib.gK[2] == 0).all() and (eK[2] == 0).all()  # the forward never reads row 2
    # the INTR variants leave every other output of the per-point kernel bit-identical
    assert np.array_equal(calib.gx, default[0]) and np.array_equal(calib.gf, default[1])
    if pose_only is not None:
        for got, want in ((calib.gq, eq), (calib.gt, et)):
            ok = grad_close(got, want)
            assert ok[0], (got, want, ok)
        assert np.array_equal(calib.gq, pose_only.gq) and np.array_equal(calib.gt, pose_only.gt)


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_emulated_intrinsics_gradient_matches_dense_autograd(emus, seed, band, exact, kind, pose):
    sc = _scene(seed)
    _check(*_case(emus, sc, exact, band, kind, seed, pose=pose))


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_emulated_intrinsics_gradient_with_skew_and_off_centre_principal_point(emus, kind, pose):
    sc = _general_K(_scene(14))
    default, pose_only, calib, eK, eq, et = _case(emus, sc, False, 3, kind, 14, pose=pose)
    assert (np.abs(eK[:2]) > 0).all()  # every entry of rows 0 and 1 gets a gradient
    _check(default, pose_only, calib, eK, eq, et)


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_emulated_intrinsics_gradient_of_interleaved_objects(emus, kind, pose):
    """Three objects whose points alternate row by row: every warp holds points of all three, and K is shared."""
    sc = _scene(17, objects=3)
    _check(*_case(emus, sc, False, 3, kind, 17, pose=pose))


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("exact", [True, False])
def test_emulated_intrinsics_gradient_under_the_butterfly_loop_a(emus, exact, pose):
    sc = _general_K(_scene(11, objects=2))
    _check(*_case(emus, sc, exact, 3, "image", 11, transposed=False, pose=pose))


def test_intrinsics_gradient_is_deterministic_and_sums_the_partials_in_block_order(emus):
    sc = _scene(12, n=1500, objects=2)  # 12 CTAs of partial rows
    emu, demu = emus["emu"], emus["demu"]
    st = emulated_forward(emu, sc, exact=False)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(5)).numpy()
    _, _, accum, _ = emulated_backward_depth(emu, demu, st, g_img, None)
    for pose in (False, True):
        a = emulated_points_calib(emu, emus["iemu"], st, accum, pose=pose)
        b = emulated_points_calib(emu, emus["iemu"], st, accum, pose=pose)
        assert a.blocks == 12
        for k in ("gx", "gf", "gK", "gq", "gt", "partials"):
            assert (getattr(a, k) is None and getattr(b, k) is None) or np.array_equal(getattr(a, k), getattr(b, k)), k
        # every partial row is written, and the finishing kernel's result is their sum (up to the order's rounding)
        assert np.isfinite(a.partials).all() and not (a.partials == 7.0).any()
        ok = grad_close(a.gK[:2].reshape(-1), a.partials.astype(np.float64).sum(0), rtol=1e-5)
        assert ok[0], ok
    # the combined pass gives the intrinsics gradient of the intrinsics-only pass, bit for bit
    assert np.array_equal(emulated_points_calib(emu, emus["iemu"], st, accum, pose=True).gK, a.gK)


# ------------------------------------------------------------------ C ABI
def _args(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1):
    return _lib.GsbBackwardArgs(flags=flags, num_objects=num_objects)


def test_c_entry_point_checks_its_arguments_without_a_gpu():
    lib = _lib.load()
    for name in ("gsb200_backward_calib", "gsb200_intrinsics_grad_temp_bytes"):
        assert hasattr(lib, name) and name in _lib.EXPORTS
    assert lib.gsb200_intrinsics_grad_temp_bytes() == 2048 * 6 * 4
    fake = ctypes.c_void_p(256)  # never dereferenced: the checks come before any CUDA call
    full = dict(grad_camera_intrinsics=fake, temp=fake)
    for missing in full:
        intr = _lib.GsbIntrinsicsGradArgs(**{k: (None if k == missing else v) for k, v in full.items()})
        assert lib.gsb200_backward_calib(ctypes.byref(_args()), None, None, None, None, None, ctypes.byref(intr)) == -1
        assert b"backward_calib: null" in lib.gsb200_last_error()
    intr = _lib.GsbIntrinsicsGradArgs(**dict(full, temp=ctypes.c_void_p(264)))
    assert lib.gsb200_backward_calib(ctypes.byref(_args()), None, None, None, None, None, ctypes.byref(intr)) == -1
    assert b"16-byte aligned" in lib.gsb200_last_error()
    intr = _lib.GsbIntrinsicsGradArgs(**full)
    compact = _args(_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS)
    assert lib.gsb200_backward_calib(ctypes.byref(compact), None, None, None, None, None, ctypes.byref(intr)) == -4
    assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # the pose rules still apply next to the intrinsics
    pose = _lib.GsbPoseGradArgs(q_pointcloud_camera=fake, grad_q_pointcloud_camera=fake, grad_t_pointcloud_camera=fake,
                                temp=fake)
    assert lib.gsb200_backward_calib(ctypes.byref(_args(num_objects=65)), None, None, None, None, ctypes.byref(pose),
                                     ctypes.byref(intr)) == -4
    assert b"GSB_POSE_MAX_OBJECTS" in lib.gsb200_last_error()
    # the depth, alpha and feature terms keep their requirement of the transposed kernel; an image loss does not have it
    assert lib.gsb200_backward_calib(ctypes.byref(_args(0)), fake, fake, None, None, None, ctypes.byref(intr)) == -4
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    assert lib.gsb200_backward_calib(ctypes.byref(_args(0)), None, None, None, None, None, ctypes.byref(intr)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()
    assert lib.gsb200_backward_calib(None, None, None, None, None, None, ctypes.byref(intr)) == -1


def test_null_intrinsics_is_exactly_backward_pose():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ext = _lib.GsbExtraFeatureArgs(channels=0, features=fake, grad_rasterized=fake, grad_features=fake)
    pose = _lib.GsbPoseGradArgs(q_pointcloud_camera=fake, grad_q_pointcloud_camera=None, grad_t_pointcloud_camera=fake,
                                temp=fake)
    cases = [(_args(), (None, None, None, None, None)), (_args(), (fake, None, None, None, None)),
             (_args(0), (fake, fake, None, None, None)), (_args(), (None, None, None, ctypes.byref(ext), None)),
             (_args(), (None, None, None, None, ctypes.byref(pose))), (_args(num_objects=0), (None, None, None, None, None))]
    for args, extra in cases:
        want = lib.gsb200_backward_pose(ctypes.byref(args), *extra)
        want_msg = lib.gsb200_last_error()
        assert lib.gsb200_backward_calib(ctypes.byref(args), *extra, None) == want != 0
        assert lib.gsb200_last_error() == want_msg


def test_abi_size_of_the_intrinsics_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 10)()
    lib.gsb200_abi_sizes_ext(sizes, 10)
    assert sizes[9] == ctypes.sizeof(_lib.GsbIntrinsicsGradArgs) == 16
    first9 = (ctypes.c_int64 * 9)()
    lib.gsb200_abi_sizes_ext(first9, 9)
    assert list(first9) == list(sizes)[:9]


# ------------------------------------------------------------------ operator and trainer configuration
def test_operator_option_and_its_constructor_checks():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    param = inspect.signature(G.__init__).parameters["differentiable_intrinsics"]
    assert param.kind is inspect.Parameter.KEYWORD_ONLY and param.default is False
    assert G(Config()).differentiable_intrinsics is False
    assert G(Config(), differentiable_intrinsics=True).differentiable_intrinsics is True
    assert G(Config(), backward_impl="butterfly", differentiable_intrinsics=True).differentiable_intrinsics is True
    both = G(Config(), differentiable_intrinsics=True, differentiable_pose=True, differentiable_depth=True,
             differentiable_alpha=True)
    assert both.differentiable_intrinsics and both.differentiable_pose
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_intrinsics=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_intrinsics=True, gradient_exchange=object())
    G(Config(rgb_only=True))  # unchanged without the option
    G(Config(), gradient_exchange=object())


def _trainer(intr_lr, pose_lr=0.0, **kw):
    from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 32, 48))
    ci = sc.camera_info
    other = CameraInfo(camera_intrinsics=ci.camera_intrinsics.clone(), camera_height=32, camera_width=48, camera_id=5)
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci)] * 2 + \
        [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera, other)]
    seen = {}

    def factory(**kwargs):
        seen.update(kwargs)
        return lambda *a, **k: None

    cfg = T.TrainConfig(intrinsics_learning_rate=intr_lr, pose_learning_rate=pose_lr)
    trainer = T(cfg, scene, views, rasterisation_factory=factory, **kw)
    return trainer, seen


def test_trainer_intrinsics_configuration():
    trainer, seen = _trainer(0.0)
    assert "differentiable_intrinsics" not in seen  # injected factories get the flag only when it is on
    assert [torch.equal(K, v[3].camera_intrinsics) for K, v in zip(trainer.refined_intrinsics(), trainer.train_views)] \
        == [True] * 3
    trainer, seen = _trainer(1e-3)
    assert seen["differentiable_intrinsics"] is True and "differentiable_pose" not in seen
    corr = trainer._intrinsics
    assert sorted(corr) == [0, 5]  # one correction per camera_id
    for p in corr.values():
        assert p.is_leaf and p.requires_grad and p.shape == (4,) and torch.equal(p, torch.zeros(4))
    # the K of a view: its own full-resolution K with the camera's correction, scaled by the downsample factor
    with torch.no_grad():
        corr[0].copy_(torch.tensor([0.1, -0.05, 0.02, -0.03]))
    K0 = trainer.train_views[0][3].camera_intrinsics
    want = K0.clone()
    want[0, 0] *= float(np.exp(0.1))
    want[1, 1] *= float(np.exp(-0.05))
    want[0, 2] += 0.02 * 48
    want[1, 2] += -0.03 * 32
    assert torch.allclose(trainer.refined_intrinsics()[0], want, rtol=1e-6)
    assert torch.equal(trainer.refined_intrinsics()[2], trainer.train_views[2][3].camera_intrinsics)  # camera 5 untouched
    K4 = trainer._intrinsics_of(0, 4)
    assert K4.requires_grad and torch.allclose(K4.detach()[:2], want[:2] / 4, rtol=1e-6)
    K4.sum().backward()
    assert corr[0].grad is not None and corr[5].grad is None
    trainer, seen = _trainer(1e-3, pose_lr=1e-3)  # combines with pose refinement
    assert seen["differentiable_intrinsics"] is True and seen["differentiable_pose"] is True
    with pytest.raises(ValueError, match="fused_step"):
        _trainer(1e-3, fused_step=True)
    for bad in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="intrinsics_learning_rate"):
            _trainer(bad)
