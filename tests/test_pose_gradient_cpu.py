"""The camera-pose gradient (``differentiable_pose=True``, ``gsb200_backward_pose``) without a GPU.

The POSE instantiation of the per-point kernel and the per-object finishing kernel run under the SIMT emulator of
``tests/simt`` (the unmodified CUDA sources), on the accumulator rows of the emulated loop A (both kernels for an image
loss; the transposed one with the depth, alpha and feature terms), chained with the emulated preprocess, sort, tile ranges
and forward blend.  They are compared with torch autograd of the multi-object float64 dense evaluator
(``torch_reference_pose``) with respect to (q_pointcloud_camera, t_pointcloud_camera), taken through the pose kernel's map.
Also: determinism, the POSE variant leaves every other output bit-identical, the C entry point's argument rules, and the
operator's and trainer's configuration errors."""
import ctypes
import inspect
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth, emulated_points
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator, c, emulated_forward
from simt_pose_helpers import build_pose_emulator, emulated_points_pose
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_pose import dense_render_objects


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                pemu=build_pose_emulator())


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, objects=1):
    """The scenes of test_depth_gradient_cpu.  With objects > 1 the scene rows cycle through the objects, so the points of
    every warp belong to several objects, and the other objects get their own poses (one with a non-unit q)."""
    sc = make_scene(n, h, w, sigma, seed, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    if objects > 1:
        sc.point_object_id = (torch.arange(n) % objects).to(torch.int32)
        qs, ts = [sc.q_pointcloud_camera[0]], [sc.t_pointcloud_camera[0]]
        for k in range(1, objects):
            a = math.radians(3.0 * k) / 2
            q = torch.tensor([math.sin(a) * 0.6, math.sin(a) * 0.8, 0.0, math.cos(a)]) * (1.0 + 0.03 * k)
            qs.append(q)
            ts.append(torch.tensor([0.15 * k, -0.1 * k, 0.2 * k]))
        sc.q_pointcloud_camera = torch.stack(qs).float().contiguous()
        sc.t_pointcloud_camera = torch.stack(ts).float().contiguous()
    return sc


def _dense_pose_grads(sc, feats_n, g_img, g_dep=None, g_alpha=None, extra=None, g_map=None):
    """dL/dq_pc, dL/dt_pc of L = <image, g_img> (+ <depth, g_dep>) (+ <alpha, g_alpha>) (+ <F, g_map>) by float64 autograd."""
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    q = sc.q_pointcloud_camera.clone().double().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().double().requires_grad_(True)
    image, aux = dense_render_objects(sc.point_cloud.double(), torch.from_numpy(feats_n).double(), sc.point_invalid_mask,
                                      sc.point_object_id, sc.camera_info.camera_intrinsics, q, t, H, W)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        depth, _ = differentiable_depth(aux, H, W)
        loss = loss + (depth * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    return q.grad.numpy(), t.grad.numpy(), aux


def _loop_a_image(emu, st, g_img, transposed):
    """Loop A for an image loss alone (butterfly or transposed kernel): the accumulator rows."""
    pre, M = st.pre, st.M
    H, W = pre.H, pre.W
    accum, mag = np.zeros((max(M, 1), 12), np.float32), np.zeros((H, W, 2), np.float32)
    g = np.ascontiguousarray(g_img, dtype=np.float32)
    if st.K:
        emu.emu_blend_backward(int(transposed), int(st.exact), 1, H, W, c(st.start), c(st.end), c(st.sorted_vals),
                               c(pre.records), c(g), c(st.acc_alpha), c(st.last_effective), c(accum), c(mag))
    return accum[:M].copy()


def _case(emus, sc, exact, band, kind, seed, transposed=True):
    """Emulated loop A for the loss `kind`, the default per-point kernel and the POSE one on its rows, and the dense
    gradients.  Returns (default dense gradients, POSE result, expected dL/dq, dL/dt)."""
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
    pose = emulated_points_pose(emu, emus["pemu"], st, accum, band, depth=depth)
    eq, et, aux = _dense_pose_grads(sc, st.pre.feats, g_img, g_dep, g_alpha, extra, g_map)
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()  # multi-splat blending and saturated pixels
    assert np.array_equal(aux["count"].numpy(), st.count)  # the evaluator composites the same pairs
    return default, pose, eq, et


def _assert_pose_close(pose, eq, et):
    for got, want in ((pose.gq, eq), (pose.gt, et)):
        ok = grad_close(got, want)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
        assert ok[0], (got, want, ok)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_emulated_pose_gradient_matches_dense_autograd(emus, seed, band, exact, kind):
    sc = _scene(seed)
    default, pose, eq, et = _case(emus, sc, exact, band, kind, seed)
    _assert_pose_close(pose, eq, et)
    # the POSE variant leaves every other output of the per-point kernel bit-identical
    assert np.array_equal(pose.gx, default[0]) and np.array_equal(pose.gf, default[1])
    # one object, unit q: dL/dt_pc = -sum_i dL/dxyz_i (translating the camera = translating every point the other way)
    ok = grad_close(pose.gt[0], -default[0].astype(np.float64).sum(0))
    assert ok[0], ok


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_emulated_pose_gradient_of_interleaved_objects(emus, kind):
    """Three objects whose points alternate row by row: every warp holds points of all three."""
    sc = _scene(17, objects=3)
    default, pose, eq, et = _case(emus, sc, False, 3, kind, 17)
    assert np.abs(eq).min(axis=1).max() > 0 and (np.abs(et).max(axis=1) > 0).all()  # every object is seen
    _assert_pose_close(pose, eq, et)
    assert np.array_equal(pose.gx, default[0]) and np.array_equal(pose.gf, default[1])


@pytest.mark.parametrize("exact", [True, False])
def test_emulated_pose_gradient_under_the_butterfly_loop_a(emus, exact):
    sc = _scene(11, objects=2)
    default, pose, eq, et = _case(emus, sc, exact, 3, "image", 11, transposed=False)
    _assert_pose_close(pose, eq, et)
    assert np.array_equal(pose.gx, default[0]) and np.array_equal(pose.gf, default[1])


def test_pose_gradient_is_deterministic_and_sums_the_partials_in_block_order(emus):
    sc = _scene(12, n=1500, objects=2)  # 12 CTAs of partial rows
    emu, demu = emus["emu"], emus["demu"]
    st = emulated_forward(emu, sc, exact=False)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(5)).numpy()
    _, _, accum, _ = emulated_backward_depth(emu, demu, st, g_img, None)
    a = emulated_points_pose(emu, emus["pemu"], st, accum)
    b = emulated_points_pose(emu, emus["pemu"], st, accum)
    assert a.blocks == 12
    for k in ("gx", "gf", "gq", "gt", "partials"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    # the finishing kernel's input: the per-CTA rows add up (in any order, up to rounding) to the per-object sums of the
    # points' 12 values, and no row is left unwritten
    assert np.isfinite(a.partials).all() and not (a.partials == 7.0).any()


# ------------------------------------------------------------------ C ABI
def _args(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1):
    return _lib.GsbBackwardArgs(flags=flags, num_objects=num_objects)


def test_c_entry_point_checks_its_arguments_without_a_gpu():
    lib = _lib.load()
    for name in ("gsb200_backward_pose", "gsb200_pose_grad_temp_bytes"):
        assert hasattr(lib, name) and name in _lib.EXPORTS
    assert lib.gsb200_pose_grad_temp_bytes(1) == 2048 * 12 * 4
    assert lib.gsb200_pose_grad_temp_bytes(3) == 3 * 2048 * 12 * 4
    assert lib.gsb200_pose_grad_temp_bytes(0) == 0
    fake = ctypes.c_void_p(256)  # never dereferenced: the checks come before any CUDA call
    full = dict(q_pointcloud_camera=fake, grad_q_pointcloud_camera=fake, grad_t_pointcloud_camera=fake, temp=fake)
    for missing in full:
        pose = _lib.GsbPoseGradArgs(**{k: (None if k == missing else v) for k, v in full.items()})
        assert lib.gsb200_backward_pose(ctypes.byref(_args()), None, None, None, None, ctypes.byref(pose)) == -1  # EINVAL
        assert b"backward_pose: null" in lib.gsb200_last_error()
    pose = _lib.GsbPoseGradArgs(**dict(full, temp=ctypes.c_void_p(264)))
    assert lib.gsb200_backward_pose(ctypes.byref(_args()), None, None, None, None, ctypes.byref(pose)) == -1
    assert b"16-byte aligned" in lib.gsb200_last_error()
    pose = _lib.GsbPoseGradArgs(**full)
    assert lib.gsb200_backward_pose(ctypes.byref(_args(num_objects=0)), None, None, None, None, ctypes.byref(pose)) == -1
    assert b"num_objects >= 1" in lib.gsb200_last_error()
    assert lib.gsb200_backward_pose(ctypes.byref(_args(num_objects=65)), None, None, None, None, ctypes.byref(pose)) == -4
    assert b"GSB_POSE_MAX_OBJECTS" in lib.gsb200_last_error()
    compact = _args(_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS)
    assert lib.gsb200_backward_pose(ctypes.byref(compact), None, None, None, None, ctypes.byref(pose)) == -4
    assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # the depth, alpha and feature terms keep their requirement of the transposed kernel; an image loss does not have it
    assert lib.gsb200_backward_pose(ctypes.byref(_args(0)), fake, fake, None, None, ctypes.byref(pose)) == -4
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    assert lib.gsb200_backward_pose(ctypes.byref(_args(0)), None, None, None, None, ctypes.byref(pose)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()
    assert lib.gsb200_backward_pose(None, None, None, None, None, ctypes.byref(pose)) == -1


def test_null_pose_is_exactly_backward_ext():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ext = _lib.GsbExtraFeatureArgs(channels=0, features=fake, grad_rasterized=fake, grad_features=fake)
    cases = [(_args(), (None, None, None, None)), (_args(), (fake, None, None, None)), (_args(0), (fake, fake, None, None)),
             (_args(), (None, None, None, ctypes.byref(ext))), (_args(), (None, None, None, None))]
    for args, extra in cases:
        want = lib.gsb200_backward_ext(ctypes.byref(args), *extra)
        want_msg = lib.gsb200_last_error()
        assert lib.gsb200_backward_pose(ctypes.byref(args), *extra, None) == want != 0
        assert lib.gsb200_last_error() == want_msg


def test_abi_size_of_the_pose_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 9)()
    lib.gsb200_abi_sizes_ext(sizes, 9)
    assert sizes[8] == ctypes.sizeof(_lib.GsbPoseGradArgs) == 32
    first8 = (ctypes.c_int64 * 8)()
    lib.gsb200_abi_sizes_ext(first8, 8)
    assert list(first8) == list(sizes)[:8]


# ------------------------------------------------------------------ operator and trainer configuration
def test_operator_option_and_its_constructor_checks():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    param = inspect.signature(G.__init__).parameters["differentiable_pose"]
    assert param.kind is inspect.Parameter.KEYWORD_ONLY and param.default is False
    assert G(Config()).differentiable_pose is False
    assert G(Config(), differentiable_pose=True).differentiable_pose is True
    assert G(Config(), backward_impl="butterfly", differentiable_pose=True).differentiable_pose is True
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_pose=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_pose=True, gradient_exchange=object())
    G(Config(rgb_only=True))  # unchanged without the option
    G(Config(), gradient_exchange=object())


def _trainer(pose_lr, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 32, 48))
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera, sc.camera_info)] * 2
    seen = {}

    def factory(**kwargs):
        seen.update(kwargs)
        return lambda *a, **k: None

    trainer = T(T.TrainConfig(pose_learning_rate=pose_lr), scene, views, rasterisation_factory=factory, **kw)
    return trainer, seen


def test_trainer_pose_configuration():
    trainer, seen = _trainer(0.0)
    assert "differentiable_pose" not in seen  # injected factories get the flag only when it is on
    assert all(q is v[1] and t is v[2] for (q, t), v in zip(trainer._poses, trainer.train_views))
    trainer, seen = _trainer(1e-3)
    assert seen["differentiable_pose"] is True
    (q0, t0), (q1, t1) = trainer._poses
    assert q0 is trainer.train_views[0][1] and not q0.requires_grad  # view 0 is the gauge
    assert q1.requires_grad and t1.requires_grad and q1.is_leaf and torch.equal(q1, trainer.train_views[1][1])
    assert [torch.equal(a, b) for p, r in zip(trainer.refined_poses(), trainer._poses) for a, b in zip(p, r)] == [True] * 4
    with pytest.raises(ValueError, match="fused_step"):
        _trainer(1e-3, fused_step=True)
    for bad in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="pose_learning_rate"):
            _trainer(bad)
