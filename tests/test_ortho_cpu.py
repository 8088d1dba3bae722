"""Orthographic views (``gsb200_forward_ortho`` / ``gsb200_backward_ortho``) on the CPU: the unmodified kernels under the SIMT
emulator (``tests/simt/emu_ortho.cpp``) against the float64 evaluator (``torch_reference_ortho``) and autograd on it -- records,
images, the point, pose and intrinsics gradients, with depth, alpha, features and the 3D filter --, the projection's
invariances, the pinhole limit, the C ABI's argument checks, and the Python surface (``LensDistortion``,
``orthographic_view``, the dataset, and the operator's, ``parallel.render_views``', ``mip_filter``'s and the trainer's
refusals)."""
import ctypes
import json
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import (CameraInfo, Defocus, LensDistortion, MotionBlur, RollingShutter,
                                                      orthographic_view)
from taichi_3d_gaussian_splatting_b200.synthetic import make_aerial_scene, make_scene

from simt_helpers import build_emulator
from simt_ortho_helpers import build_ortho_emulator, emulated_backward_ortho, emulated_forward_ortho
from torch_reference import postprocess_feature_grads
from torch_reference_ortho import dense_render_ortho
from torch_reference_pose import dense_render_objects


@pytest.fixture(scope="module")
def emus():
    return build_emulator(), build_ortho_emulator()


def _scene(H=32, W=48, n=220, seed=4, sigma=0.12, skew=True):
    """A box of Gaussians (make_scene's) seen by an orthographic camera 6 units in front of it, turned by a few degrees, with a
    little skew in K so that every entry of K[:2,:2] reaches J; plus hand-placed points behind the near plane (culled) and
    beyond the image's boundary tiles (culled)."""
    sc = make_scene(n, H, W, sigma, seed, sh_degree=2)
    K = torch.tensor([[W / 8.0, 0.3 if skew else 0.0, W / 2.0], [-0.2 if skew else 0.0, W / 8.0, H / 2.0], [0.0, 0.0, 1.0]])
    ci = CameraInfo(K, H, W, 0, LensDistortion("orthographic", ()))
    extra = torch.tensor([[0.0, 0.0, -7.0],     # z < near after the camera's shift: culled
                          [40.0, 0.0, 6.0]],    # u far outside the image: culled
                         dtype=torch.float32)
    sc.point_cloud = torch.cat([sc.point_cloud, extra]).contiguous()
    sc.point_cloud_features = torch.cat([sc.point_cloud_features, sc.point_cloud_features[:2]]).contiguous()
    N = sc.point_cloud.shape[0]
    sc.point_invalid_mask = torch.zeros(N, dtype=torch.int8)
    sc.point_object_id = torch.zeros(N, dtype=torch.int32)
    sc.camera_info = ci
    a = math.radians(4.0) / 2
    sc.q_pointcloud_camera = torch.tensor([[math.sin(a) * 0.6, math.sin(a) * 0.8, 0.0, math.cos(a)]], dtype=torch.float32)
    sc.t_pointcloud_camera = torch.tensor([[0.1, -0.2, -4.0]], dtype=torch.float32)
    return sc


def _dense(sc, extra=None, filter3d=None, requires_grad=False):
    ci = sc.camera_info
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = sc.point_cloud_features.clone().double().requires_grad_(requires_grad)
    q = sc.q_pointcloud_camera.clone().double().requires_grad_(requires_grad)
    t = sc.t_pointcloud_camera.clone().double().requires_grad_(requires_grad)
    K = ci.camera_intrinsics.clone().double().requires_grad_(requires_grad)
    ef = None if extra is None else torch.from_numpy(extra).double().requires_grad_(requires_grad)
    f3 = None if filter3d is None else torch.from_numpy(filter3d)
    out = dense_render_ortho(xyz, feats, sc.point_invalid_mask, sc.point_object_id, K, q, t, ci.camera_height,
                             ci.camera_width, extra_features=ef, filter3d=f3)
    return dict(xyz=xyz, feats=feats, q=q, t=t, K=K, ef=ef), out


def _filter(N, seed=2):
    f = np.random.default_rng(seed).uniform(0.0, 0.15, N).astype(np.float32)
    f[::3] = 0.0  # sigma = 0 leaves a row untouched
    return f


@pytest.mark.parametrize("with_filter", [False, True])
def test_per_point_records_follow_the_model(emus, with_filter):
    emu, oemu = emus
    sc = _scene()
    N = sc.point_cloud.shape[0]
    f3 = _filter(N) if with_filter else None
    st = emulated_forward_ortho(emu, oemu, sc, filter3d=f3, filter_tiles=False)
    _, (_, _, _, _, aux) = _dense(sc, filter3d=f3)
    ids = aux["ids"].numpy()
    po = st.pre.point_offset
    assert sorted(np.nonzero(po >= 0)[0].tolist()) == ids.tolist()
    assert po[N - 2] < 0 and po[N - 1] < 0
    rec = st.pre.records[po[ids]]
    np.testing.assert_allclose(rec[:, 0:2], aux["uv"].detach().numpy(), atol=2e-4)
    np.testing.assert_allclose(rec[:, 7], aux["depth"].detach().numpy(), rtol=1e-6)
    np.testing.assert_allclose(st.pre.pic[po[ids]], aux["pc"].detach().numpy(), atol=2e-5)
    np.testing.assert_allclose(rec[:, 2:6], aux["conic"].detach().numpy(), rtol=2e-3, atol=1e-6)
    np.testing.assert_allclose(rec[:, 8:11], aux["color"].detach().numpy(), atol=2e-6)
    np.testing.assert_allclose(rec[:, 11], aux["radius"].numpy(), rtol=2e-3)
    np.testing.assert_array_equal(st.pre.num_tiles[po[ids]], ((aux["max_tu"] - aux["min_tu"]) *
                                                              (aux["max_tv"] - aux["min_tv"])).numpy())
    assert int(st.pre.counters[4]) == int((rec[:, 7] * np.float32(100.0)).astype(np.int32).max())


@pytest.mark.parametrize("with_filter", [False, True])
@pytest.mark.parametrize("exact", [True, False])
def test_images_match_the_evaluator(emus, exact, with_filter):
    emu, oemu = emus
    sc = _scene()
    N = sc.point_cloud.shape[0]
    f3 = _filter(N) if with_filter else None
    extra = np.random.default_rng(1).standard_normal((N, 5)).astype(np.float32)
    st = emulated_forward_ortho(emu, oemu, sc, exact=exact, features=extra, filter3d=f3)
    _, (C, D, S, F, _) = _dense(sc, extra, f3)
    tol = 2e-5 if exact else 2e-3
    np.testing.assert_allclose(st.image, C.detach().numpy(), atol=tol)
    np.testing.assert_allclose(st.acc_alpha, S.detach().numpy(), atol=tol)
    np.testing.assert_allclose(st.fmap, F.detach().numpy(), atol=10 * tol)
    np.testing.assert_allclose(st.depth, D.detach().numpy(), atol=100 * tol, rtol=tol)
    assert st.acc_alpha.max() > 0.5


@pytest.mark.parametrize("terms", ["image", "depth", "alpha", "features", "all", "filter", "filter_all"])
@pytest.mark.parametrize("camera", ["none", "pose", "intr", "both"])
def test_gradients_match_autograd(emus, terms, camera):
    if terms.startswith("filter") and camera != "none":
        pytest.skip("the 3D filter is not implemented with camera gradients")
    emu, oemu = emus
    sc = _scene()
    N = sc.point_cloud.shape[0]
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    rng = np.random.default_rng(5)
    full = terms in ("all", "filter_all")
    f3 = _filter(N) if terms.startswith("filter") else None
    extra = rng.standard_normal((N, 3)).astype(np.float32) if terms == "features" or full else None
    st = emulated_forward_ortho(emu, oemu, sc, exact=True, features=extra, filter3d=f3)
    g = rng.standard_normal((H, W, 3)).astype(np.float32)
    gd = 0.1 * rng.standard_normal((H, W)).astype(np.float32) if terms == "depth" or full else None
    ga = rng.standard_normal((H, W)).astype(np.float32) if terms == "alpha" or full else None
    gF = rng.standard_normal((H, W, 3)).astype(np.float32) if extra is not None else None
    pose, intr = camera in ("pose", "both"), camera in ("intr", "both")
    out = emulated_backward_ortho(emu, oemu, st, g, grad_depth=gd, grad_alpha=ga, grad_feature_map=gF, pose=pose, intr=intr)
    leaves, (C, D, S, F, _) = _dense(sc, extra, f3, requires_grad=True)
    loss = (C * torch.from_numpy(g).double()).sum()
    if gd is not None:
        loss = loss + (D * torch.from_numpy(gd).double()).sum()
    if ga is not None:
        loss = loss + (S * torch.from_numpy(ga).double()).sum()
    if gF is not None:
        loss = loss + (F * torch.from_numpy(gF).double()).sum()
    loss.backward()
    want_x = leaves["xyz"].grad.numpy()
    want_f = postprocess_feature_grads(leaves["feats"].grad, 3).numpy()
    np.testing.assert_allclose(out.gx, want_x, atol=2e-5 * np.abs(want_x).max() + 1e-6)
    np.testing.assert_allclose(out.gf, want_f, atol=2e-5 * np.abs(want_f).max() + 1e-6)
    if out.gext is not None:
        want_e = leaves["ef"].grad.numpy()
        np.testing.assert_allclose(out.gext, want_e, atol=1e-5 * np.abs(want_e).max() + 1e-6)
    if pose:
        want_q, want_t = leaves["q"].grad.numpy(), leaves["t"].grad.numpy()
        np.testing.assert_allclose(out.gq, want_q, atol=1e-4 * np.abs(want_q).max() + 1e-6)
        np.testing.assert_allclose(out.gt, want_t, atol=1e-4 * np.abs(want_t).max() + 1e-6)
    if intr:
        want_K = leaves["K"].grad.numpy()
        want_K[2] = 0.0  # the forward does not read K's last row
        np.testing.assert_allclose(out.gK, want_K, atol=1e-4 * np.abs(want_K).max() + 1e-6)
        assert (out.gK[0, :2] != 0).all() and (out.gK[1, :2] != 0).all()  # the skew entries reach J
    assert (out.gx[st.pre.point_offset < 0] == 0).all()


def test_footprint_and_colour_do_not_change_along_the_viewing_axis(emus):
    """Move every Gaussian along the camera's forward axis: (u, v), the conic, rescale, radius and the SH colour stay as they
    were, only the depth changes by the shift; and the SH colour is the same at every position."""
    emu, oemu = emus
    sc = _scene(skew=False)
    a = emulated_forward_ortho(emu, oemu, sc, filter_tiles=False)
    from torch_reference_pose import camera_from_pose
    Rc, _ = camera_from_pose(sc.q_pointcloud_camera.double(), sc.t_pointcloud_camera.double())
    forward = Rc[0, 2].float()  # row 2 of W: the forward axis in the scene frame
    moved = _scene(skew=False)
    moved.point_cloud = (sc.point_cloud + 1.5 * forward).contiguous()
    b = emulated_forward_ortho(emu, oemu, moved, filter_tiles=False)
    ia, ib = a.pre.point_offset, b.pre.point_offset
    both = np.nonzero((ia >= 0) & (ib >= 0))[0]
    assert len(both) > 150
    ra, rb = a.pre.records[ia[both]], b.pre.records[ib[both]]
    np.testing.assert_allclose(rb[:, 0:2], ra[:, 0:2], atol=2e-4)
    np.testing.assert_allclose(rb[:, 2:7], ra[:, 2:7], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(rb[:, 8:12], ra[:, 8:12], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(rb[:, 7] - ra[:, 7], 1.5, atol=1e-4)
    # one feature row at several positions: one colour
    same = _scene(skew=False)
    same.point_cloud_features = same.point_cloud_features[:1].repeat(same.point_cloud.shape[0], 1).contiguous()
    c = emulated_forward_ortho(emu, oemu, same, filter_tiles=False)
    cols = c.pre.records[c.pre.point_offset[c.pre.point_offset >= 0], 8:11]
    assert np.abs(cols - cols[0]).max() == 0.0


def test_pinhole_far_away_converges_to_the_orthographic_render(emus):
    """A pinhole d units behind the orthographic camera with f = fx d renders the same scene ever closer as d grows: the
    mean image error falls roughly as 1/d (measured: 0.070, 0.021, 0.0065 at d = 80, 320, 1280; the splats' screen offsets
    shrink as z / d, z the ortho depth)."""
    emu, oemu = emus
    H, W = 32, 48
    sc = _scene(H, W, n=150, skew=False, sigma=0.2)
    ortho = emulated_forward_ortho(emu, oemu, sc, exact=True).image.astype(np.float64)
    K = sc.camera_info.camera_intrinsics
    errs = []
    for d in (80.0, 320.0, 1280.0):
        Kp = torch.tensor([[float(K[0, 0]) * d, 0.0, float(K[0, 2])], [0.0, float(K[1, 1]) * d, float(K[1, 2])], [0.0, 0.0, 1.0]])
        # the camera moved back by d along its axis: pc' = pc + (0, 0, d), i.e. t_pc' = t_pc - d * forward
        from torch_reference_pose import camera_from_pose
        Rc, _ = camera_from_pose(sc.q_pointcloud_camera.double(), sc.t_pointcloud_camera.double())
        t = (sc.t_pointcloud_camera.double() - d * Rc[0, 2]).float()
        img, _ = dense_render_objects(sc.point_cloud, sc.point_cloud_features, sc.point_invalid_mask, sc.point_object_id, Kp,
                                      sc.q_pointcloud_camera, t, H, W, far=1000.0 + d)
        errs.append(float(np.abs(img.detach().numpy() - ortho).mean()))
    assert errs[0] > errs[1] > errs[2], errs
    assert errs[2] < 0.01 and errs[1] / errs[2] > 2.5 and errs[0] / errs[1] > 2.5, errs


# ------------------------------------------------------------------ C ABI
def test_c_entry_points_check_their_arguments_before_any_cuda_call():
    lib = _lib.load()
    ok = ctypes.c_void_p(256)
    odd = _lib.GsbFilter3dArgs(filter3d=ctypes.c_void_p(258))
    fargs = _lib.GsbForwardArgs(camera_width=64, camera_height=32, camera_intrinsics=ok, rasterized_image=ok, rgb_only=1)
    assert lib.gsb200_forward_ortho(ctypes.byref(fargs), None, ctypes.byref(odd)) == -1
    assert b"4-byte aligned" in lib.gsb200_last_error()
    assert lib.gsb200_forward_ortho(ctypes.byref(_lib.GsbForwardArgs()), None, None) == -1
    assert b"null camera_intrinsics" in lib.gsb200_last_error()
    ext = _lib.GsbExtraFeatureArgs(channels=17, features=ok, rasterized=ok)
    assert lib.gsb200_forward_ortho(ctypes.byref(fargs), ctypes.byref(ext), None) == -1
    assert b"channels must be in 1..16" in lib.gsb200_last_error()
    assert lib.gsb200_forward_ortho(None, None, None) == -1
    flt = _lib.GsbFilter3dArgs(filter3d=ok)
    pose = _lib.GsbPoseGradArgs(q_pointcloud_camera=ok, grad_q_pointcloud_camera=ok, grad_t_pointcloud_camera=ok, temp=ok)
    intr = _lib.GsbIntrinsicsGradArgs(grad_camera_intrinsics=ok, temp=ok)
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, camera_width=64,
                                   camera_intrinsics=ok)
    assert lib.gsb200_backward_ortho(ctypes.byref(compact), None, None, None, None, None, None, None) == -4
    assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1, camera_width=64, camera_intrinsics=ok)
    for p, i in ((pose, None), (None, intr), (pose, intr)):
        assert lib.gsb200_backward_ortho(ctypes.byref(bargs), None, None, None, None, ctypes.byref(flt),
                                         ctypes.byref(p) if p else None, ctypes.byref(i) if i else None) == -4
        assert b"3D filter" in lib.gsb200_last_error()
    assert lib.gsb200_backward_ortho(ctypes.byref(bargs), None, None, None, None, ctypes.byref(odd), None, None) == -1
    assert b"4-byte aligned" in lib.gsb200_last_error()
    assert lib.gsb200_backward_ortho(ctypes.byref(bargs), ok, None, None, None, None, None, None) == -1
    assert b"both NULL or both set" in lib.gsb200_last_error()
    butterfly = _lib.GsbBackwardArgs(num_objects=1, camera_width=64, camera_intrinsics=ok)
    assert lib.gsb200_backward_ortho(ctypes.byref(butterfly), ok, ok, None, None, None, None, None) == -4
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    bad_pose = _lib.GsbPoseGradArgs(q_pointcloud_camera=ok, temp=ok)
    assert lib.gsb200_backward_ortho(ctypes.byref(bargs), None, None, None, None, None, ctypes.byref(bad_pose), None) == -1
    assert b"backward_pose: null" in lib.gsb200_last_error()
    bad_intr = _lib.GsbIntrinsicsGradArgs(temp=ok)
    assert lib.gsb200_backward_ortho(ctypes.byref(bargs), None, None, None, None, None, None, ctypes.byref(bad_intr)) == -1
    assert b"backward_calib: null" in lib.gsb200_last_error()
    assert lib.gsb200_backward_ortho(None, None, None, None, None, None, None, None) == -1


# ------------------------------------------------------------------ Python surface
def test_lens_distortion_record_intrinsics_and_view():
    d = LensDistortion("orthographic", ())
    assert d.coefficients == ()
    with pytest.raises(ValueError, match="0 coefficients"):
        LensDistortion("orthographic", (0.1,))
    K = LensDistortion.orthographic_intrinsics(640, 480, 0.05)
    assert K.dtype == torch.float32 and K.shape == (3, 3)
    assert K[0, 0] == pytest.approx(20.0) and K[1, 1] == pytest.approx(20.0)
    assert K[0, 2] == 320 and K[1, 2] == 240 and K[0, 1] == 0 and K[1, 0] == 0 and K[2].tolist() == [0, 0, 1]
    for bad in ((0, 16, 0.1), (16, 16, 0.0), (16, 16, float("nan"))):
        with pytest.raises(ValueError):
            LensDistortion.orthographic_intrinsics(*bad)
    with pytest.raises(KeyError):
        _lib.lens_args(d)
    # a nadir view over z = 0 with +y toward the top of the image: scene x grows with u, scene y shrinks with v
    q, t, ci = orthographic_view((1.0, 2.0, 10.0), (0.0, 0.0, -1.0), (0.0, 1.0, 0.0), 64, 32, 0.5)
    assert ci.distortion.model == "orthographic" and (ci.camera_height, ci.camera_width) == (32, 64)
    assert q.shape == (1, 4) and t.tolist() == [[1.0, 2.0, 10.0]]
    from torch_reference_pose import camera_from_pose
    Rc, tc = camera_from_pose(q.double(), t.double())
    pts = torch.tensor([[1.0, 2.0, 0.0], [3.0, 2.0, 0.0], [1.0, 3.0, 0.0], [1.0, 2.0, 4.0]], dtype=torch.float64)
    pc = pts @ Rc[0].T + tc[0]
    uv = pc[:, :2] @ ci.camera_intrinsics[:2, :2].double().T + ci.camera_intrinsics[:2, 2].double()
    np.testing.assert_allclose(uv.numpy(), [[32, 16], [36, 16], [32, 14], [32, 16]], atol=1e-5)
    np.testing.assert_allclose(pc[:, 2].numpy(), [10, 10, 10, 6], atol=1e-6)  # depth: height = 10 - depth
    with pytest.raises(ValueError, match="parallel"):
        orthographic_view((0, 0, 1), (0, 0, -1), (0, 0, 2), 16, 16, 0.1)
    with pytest.raises(ValueError, match="forward"):
        orthographic_view((0, 0, 1), (0, 0, 0), (0, 1, 0), 16, 16, 0.1)


def test_aerial_scene_sits_under_its_nadir_camera():
    from taichi_3d_gaussian_splatting_b200.synthetic import AERIAL_BLOCKS, aerial_height
    sc = make_aerial_scene(2000, 32, 48, 0, pixel_size=0.05, altitude=4.0)
    assert sc.camera_info.distortion.model == "orthographic"
    xyz = sc.point_cloud
    assert (xyz[:, 2] >= 0).all() and float(xyz[:, 2].max()) == pytest.approx(max(b[4] for b in AERIAL_BLOCKS) * 4.0)
    gw = 1.1 * 48 * 0.05
    torch.testing.assert_close(aerial_height(xyz[:, 0], xyz[:, 1], gw, 4.0), xyz[:, 2])
    assert sc.point_cloud_features.shape == (2000, 56)


def _input(sc=None, **camera):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = sc or make_aerial_scene(64, 32, 48, 3, pixel_size=0.1)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, ci.distortion, camera.get("rs"),
                    camera.get("mb"), camera.get("df"))
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_refuses_what_the_orthographic_view_does_not_combine_with():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    from taichi_3d_gaussian_splatting_b200 import parallel
    from taichi_3d_gaussian_splatting_b200.mip_filter import compute_filter_3d
    Config = G.GaussianPointCloudRasterisationConfig
    inp = _input()
    for option in ("differentiable_distortion", "differentiable_rolling_shutter", "differentiable_motion_blur",
                   "differentiable_defocus"):
        with pytest.raises(ValueError, match=option):
            G(Config(), **{option: True})(inp)
    with pytest.raises(ValueError, match="gradient_exchange"):
        op = G(Config())
        op.gradient_exchange = object()
        op(inp)
    for camera, msg in ((dict(rs=RollingShutter((0.1, 0, 0), (0, 0, 0))), "rolling shutter"),
                        (dict(mb=MotionBlur((0.1, 0, 0), (0, 0, 0))), "motion blur"),
                        (dict(df=Defocus(0.05, 2.0)), "defocus")):
        with pytest.raises(ValueError, match=msg):
            G(Config())(_input(**camera))
    for option in ("differentiable_pose", "differentiable_intrinsics"):
        with pytest.raises(ValueError, match="point_filter_3d"):
            G(Config(), **{option: True})(inp, point_filter_3d=torch.zeros(64))
    with pytest.raises(ValueError, match="parallel.render_views"):
        parallel.render_views(G(Config()), lambda i: inp, [0])
    sc = make_aerial_scene(64, 32, 48, 3, pixel_size=0.1)
    with pytest.raises(ValueError, match="orthographic"):
        compute_filter_3d(sc.point_cloud, sc.point_invalid_mask, sc.point_object_id,
                          [(sc.q_pointcloud_camera, sc.t_pointcloud_camera, sc.camera_info)], 0.8)


def _trainer(fused_step=False, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_aerial_scene(64, 32, 48, 3, pixel_size=0.1)
    pin = make_scene(64, 32, 48, 0.1, 1)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    views = [(torch.zeros((3, 32, 48)), sc.q_pointcloud_camera, sc.t_pointcloud_camera, sc.camera_info),
             (torch.zeros((3, 32, 48)), pin.q_pointcloud_camera, pin.t_pointcloud_camera, pin.camera_info)]

    class Factory:
        gradient_exchange = None

        def __init__(self, **kwargs):
            pass

    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=Factory, fused_step=fused_step)


def test_trainer_refines_poses_and_intrinsics_and_refuses_the_rest():
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(mip_filter_3d=True), "mip_filter_3d"),
                    (dict(distortion_learning_rate=1e-3), "distortion"),
                    (dict(rolling_shutter_learning_rate=1e-3), "rolling_shutter_learning_rate"),
                    (dict(motion_blur_learning_rate=1e-3), "motion_blur_learning_rate"),
                    (dict(defocus_learning_rate=1e-3), "defocus_learning_rate")):
        with pytest.raises(ValueError, match=msg):
            _trainer(**kw)
    _trainer()
    _trainer(pose_learning_rate=1e-3, intrinsics_learning_rate=1e-3)


def test_dataset_scales_an_orthographic_k_like_a_pinhole_k(tmp_path):
    """Crop to tiles, the on-disk size and autoscale act on an orthographic K exactly as on a pinhole K: the same record with
    and without the distortion key gives the same K, size and image."""
    from PIL import Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    records = []
    for i, (h, w, rec_h, rec_w) in enumerate(((100, 200, 100, 200), (1000, 2000, 500, 1000), (40, 50, 40, 50))):
        img = tmp_path / f"p{i}.png"
        Image.fromarray(np.random.default_rng(i).integers(0, 255, (h, w, 3), dtype=np.uint8)).save(img)
        K = [[1.0 / 0.05, 0.0, rec_w / 2.0], [0.0, 1.0 / 0.05, rec_h / 2.0], [0.0, 0.0, 1.0]]
        base = {"image_path": str(img), "T_pointcloud_camera": np.eye(4).tolist(), "camera_intrinsics": K,
                "camera_height": rec_h, "camera_width": rec_w, "camera_id": 0}
        records.append(dict(base, distortion={"model": "orthographic", "coefficients": []}))
        records.append(base)
    path = tmp_path / "poses.json"
    path.write_text(json.dumps(records))
    ds = ImagePoseDataset(str(path))
    for i in range(3):
        image_o, _, _, ci_o = ds[2 * i]
        image_p, _, _, ci_p = ds[2 * i + 1]
        assert ci_o.distortion.model == "orthographic" and ci_p.distortion is None
        assert (ci_o.camera_height, ci_o.camera_width) == (ci_p.camera_height, ci_p.camera_width)
        assert ci_o.camera_height % 16 == 0 and ci_o.camera_width % 16 == 0
        torch.testing.assert_close(ci_o.camera_intrinsics, ci_p.camera_intrinsics)
        torch.testing.assert_close(image_o, image_p)
    # the on-disk size decides: an image twice the recorded size has twice the pixels per scene unit
    assert float(ds[2][3].camera_intrinsics[0, 0]) != pytest.approx(20.0)


def test_trainer_steps_render_orthographic_views_as_orthographic():
    """A trainer step rebuilds the camera of each view with its intrinsics as trained: the rebuilt camera keeps the view's
    orthographic projection (and the trained K reaches the rasteriser), with and without intrinsics refinement, for an
    orthographic view trained beside a pinhole view of another camera_id."""
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_aerial_scene(64, 32, 48, 3, pixel_size=0.1)
    pin = make_scene(64, 32, 48, 0.1, 1)
    q, t, ci = orthographic_view((0.0, 0.0, 5.0), (0.0, 0.0, -1.0), (0.0, 1.0, 0.0), 48, 32, 0.1, camera_id=7)
    assert ci.camera_id == 7
    for intr_lr in (0.0, 1e-3):
        seen = []

        class Recorder(torch.nn.Module):
            gradient_exchange = None

            def __init__(self, **kwargs):
                super().__init__()

            def forward(self, inp, **kw):
                c = inp.camera_info
                seen.append((c.camera_id, getattr(c.distortion, "model", None), c.camera_intrinsics.requires_grad))
                H, W = c.camera_height, c.camera_width
                v = torch.sigmoid(inp.point_cloud_features[:, 8].mean() + 1e-3 * c.camera_intrinsics.sum() +
                                  inp.point_cloud.sum() * 0.0 + (inp.q_pointcloud_camera.sum() + inp.t_pointcloud_camera.sum()) * 0.0)
                return v.expand(H, W, 3), torch.zeros((H, W)), torch.zeros((H, W), dtype=torch.int32)

        scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                      sc.point_invalid_mask, sc.point_object_id)
        views = [(torch.full((3, 32, 48), 0.3), q, t, ci),
                 (torch.full((3, 32, 48), 0.3), pin.q_pointcloud_camera, pin.t_pointcloud_camera, pin.camera_info)]
        cfg = T.TrainConfig(num_iterations=4, intrinsics_learning_rate=intr_lr, initial_downsample_factor=1)
        cfg.adaptive_controller_config.num_iterations_warm_up = 10 ** 9
        trainer = T(cfg, scene, views, rasterisation_factory=Recorder)
        trainer.train()
        assert {(7, "orthographic", intr_lr > 0), (0, None, intr_lr > 0)} == set(seen), seen
        if intr_lr > 0:
            assert sorted(trainer._intrinsics) == [0, 7]  # the orthographic camera has a correction of its own
