"""Equirectangular panoramas (``gsb200_forward_equirect`` / ``gsb200_backward_equirect``) on the CPU: the unmodified kernels
under the SIMT emulator (``tests/simt/emu_equirect.cpp``) against the float64 dense evaluator (``equirect_reference``) and
autograd on it, the seam's roll invariance, the convention against pinhole views along the same rays, the C ABI's argument
checks, and the Python surface (``LensDistortion``, the dataset, the operator's, ``parallel.render_views``' and the
trainer's refusals)."""
import ctypes
import json
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, Defocus, LensDistortion, MotionBlur, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import make_panorama_scene, make_scene

from equirect_reference import dense_render_equirect, keyed_tiles
from simt_equirect_helpers import build_equirect_emulator, emulated_backward_equirect, emulated_forward_equirect
from simt_helpers import build_emulator
from torch_reference import postprocess_feature_grads
from torch_reference_pose import dense_render_objects


@pytest.fixture(scope="module")
def emus():
    return build_emulator(), build_equirect_emulator()


def _scene(H=32, W=64, n=240, seed=3, sigma=0.15):
    """The shell scene plus hand-placed points: behind the camera, across the seam, inside the near sphere (culled), in the
    polar cone (culled) and just outside it (drawn)."""
    sc = make_panorama_scene(n, H, W, sigma, seed, sh_degree=2, radius=3.0, seam_fraction=0.2, pole_fraction=0.05)
    extra = torch.tensor([[0.0, 0.3, -2.5],          # behind the camera, on the seam
                          [0.05, -0.2, -2.0],        # straddles the seam
                          [0.3, 0.1, 0.2],           # inside the near sphere (r < 0.8): culled
                          [1e-4, 2.5, 1e-4],         # rho / r < 1e-3: culled
                          [0.02, -2.0, 0.01]],       # 0.6 degrees from the pole: drawn across its rows
                         dtype=torch.float32)
    f = sc.point_cloud_features[:extra.shape[0]].clone()
    f[:, 4:7] = math.log(0.2)
    f[:, 7] = 2.0
    sc.point_cloud = torch.cat([sc.point_cloud, extra]).contiguous()
    sc.point_cloud_features = torch.cat([sc.point_cloud_features, f]).contiguous()
    sc.point_invalid_mask = torch.zeros(sc.point_cloud.shape[0], dtype=torch.int8)
    sc.point_object_id = torch.zeros(sc.point_cloud.shape[0], dtype=torch.int32)
    return sc


def _dense(sc, extra=None, requires_grad=False):
    ci = sc.camera_info
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = sc.point_cloud_features.clone().double().requires_grad_(requires_grad)
    ef = None if extra is None else torch.from_numpy(extra).double().requires_grad_(requires_grad)
    out = dense_render_equirect(xyz, feats, sc.point_invalid_mask, sc.point_object_id, ci.camera_intrinsics,
                                sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci.camera_height, ci.camera_width,
                                extra_features=ef)
    return (xyz, feats, ef) + out


def test_per_point_records_and_keys_follow_the_model(emus):
    emu, qemu = emus
    sc = _scene()
    N = sc.point_cloud.shape[0]
    st = emulated_forward_equirect(emu, qemu, sc, filter_tiles=False)
    *_, aux = _dense(sc)
    ids = aux["ids"].numpy()
    po = st.pre.point_offset
    assert sorted(np.nonzero(po >= 0)[0].tolist()) == ids.tolist()
    assert po[N - 3] < 0 and po[N - 2] < 0 and po[N - 1] >= 0 and po[N - 5] >= 0  # near sphere, polar cone; behind: in view
    rec = st.pre.records[po[ids]]
    du = (rec[:, 0] - aux["uv"][:, 0].detach().numpy() + 32.0) % 64.0 - 32.0  # u on the seam may round to either side
    assert np.abs(du).max() < 2e-4
    np.testing.assert_allclose(rec[:, 1], aux["uv"][:, 1].detach().numpy(), atol=2e-4)
    assert (rec[:, 0] >= 0).all() and (rec[:, 0] < 64).all()
    np.testing.assert_allclose(rec[:, 7], aux["depth"].detach().numpy(), rtol=1e-6)
    conic = aux["conic"].detach().numpy()
    np.testing.assert_allclose(rec[:, 2:6], conic, rtol=2e-3, atol=1e-6)
    np.testing.assert_allclose(rec[:, 11], aux["radius"].numpy(), rtol=2e-3)
    # every tile of the footprint is keyed (the reach filter is off), the columns modulo W/16; at most the full width
    keys = st.pre.keys[:st.K].astype(np.int64)
    tiles = keys >> st.pre.depth_bits
    depth_keys = keys & ((1 << st.pre.depth_bits) - 1)
    vals = st.pre.vals[:st.K]
    for j, m in enumerate(ids):
        o = po[m]
        mine = vals == o
        assert set(tiles[mine].tolist()) == keyed_tiles(aux, 64, j)
        assert len(tiles[mine]) == len(set(tiles[mine].tolist()))
        assert (depth_keys[mine] == int(np.float32(rec[j, 7]) * np.float32(100.0))).all()
    assert int(st.pre.counters[4]) == int((rec[:, 7] * np.float32(100.0)).astype(np.int32).max())
    # the seam: some splats key columns on both sides of it, and the near-pole splat keys whole rows
    pole = np.nonzero(ids == N - 1)[0][0]
    assert int(aux["max_tu"][pole] - aux["min_tu"][pole]) == 4
    assert any(aux["min_tu"][j] < 0 or aux["max_tu"][j] > 4 for j in range(len(ids)))


@pytest.mark.parametrize("size", [(32, 64), (64, 128)])
@pytest.mark.parametrize("exact", [True, False])
def test_images_match_the_evaluator(emus, size, exact):
    emu, qemu = emus
    H, W = size
    sc = _scene(H, W, n=200 if W == 64 else 400)
    N = sc.point_cloud.shape[0]
    extra = np.random.default_rng(1).standard_normal((N, 5)).astype(np.float32)
    st = emulated_forward_equirect(emu, qemu, sc, exact=exact, features=extra)
    _, _, _, C, D, S, F, aux = _dense(sc, extra)
    tol = 2e-5 if exact else 2e-3
    np.testing.assert_allclose(st.image, C.detach().numpy(), atol=tol)
    np.testing.assert_allclose(st.acc_alpha, S.detach().numpy(), atol=tol)
    np.testing.assert_allclose(st.fmap, F.detach().numpy(), atol=10 * tol)
    np.testing.assert_allclose(st.depth, D.detach().numpy(), atol=100 * tol, rtol=tol)
    assert np.isfinite(st.image).all() and st.acc_alpha.max() > 0.5


@pytest.mark.parametrize("terms", ["image", "depth", "alpha", "features", "all"])
def test_gradients_match_autograd(emus, terms):
    emu, qemu = emus
    sc = _scene(32, 64)
    N = sc.point_cloud.shape[0]
    rng = np.random.default_rng(5)
    extra = rng.standard_normal((N, 3)).astype(np.float32) if terms in ("features", "all") else None
    st = emulated_forward_equirect(emu, qemu, sc, exact=True, features=extra)
    g = rng.standard_normal((32, 64, 3)).astype(np.float32)
    gd = 0.1 * rng.standard_normal((32, 64)).astype(np.float32) if terms in ("depth", "all") else None
    ga = rng.standard_normal((32, 64)).astype(np.float32) if terms in ("alpha", "all") else None
    gF = rng.standard_normal((32, 64, 3)).astype(np.float32) if extra is not None else None
    gx, gf, gext, _ = emulated_backward_equirect(emu, qemu, st, g, grad_depth=gd, grad_alpha=ga, grad_feature_map=gF)
    xyz, feats, ef, C, D, S, F, aux = _dense(sc, extra, requires_grad=True)
    loss = (C * torch.from_numpy(g).double()).sum()
    if gd is not None:
        loss = loss + (D * torch.from_numpy(gd).double()).sum()
    if ga is not None:
        loss = loss + (S * torch.from_numpy(ga).double()).sum()
    if gF is not None:
        loss = loss + (F * torch.from_numpy(gF).double()).sum()
    loss.backward()
    want_x = xyz.grad.numpy()
    want_f = postprocess_feature_grads(feats.grad, 3).numpy()
    scale_x, scale_f = np.abs(want_x).max(), np.abs(want_f).max()
    np.testing.assert_allclose(gx, want_x, atol=2e-5 * scale_x + 1e-6)
    np.testing.assert_allclose(gf, want_f, atol=2e-5 * scale_f + 1e-6)
    if gext is not None:
        np.testing.assert_allclose(gext, ef.grad.numpy(), atol=1e-5 * np.abs(ef.grad.numpy()).max() + 1e-6)
    assert np.isfinite(gx).all() and np.isfinite(gf).all()
    assert (gx[st.pre.point_offset < 0] == 0).all()


@pytest.mark.parametrize("size", [(32, 64), (64, 128)])
def test_a_yaw_of_k_columns_rolls_the_image(emus, size):
    """Yaw the camera by 2 pi k / W: the panorama rolls by k columns (k = a quarter turn, a multiple of the tile width, so
    the splats across the seam of one image lie mid-image in the other)."""
    emu, qemu = emus
    H, W = size
    k = W // 4
    base = _scene(H, W, n=300)
    turned = _scene(H, W, n=300)
    half = (2 * math.pi * k / W) / 2
    turned.q_pointcloud_camera = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], dtype=torch.float32)
    a = emulated_forward_equirect(emu, qemu, base, exact=False)
    b = emulated_forward_equirect(emu, qemu, turned, exact=False)
    want = np.roll(a.image, -k, axis=1)
    assert np.abs(b.image - want).max() < 2e-3
    assert np.abs(b.image - a.image).max() > 0.1  # the yaw did move the image
    np.testing.assert_allclose(b.acc_alpha, np.roll(a.acc_alpha, -k, axis=1), atol=2e-3)


def test_convention_matches_pinhole_views_along_the_same_rays(emus):
    """Large smooth Gaussians at |lat| <= 45 degrees: an equirectangular pixel equals a pinhole render along its ray, which
    pins the signs of lon and lat and the placement of (cx, cy).  Pinhole views look along +z, +x, -z and -x (yaw 0, 90, 180,
    270 degrees); each pinhole pixel is compared with the panorama sampled bilinearly at its ray's (u, v)."""
    emu, qemu = emus
    H, W = 64, 128
    g = torch.Generator().manual_seed(11)
    n = 30
    lon = torch.rand(n, generator=g) * 2 * math.pi
    lat = (torch.rand(n, generator=g) * 2 - 1) * math.radians(35.0)
    d = torch.stack([torch.cos(lat) * torch.sin(lon), torch.sin(lat), torch.cos(lat) * torch.cos(lon)], -1)
    xyz = (d * 6.0).float()
    sc = make_panorama_scene(n, H, W, 0.5, 2, sh_degree=0)
    sc.point_cloud = xyz.contiguous()
    f = sc.point_cloud_features.clone()
    f[:, 4:7] = math.log(0.5)  # sigma ~4.8 degrees: 2.3 panorama pixels, 3 pinhole pixels
    f[:, 7] = 0.5
    sc.point_cloud_features = f
    pano = emulated_forward_equirect(emu, qemu, sc, exact=True).image.astype(np.float64)
    Hp = Wp = 32
    fp = 24.0
    Kp = torch.tensor([[fp, 0.0, Wp / 2], [0.0, fp, Hp / 2], [0.0, 0.0, 1.0]])
    ys, xs = np.meshgrid(np.arange(Hp) + 0.5, np.arange(Wp) + 0.5, indexing="ij")
    worst = 0.0
    for yaw in (0.0, 90.0, 180.0, 270.0):
        half = math.radians(yaw) / 2
        q = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]])
        img, _ = dense_render_objects(sc.point_cloud, f, sc.point_invalid_mask, sc.point_object_id, Kp, q,
                                      torch.zeros(1, 3), Hp, Wp)
        img = img.detach().numpy()
        # the ray of each pinhole pixel in the panorama's frame: camera yawed by `yaw` about +y
        c, s = math.cos(math.radians(yaw)), math.sin(math.radians(yaw))
        dx, dy, dz = (xs - Wp / 2) / fp, (ys - Hp / 2) / fp, np.ones_like(xs)
        wx, wz = c * dx + s * dz, -s * dx + c * dz
        u = W / (2 * math.pi) * np.arctan2(wx, wz) + W / 2
        v = H / math.pi * np.arctan2(dy, np.hypot(wx, wz)) + H / 2
        uu, vv = (u - 0.5) % W, np.clip(v - 0.5, 0, H - 1.001)
        u0, v0 = np.floor(uu).astype(int), np.floor(vv).astype(int)
        fu, fv = (uu - u0)[..., None], (vv - v0)[..., None]
        u1 = (u0 + 1) % W
        sample = (pano[v0, u0] * (1 - fu) * (1 - fv) + pano[v0, u1] * fu * (1 - fv) + pano[v0 + 1, u0] * (1 - fu) * fv +
                  pano[v0 + 1, u1] * fu * fv)
        worst = max(worst, float(np.abs(sample - img).mean()))
        assert img.std() > 0.02
    # the mean absolute error of the bilinear comparison per view is at most 0.008 here (the panorama's pixels are 2.8
    # degrees, the pinhole's 2.4, and the two projections order overlapping splats by r and by z respectively); a mirrored
    # longitude, a flipped latitude or a cx shifted by 8 pixels gives 0.04 or more on this scene
    assert worst < 0.015, worst


# ------------------------------------------------------------------ C ABI
def test_c_entry_points_check_their_arguments_before_any_cuda_call():
    lib = _lib.load()
    ok = ctypes.c_void_p(256)
    fargs = _lib.GsbForwardArgs(camera_width=100, camera_height=64, camera_intrinsics=ok, rasterized_image=ok, rgb_only=1)
    assert lib.gsb200_forward_equirect(ctypes.byref(fargs), None) == -1
    assert b"multiple of 16" in lib.gsb200_last_error()
    assert lib.gsb200_forward_equirect(ctypes.byref(_lib.GsbForwardArgs()), None) == -1
    assert b"null camera_intrinsics" in lib.gsb200_last_error()
    fargs.camera_width = 128
    ext = _lib.GsbExtraFeatureArgs(channels=17, features=ok, rasterized=ok)
    assert lib.gsb200_forward_equirect(ctypes.byref(fargs), ctypes.byref(ext)) == -1
    assert b"channels must be in 1..16" in lib.gsb200_last_error()
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, camera_width=100, camera_intrinsics=ok)
    assert lib.gsb200_backward_equirect(ctypes.byref(bargs), None, None, None, None) == -1
    assert b"multiple of 16" in lib.gsb200_last_error()
    bargs.camera_width = 128
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, camera_width=128,
                                   camera_intrinsics=ok)
    assert lib.gsb200_backward_equirect(ctypes.byref(compact), None, None, None, None) == -4
    assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    butterfly = _lib.GsbBackwardArgs(camera_width=128, camera_intrinsics=ok)
    assert lib.gsb200_backward_equirect(ctypes.byref(butterfly), None, None, None, None) == -4
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    assert lib.gsb200_backward_equirect(ctypes.byref(bargs), ok, None, None, None) == -1
    assert b"both NULL or both set" in lib.gsb200_last_error()
    assert lib.gsb200_backward_equirect(None, None, None, None, None) == -1
    # lens model 3 stays unknown to the lens calls: the panorama has its own entry points
    lens = _lib.GsbLensArgs(model=3)
    assert lib.gsb200_forward_lens(ctypes.byref(_lib.GsbForwardArgs()), None, ctypes.byref(lens)) == -1
    assert b"unknown lens model 3" in lib.gsb200_last_error()


# ------------------------------------------------------------------ Python surface
def test_lens_distortion_record_and_intrinsics():
    d = LensDistortion("equirectangular", ())
    assert d.coefficients == ()
    with pytest.raises(ValueError, match="0 coefficients"):
        LensDistortion("equirectangular", (0.1,))
    K = LensDistortion.equirectangular_intrinsics(2048, 1024)
    assert K.dtype == torch.float32 and K.shape == (3, 3)
    assert abs(2 * math.pi * float(K[0, 0]) - 2048) < 1e-3 and abs(math.pi * float(K[1, 1]) - 1024) < 1e-3
    assert K[0, 2] == 1024 and K[1, 2] == 512 and K[0, 1] == 0 and K[2].tolist() == [0, 0, 1]
    with pytest.raises(ValueError):
        LensDistortion.equirectangular_intrinsics(0, 16)
    with pytest.raises(KeyError):
        _lib.lens_args(d)


def _input(**camera):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_panorama_scene(64, 32, 64, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, ci.distortion, camera.get("rs"),
                    camera.get("mb"), camera.get("df"))
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_refuses_what_the_panorama_does_not_combine_with():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    from taichi_3d_gaussian_splatting_b200 import parallel
    Config = G.GaussianPointCloudRasterisationConfig
    inp = _input()
    for option in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion",
                   "differentiable_rolling_shutter", "differentiable_motion_blur", "differentiable_defocus"):
        with pytest.raises(ValueError, match=option):
            G(Config(), **{option: True})(inp)
    with pytest.raises(ValueError, match="gradient_exchange"):
        op = G(Config())
        op.gradient_exchange = object()
        op(inp)
    with pytest.raises(ValueError, match="butterfly"):
        G(Config(), backward_impl="butterfly")(inp)
    for camera, msg in ((dict(rs=RollingShutter((0.1, 0, 0), (0, 0, 0))), "rolling shutter"),
                        (dict(mb=MotionBlur((0.1, 0, 0), (0, 0, 0))), "motion blur"),
                        (dict(df=Defocus(0.05, 2.0)), "defocus")):
        with pytest.raises(ValueError, match=msg):
            G(Config())(_input(**camera))
    with pytest.raises(ValueError, match="point_filter_3d"):
        G(Config())(inp, point_filter_3d=torch.zeros(64))
    with pytest.raises(ValueError, match="parallel.render_views"):
        parallel.render_views(G(Config()), lambda i: inp, [0])


def _trainer(fused_step=False, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_panorama_scene(64, 32, 64, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    views = [(torch.zeros((3, 32, 64)), sc.q_pointcloud_camera, sc.t_pointcloud_camera, sc.camera_info)]

    class Factory:
        gradient_exchange = None

        def __init__(self, **kwargs):
            pass

    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=Factory, fused_step=fused_step)


def test_trainer_refuses_what_the_panorama_does_not_combine_with():
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(mip_filter_3d=True), "mip_filter_3d"),
                    (dict(pose_learning_rate=1e-3), "pose"), (dict(intrinsics_learning_rate=1e-3), "intrinsics"),
                    (dict(distortion_learning_rate=1e-3), "distortion"),
                    (dict(rolling_shutter_learning_rate=1e-3), "rolling_shutter_learning_rate"),
                    (dict(motion_blur_learning_rate=1e-3), "motion_blur_learning_rate"),
                    (dict(defocus_learning_rate=1e-3), "defocus_learning_rate")):
        with pytest.raises(ValueError, match=msg):
            _trainer(**kw)
    _trainer()


def test_dataset_and_downsampling_keep_a_full_turn(tmp_path):
    from PIL import Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets
    from taichi_3d_gaussian_splatting_b200.trainer import downsample_image_and_camera_info, downsample_targets
    records = []
    for i, (h, w) in enumerate(((100, 200), (1000, 2000), (40, 48))):
        img = tmp_path / f"p{i}.png"
        Image.fromarray(np.random.default_rng(i).integers(0, 255, (h, w, 3), dtype=np.uint8)).save(img)
        K = LensDistortion.equirectangular_intrinsics(w, h).tolist()
        rec = {"image_path": str(img), "T_pointcloud_camera": np.eye(4).tolist(), "camera_intrinsics": K,
               "camera_height": h, "camera_width": w, "camera_id": 0,
               "distortion": {"model": "equirectangular", "coefficients": []}}
        if i == 0:
            mask = tmp_path / "m0.png"
            Image.fromarray(np.full((h, w), 255, np.uint8)).save(mask)
            np.save(tmp_path / "d0.npy", np.full((h, w), 2.0, np.float32))
            rec.update(loss_weight_path=str(mask), depth_path=str(tmp_path / "d0.npy"))
        records.append(rec)
    path = tmp_path / "poses.json"
    path.write_text(json.dumps(records))
    ds = ImagePoseDataset(str(path), with_targets=True)
    for i, (h, w) in enumerate(((96, 192), (784, 1600), (32, 48))):
        image, _, _, ci, targets = ds[i]
        assert ci.distortion.model == "equirectangular"
        assert (ci.camera_height, ci.camera_width) == (h, w) and tuple(image.shape) == (3, h, w)
        assert abs(2 * math.pi * float(ci.camera_intrinsics[0, 0]) - w) < 1e-3 * w / 1000
        assert float(ci.camera_intrinsics[0, 2]) == pytest.approx(w / 2)
        assert float(ci.camera_intrinsics[1, 1]) == pytest.approx(h / math.pi, rel=1e-5)
        for factor in (2, 3):
            if ci.camera_height // factor < 16:
                continue
            im2, c2 = downsample_image_and_camera_info(image, ci, factor)
            assert c2.camera_width % 16 == 0 and c2.camera_height % 16 == 0
            assert tuple(im2.shape) == (3, c2.camera_height, c2.camera_width)
            assert abs(2 * math.pi * float(c2.camera_intrinsics[0, 0]) - c2.camera_width) < 1e-4 * c2.camera_width
            if i == 0:
                t2 = downsample_targets(targets, ci, factor)
                assert tuple(t2.loss_weight.shape) == (c2.camera_height, c2.camera_width)
                assert tuple(t2.depth.shape) == (c2.camera_height, c2.camera_width) and (t2.depth == 2.0).all()
    assert isinstance(ds[0][4], SupervisionTargets) and tuple(ds[0][4].loss_weight.shape) == (96, 192)
    # a pinhole view keeps today's crop
    _, ci = downsample_image_and_camera_info(torch.zeros((3, 100, 200)), make_scene(4, 100, 200, 0.1, 0).camera_info, 3)
    assert (ci.camera_height, ci.camera_width) == (32, 64)
