"""The 3D smoothing filter on the CPU: the torch rule of the views kernel and the bake against the loop reference, the C ABI's
argument rules (checked before any CUDA call), the trainer's recomputation and refusals on the oracle-backed module, and
the export."""
import ctypes
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.mcmc import MCMCConfig
from taichi_3d_gaussian_splatting_b200.mip_filter import _pose_matrices, bake_filter_3d, compute_filter_3d
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T

from mip_filter_reference import FilteredOracleModule, bake_reference, filter_reference, random_views
from oracle_module import OracleRasterisationModule
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR


def _rule_inputs(views):
    V, n_obj = len(views), views[0][0].shape[0]
    q = torch.cat([v[0] for v in views])
    t = torch.cat([v[1] for v in views])
    poses = _pose_matrices(q, t).view(V, n_obj, 3, 4).numpy()
    K = np.stack([v[2].camera_intrinsics.numpy() for v in views])
    sizes = [(v[2].camera_width, v[2].camera_height) for v in views]
    return poses, K, sizes


def test_torch_rule_is_the_loop_reference():
    g = torch.Generator().manual_seed(2)
    N = 700
    xyz = torch.rand((N, 3), generator=g) * torch.tensor([12.0, 8.0, 14.0]) - torch.tensor([6.0, 4.0, 3.0])
    mask = (torch.rand(N, generator=g) < 0.1).to(torch.int8)
    obj = torch.randint(0, 3, (N,), generator=g, dtype=torch.int32)
    views = random_views(7, 3, g)
    got = compute_filter_3d(xyz, mask, obj, views, 0.5, 0.2).numpy()
    ref = filter_reference(xyz.numpy(), mask.numpy(), obj.numpy(), *_rule_inputs(views), 0.5, 0.2)
    np.testing.assert_array_equal(got.view(np.int32), ref.view(np.int32))
    assert (got[mask.numpy() == 1] == 0).all() and (got[mask.numpy() == 0] > 0).all()


def test_margins_near_plane_unseen_and_no_row_seen():
    W, H = 64, 48
    K = torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.5, 0.0], [0.0, 0.0, 1.0]])  # u = x / z, v = 0.5 y / z
    view = (torch.tensor([[0.0, 0.0, 0.0, 1.0]]), torch.zeros((1, 3)), CameraInfo(K, H, W, 0))
    lo_w, hi_w = np.float32(-0.15) * np.float32(W), np.float32(1.15) * np.float32(W)
    lo_h = np.float32(-0.15) * np.float32(H)
    pts = [
        (lo_w, 0.0, 1.0),                                   # on the left margin: seen
        (np.nextafter(lo_w, np.float32(-1e9)), 0.0, 1.0),   # just outside: unseen
        (hi_w, 0.0, 1.0),                                   # on the right margin: seen
        (0.0, 2 * lo_h, 1.0),                               # on the top margin: seen
        (0.0, 0.0, 0.5),                                    # on the near plane: unseen
        (0.0, 0.0, float(np.nextafter(np.float32(0.5), np.float32(1)))),  # just beyond it: seen
        (0.0, 0.0, -2.0),                                   # behind the camera: unseen
        (1.0, 1.0, 4.0),                                    # seen, the largest d
    ]
    xyz = torch.tensor(pts, dtype=torch.float32)
    mask = torch.zeros(len(pts), dtype=torch.int8)
    obj = torch.zeros(len(pts), dtype=torch.int32)
    got = compute_filter_3d(xyz, mask, obj, [view], 0.5, 0.2).numpy()
    sv = np.sqrt(np.float32(0.2))
    seen = [True, False, True, True, False, True, False, True]
    for i, s in enumerate(seen):
        d = np.float32(pts[i][2]) / np.float32(1.0) if s else np.float32(4.0)
        assert got[i] == sv * d, (i, got[i], sv * d)
    # no row seen: every row 0
    got = compute_filter_3d(xyz[[1, 4, 6]], mask[:3], obj[:3], [view], 0.5, 0.2)
    assert (got == 0).all()
    # several focal lengths: the finest view (largest f) wins
    K2 = K.clone()
    K2[0, 0] = 4.0
    got = compute_filter_3d(xyz[[7]], mask[:1], obj[:1], [view, (view[0], view[1], CameraInfo(K2, H, W, 0))], 0.5, 0.2)
    assert float(got[0]) == float(sv * (np.float32(4.0) / np.float32(4.0)))


def test_bake_is_the_float64_reference():
    g = torch.Generator().manual_seed(4)
    feats = torch.randn((50, 56), generator=g)
    feats[:, 4:7] = feats[:, 4:7] * 0.5 - 3.0
    sigma = torch.rand(50, generator=g) * 0.1
    sigma[::4] = 0.0
    sigma[1] = float("nan")
    sigma[2] = -0.3
    got = bake_filter_3d(feats, sigma).numpy()
    ref = bake_reference(feats.numpy(), sigma.numpy())
    np.testing.assert_allclose(got, ref.astype(np.float32), rtol=2e-7, atol=2e-7)
    keep = (sigma.nan_to_num(0) <= 0).numpy()
    np.testing.assert_array_equal(got[keep], feats.numpy()[keep])
    # the opacity only goes down and the scales only up
    on = ~keep
    assert (got[on, 7] < feats.numpy()[on, 7]).all() and (got[on, 4:7] > feats.numpy()[on, 4:7]).all()


def test_abi_sizes_and_argument_rules():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 2)()
    lib.gsb200_abi_sizes_filter3d(sizes)
    assert tuple(sizes) == (ctypes.sizeof(_lib.GsbFilter3dArgs), ctypes.sizeof(_lib.GsbFilter3dViewsArgs))
    assert lib.gsb200_filter3d_temp_bytes(3, 2) == 256 + 6 * 80 and lib.gsb200_filter3d_temp_bytes(0, 1) == 0
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    temp = (ctypes.c_uint8 * 1024)()
    tp = (ctypes.addressof(temp) + 15) // 16 * 16

    def views(**kw):
        a = dict(num_points=4, pointcloud=p, point_invalid_mask=p, point_object_id=p, num_objects=1, num_views=2,
                 q_pointcloud_camera=p, t_pointcloud_camera=p, camera_intrinsics=p, camera_size=p, near_plane=0.1,
                 variance=0.2, filter3d=p, temp=tp, temp_bytes=512, stream=None)
        a.update(kw)
        return lib.gsb200_filter3d_from_views(ctypes.byref(_lib.GsbFilter3dViewsArgs(**a)))

    assert lib.gsb200_filter3d_from_views(None) == -1
    for bad in (dict(num_points=-1), dict(num_views=0), dict(num_objects=0), dict(pointcloud=None), dict(filter3d=None),
                dict(camera_size=None), dict(q_pointcloud_camera=p + 2), dict(filter3d=p + 1), dict(temp=None),
                dict(temp=tp + 4), dict(temp_bytes=100), dict(near_plane=-1.0), dict(near_plane=math.nan),
                dict(variance=-0.1), dict(variance=math.inf)):
        assert views(**bad) == -1, bad
    assert "filter3d_from_views" in lib.gsb200_last_error().decode()
    assert views(num_views=1 << 16, num_objects=1 << 15) == -4  # GSB_EUNSUPPORTED
    # the frame calls: a NULL or misaligned filter array is refused before anything else
    for fn, args in ((lib.gsb200_forward_filter3d, (None, None, None, None)),
                     (lib.gsb200_backward_filter3d, (None, None, None, None, None, None, None)),
                     (lib.gsb200_train_step_filter3d, (None, None, None, None, None))):
        for arr in (None, p + 2):
            rc = fn(*args, ctypes.byref(_lib.GsbFilter3dArgs(filter3d=arr)))
            assert rc == -1 and "filter3d" in lib.gsb200_last_error().decode()
    # the compact rows of the view-parallel exchange
    b = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_COMPACT_GRADS)
    assert lib.gsb200_backward_filter3d(ctypes.byref(b), None, None, None, None, None, None,
                                        ctypes.byref(_lib.GsbFilter3dArgs(filter3d=p))) == -4


@pytest.fixture(scope="module")
def problem():
    hidden = hidden_scene(n=200)
    return hidden, render_views(OracleRasterisationModule(GPCR.GaussianPointCloudRasterisationConfig()), hidden)


def _config(iters, **kw):
    cfg = train_config(iters, densify=kw.pop("densify", False))
    cfg.mip_filter_3d = True
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _recomputes(monkeypatch, trainer):
    at = []
    orig = trainer._update_filter_3d

    def spy():
        at.append(len(trainer.history))
        orig()
    monkeypatch.setattr(trainer, "_update_filter_3d", spy)
    return at


def test_trainer_recomputes_at_start_interval_and_refinements(problem, monkeypatch):
    hidden, views = problem
    FilteredOracleModule.calls.clear()
    cfg = _config(12, mip_filter_interval=5)
    trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=FilteredOracleModule)
    at = _recomputes(monkeypatch, trainer)
    trainer.train(log_interval=1)
    assert at == [0, 4, 9]  # before the first iteration, then after the 5th and the 10th (history entries so far)
    assert len(FilteredOracleModule.calls) == 12 and all(c is not None for c in FilteredOracleModule.calls)
    f = trainer.filter_3d()
    s = trainer.scene
    assert (f[s.point_invalid_mask == 1] == 0).all() and (f[s.point_invalid_mask == 0] > 0).all()
    FilteredOracleModule.calls.clear()
    trainer.validation()
    assert len(FilteredOracleModule.calls) == len(views) and all(torch.equal(c, trainer._filter_3d)
                                                                 for c in FilteredOracleModule.calls)


def test_trainer_recomputes_after_densification_and_mcmc(problem, monkeypatch):
    hidden, views = problem
    cfg = _config(25, densify=True, mip_filter_interval=1000)
    trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=FilteredOracleModule)
    at = _recomputes(monkeypatch, trainer)
    trainer.train(log_interval=1)
    ac = cfg.adaptive_controller_config
    assert at == [0] + [i for i in range(25) if i >= ac.num_iterations_warm_up and i % ac.num_iterations_densify == 0]
    cfg = _config(25, mip_filter_interval=1000, densification="mcmc",
                  mcmc_config=MCMCConfig(cap_max=300, refine_start=5, refine_every=5))
    trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=FilteredOracleModule)
    at = _recomputes(monkeypatch, trainer)
    trainer.train(log_interval=1)
    assert at == [0, 5, 10, 15, 20]  # after each refinement (the controller counts from iteration 0)
    s = trainer.scene
    f = trainer.filter_3d()
    assert int((s.point_invalid_mask == 0).sum()) > 200
    assert (f[s.point_invalid_mask == 0] > 0).all() and (f[s.point_invalid_mask == 1] == 0).all()


def test_trainer_refusals(problem):
    hidden, views = problem
    for kw, word in ((dict(pose_learning_rate=1e-3), "pose refinement"),
                     (dict(intrinsics_learning_rate=1e-3), "intrinsics refinement"),
                     (dict(mip_filter_variance=-1.0), "mip_filter_variance"),
                     (dict(mip_filter_variance=math.nan), "mip_filter_variance"),
                     (dict(mip_filter_interval=0), "mip_filter_interval")):
        with pytest.raises(ValueError, match=word):
            T(_config(2, **kw), initial_scene(hidden), views, rasterisation_factory=FilteredOracleModule)
    fish = [(v[0], v[1], v[2], CameraInfo(v[3].camera_intrinsics, v[3].camera_height, v[3].camera_width, 0,
                                          LensDistortion("fisheye", (0.01, 0.0, 0.0, 0.0)))) for v in views]
    with pytest.raises(ValueError, match="fisheye"):
        T(_config(2), initial_scene(hidden), fish, rasterisation_factory=FilteredOracleModule)
    ocv = [(v[0], v[1], v[2], CameraInfo(v[3].camera_intrinsics, v[3].camera_height, v[3].camera_width, 0,
                                         LensDistortion("opencv", (0.01, 0.0, 0.0, 0.0, 0.0)))) for v in views]
    with pytest.raises(ValueError, match="distortion refinement"):
        T(_config(2, distortion_learning_rate=1e-3), initial_scene(hidden), ocv, rasterisation_factory=FilteredOracleModule)

    class Exchanging(FilteredOracleModule):
        gradient_exchange = object()
    with pytest.raises(ValueError, match="view-parallel"):
        T(_config(2), initial_scene(hidden), views, rasterisation_factory=Exchanging)


def test_to_ply_bakes_the_filter_and_keeps_todays_bytes_without_it(tmp_path):
    from taichi_3d_gaussian_splatting_b200.scene_io import GaussianPointCloudScene, read_ply_vertices
    g = torch.Generator().manual_seed(8)
    n = 40
    feats = torch.randn((n, 56), generator=g)
    feats[:, 4:7] -= 3.0
    scene = GaussianPointCloudScene(torch.randn((n, 3), generator=g).numpy(), GaussianPointCloudScene.PointCloudSceneConfig(),
                                    point_cloud_features=feats)
    scene.point_invalid_mask[::6] = 1
    plain, again = tmp_path / "a.ply", tmp_path / "b.ply"
    scene.to_ply(str(plain))
    scene.to_ply(str(again), filter_3d=None)
    assert plain.read_bytes() == again.read_bytes()
    sigma = torch.rand(n, generator=g) * 0.05
    baked_path = tmp_path / "c.ply"
    scene.to_ply(str(baked_path), filter_3d=sigma)
    v = read_ply_vertices(str(baked_path))
    keep = (scene.point_invalid_mask == 0).numpy()
    ref = bake_reference(scene.point_cloud_features.detach().numpy()[keep], sigma.numpy()[keep])
    np.testing.assert_allclose(v["opacity"], ref[:, 7], rtol=1e-6, atol=1e-6)
    for i in range(3):
        np.testing.assert_allclose(v[f"scale_{i}"], ref[:, 4 + i], rtol=1e-6, atol=1e-6)
    p0 = read_ply_vertices(str(plain))
    np.testing.assert_array_equal(v["x"], p0["x"])
    np.testing.assert_array_equal(v["f_dc_0"], p0["f_dc_0"])


def test_operator_and_compute_refuse_what_the_filter_does_not_take():
    from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
    sc = make_scene(20, 32, 32, 0.05, 0)
    f3d = torch.zeros(20)
    inp = GPCR.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=sc.camera_info, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)
    for kw, word in ((dict(lens_coefficients=torch.zeros(5)), "lens_coefficients"),
                     (dict(rolling_shutter_motion=torch.zeros(6)), "rolling_shutter_motion")):
        op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
        with pytest.raises(ValueError, match=word):
            op(inp, point_filter_3d=f3d, **kw)
    for flag in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion",
                 "differentiable_rolling_shutter"):
        op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), **{flag: True})
        with pytest.raises(ValueError, match=flag):
            op(inp, point_filter_3d=f3d)
    view = [(sc.q_pointcloud_camera, sc.t_pointcloud_camera, sc.camera_info)]
    for args, word in (((sc.point_cloud, sc.point_invalid_mask, sc.point_object_id.long()), "point_object_id"),
                       ((sc.point_cloud, sc.point_invalid_mask.int(), sc.point_object_id), "point_invalid_mask"),
                       ((sc.point_cloud, sc.point_invalid_mask, sc.point_object_id[:10]), "point_object_id"),
                       ((sc.point_cloud.double(), sc.point_invalid_mask, sc.point_object_id), "point_cloud")):
        with pytest.raises(ValueError, match=word):
            compute_filter_3d(*args, view, 0.8)
