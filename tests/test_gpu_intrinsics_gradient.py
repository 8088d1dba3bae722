"""-m gpu: the camera-intrinsics gradient of the CUDA operator (``differentiable_intrinsics=True``, ``gsb200_backward_calib``).

Against torch autograd of the multi-object float64 dense evaluator (``torch_reference_pose``) under the gradient gate of
test_gpu_parity (|a - b| <= 1e-3 |b| + 1e-5 max|b|), for image, depth, alpha and feature-map losses, intrinsics alone and
with the pose, a K with skew and an off-centre principal point, objects whose points share warps, and an image loss under
both loop-A kernels; at C3 full size the principal-point identity dL/dc = sum dL/duv, row 2 zero and bit-identical repeats;
the default operator unchanged; a calibration fit; and intrinsics refinement in the trainer."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer

from gpu_helpers import cuda_scene, n
from helpers import grad_close
from test_gpu_pose_gradient import _same_or_close, _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_pose import dense_render_objects

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput


def _general_K(scene):
    """The scene's K with skew, a non-zero K[1,0] and an off-centre principal point."""
    K = scene.camera_info.camera_intrinsics.clone()
    K[0, 1], K[1, 0] = 2.5, -1.5
    K[0, 2] += 5.0
    K[1, 2] -= 4.0
    scene.camera_info.camera_intrinsics = K.contiguous()
    return scene


def _render(op, sc, K, q=None, t=None, band=3, extra=None):
    ci = sc.camera_info
    inp = Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                point_invalid_mask=sc.point_invalid_mask,
                camera_info=CameraInfo(K, ci.camera_height, ci.camera_width, ci.camera_id),
                q_pointcloud_camera=sc.q_pointcloud_camera if q is None else q,
                t_pointcloud_camera=sc.t_pointcloud_camera if t is None else t, color_max_sh_band=band)
    return op(inp) if extra is None else op(inp, point_extra_features=extra)


def _cuda_and_dense(scene, kind, exact_exp, seed, backward_impl="transposed", band=3, pose=False):
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    K = sc.camera_info.camera_intrinsics.clone().requires_grad_(True)
    q = sc.q_pointcloud_camera.clone().requires_grad_(pose)
    t = sc.t_pointcloud_camera.clone().requires_grad_(pose)
    op = GPCR(Config(), exact_exp=exact_exp, backward_impl=backward_impl, differentiable_intrinsics=True,
              differentiable_pose=pose, differentiable_depth=kind == "depth", differentiable_alpha=kind == "alpha")
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    extra = g_map = None
    if kind == "features":
        extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g)
        g_map = torch.randn((H, W, 5), generator=g)
    outs = _render(op, sc, K, q, t, band, None if extra is None else extra.cuda())
    loss = (outs[0] * g_img.cuda()).sum()
    g_aux = None
    if kind == "depth":
        g_aux = torch.randn((H, W), generator=g)
        loss = loss + (outs[1] * g_aux.cuda()).sum()
    elif kind == "alpha":
        g_aux = torch.randn((H, W), generator=g)
        loss = loss + (outs[3] * g_aux.cuda()).sum()
    elif kind == "features":
        loss = loss + (outs[-1] * g_map.cuda()).sum()
    loss.backward()
    # float64 autograd on the quaternions the forward normalised in place
    Kd = scene.camera_info.camera_intrinsics.clone().double().requires_grad_(True)
    qd = scene.q_pointcloud_camera.clone().double().requires_grad_(True)
    td = scene.t_pointcloud_camera.clone().double().requires_grad_(True)
    image, aux = dense_render_objects(scene.point_cloud.double(), sc.point_cloud_features.detach().cpu().double(),
                                      scene.point_invalid_mask, scene.point_object_id, Kd, qd, td, H, W)
    dl = (image * g_img.double()).sum()
    if kind == "depth":
        dl = dl + (differentiable_depth(aux, H, W)[0] * g_aux.double()).sum()
    elif kind == "alpha":
        dl = dl + (aux["acc_alpha"] * g_aux.double()).sum()
    elif kind == "features":
        dl = dl + (feature_map(aux, extra.double(), H, W) * g_map.double()).sum()
    dl.backward()
    return K, q, t, Kd.grad.numpy(), qd.grad.numpy(), td.grad.numpy()


def _check(K, q, t, eK, eq, et, pose):
    ok = grad_close(n(K.grad), eK)
    assert ok[0], (n(K.grad), eK, ok)
    assert (n(K.grad)[2] == 0).all()
    if pose:
        for got, want in ((n(q.grad), eq), (n(t.grad), et)):
            ok = grad_close(got, want)
            assert ok[0], (got, want, ok)
    else:
        assert q.grad is None and t.grad is None


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("exact_exp", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_intrinsics_gradient_matches_dense_autograd(seed, band, exact_exp, kind, pose):
    _check(*_cuda_and_dense(_scene(seed), kind, exact_exp, seed, band=band, pose=pose), pose)


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_intrinsics_gradient_with_skew_and_off_centre_principal_point(kind, pose):
    K, q, t, eK, eq, et = _cuda_and_dense(_general_K(_scene(14)), kind, False, 14, pose=pose)
    assert (np.abs(eK[:2]) > 0).all()
    _check(K, q, t, eK, eq, et, pose)


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_intrinsics_gradient_of_interleaved_objects(kind, pose):
    _check(*_cuda_and_dense(_scene(17, objects=3), kind, False, 17, pose=pose), pose)


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("backward_impl", ["butterfly", "transposed"])
def test_image_loss_intrinsics_gradient_under_both_loop_a_kernels(backward_impl, pose):
    _check(*_cuda_and_dense(_general_K(_scene(11, objects=2)), "image", False, 11, backward_impl=backward_impl, pose=pose),
           pose)


def test_frozen_scene_and_a_K_built_from_parameters():
    """Only (fx, fy, cx, cy) require grad, and K is assembled from them by torch ops: the backward runs and returns the
    gradient to the parameters through K."""
    scene = _scene(12)
    sc = cuda_scene(scene)
    K0 = sc.camera_info.camera_intrinsics
    p = torch.stack([K0[0, 0], K0[1, 1], K0[0, 2], K0[1, 2]]).clone().requires_grad_(True)
    zero = torch.zeros((), device="cuda")
    K = torch.stack([torch.stack([p[0], zero, p[2]]), torch.stack([zero, p[1], p[3]]),
                     torch.stack([zero, zero, zero + 1])])
    image = _render(GPCR(Config(), differentiable_intrinsics=True), sc, K)[0]
    image.sum().backward()
    assert p.grad is not None and float(p.grad.abs().sum()) > 0


def test_full_size_principal_point_identity_determinism_and_flag_off():
    """C3: dL/dK[0,2] = sum dL/du and dL/dK[1,2] = sum dL/dv over the backward hook's (M,2) dL/duv, summed in float64, to
    1e-5 of sum |dL/duv|; row 2 exactly 0; repeated backward passes give bit-identical intrinsics gradients whenever loop
    A's rows are the same.  With the flag off, the image and the scene gradients equal the flag-on run's and K gets no
    gradient."""
    base = make_scene(**CONFIGS["C3"]).to("cuda")
    feats0 = base.point_cloud_features.clone()
    ci = base.camera_info
    runs = []
    for on in (True, False):
        xyz = base.point_cloud.clone().requires_grad_(True)
        feats = feats0.clone().requires_grad_(True)  # each forward normalises its own copy in place
        K = ci.camera_intrinsics.clone().requires_grad_(True)
        seen = []
        op = GPCR(Config(), backward_valid_point_hook=lambda h: seen.append(h.grad_viewspace.double().clone()),
                  differentiable_intrinsics=on)
        image = op(Input(point_cloud=xyz, point_cloud_features=feats, point_object_id=base.point_object_id,
                         point_invalid_mask=base.point_invalid_mask,
                         camera_info=CameraInfo(K, ci.camera_height, ci.camera_width, ci.camera_id),
                         q_pointcloud_camera=base.q_pointcloud_camera, t_pointcloud_camera=base.t_pointcloud_camera,
                         color_max_sh_band=3))[0]
        g_img = torch.randn(image.shape, generator=torch.Generator().manual_seed(3)).cuda()
        rs = [torch.autograd.grad([image], [xyz, feats, K], [g_img], retain_graph=True, allow_unused=True)
              for _ in range(3)]
        if on:
            for r, guv in zip(rs, seen):
                gK = n(r[2]).astype(np.float64)
                want, scale = n(guv.sum(0)), n(guv.abs().sum(0))
                print(f"C3 dL/dK[:2,2] {gK[:2, 2]}  sum dL/duv {want}  sum |dL/duv| {scale}")
                assert (np.abs(gK[:2, 2] - want) <= 1e-5 * scale).all()
                assert (gK[2] == 0).all()
            for r in rs[1:]:
                same_rows = torch.equal(r[0], rs[0][0]) and torch.equal(r[1], rs[0][1])
                for a, b in zip(r, rs[0]):
                    assert torch.equal(a, b) if same_rows else _same_or_close(a, b)
        else:
            assert all(r[2] is None for r in rs)  # off: K gets no gradient, as before
        runs.append((image.detach(), rs[0]))
    (image_1, r1), (image_0, r0) = runs
    assert torch.equal(image_1, image_0)
    assert _same_or_close(r1[0], r0[0]) and _same_or_close(r1[1], r0[1])


def test_calibration_fit_recovers_focal_lengths_and_principal_point():
    """Frozen scene, true pose, targets rendered with the true K.  Start with fx and fy 5 % high and cx, cy 6 px off, and
    fit (fx, fy, cx, cy) alone with Adam on the image L1; each error must fall to at most 5 % of its initial value.  On an
    H100 80GB HBM3 (700 W) the errors went (2.88, 2.88, 6, 6) px -> (0.0002, 0.0001, 0.0001, 0.0007) px in 300 steps and the L1
    0.091 -> 0.00002."""
    scene = make_scene(3000, 64, 96, 0.08, 21, sh_degree=0)
    scene.point_cloud_features[:, 7] += 2.0
    sc = cuda_scene(scene)
    op = GPCR(Config(), differentiable_intrinsics=True)
    K_true = sc.camera_info.camera_intrinsics.clone()
    true = torch.stack([K_true[0, 0], K_true[1, 1], K_true[0, 2], K_true[1, 2]])
    with torch.no_grad():
        target = _render(op, sc, K_true)[0]
    p0 = true * torch.tensor([1.05, 1.05, 1.0, 1.0], device="cuda") + torch.tensor([0.0, 0.0, 6.0, -6.0], device="cuda")
    p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p], lr=0.1)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.99)
    zero = torch.zeros((), device="cuda")
    errs, losses = [], []
    for _ in range(300):
        K = torch.stack([torch.stack([p[0], zero, p[2]]), torch.stack([zero, p[1], p[3]]),
                         torch.stack([zero, zero, zero + 1])])
        loss = (_render(op, sc, K)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        losses.append(float(loss.detach()))
        errs.append(n((p.detach() - true).abs()))
    err0 = n((p0 - true).abs())
    print(f"calibration: |error| (fx, fy, cx, cy) {err0} -> {errs[-1]}, L1 {losses[0]:.5f} -> {losses[-1]:.5f}; every 50 "
          f"steps {[np.round(e, 4).tolist() for e in errs[::50]]}")
    assert np.isfinite(losses).all()
    assert (errs[-1] <= 0.05 * err0).all(), (err0, errs[-1])


def _camera_views(hidden):
    """The four views of trainer_helpers, views 0 and 2 from camera 0 and views 1 and 3 from camera 1, both cameras with
    the hidden scene's K.  Returns the views and the per-camera perturbed K."""
    from trainer_helpers import render_views
    views = render_views(GPCR(Config()), hidden, device="cuda")
    K = views[0][3].camera_intrinsics
    bad = {0: K.clone(), 1: K.clone()}
    bad[0][0, 0] *= 1.04
    bad[0][0, 2] += 3.0
    bad[1][1, 1] *= 0.96
    bad[1][1, 2] -= 3.0
    bad[1][0, 2] -= 2.0
    out = []
    for k, (img, q, t, cam) in enumerate(views):
        out.append((img, q.contiguous(), t.contiguous(),
                    CameraInfo(bad[k % 2].contiguous(), cam.camera_height, cam.camera_width, k % 2)))
    return out, K


def _frozen_config(iters, intr_lr):
    C = GaussianPointCloudTrainer.TrainConfig
    cfg = C(num_iterations=iters, feature_learning_rate=0.0, position_learning_rate=0.0, initial_downsample_factor=1,
            intrinsics_learning_rate=intr_lr)
    cfg.adaptive_controller_config.num_iterations_warm_up = 10 ** 9
    cfg.loss_function_config.enable_regularization = False
    return cfg


def test_trainer_refines_the_intrinsics_of_each_camera_on_a_frozen_scene():
    """Views 0 and 2 from camera 0 (fx 4 % high, cx 3 px off), views 1 and 3 from camera 1 (fy 4 % low, cx and cy off), on
    the frozen scene that rendered them with the true K.  On an H100 80GB HBM3 (700 W) 240 iterations took the per-camera
    |fx| + |fy| + |cx| + |cy| error from 5.30 and 7.30 px to 0.015 and 0.053 px."""
    from trainer_helpers import hidden_scene
    from taichi_3d_gaussian_splatting_b200.trainer import Scene
    hidden = hidden_scene(n=600)
    views, K_true = _camera_views(hidden)
    scene = Scene(hidden.point_cloud.cuda().requires_grad_(True), hidden.point_cloud_features.cuda().requires_grad_(True),
                  hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda())
    K_view0 = views[0][3].camera_intrinsics.clone()
    trainer = GaussianPointCloudTrainer(_frozen_config(240, 2e-3), scene, views)

    def err(Ks):  # per camera: |fx| + |fy| + |cx| + |cy| error in pixels
        return [float((Ks[k] - K_true)[[0, 1, 0, 1], [0, 1, 2, 2]].abs().sum()) for k in (0, 1)]

    before = err(trainer.refined_intrinsics())
    trainer.train()
    after = err(trainer.refined_intrinsics())
    print(f"trainer intrinsics refinement: per-camera error {before} -> {after} px")
    assert all(a < 0.5 * b for a, b in zip(after, before))
    Ks = trainer.refined_intrinsics()
    assert torch.equal(Ks[0], Ks[2]) and torch.equal(Ks[1], Ks[3])  # one correction per camera
    assert torch.equal(views[0][3].camera_intrinsics, K_view0)  # the views' own K is left as given


def test_trainer_history_without_intrinsics_refinement_is_unchanged():
    """intrinsics_learning_rate = 0 runs the trainer's previous loop.  Loop A adds a splat's partials with float atomics,
    so two runs agree up to rounding; the bound is far below any change of the loop."""
    from trainer_helpers import hidden_scene, initial_scene, render_views, train_config
    hidden = hidden_scene(n=400)
    views = render_views(GPCR(Config()), hidden, device="cuda")
    hist = []
    for cfg in (train_config(30), train_config(30)):
        if hist:
            cfg.intrinsics_learning_rate = 0.0
        tr = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views)
        hist.append(tr.train(log_interval=1))
    assert [h["num_valid_points"] for h in hist[0]] == [h["num_valid_points"] for h in hist[1]]
    for key in ("loss", "l1", "psnr"):
        a, b = np.array([h[key] for h in hist[0]]), np.array([h[key] for h in hist[1]])
        assert np.abs(a - b).max() <= 1e-5 * np.abs(a).max(), key
