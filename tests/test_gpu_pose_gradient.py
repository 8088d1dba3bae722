"""-m gpu: the camera-pose gradient of the CUDA operator (``differentiable_pose=True``, ``gsb200_backward_pose``).

Against torch autograd of the multi-object float64 dense evaluator (``torch_reference_pose``) under the gradient gate of
test_gpu_parity (|a - b| <= 1e-3 |b| + 1e-5 max|b|), for image, depth, alpha and feature-map losses and for objects whose
points share warps; an image loss under both loop-A kernels; at C3 full size dL/dt_pc = -sum dL/dxyz and bit-identical
repeats; a relocalisation fit; and pose refinement in the trainer."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer

from gpu_helpers import cuda_scene, n
from helpers import grad_close
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_pose import dense_render_objects

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, objects=1):
    """As in test_pose_gradient_cpu: with objects > 1 the scene rows cycle through the objects (one with a non-unit q)."""
    sc = make_scene(n, h, w, sigma, seed, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    if objects > 1:
        sc.point_object_id = (torch.arange(n) % objects).to(torch.int32)
        qs, ts = [sc.q_pointcloud_camera[0]], [sc.t_pointcloud_camera[0]]
        for k in range(1, objects):
            a = math.radians(3.0 * k) / 2
            qs.append(torch.tensor([math.sin(a) * 0.6, math.sin(a) * 0.8, 0.0, math.cos(a)]) * (1.0 + 0.03 * k))
            ts.append(torch.tensor([0.15 * k, -0.1 * k, 0.2 * k]))
        sc.q_pointcloud_camera = torch.stack(qs).float().contiguous()
        sc.t_pointcloud_camera = torch.stack(ts).float().contiguous()
    return sc


def _render(op, sc, q, t, band=3, extra=None):
    inp = Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                point_invalid_mask=sc.point_invalid_mask, camera_info=sc.camera_info, q_pointcloud_camera=q,
                t_pointcloud_camera=t, color_max_sh_band=band)
    return op(inp) if extra is None else op(inp, point_extra_features=extra)


def _cuda_and_dense(scene, kind, exact_exp, seed, backward_impl="transposed", band=3):
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    q = sc.q_pointcloud_camera.clone().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().requires_grad_(True)
    op = GPCR(Config(), exact_exp=exact_exp, backward_impl=backward_impl, differentiable_pose=True,
              differentiable_depth=kind == "depth", differentiable_alpha=kind == "alpha")
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    extra = g_map = None
    if kind == "features":
        extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g)
        g_map = torch.randn((H, W, 5), generator=g)
    outs = _render(op, sc, q, t, band, None if extra is None else extra.cuda())
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
    qd = scene.q_pointcloud_camera.clone().double().requires_grad_(True)
    td = scene.t_pointcloud_camera.clone().double().requires_grad_(True)
    image, aux = dense_render_objects(scene.point_cloud.double(), sc.point_cloud_features.detach().cpu().double(),
                                      scene.point_invalid_mask, scene.point_object_id, scene.camera_info.camera_intrinsics,
                                      qd, td, H, W)
    dl = (image * g_img.double()).sum()
    if kind == "depth":
        dl = dl + (differentiable_depth(aux, H, W)[0] * g_aux.double()).sum()
    elif kind == "alpha":
        dl = dl + (aux["acc_alpha"] * g_aux.double()).sum()
    elif kind == "features":
        dl = dl + (feature_map(aux, extra.double(), H, W) * g_map.double()).sum()
    dl.backward()
    return sc, q, t, qd.grad.numpy(), td.grad.numpy()


def _check(q, t, eq, et):
    for got, want in ((n(q.grad), eq), (n(t.grad), et)):
        ok = grad_close(got, want)
        assert ok[0], (got, want, ok)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("exact_exp", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_pose_gradient_matches_dense_autograd(seed, band, exact_exp, kind):
    sc, q, t, eq, et = _cuda_and_dense(_scene(seed), kind, exact_exp, seed, band=band)
    _check(q, t, eq, et)
    ok = grad_close(n(t.grad)[0], -n(sc.point_cloud.grad).astype(np.float64).sum(0))  # one object, unit q
    assert ok[0], ok


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
def test_pose_gradient_of_interleaved_objects(kind):
    _, q, t, eq, et = _cuda_and_dense(_scene(17, objects=3), kind, False, 17)
    _check(q, t, eq, et)


@pytest.mark.parametrize("backward_impl", ["butterfly", "transposed"])
def test_image_loss_pose_gradient_under_both_loop_a_kernels(backward_impl):
    _, q, t, eq, et = _cuda_and_dense(_scene(11, objects=2), "image", False, 11, backward_impl=backward_impl)
    _check(q, t, eq, et)


def test_frozen_scene_and_default_operator():
    scene = _scene(12)
    sc = cuda_scene(scene)  # the scene needs no gradient: relocalisation
    q = sc.q_pointcloud_camera.clone().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().requires_grad_(True)
    image = _render(GPCR(Config(), differentiable_pose=True), sc, q, t)[0]
    image.sum().backward()
    assert q.grad is not None and t.grad is not None and float(t.grad.abs().sum()) > 0
    q2 = sc.q_pointcloud_camera.clone().requires_grad_(True)
    sc2 = cuda_scene(scene, requires_grad=True)
    image = _render(GPCR(Config()), sc2, q2, sc2.t_pointcloud_camera)[0]
    image.sum().backward()
    assert q2.grad is None  # off by default: as before


def _same_or_close(a, b):
    """Loop A adds each splat's partials with float atomics, so two backward passes of one frame may differ in the last
    bits of the accumulator rows.  Where the dense gradients of both passes are bit-identical (the per-point kernels read
    the same rows), the compared tensor must be bit-identical too; otherwise it agrees up to that rounding."""
    return torch.equal(a, b) or bool(torch.allclose(a, b, rtol=1e-4, atol=1e-5 * float(b.abs().max())))


def test_full_size_translation_identity_determinism_and_other_outputs():
    """C3: dL/dt_pc = -sum_i dL/dxyz_i (one object, unit q) to the gradient criterion; repeated backward passes give
    bit-identical pose gradients whenever loop A's rows are the same; the image and the dense gradients equal the default
    operator's on the same inputs."""
    base = make_scene(**CONFIGS["C3"]).to("cuda")
    feats0 = base.point_cloud_features.clone()
    runs = []
    for pose in (True, False):
        xyz = base.point_cloud.clone().requires_grad_(True)
        feats = feats0.clone().requires_grad_(True)  # each forward normalises its own copy in place
        q = base.q_pointcloud_camera.clone().requires_grad_(pose)
        t = base.t_pointcloud_camera.clone().requires_grad_(pose)
        op = GPCR(Config(), differentiable_pose=pose)
        image = op(Input(point_cloud=xyz, point_cloud_features=feats, point_object_id=base.point_object_id,
                         point_invalid_mask=base.point_invalid_mask, camera_info=base.camera_info, q_pointcloud_camera=q,
                         t_pointcloud_camera=t, color_max_sh_band=3))[0]
        g_img = torch.randn(image.shape, generator=torch.Generator().manual_seed(3)).cuda()
        inputs = [xyz, feats] + ([q, t] if pose else [])
        rs = [torch.autograd.grad([image], inputs, [g_img], retain_graph=True) for _ in range(3)]
        for r in rs[1:]:
            same_rows = torch.equal(r[0], rs[0][0]) and torch.equal(r[1], rs[0][1])
            for a, b in zip(r, rs[0]):
                assert torch.equal(a, b) if same_rows else _same_or_close(a, b)
        runs.append((image.detach(), rs[0]))
    (image_p, rp), (image_0, r0) = runs
    ok = grad_close(n(rp[3])[0], -n(rp[0]).astype(np.float64).sum(0))
    print(f"C3 dL/dt_pc {n(rp[3])[0]}  -sum dL/dxyz {-n(rp[0]).astype(np.float64).sum(0)}  dL/dq_pc {n(rp[2])[0]}")
    assert ok[0], ok
    assert torch.equal(image_p, image_0)
    assert _same_or_close(rp[0], r0[0]) and _same_or_close(rp[1], r0[1])


def _quat_mul(a, b):
    x0, y0, z0, w0 = a.unbind(-1)
    x1, y1, z1, w1 = b.unbind(-1)
    return torch.stack([w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1, w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1,
                        w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1, w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1], -1)


def _perturb(q, t, deg, shift, axis):
    a = torch.tensor(axis, dtype=torch.float32)
    a = a / a.norm()
    half = math.radians(deg) / 2
    dq = torch.cat([a * math.sin(half), torch.tensor([math.cos(half)])]).to(q.device)
    return _quat_mul(dq[None], q), t + torch.tensor(shift, dtype=torch.float32, device=t.device)[None]


def _rot_err_deg(q, q_true):
    qn = q / q.norm(dim=-1, keepdim=True)
    return float(2 * torch.rad2deg(torch.acos(torch.clamp((qn * q_true).sum(-1).abs(), max=1.0))).mean())


def test_relocalisation_fit_recovers_the_pose():
    """Render a scene from a known pose, perturb the pose by 2 deg and by 2 % of the scene depth (0.12 on a mean depth of
    about 6), and fit (q, t) alone with Adam on the image L1.  On an H100 80GB HBM3 (700 W) the rotation error went
    2.000 -> 1.890, 0.358, 0.105, 0.040, 0.000 deg at steps 1, 21, 41, 61, 81 and 0.0000 deg after 100 steps; the translation
    error 0.1175 -> 0.1161, 0.0602, 0.0132, 0.0029, 0.0009 and 0.00056; the L1 0.0731 -> 0.0007."""
    scene = make_scene(3000, 64, 96, 0.08, 21, sh_degree=0)
    scene.point_cloud_features[:, 7] += 2.0
    sc = cuda_scene(scene)
    op = GPCR(Config(), differentiable_pose=True)
    q_true, t_true = sc.q_pointcloud_camera.clone(), sc.t_pointcloud_camera.clone()
    with torch.no_grad():
        target = _render(op, sc, q_true, t_true)[0]
    q0, t0 = _perturb(q_true, t_true, 2.0, (0.07, -0.05, 0.08), (0.3, 1.0, 0.2))
    q, t = q0.clone().requires_grad_(True), t0.clone().requires_grad_(True)
    opt = torch.optim.Adam([{"params": [q], "lr": 1e-3}, {"params": [t], "lr": 5e-3}])
    rot, trans, losses = [], [], []
    for _ in range(100):
        loss = (_render(op, sc, q, t)[0] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        with torch.no_grad():
            q.div_(q.norm(dim=-1, keepdim=True))
        losses.append(float(loss.detach()))
        rot.append(_rot_err_deg(q.detach(), q_true))
        trans.append(float((t.detach() - t_true).norm()))
    rot0, trans0 = _rot_err_deg(q0, q_true), float((t0 - t_true).norm())
    print(f"relocalisation: rotation {rot0:.3f} -> {rot[-1]:.4f} deg, translation {trans0:.4f} -> {trans[-1]:.5f}, "
          f"L1 {losses[0]:.5f} -> {losses[-1]:.5f}; rotation every 20 steps {[round(r, 4) for r in rot[::20]]}, "
          f"translation {[round(x, 5) for x in trans[::20]]}")
    assert np.isfinite(losses).all()
    assert rot[-1] < 0.25 * rot0 and trans[-1] < 0.25 * trans0


def _trainer_views(hidden, perturb):
    from trainer_helpers import poses, render_views
    views = render_views(GPCR(Config()), hidden, device="cuda")
    out = []
    for k, (img, q, t, cam) in enumerate(views):
        if perturb and k > 0:
            q, t = _perturb(q, t, 1.5, (0.04 * (-1) ** k, 0.03, -0.04), (1.0, 0.5 * k, -0.3))
        out.append((img, q.contiguous(), t.contiguous(), cam))
    return out, [(q.cuda(), t.cuda()) for q, t in poses()]


def _frozen_config(iters, pose_lr):
    C = GaussianPointCloudTrainer.TrainConfig
    cfg = C(num_iterations=iters, feature_learning_rate=0.0, position_learning_rate=0.0, initial_downsample_factor=1,
            pose_learning_rate=pose_lr)
    cfg.adaptive_controller_config.num_iterations_warm_up = 10 ** 9
    cfg.loss_function_config.enable_regularization = False
    return cfg


def _pose_errors(poses, truth):
    rot = [_rot_err_deg(q, qt) for (q, _), (qt, _) in zip(poses[1:], truth[1:])]
    trans = [float((t - tt).norm()) for (_, t), (_, tt) in zip(poses[1:], truth[1:])]
    return float(np.mean(rot)), float(np.mean(trans))


def test_trainer_refines_perturbed_poses_of_a_frozen_scene():
    """Views 1..3 rendered from their poses, then perturbed by 1.5 deg and about 0.06; the scene is the one that rendered
    them and stays frozen.  On an H100 80GB HBM3 (700 W) 240 iterations took the mean rotation error from 1.500 to 0.158 deg
    and the mean translation error from 0.0640 to 0.0126."""
    from trainer_helpers import hidden_scene
    from taichi_3d_gaussian_splatting_b200.trainer import Scene
    hidden = hidden_scene(n=600)
    views, truth = _trainer_views(hidden, perturb=True)
    scene = Scene(hidden.point_cloud.cuda().requires_grad_(True), hidden.point_cloud_features.cuda().requires_grad_(True),
                  hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda())
    trainer = GaussianPointCloudTrainer(_frozen_config(240, 2e-3), scene, views)
    rot0, trans0 = _pose_errors(trainer.refined_poses(), truth)
    trainer.train()
    rot1, trans1 = _pose_errors(trainer.refined_poses(), truth)
    print(f"trainer pose refinement: mean rotation error {rot0:.3f} -> {rot1:.4f} deg, translation {trans0:.4f} -> {trans1:.5f}")
    assert rot1 < 0.25 * rot0 and trans1 < 0.25 * trans0
    assert torch.equal(trainer.refined_poses()[0][0], views[0][1])  # view 0 is the fixed reference frame


def test_trainer_history_without_pose_refinement_is_unchanged():
    """pose_learning_rate = 0 runs the trainer's previous loop.  Loop A adds a splat's partials with float atomics, so two
    runs agree up to rounding; the bound is far below any change of the loop."""
    from trainer_helpers import hidden_scene, initial_scene, train_config
    hidden = hidden_scene(n=400)
    views, _ = _trainer_views(hidden, perturb=False)
    hist = []
    for cfg in (train_config(30), train_config(30)):
        if hist:
            cfg.pose_learning_rate = 0.0
        tr = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views)
        hist.append(tr.train(log_interval=1))
    assert [h["num_valid_points"] for h in hist[0]] == [h["num_valid_points"] for h in hist[1]]
    for key in ("loss", "l1", "psnr"):
        a, b = np.array([h[key] for h in hist[0]]), np.array([h[key] for h in hist[1]])
        assert np.abs(a - b).max() <= 1e-5 * np.abs(a).max(), key
