"""Equirectangular panoramas on the GPU (``gsb200_forward_equirect`` / ``gsb200_backward_equirect`` through the operator):
the per-point records at 2048 x 1024 with 1e5 Gaussians and the images and gradients of small panoramas against the float64
evaluator (``equirect_reference``), roll invariance at full size, and a fit: a scene trained from panoramas of the shell
scene with the autograd trainer, checked on held-out pinhole views."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import CameraInfo
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import LensDistortion
from taichi_3d_gaussian_splatting_b200.synthetic import make_panorama_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from equirect_reference import dense_render_equirect, jacobian, project
from torch_reference import postprocess_feature_grads, quat_to_rot
from torch_reference_pose import camera_from_pose

pytestmark = pytest.mark.gpu


def _input(sc, device="cuda", q=None, t=None, camera_info=None):
    ci = camera_info or sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics.to(device), ci.camera_height, ci.camera_width, ci.camera_id, ci.distortion)
    return GPCR.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud.to(device), point_cloud_features=sc.point_cloud_features.to(device),
        point_object_id=sc.point_object_id.to(device), point_invalid_mask=sc.point_invalid_mask.to(device),
        camera_info=ci, q_pointcloud_camera=(sc.q_pointcloud_camera if q is None else q).to(device),
        t_pointcloud_camera=(sc.t_pointcloud_camera if t is None else t).to(device), color_max_sh_band=3)


def test_records_at_full_size_match_the_model():
    H, W = 1024, 2048
    sc = make_panorama_scene(100_000, H, W, 0.01, 5, radius=4.0)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        image, depth, _ = op(_input(sc))
    torch.cuda.synchronize()
    assert torch.isfinite(image).all() and torch.isfinite(depth).all()
    frame = op.last_frame
    ids = frame.point_id_in_camera_list.long().cpu()
    rec = frame.records.cpu().double()
    assert ids.shape[0] > 0.99 * 100_000  # the whole shell is in view, but for the polar cones
    dt = torch.float64
    Rc, tc = camera_from_pose(sc.q_pointcloud_camera.to(dt), sc.t_pointcloud_camera.to(dt))
    pc = (Rc[0] @ sc.point_cloud.to(dt)[ids, :, None])[..., 0] + tc[0]
    K = sc.camera_info.camera_intrinsics.to(dt)
    uv = project(pc, K, W)
    du = (rec[:, 0] - uv[:, 0] + W / 2) % W - W / 2
    assert float(du.abs().max()) < 5e-3 and float((rec[:, 1] - uv[:, 1]).abs().max()) < 5e-3
    assert float((rec[:, 7] / pc.norm(dim=-1) - 1).abs().max()) < 1e-6
    f = sc.point_cloud_features.to(dt)[ids]
    R = quat_to_rot(f[:, 0:4] / f[:, 0:4].norm(dim=-1, keepdim=True))
    Sigma = R @ torch.diag_embed(torch.exp(2 * f[:, 4:7])) @ R.transpose(-1, -2)
    U = jacobian(pc, K) @ Rc[0]
    cov = U @ Sigma @ U.transpose(-1, -2)
    a, b, d = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * d - b * b
    conic = torch.stack([d / det, -b / det, a / det], -1)
    rel = ((rec[:, 2:5] - conic).abs() / conic.abs().amax(-1, keepdim=True)).amax(-1)
    assert float(torch.quantile(rel, 0.999)) < 2e-3 and float(rel.max()) < 2e-2


@pytest.mark.parametrize("terms", ["image", "all"])
def test_images_and_gradients_match_the_evaluator(terms):
    H, W = 64, 128
    sc = make_panorama_scene(400, H, W, 0.15, 3, sh_degree=2, radius=3.0, seam_fraction=0.2, pole_fraction=0.05)
    N = sc.point_cloud.shape[0]
    rng = np.random.default_rng(2)
    extra = torch.from_numpy(rng.standard_normal((N, 4)).astype(np.float32))
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_depth=True, differentiable_alpha=True)
    inp = _input(sc)
    inp.point_cloud.requires_grad_(True)
    inp.point_cloud_features.requires_grad_(True)
    ef = extra.cuda().requires_grad_(True)
    image, depth, _, alpha, fmap = op(inp, point_extra_features=ef)
    g = torch.from_numpy(rng.standard_normal((H, W, 3)).astype(np.float32))
    gd = torch.from_numpy(0.1 * rng.standard_normal((H, W)).astype(np.float32))
    ga = torch.from_numpy(rng.standard_normal((H, W)).astype(np.float32))
    gF = torch.from_numpy(rng.standard_normal((H, W, 4)).astype(np.float32))
    loss = (image * g.cuda()).sum()
    if terms == "all":
        loss = loss + (depth * gd.cuda()).sum() + (alpha * ga.cuda()).sum() + (fmap * gF.cuda()).sum()
    loss.backward()
    xyz = sc.point_cloud.double().requires_grad_(True)
    feats = sc.point_cloud_features.double().requires_grad_(True)
    efd = extra.double().requires_grad_(True)
    C, D, S, F, _ = dense_render_equirect(xyz, feats, sc.point_invalid_mask, sc.point_object_id, sc.camera_info.camera_intrinsics,
                                          sc.q_pointcloud_camera, sc.t_pointcloud_camera, H, W, extra_features=efd)
    assert float((image.detach().cpu().double() - C).abs().max()) < 2e-3
    assert float((alpha.detach().cpu().double() - S).abs().max()) < 2e-3
    assert float((fmap.detach().cpu().double() - F).abs().max()) < 2e-2
    ref = (C * g.double()).sum()
    if terms == "all":
        ref = ref + (D * gd.double()).sum() + (S * ga.double()).sum() + (F * gF.double()).sum()
    ref.backward()
    gx, want_x = inp.point_cloud.grad.cpu().double(), xyz.grad
    gf, want_f = inp.point_cloud_features.grad.cpu().double(), postprocess_feature_grads(feats.grad, 3)
    assert float((gx - want_x).abs().max()) < 5e-3 * float(want_x.abs().max())
    assert float((gf - want_f).abs().max()) < 5e-3 * float(want_f.abs().max())
    if terms == "all":
        assert float((ef.grad.cpu().double() - efd.grad).abs().max()) < 5e-3 * float(efd.grad.abs().max())


def test_a_quarter_turn_rolls_the_full_size_panorama():
    H, W = 1024, 2048
    base = make_panorama_scene(100_000, H, W, 0.01, 7, radius=4.0)
    turned = make_panorama_scene(100_000, H, W, 0.01, 7, radius=4.0, yaw_degrees=90.0)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        a, _, _ = op(_input(base))
        b, _, _ = op(_input(turned))
    err = (b - torch.roll(a, -W // 4, dims=1)).abs()
    # the yaw moves every point's camera-frame position by a float rounding, which can flip a depth key and swap two
    # overlapping splats of nearly the same depth on a handful of pixels
    assert float(err.mean()) < 1e-5 and float((err > 1e-2).float().mean()) < 1e-4, (float(err.mean()), float(err.max()))
    assert float((b - a).abs().mean()) > 0.01


def _cube_faces(pano, size):
    """Six 90-degree pinhole crops of an (H, W, 3) panorama (bilinear), with their (q, t, K): yaws 0/90/180/270, up, down."""
    H, W = pano.shape[:2]
    f = size / 2.0
    ys, xs = torch.meshgrid(torch.arange(size, dtype=torch.float64) + 0.5, torch.arange(size, dtype=torch.float64) + 0.5,
                            indexing="ij")
    d = torch.stack([(xs - size / 2) / f, (ys - size / 2) / f, torch.ones_like(xs)], -1)
    out = []
    rots = [(0.0, 1.0, 0.0, a) for a in (0.0, 90.0, 180.0, 270.0)] + [(1.0, 0.0, 0.0, 90.0), (1.0, 0.0, 0.0, -90.0)]
    for ax, ay, az, deg in rots:
        h = math.radians(deg) / 2
        q = torch.tensor([[ax * math.sin(h), ay * math.sin(h), az * math.sin(h), math.cos(h)]], dtype=torch.float32)
        Rcam = quat_to_rot(q.double())[0]  # camera -> panorama frame
        w = d @ Rcam.T
        u = W / (2 * math.pi) * torch.atan2(w[..., 0], w[..., 2]) + W / 2
        v = H / math.pi * torch.atan2(w[..., 1], torch.hypot(w[..., 0], w[..., 2])) + H / 2
        uu, vv = (u - 0.5) % W, torch.clamp(v - 0.5, 0, H - 1.001)
        u0, v0 = uu.floor().long(), vv.floor().long()
        fu, fv = (uu - u0)[..., None], (vv - v0)[..., None]
        u1 = (u0 + 1) % W
        img = (pano[v0, u0] * (1 - fu) * (1 - fv) + pano[v0, u1] * fu * (1 - fv) + pano[v0 + 1, u0] * (1 - fu) * fv +
               pano[v0 + 1, u1] * fu * fv)
        K = torch.tensor([[f, 0.0, size / 2], [0.0, f, size / 2], [0.0, 0.0, 1.0]], dtype=torch.float32)
        out.append((img.float(), q, K))
    return out


def _train(views, hidden, iters):
    cfg = GaussianPointCloudTrainer.TrainConfig(num_iterations=iters, feature_learning_rate=5e-3, position_learning_rate=2e-4,
                                                initial_downsample_factor=1, increase_color_max_sh_band_interval=100.0)
    cfg.adaptive_controller_config.num_iterations_warm_up = 10 ** 9
    cfg.loss_function_config.enable_regularization = False
    g = torch.Generator().manual_seed(9)
    n = hidden.point_cloud.shape[0]
    pc = hidden.point_cloud + 0.03 * torch.randn((n, 3), generator=g)
    feat = hidden.point_cloud_features.clone()
    feat[:, 4:7] += 0.3 * torch.randn((n, 3), generator=g)
    feat[:, 8:] = 0.5 * feat[:, 8:]
    feat[:, 7] = 0.5
    scene = Scene(point_cloud=pc.cuda().requires_grad_(True), point_cloud_features=feat.cuda().requires_grad_(True),
                  point_invalid_mask=torch.zeros(n, dtype=torch.int8, device="cuda"),
                  point_object_id=torch.zeros(n, dtype=torch.int32, device="cuda"))
    trainer = GaussianPointCloudTrainer(cfg, scene, views)
    trainer.train()
    return trainer


def test_fit_from_panoramas_renders_held_out_pinhole_views():
    """Panoramas of the shell scene from four positions near its centre train a perturbed copy of it; pinhole views from
    other positions and directions are the check.  The same panoramas cut into cube faces train a second copy (reported
    beside it, not gated)."""
    H, W = 256, 512
    hidden = make_panorama_scene(3000, H, W, 0.08, 4, sh_degree=1, radius=4.0)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    K = LensDistortion.equirectangular_intrinsics(W, H)
    pano_views, cube_views = [], []
    for k, t in enumerate(((0.0, 0.0, 0.0), (0.3, 0.0, 0.1), (-0.2, 0.1, -0.2), (0.1, -0.1, 0.3))):
        tt = torch.tensor([t], dtype=torch.float32)
        ci = CameraInfo(K.cuda(), H, W, 0, LensDistortion("equirectangular", ()))
        with torch.no_grad():
            img, _, _ = op(_input(hidden, q=hidden.q_pointcloud_camera, t=tt, camera_info=ci))
        img = img.clamp(0, 1)
        pano_views.append((img.permute(2, 0, 1).contiguous(), hidden.q_pointcloud_camera.cuda(), tt.cuda(), ci))
        for face, q, Kf in _cube_faces(img.cpu().double(), 128):
            cube_views.append((face.permute(2, 0, 1).contiguous().cuda(), q.cuda(), tt.cuda(),
                               CameraInfo(Kf.cuda(), 128, 128, 1)))
    held = []
    Kp = torch.tensor([[80.0, 0.0, 64.0], [0.0, 80.0, 48.0], [0.0, 0.0, 1.0]])
    for yaw, t in ((30.0, (0.15, 0.05, 0.0)), (135.0, (-0.1, 0.0, 0.1)), (250.0, (0.0, -0.05, -0.1)), (315.0, (0.1, 0.1, 0.1))):
        h = math.radians(yaw) / 2
        q = torch.tensor([[0.0, math.sin(h), 0.0, math.cos(h)]])
        tt = torch.tensor([t], dtype=torch.float32)
        ci = CameraInfo(Kp.cuda(), 96, 128, 2)
        with torch.no_grad():
            img, _, _ = op(_input(hidden, q=q, t=tt, camera_info=ci))
        held.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q.cuda(), tt.cuda(), ci))
    iters = 400
    pano = _train(pano_views, hidden, iters)
    psnr_pano = pano.validation(held)
    cube = _train(cube_views, hidden, iters)
    psnr_cube = cube.validation(held)
    print(f"held-out pinhole PSNR: trained on panoramas {psnr_pano:.2f} dB, on cube faces {psnr_cube:.2f} dB")
    # measured 46.2 dB (and 37.0 dB from the cube faces) on an H100; the margin covers run-to-run variation of the training
    assert psnr_pano > 40.0, (psnr_pano, psnr_cube)
