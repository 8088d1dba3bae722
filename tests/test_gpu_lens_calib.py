"""-m gpu: pose and intrinsics gradients through a lens in the CUDA operator (``differentiable_pose`` /
``differentiable_intrinsics`` on OpenCV and fisheye views, ``gsb200_backward_lens_calib``) and joint camera refinement in the
trainer.

dL/dq, dL/dt, dL/dK and dL/dk against torch autograd of the float64 dense evaluator (``torch_reference_lens_grad``) for both
lenses and image, depth, alpha and feature-map losses; the scene's gradients against the LENS call's; the same camera
gradients from the full-frame emulator; two C3 calls; pose refinement through a lens in the trainer; intrinsics recovery
through a known lens; and joint self-calibration of K and the lens from a pinhole start."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from gpu_helpers import cuda_scene, n
from helpers import grad_close
from test_gpu_pose_gradient import _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_lens import r2_bound
from torch_reference_lens_grad import dense_render_lens_k, project_k

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput
LENSES = {
    "opencv": LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": LensDistortion("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
FIT_LENSES = {  # the capture lenses of the fits: a strong barrel lens and a fisheye
    "opencv": LensDistortion("opencv", (-0.2, 0.03, 0.0, 0.0, 0.0)),
    "fisheye": LensDistortion("fisheye", (0.05, -0.01, 0.0, 0.0)),
}


def _input(sc, lens, K=None, q=None, t=None, band=3):
    ci = sc.camera_info
    return Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                 point_invalid_mask=sc.point_invalid_mask,
                 camera_info=CameraInfo(ci.camera_intrinsics if K is None else K, ci.camera_height, ci.camera_width,
                                        ci.camera_id, lens),
                 q_pointcloud_camera=sc.q_pointcloud_camera if q is None else q,
                 t_pointcloud_camera=sc.t_pointcloud_camera if t is None else t, color_max_sh_band=band)


def _loss(outs, g_img, g_dep, g_alpha, g_map):
    loss = (outs[0] * g_img.cuda()).sum()
    if g_dep is not None:
        loss = loss + (outs[1] * g_dep.cuda()).sum()
    if g_alpha is not None:
        loss = loss + (outs[3] * g_alpha.cuda()).sum()
    if g_map is not None:
        loss = loss + (outs[-1] * g_map.cuda()).sum()
    return loss


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_cuda_camera_gradients_through_a_lens_match_dense_autograd(lens, kind, backward_impl="transposed", seed=61,
                                                                   objects=1):
    scene = _scene(seed, objects=objects)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    dist = LENSES[lens]
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    g_dep = torch.randn((H, W), generator=g) if kind == "depth" else None
    g_alpha = torch.randn((H, W), generator=g) if kind == "alpha" else None
    extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g) if kind == "features" else None
    g_map = torch.randn((H, W, 5), generator=g) if kind == "features" else None
    runs = []
    for joint in (True, False):
        sc = cuda_scene(scene, requires_grad=True)
        op = GPCR(Config(), exact_exp=True, backward_impl=backward_impl, differentiable_depth=kind == "depth",
                  differentiable_alpha=kind == "alpha", differentiable_pose=joint, differentiable_intrinsics=joint,
                  differentiable_distortion=joint, camera_gradients_through_lens=joint)
        q = sc.q_pointcloud_camera.clone().requires_grad_(joint)
        t = sc.t_pointcloud_camera.clone().requires_grad_(joint)
        K = sc.camera_info.camera_intrinsics.clone().requires_grad_(joint)
        kw = dict(lens_coefficients=torch.tensor(dist.coefficients, requires_grad=True)) if joint else {}
        if extra is not None:
            kw["point_extra_features"] = extra.cuda()
        outs = op(_input(sc, dist, K, q, t), **kw)
        _loss(outs, g_img, g_dep, g_alpha, g_map).backward()
        runs.append((sc, q, t, K, kw.get("lens_coefficients")))
    (sc, q, t, K, k), (sc0, *_) = runs
    # the scene's gradients are the LENS call's (loop A's float atomics: equal up to rounding)
    for a, b in ((sc.point_cloud.grad, sc0.point_cloud.grad), (sc.point_cloud_features.grad, sc0.point_cloud_features.grad)):
        assert np.abs(n(a) - n(b)).max() <= 1e-5 * max(np.abs(n(b)).max(), 1e-30)
    qq = scene.q_pointcloud_camera.clone().double().requires_grad_(True)
    tt = scene.t_pointcloud_camera.clone().double().requires_grad_(True)
    KK = scene.camera_info.camera_intrinsics.clone().double().requires_grad_(True)
    kk = torch.tensor(dist.coefficients, dtype=torch.float64, requires_grad=True)
    feats = sc.point_cloud_features.detach().cpu().double()  # q normalised in place by the forward
    ref, aux = dense_render_lens_k(scene.point_cloud.double(), feats, scene.point_invalid_mask, scene.point_object_id,
                                   KK, qq, tt, H, W, dist.model, kk)
    rloss = (ref * g_img.double()).sum()
    if g_dep is not None:
        rloss = rloss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        rloss = rloss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        rloss = rloss + (feature_map(aux, extra.double(), H, W) * g_map.double()).sum()
    rloss.backward()
    for got, want in ((q.grad, qq.grad), (t.grad, tt.grad), (K.grad, KK.grad)):
        ok = grad_close(n(got), want.numpy())
        assert ok[0], (n(got), want.numpy(), ok)
    assert (n(K.grad)[2] == 0).all()
    got, want = k.grad.numpy(), kk.grad.numpy()
    assert (np.abs(got - want) <= 2e-3 * np.abs(want) + 2e-4 * np.abs(want).max()).all(), (got, want)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_image_loss_camera_gradients_under_the_butterfly_loop_a_with_three_objects(lens):
    test_cuda_camera_gradients_through_a_lens_match_dense_autograd(lens, "image", backward_impl="butterfly", seed=63,
                                                                   objects=3)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_cuda_camera_gradients_match_the_emulator(lens):
    """The same frame through the CUDA call and through the emulated pipeline (the unmodified kernel sources on the CPU):
    the loop-A rows differ only by float atomics, so the camera gradients agree to the gradient criterion."""
    from simt_helpers import build_emulator
    from simt_lens_calib_helpers import build_lens_calib_emulator, emulated_points_lens_calib
    from simt_lens_helpers import build_lens_emulator, emulated_forward_lens
    from test_pose_gradient_cpu import _loop_a_image
    emu, lemu, cemu = build_emulator(), build_lens_emulator(), build_lens_calib_emulator()
    scene = _scene(65)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    dist = LENSES[lens]
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(7))
    st = emulated_forward_lens(emu, lemu, scene, dist.model, dist.coefficients, exact=True)
    res = emulated_points_lens_calib(emu, cemu, st, _loop_a_image(emu, st, g_img.numpy(), True), pose=True, intr=True,
                                     lgrad=True)
    sc = cuda_scene(scene)
    q = sc.q_pointcloud_camera.clone().requires_grad_(True)
    t = sc.t_pointcloud_camera.clone().requires_grad_(True)
    K = sc.camera_info.camera_intrinsics.clone().requires_grad_(True)
    k = torch.tensor(dist.coefficients, requires_grad=True)
    op = GPCR(Config(), exact_exp=True, differentiable_pose=True, differentiable_intrinsics=True,
              differentiable_distortion=True, camera_gradients_through_lens=True)
    outs = op(_input(sc, dist, K, q, t), lens_coefficients=k)
    (outs[0] * g_img.cuda()).sum().backward()
    for got, want in ((q.grad, res.gq), (t.grad, res.gt), (K.grad, res.gK)):
        ok = grad_close(n(got), want)
        assert ok[0], (n(got), want, ok)
    nk = len(dist.coefficients)
    assert np.allclose(k.grad.numpy(), res.gk[:nk], rtol=1e-3, atol=1e-4 * np.abs(res.gk).max())


def _c3():
    scene = make_scene(**CONFIGS["C3"]).to("cuda")
    return scene, scene.point_cloud_features.detach().clone()


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_full_size_camera_gradients_repeat(lens):
    """Two C3 calls with pose, intrinsics and coefficient gradients: the same per-point records, and camera gradients equal
    up to loop A's float atomics."""
    scene, feats0 = _c3()
    dist = LENSES[lens]
    op = GPCR(Config(), differentiable_pose=True, differentiable_intrinsics=True, differentiable_distortion=True,
              camera_gradients_through_lens=True)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(3)).cuda()
    out = []
    for _ in range(2):
        with torch.no_grad():
            scene.point_cloud_features.copy_(feats0)
        q = scene.q_pointcloud_camera.clone().requires_grad_(True)
        t = scene.t_pointcloud_camera.clone().requires_grad_(True)
        K = scene.camera_info.camera_intrinsics.clone().requires_grad_(True)
        k = torch.tensor(dist.coefficients, requires_grad=True)
        image = op(_input(scene, dist, K, q, t), lens_coefficients=k)[0]
        grads = torch.autograd.grad([(image * g_img).sum()], [q, t, K, k])
        out.append(([g.cpu().numpy().copy() for g in grads], n(op.last_frame.records),
                    n(op.last_frame.point_id_in_camera_list)))
    (a, ra, oa), (b, rb, ob) = out
    assert np.array_equal(ra, rb) and np.array_equal(oa, ob)
    for x, y in zip(a, b):
        print(f"C3 {lens}: {x.reshape(-1)[:6].tolist()} / {y.reshape(-1)[:6].tolist()}, bit-identical: {np.array_equal(x, y)}")
        assert np.abs(x - y).max() <= 1e-4 * np.abs(x).max() and np.abs(x).max() > 0


# ------------------------------------------------------------------ fits
def _qmul(a, b):
    w0, v0 = a[..., 3], a[..., :3]
    w1, v1 = b[..., 3], b[..., :3]
    return torch.cat([w0[..., None] * v1 + w1[..., None] * v0 + torch.linalg.cross(v0, v1),
                      (w0 * w1 - (v0 * v1).sum(-1))[..., None]], -1)


def _angle_deg(q0, q1):
    q0, q1 = q0 / q0.norm(dim=-1, keepdim=True), q1 / q1.norm(dim=-1, keepdim=True)
    return float(torch.rad2deg(2 * torch.acos((q0 * q1).sum(-1).abs().clamp(max=1.0))).reshape(-1)[0])


def _fit_views(hidden, lens, yaws, K):
    from trainer_helpers import H, W
    op = GPCR(Config())
    pc, feat = hidden.point_cloud.cuda(), hidden.point_cloud_features.clone().cuda()
    mask, obj = hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda()
    views = []
    for yaw in yaws:
        half = math.radians(yaw) / 2
        q, t = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]]), torch.zeros((1, 3))
        with torch.no_grad():
            img = op(Input(point_cloud=pc, point_cloud_features=feat, point_object_id=obj, point_invalid_mask=mask,
                           camera_info=CameraInfo(K.cuda(), H, W, 0, lens), q_pointcloud_camera=q.cuda(),
                           t_pointcloud_camera=t.cuda(), color_max_sh_band=3))[0]
        views.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q.cuda(), t.cuda(), CameraInfo(K.cuda(), H, W, 0, lens)))
    return views


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_pose_refinement_through_a_lens(lens):
    """Five views of the trainer's synthetic scene through the lens; views 1..4 recorded with poses rotated by about 1 degree
    and shifted by 0.03 (about 3 % of the scene's extent).  A perturbed copy of the scene trains with and without pose
    refinement; with it the median rotation and translation errors must at least halve, and the held-out PSNR rise."""
    from trainer_helpers import hidden_scene, train_config
    dist = FIT_LENSES[lens]
    hidden = hidden_scene(n=600)
    K = hidden.camera_info.camera_intrinsics.clone()
    train = _fit_views(hidden, dist, (0.0, -6.0, -2.0, 2.0, 6.0), K)
    held = _fit_views(hidden, dist, (-4.0, 4.0), K)
    g = torch.Generator().manual_seed(5)
    truth, recorded = [], []
    for i, (img, q, t, ci) in enumerate(train):
        truth.append((q.cpu(), t.cpu()))
        if i:
            axis = torch.randn(3, generator=g)
            half = math.radians(1.0) / 2
            dq = torch.cat([axis / axis.norm() * math.sin(half), torch.tensor([math.cos(half)])])[None]
            q = _qmul(dq, q.cpu())
            d = torch.randn((1, 3), generator=g)
            t = t.cpu() + 0.03 * d / d.norm()
        recorded.append((img, q.float().cuda(), t.float().cuda(), ci))
    psnr, errors = {}, {}
    for pose_lr in (0.0, 1e-3):
        cfg = train_config(600)
        cfg.initial_downsample_factor = 1
        cfg.pose_learning_rate = pose_lr
        cfg.camera_refinement_through_lens = True
        cfg.loss_function_config.enable_regularization = False
        gg = torch.Generator().manual_seed(9)
        npts = hidden.point_cloud.shape[0]
        pc = hidden.point_cloud + 0.01 * torch.randn((npts, 3), generator=gg)
        feat = hidden.point_cloud_features.clone()
        feat[:, 8:] = 0.5 * feat[:, 8:]
        scene = Scene(pc.cuda().requires_grad_(True), feat.cuda().requires_grad_(True), hidden.point_invalid_mask.cuda(),
                      hidden.point_object_id.cuda())
        trainer = GaussianPointCloudTrainer(cfg, scene, recorded)
        trainer.train()
        psnr[pose_lr] = trainer.validation(held)
        refined = trainer.refined_poses()
        errors[pose_lr] = (np.median([_angle_deg(q.cpu(), tq) for (q, _), (tq, _) in zip(refined[1:], truth[1:])]),
                           np.median([float((t.cpu() - tt).norm()) for (_, t), (_, tt) in zip(refined[1:], truth[1:])]))
    print(f"pose refinement through the {lens} lens: median rotation error {errors[0.0][0]:.3f} -> {errors[1e-3][0]:.3f} deg, "
          f"translation {errors[0.0][1]:.4f} -> {errors[1e-3][1]:.4f}; held-out PSNR {psnr[0.0]:.2f} -> {psnr[1e-3]:.2f} dB")
    assert errors[1e-3][0] <= 0.5 * errors[0.0][0] and errors[1e-3][1] <= 0.5 * errors[0.0][1], errors
    assert psnr[1e-3] > psnr[0.0], psnr


def _ray_grid_error(K_a, lens_a, K_b, lens_b, H, W, step=8):
    """Largest |uv_a - uv_b| in pixels of a grid of rays over the image (the hidden camera's pixel grid, unprojected through
    its pinhole part), projected through camera a and camera b (rays beyond either lens's r_max skipped)."""
    K_a = torch.as_tensor(K_a, dtype=torch.float64).cpu()
    K_b = torch.as_tensor(K_b, dtype=torch.float64).cpu()
    v, u = torch.meshgrid(torch.arange(0.5, H, step, dtype=torch.float64), torch.arange(0.5, W, step, dtype=torch.float64),
                          indexing="ij")
    yn = (v.reshape(-1) - K_b[1, 2]) / K_b[1, 1]
    xn = (u.reshape(-1) - K_b[0, 2] - K_b[0, 1] * yn) / K_b[0, 0]
    keep = xn * xn + yn * yn <= min(r2_bound(lens_a.model, lens_a.coefficients), r2_bound(lens_b.model, lens_b.coefficients))
    pc = torch.stack([xn, yn, torch.ones_like(xn)], -1)[keep]
    ua = project_k(pc, K_a, lens_a.model, torch.tensor(lens_a.coefficients, dtype=torch.float64))
    ub = project_k(pc, K_b, lens_b.model, torch.tensor(lens_b.coefficients, dtype=torch.float64))
    return float((ua - ub).norm(dim=-1).max())


def _calibrate(scene, feats0, views, lens0, K0, steps, pose, lr0=1e-2, lr1=1e-5, intr=True, lgrad=True):
    """Adam through the operator on a frozen scene: K = K0 with (log fx, log fy) scales and (cx, cy) shifts, the
    coefficients, and with ``pose`` the (q, t) of every view but the first.  Returns (K, lens, poses)."""
    op = GPCR(Config(), differentiable_pose=pose, differentiable_intrinsics=intr, differentiable_distortion=lgrad,
              camera_gradients_through_lens=True)
    corr = torch.zeros(4, device="cuda", requires_grad=True)
    k = torch.tensor(lens0.coefficients, dtype=torch.float32, requires_grad=True)
    poses = [(q.clone().requires_grad_(pose and i > 0), t.clone().requires_grad_(pose and i > 0))
             for i, (_, q, t) in enumerate(views)]
    groups = [{"params": ([corr] if intr else []) + ([k] if lgrad else []), "scale": 1.0}]
    if pose:  # a tenth of the rate: 1e-3 on a unit quaternion is about 0.1 degree per step
        groups.append({"params": [x for qt in poses[1:] for x in qt], "scale": 0.1})
    opt = torch.optim.Adam(groups, lr=lr0)
    rows = torch.tensor([0, 1], device="cuda")
    W, H = scene.camera_info.camera_width, scene.camera_info.camera_height

    def K_of():
        scale = torch.ones_like(K0).index_put((rows, rows), torch.exp(corr[:2]))
        shift = torch.zeros_like(K0).index_put((rows, torch.tensor([2, 2], device="cuda")),
                                                corr[2:] * torch.tensor([float(W), float(H)], device="cuda"))
        return K0 * scale + shift
    for it in range(steps):
        for group in opt.param_groups:
            group["lr"] = group["scale"] * lr0 * (lr1 / lr0) ** (it / steps)
        opt.zero_grad()
        for (target, _, _), (q, t) in zip(views, poses):
            with torch.no_grad():
                scene.point_cloud_features.copy_(feats0)
            lens = LensDistortion(lens0.model, k.detach().tolist())
            kw = dict(lens_coefficients=k) if lgrad else {}
            image = op(_input(scene, lens, K_of() if intr else K0, q, t), **kw)[0]
            ((image - target) ** 2).mean().backward()
        opt.step()
        with torch.no_grad():
            for q, _ in poses[1:]:
                q.div_(q.norm(dim=-1, keepdim=True))
    with torch.no_grad():
        return K_of().detach(), LensDistortion(lens0.model, k.detach().tolist()), poses


def _c3_views(scene, feats0, lens, K, yaws):
    op = GPCR(Config())
    views = []
    for yaw in yaws:
        half = math.radians(yaw) / 2
        q = _qmul(torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device="cuda"), scene.q_pointcloud_camera)
        t = scene.t_pointcloud_camera.clone()
        with torch.no_grad():
            scene.point_cloud_features.copy_(feats0)
            views.append((op(_input(scene, lens, K, q, t))[0].clone(), q, t))
    return views


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_intrinsics_fit_through_a_known_lens(lens):
    """C3 views recorded through a known lens with fx, fy 4 % too large; intrinsics refinement alone brings fx and fy back
    to within 1 %."""
    scene, feats0 = _c3()
    dist = FIT_LENSES[lens]
    K = scene.camera_info.camera_intrinsics.clone()
    views = _c3_views(scene, feats0, dist, K, (0.0, 2.0))
    K0 = K.clone()
    K0[0, 0] *= 1.04
    K0[1, 1] *= 1.04
    Kf, _, _ = _calibrate(scene, feats0, views, dist, K0, 400, pose=False, lr0=3e-3, lgrad=False)
    err = [abs(float(Kf[i, i] / K[i, i]) - 1.0) for i in (0, 1)]
    print(f"intrinsics fit through the {lens} lens: fx, fy relative error 0.040 -> {err[0]:.4f}, {err[1]:.4f}")
    assert max(err) < 0.01, err


@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_joint_self_calibration_from_a_pinhole_start(lens, pose):
    """C3 views through the hidden lens; the fit starts from k = 0 and a K 3 % off (fx, fy too large, the principal point
    shifted), and refines K and k together, with pose refinement of the second view (recorded 0.5 degree off) or without.
    fx and k1 trade off, so the result is judged by the cameras' projections of a grid of rays over the image."""
    scene, feats0 = _c3()
    hidden = FIT_LENSES[lens]
    K = scene.camera_info.camera_intrinsics.clone()
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    views = _c3_views(scene, feats0, hidden, K, (0.0, 2.0))
    q_true = views[1][1].detach().cpu()
    if pose:  # the second view's recorded pose is off by 0.5 degree
        half = math.radians(0.5) / 2
        target, q, t = views[1]
        views[1] = (target, _qmul(torch.tensor([[math.sin(half), 0.0, 0.0, math.cos(half)]], device="cuda"), q), t)
    K0 = K.clone()
    K0[0, 0] *= 1.03
    K0[1, 1] *= 1.03
    K0[0, 2] += 0.01 * W
    zero = LensDistortion(hidden.model, (0.0,) * len(hidden.coefficients))
    before = _ray_grid_error(K0, zero, K, hidden, H, W)
    Kf, fitted, poses = _calibrate(scene, feats0, views, zero, K0, 3000, pose=pose)
    after = _ray_grid_error(Kf, fitted, K, hidden, H, W)
    msg, rot = "", 0.0
    if pose:
        rot = _angle_deg(poses[1][0].detach().cpu(), q_true)
        msg = f", view 1 rotation error 0.500 -> {rot:.3f} deg"
    print(f"self-calibration {lens} (pose {pose}): ray-grid error {before:.2f} px -> {after:.3f} px; K diag "
          f"{[round(float(Kf[i, i]), 2) for i in (0, 1)]} vs {[round(float(K[i, i]), 2) for i in (0, 1)]}, "
          f"k {fitted.coefficients} vs {hidden.coefficients}{msg}")
    assert after < 0.5 and rot < 0.1, (before, after, rot)
