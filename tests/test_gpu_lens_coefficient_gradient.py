"""-m gpu: lens-coefficient gradients in the CUDA operator (``differentiable_distortion``, ``gsb200_backward_lens_grad``) and
lens refinement in the trainer (``TrainConfig.distortion_learning_rate``).

dL/dk against torch autograd of the float64 dense evaluator with k as a leaf (``torch_reference_lens_grad``) on small scenes,
for both models, image, depth, alpha and feature-map losses, and an image loss under both loop-A kernels; the other outputs
against the LENS call's; at C3 full size two calls; a calibration fit of the coefficients alone through the operator; and
the trainer refining a lens from zero against a frozen scene."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from gpu_helpers import cuda_scene, n
from test_gpu_pose_gradient import _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_lens import r2_bound
from torch_reference_lens_grad import dense_render_lens_k, project_k

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput
LENSES = {  # the lenses of scripts/bench_lens.py
    "opencv": LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": LensDistortion("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}


def _input(sc, lens, band=3):
    ci = sc.camera_info
    return Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                 point_invalid_mask=sc.point_invalid_mask,
                 camera_info=CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, lens),
                 q_pointcloud_camera=sc.q_pointcloud_camera, t_pointcloud_camera=sc.t_pointcloud_camera,
                 color_max_sh_band=band)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_cuda_coefficient_gradient_matches_dense_autograd(lens, kind, backward_impl="transposed", seed=41):
    scene = _scene(seed)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    dist = LENSES[lens]
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    g_dep = torch.randn((H, W), generator=g) if kind == "depth" else None
    g_alpha = torch.randn((H, W), generator=g) if kind == "alpha" else None
    extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g) if kind == "features" else None
    g_map = torch.randn((H, W, 5), generator=g) if kind == "features" else None
    runs = []
    for with_k in (True, False):
        sc = cuda_scene(scene, requires_grad=True)
        op = GPCR(Config(), exact_exp=True, backward_impl=backward_impl, differentiable_depth=kind == "depth",
                  differentiable_alpha=kind == "alpha", differentiable_distortion=True)
        k = torch.tensor(dist.coefficients, dtype=torch.float32, requires_grad=True) if with_k else None
        kw = dict(lens_coefficients=k) if with_k else {}
        outs = op(_input(sc, dist), **kw) if extra is None else op(_input(sc, dist), point_extra_features=extra.cuda(), **kw)
        loss = (outs[0] * g_img.cuda()).sum()
        if g_dep is not None:
            loss = loss + (outs[1] * g_dep.cuda()).sum()
        if g_alpha is not None:
            loss = loss + (outs[3] * g_alpha.cuda()).sum()
        if g_map is not None:
            loss = loss + (outs[-1] * g_map.cuda()).sum()
        loss.backward()
        runs.append((sc, k))
    (sc, k), (sc0, _) = runs
    assert k.grad is not None and k.grad.device.type == "cpu" and k.grad.shape == (len(dist.coefficients),)
    # the scene's gradients are the LENS call's (loop A's float atomics: equal up to rounding)
    for a, b in ((sc.point_cloud.grad, sc0.point_cloud.grad), (sc.point_cloud_features.grad, sc0.point_cloud_features.grad)):
        assert np.abs(n(a) - n(b)).max() <= 1e-5 * max(np.abs(n(b)).max(), 1e-30)
    kk = torch.tensor(dist.coefficients, dtype=torch.float64, requires_grad=True)
    feats = sc.point_cloud_features.detach().cpu().double()  # q normalised in place by the forward
    ref, aux = dense_render_lens_k(scene.point_cloud.double(), feats, scene.point_invalid_mask, scene.point_object_id,
                                   scene.camera_info.camera_intrinsics, scene.q_pointcloud_camera, scene.t_pointcloud_camera,
                                   H, W, dist.model, kk)
    rloss = (ref * g_img.double()).sum()
    if g_dep is not None:
        rloss = rloss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        rloss = rloss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        rloss = rloss + (feature_map(aux, extra.double(), H, W) * g_map.double()).sum()
    rloss.backward()
    got, want = k.grad.numpy(), kk.grad.numpy()
    assert (np.abs(got - want) <= 2e-3 * np.abs(want) + 2e-4 * np.abs(want).max()).all(), (got, want)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_image_loss_coefficient_gradient_under_the_butterfly_loop_a(lens):
    test_cuda_coefficient_gradient_matches_dense_autograd(lens, "image", backward_impl="butterfly", seed=43)


def _c3():
    scene = make_scene(**CONFIGS["C3"]).to("cuda")
    return scene, scene.point_cloud_features.detach().clone()


def _c3_step(op, scene, feats0, dist, k, target=None, g_img=None):
    with torch.no_grad():
        scene.point_cloud_features.copy_(feats0)
    image = op(_input(scene, dist), lens_coefficients=k)[0]
    loss = ((image - target) ** 2).mean() if target is not None else (image * g_img).sum()
    (gk,) = torch.autograd.grad([loss], [k])
    return loss.detach(), gk


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_full_size_coefficient_gradient_repeats(lens):
    """Two C3 calls: the same per-point records, and coefficient gradients equal up to loop A's float atomics (rows
    that are equal give bit-identical gradients: the per-point sum has a fixed order, see the emulated test)."""
    scene, feats0 = _c3()
    dist = LENSES[lens]
    op = GPCR(Config(), differentiable_distortion=True)
    g_img = torch.randn((scene.camera_info.camera_height, scene.camera_info.camera_width, 3),
                        generator=torch.Generator().manual_seed(3)).cuda()
    k = torch.tensor(dist.coefficients, dtype=torch.float32, requires_grad=True)
    out = []
    for _ in range(2):
        _, gk = _c3_step(op, scene, feats0, dist, k, g_img=g_img)
        out.append((gk.numpy().copy(), n(op.last_frame.records), n(op.last_frame.point_id_in_camera_list)))
    (a, ra, oa), (b, rb, ob) = out
    assert np.array_equal(ra, rb) and np.array_equal(oa, ob)
    print(f"C3 {lens}: dL/dk {a.tolist()} / {b.tolist()}, bit-identical: {np.array_equal(a, b)}")
    assert np.abs(a - b).max() <= 1e-4 * np.abs(a).max() and np.abs(a).max() > 0


def max_displacement(K, a, b, H, W, step=8):
    """Largest |uv_a - uv_b| in pixels over a grid of the image's normalised points (within both lenses' r_max)."""
    K = torch.as_tensor(K, dtype=torch.float64).cpu()
    v, u = torch.meshgrid(torch.arange(0.5, H, step, dtype=torch.float64), torch.arange(0.5, W, step, dtype=torch.float64),
                          indexing="ij")
    yn = (v.reshape(-1) - K[1, 2]) / K[1, 1]
    xn = (u.reshape(-1) - K[0, 2] - K[0, 1] * yn) / K[0, 0]
    keep = xn * xn + yn * yn <= min(r2_bound(a.model, a.coefficients), r2_bound(b.model, b.coefficients))
    pc = torch.stack([xn, yn, torch.ones_like(xn)], -1)[keep]
    ua = project_k(pc, K, a.model, torch.tensor(a.coefficients, dtype=torch.float64))
    ub = project_k(pc, K, b.model, torch.tensor(b.coefficients, dtype=torch.float64))
    return float((ua - ub).norm(dim=-1).max())


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_calibration_fit_recovers_the_hidden_lens(lens):
    """Targets rendered through the hidden lens at C3; the coefficients alone fitted with Adam through the operator, from
    zero (opencv) or from perturbed values (fisheye)."""
    scene, feats0 = _c3()
    ci = scene.camera_info
    H, W = ci.camera_height, ci.camera_width
    hidden = LENSES[lens]
    op = GPCR(Config(), differentiable_distortion=True)
    with torch.no_grad():
        target = op(_input(scene, hidden))[0].clone()
    start = [0.0] * 5 if lens == "opencv" else [c + d for c, d in zip(hidden.coefficients, (0.03, -0.01, 0.005, -0.002))]
    k = torch.tensor(start, dtype=torch.float32, requires_grad=True)
    before = max_displacement(ci.camera_intrinsics, LensDistortion(hidden.model, start), hidden, H, W)
    # k1, k2, k3 are correlated (a long valley): a learning rate decaying exponentially from 1e-2 to 1e-5.  On an H100 80GB
    # HBM3 (700 W) this schedule reached 0.000 px (opencv) and 0.014 px (fisheye) after 3000 steps, both below 0.02 px after
    # 1000; 300 steps from 2e-3 stopped at 0.80 px and 0.16 px.
    steps, lr0, lr1 = 2000, 1e-2, 1e-5
    opt = torch.optim.Adam([k], lr=lr0)
    for it in range(steps):
        for group in opt.param_groups:
            group["lr"] = lr0 * (lr1 / lr0) ** (it / steps)
        opt.zero_grad()
        loss, gk = _c3_step(op, scene, feats0, LensDistortion(hidden.model, k.detach().tolist()), k, target=target)
        k.grad = gk
        opt.step()
    fitted = LensDistortion(hidden.model, k.detach().tolist())
    after = max_displacement(ci.camera_intrinsics, fitted, hidden, H, W)
    print(f"calibration fit {lens}: largest displacement {before:.3f} px -> {after:.4f} px, loss {float(loss):.3e}, "
          f"fitted {fitted.coefficients} hidden {hidden.coefficients}")
    assert after < 0.05


def test_trainer_refines_a_lens_from_zero():
    """A frozen scene (learning rates 0) and views rendered through the hidden opencv lens; the trainer starts from zero
    coefficients.  The refined lens's largest displacement from the hidden one must be at most 25 % of the zero lens's, and
    the validation PSNR through it must beat the zero lens's."""
    from trainer_helpers import H, W, hidden_scene, poses, train_config
    hidden = hidden_scene(n=600)
    dist = LENSES["opencv"]
    K = hidden.camera_info.camera_intrinsics.clone()
    op = GPCR(Config())
    pc, feat = hidden.point_cloud.cuda(), hidden.point_cloud_features.clone().cuda()
    mask, obj = hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda()
    zero = LensDistortion("opencv", (0.0,) * 5)
    targets = []
    for q, t in poses():
        with torch.no_grad():
            img = op(Input(point_cloud=pc, point_cloud_features=feat, point_object_id=obj, point_invalid_mask=mask,
                           camera_info=CameraInfo(K.cuda(), H, W, 0, dist), q_pointcloud_camera=q.cuda(),
                           t_pointcloud_camera=t.cuda(), color_max_sh_band=3))[0]
        targets.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q.cuda(), t.cuda()))

    def views(lens):
        return [(img, q, t, CameraInfo(K.cuda(), H, W, 0, lens)) for img, q, t in targets]

    cfg = train_config(300)
    cfg.feature_learning_rate = cfg.position_learning_rate = 0.0
    cfg.initial_downsample_factor = 1
    cfg.distortion_learning_rate = 2e-3
    scene = Scene(pc.clone().requires_grad_(True), feat.clone().requires_grad_(True), mask.clone(), obj.clone())
    trainer = GaussianPointCloudTrainer(cfg, scene, views(zero))
    trainer.train()
    refined = trainer.refined_distortion()[0]
    before = max_displacement(K, zero, dist, H, W, step=2)
    after = max_displacement(K, refined, dist, H, W, step=2)
    psnr_refined, psnr_zero = trainer.validation(views(refined)), trainer.validation(views(zero))
    print(f"trainer: largest displacement {before:.3f} px -> {after:.3f} px ({after / before:.1%}), validation PSNR "
          f"{psnr_refined:.2f} dB through the refined lens, {psnr_zero:.2f} dB through the zero lens; refined {refined}")
    assert after <= 0.25 * before
    assert psnr_refined > psnr_zero
