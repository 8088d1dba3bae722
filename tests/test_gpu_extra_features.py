"""-m gpu: per-Gaussian feature channels of the CUDA operator (``point_extra_features``, ``gsb200_forward_ext`` /
``gsb200_backward_ext``).

Against torch autograd through the float64 dense evaluator (``torch_reference_features``; the depth map of
``torch_reference_depth`` and ``dense_render``'s accumulated alpha for the combined loss) under the gradient gate of
test_gpu_parity (|a - b| <= 1e-3 |b| + 1e-5 max|b|), for every compile-time width on both arithmetic paths, with and
without a hook.  Also: a feature call leaves the frame's other outputs bit-identical, colour-valued features reproduce the
image, frozen geometry, and two short fits."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.utils import inverse_SE3_qt_torch

from gpu_helpers import Input, cuda_scene, n
from helpers import grad_close
from torch_reference import dense_render, postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, sh_degree=3):
    """As in test_gpu_alpha_gradient: dense coverage, points behind near, saturation and early stop, invalid slots."""
    sc = make_scene(n, h, w, sigma, seed, sh_degree=sh_degree, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    return sc


def _run(op, sc, F=None, band=3):
    inp = Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                point_invalid_mask=sc.point_invalid_mask, camera_info=sc.camera_info,
                q_pointcloud_camera=sc.q_pointcloud_camera, t_pointcloud_camera=sc.t_pointcloud_camera,
                color_max_sh_band=band)
    return op(inp) if F is None else op(inp, point_extra_features=F)


def _dense(scene, feats_n, F, loss_fn, band=3):
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    q_cp, t_cp = inverse_SE3_qt_torch(scene.q_pointcloud_camera, scene.t_pointcloud_camera)
    xyz = scene.point_cloud.clone().double().requires_grad_(True)
    feats = torch.from_numpy(feats_n).double().requires_grad_(True)
    Fd = F.detach().cpu().double().requires_grad_(True)
    image, aux = dense_render(xyz, feats, scene.point_invalid_mask, scene.camera_info.camera_intrinsics, q_cp, t_cp, H, W)
    depth, _ = differentiable_depth(aux, H, W)
    fmap = feature_map(aux, Fd, H, W)
    loss_fn(image, depth, aux["acc_alpha"], fmap).backward()
    return fmap.detach().numpy(), xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), Fd.grad.numpy()


def _check(gx, gf, gF, ex, ef, eF):
    for a, b, what in ((gF, eF, "dL/dF"), (gx, ex, "xyz")):
        ok = grad_close(a, b)
        assert ok[0], (what, ok)
    for sl in GROUPS:
        ok = grad_close(gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)


@pytest.mark.parametrize("with_hook", [False, True])
@pytest.mark.parametrize("exact_exp", [True, False])
@pytest.mark.parametrize("C", [1, 3, 5, 8, 16])
def test_features_match_dense_autograd(C, exact_exp, with_hook):
    seed = 11 + C
    scene = _scene(seed)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    gen = torch.Generator().manual_seed(seed + 200)
    g_img, g_dep, g_alp = torch.randn((H, W, 3), generator=gen), torch.randn((H, W), generator=gen), torch.randn((H, W), generator=gen)
    g_F = torch.randn((H, W, C), generator=gen)
    F0 = torch.randn((scene.point_cloud.shape[0], C), generator=gen)
    for loss in ("features", "features+image", "features+image+depth+alpha"):
        full = "depth" in loss
        sc = cuda_scene(scene, requires_grad=True)
        F = F0.cuda().requires_grad_(True)
        hooks = []
        op = GPCR(Config(), backward_valid_point_hook=hooks.append if with_hook else None, exact_exp=exact_exp,
                  differentiable_depth=full, differentiable_alpha=full)
        outs = _run(op, sc, F)
        image, depth, fmap = outs[0], outs[1], outs[-1]
        assert fmap.shape == (H, W, C) and fmap.dtype == torch.float32 and fmap.requires_grad
        total = (fmap * g_F.cuda()).sum()
        if "image" in loss:
            total = total + (image * g_img.cuda()).sum()
        if full:
            total = total + (depth * g_dep.cuda()).sum() + (outs[3] * g_alp.cuda()).sum()
        total.backward()

        def ref_loss(i, d, a, f):
            r = (f * g_F.double()).sum()
            if "image" in loss:
                r = r + (i * g_img.double()).sum()
            if full:
                r = r + (d * g_dep.double()).sum() + (a * g_alp.double()).sum()
            return r

        rmap, ex, ef, eF = _dense(scene, n(sc.point_cloud_features), F0, ref_loss)
        tol = (2e-6 if exact_exp else 1e-4) * float(F0.abs().max())
        assert np.abs(n(fmap) - rmap).max() <= tol
        _check(n(sc.point_cloud.grad), n(sc.point_cloud_features.grad), n(F.grad), ex, ef, eF)
        if with_hook:
            ids = hooks[0].point_id_in_camera_list.long()
            assert torch.equal(hooks[0].grad_point_in_camera, sc.point_cloud.grad[ids])


@pytest.mark.parametrize("exact_exp", [True, False])
def test_feature_call_leaves_the_other_outputs_bit_identical(exact_exp):
    scene = make_scene(20000, 128, 192, 0.04, 9, sh_degree=3)
    sc = cuda_scene(scene)
    op = GPCR(Config(), exact_exp=exact_exp, differentiable_alpha=True)
    feats = sc.point_cloud_features.clone()  # every call starts from the same rows (the forward normalises q in place)
    with torch.no_grad():
        sc.point_cloud_features = feats.clone()
        ref = [t.clone() for t in _run(op, sc)]
        for C in (1, 3, 8, 16):
            F = torch.randn((20000, C), device="cuda")
            sc.point_cloud_features = feats.clone()
            outs = _run(op, sc, F)
            for a, b in zip(outs[:4], ref):  # image, depth, count, accumulated alpha
                assert torch.equal(a, b)
            assert outs[4].shape == (128, 192, C)


def test_colour_features_reproduce_the_image():
    """Features equal to every splat's rendered colour (SH degree 0: one colour per Gaussian, sigmoid of the DC term times
    the band-0 basis): on the fast path the feature map is the image, bit for bit (same weights, same FMAs, same order)."""
    scene = make_scene(20000, 128, 192, 0.04, 9, sh_degree=0)
    sc = cuda_scene(scene)
    op = GPCR(Config())
    feats = sc.point_cloud_features.clone()  # both calls start from the same rows (the forward normalises q in place)
    with torch.no_grad():
        sc.point_cloud_features = feats.clone()
        image = _run(op, sc, band=0)[0].clone()
        frame = op.last_frame
        ids = frame.point_id_in_camera_list.long()
        F = torch.zeros((20000, 3), device="cuda")
        # the per-point stage's colours: the records' r g b of the in-camera points (the workspace view of the frame)
        F[ids] = frame.point_color.float()
        sc.point_cloud_features = feats.clone()
        fmap = _run(op, sc, F, band=0)[-1]
    assert torch.equal(fmap, image)


def test_frozen_geometry_only_the_features_train():
    scene = _scene(61)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene)  # no gradient for the scene tensors
    gen = torch.Generator().manual_seed(62)
    F0 = torch.randn((scene.point_cloud.shape[0], 4), generator=gen)
    g_F = torch.randn((H, W, 4), generator=gen)
    F = F0.cuda().requires_grad_(True)
    fmap = _run(GPCR(Config()), sc, F)[-1]
    (fmap * g_F.cuda()).sum().backward()
    assert sc.point_cloud.grad is None and sc.point_cloud_features.grad is None
    _, _, _, eF = _dense(scene, n(sc.point_cloud_features), F0, lambda i, d, a, f: (f * g_F.double()).sum())
    ok = grad_close(n(F.grad), eF)
    assert ok[0], ok


def test_feature_only_fit_on_a_fixed_scene():
    """Fit 8-channel features to the feature map of random target features, geometry frozen.  The loss must fall below 2 %
    of its start in 60 Adam steps (it is a linear least-squares problem in F)."""
    scene = make_scene(3000, 64, 96, 0.08, 17, sh_degree=0)
    sc = cuda_scene(scene)
    op = GPCR(Config())
    gen = torch.Generator().manual_seed(5)
    with torch.no_grad():
        target = _run(op, sc, torch.randn((3000, 8), generator=gen).cuda())[-1].clone()
    F = torch.zeros((3000, 8), device="cuda", requires_grad=True)
    opt = torch.optim.Adam([F], lr=0.1)
    losses = []
    for _ in range(60):
        loss = ((_run(op, sc, F)[-1] - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    print(f"feature MSE: first {losses[0]:.5f}  last {losses[-1]:.5f}")
    assert np.isfinite(losses).all() and losses[-1] < 0.02 * losses[0]


def test_joint_fit_with_the_image_loss():
    """Fit the 56 columns and 3-channel features together to a target image and feature map from perturbed colours and
    zero features.  Both losses must fall below 30 % of their start in 60 Adam steps."""
    scene = make_scene(3000, 64, 96, 0.08, 18, sh_degree=0)
    sc = cuda_scene(scene)
    op = GPCR(Config())
    gen = torch.Generator().manual_seed(6)
    with torch.no_grad():
        outs = _run(op, sc, torch.randn((3000, 3), generator=gen).cuda(), band=0)
        t_img, t_F = outs[0].clone(), outs[-1].clone()
    feats = sc.point_cloud_features.clone()
    feats[:, 8::16] += torch.randn((3000, 3), generator=gen).cuda()
    feats.requires_grad_(True)
    F = torch.zeros((3000, 3), device="cuda", requires_grad=True)
    opt = torch.optim.Adam([{"params": [feats], "lr": 0.05}, {"params": [F], "lr": 0.1}])
    li, lf = [], []
    for _ in range(60):
        sc.point_cloud_features = feats
        outs = _run(op, sc, F, band=0)
        a, b = ((outs[0] - t_img) ** 2).mean(), ((outs[-1] - t_F) ** 2).mean()
        opt.zero_grad()
        (a + b).backward()
        opt.step()
        li.append(float(a.detach()))
        lf.append(float(b.detach()))
    print(f"image MSE: {li[0]:.5f} -> {li[-1]:.5f}; feature MSE: {lf[0]:.5f} -> {lf[-1]:.5f}")
    assert li[-1] < 0.3 * li[0] and lf[-1] < 0.3 * lf[0]
