"""-m gpu: the accumulated-alpha gradient of the CUDA operator (``differentiable_alpha=True``, ``gsb200_backward_aux``).

Against torch autograd through the float64 dense evaluator (``dense_render``'s ``acc_alpha = 1 - T``, and the depth map of
``torch_reference_depth`` for the combined loss) under the gradient gate of test_gpu_parity
(|a - b| <= 1e-3 |b| + 1e-5 max|b|): with and without a hook, a loss on alpha alone, alpha + depth + image, and white or
random backgrounds composited as image + (1 - alpha) bg.  Also an image-only loss in alpha mode against the default
operator, the view-parallel exchange, and a short mask-supervised fit."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.utils import inverse_SE3_qt_torch

from gpu_helpers import cuda_scene, n, run_forward
from helpers import grad_close
from torch_reference import dense_render, postprocess_feature_grads
from torch_reference_depth import differentiable_depth

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, sh_degree=3):
    """As in test_oracle_dense_crosscheck: dense coverage, points behind near, saturation and early stop, invalid slots."""
    sc = make_scene(n, h, w, sigma, seed, sh_degree=sh_degree, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    return sc


def _grads(seed, H, W):
    g = torch.Generator().manual_seed(seed + 200)
    return torch.randn((H, W, 3), generator=g), torch.randn((H, W), generator=g), torch.randn((H, W), generator=g)


def _dense(scene, feats_n, loss_fn, band=3):
    """Dense float64 gradients of ``loss_fn(image, depth, alpha)`` (depth differentiable in z as well)."""
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    q_cp, t_cp = inverse_SE3_qt_torch(scene.q_pointcloud_camera, scene.t_pointcloud_camera)
    xyz = scene.point_cloud.clone().double().requires_grad_(True)
    feats = torch.from_numpy(feats_n).double().requires_grad_(True)
    image, aux = dense_render(xyz, feats, scene.point_invalid_mask, scene.camera_info.camera_intrinsics, q_cp, t_cp, H, W)
    depth, _ = differentiable_depth(aux, H, W)
    loss_fn(image, depth, aux["acc_alpha"]).backward()
    return xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy()


def _check(gx, gf, ex, ef):
    ok = grad_close(gx, ex)
    assert ok[0], ok
    for sl in GROUPS:
        ok = grad_close(gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)


@pytest.mark.parametrize("with_hook", [False, True])
@pytest.mark.parametrize("exact_exp", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_alpha_gradient_matches_dense_autograd(seed, band, exact_exp, with_hook):
    scene = _scene(seed)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    hooks = []
    op = GPCR(Config(), backward_valid_point_hook=hooks.append if with_hook else None, exact_exp=exact_exp,
              differentiable_alpha=True)
    image, depth, count, alpha = run_forward(op, sc, band=band)
    assert alpha.shape == (H, W) and alpha.dtype == torch.float32
    assert alpha.requires_grad and not depth.requires_grad and not count.requires_grad
    g_img, _, g_alp = _grads(seed, H, W)
    ((image * g_img.cuda()).sum() + (alpha * g_alp.cuda()).sum()).backward()
    feats_n = n(sc.point_cloud_features)  # quaternions normalised in place by the forward
    ex, ef = _dense(scene, feats_n, lambda i, d, a: (i * g_img.double()).sum() + (a * g_alp.double()).sum(), band)
    _check(n(sc.point_cloud.grad), n(sc.point_cloud_features.grad), ex, ef)
    if with_hook:
        h = hooks[0]
        ids = h.point_id_in_camera_list.long()
        assert torch.equal(h.grad_point_in_camera, sc.point_cloud.grad[ids])
        assert torch.equal(h.grad_pointfeatures_in_camera, sc.point_cloud_features.grad[ids])
    # a loss on the accumulated alpha alone
    sc2 = cuda_scene(scene, requires_grad=True)
    op2 = GPCR(Config(), exact_exp=exact_exp, differentiable_alpha=True)
    *_, alpha2 = run_forward(op2, sc2, band=band)
    (alpha2 * g_alp.cuda()).sum().backward()
    ex, ef = _dense(scene, feats_n, lambda i, d, a: (a * g_alp.double()).sum(), band)
    _check(n(sc2.point_cloud.grad), n(sc2.point_cloud_features.grad), ex, ef)


@pytest.mark.parametrize("exact_exp", [True, False])
def test_alpha_depth_and_image_losses_together(exact_exp):
    scene = _scene(41)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    hooks = []
    op = GPCR(Config(), backward_valid_point_hook=hooks.append, exact_exp=exact_exp, differentiable_depth=True,
              differentiable_alpha=True)
    image, depth, _, alpha = run_forward(op, sc)
    assert depth.requires_grad and alpha.requires_grad
    g_img, g_dep, g_alp = _grads(41, H, W)
    ((image * g_img.cuda()).sum() + (depth * g_dep.cuda()).sum() + (alpha * g_alp.cuda()).sum()).backward()
    ex, ef = _dense(scene, n(sc.point_cloud_features),
                    lambda i, d, a: (i * g_img.double()).sum() + (d * g_dep.double()).sum() + (a * g_alp.double()).sum())
    _check(n(sc.point_cloud.grad), n(sc.point_cloud_features.grad), ex, ef)
    ids = hooks[0].point_id_in_camera_list.long()
    assert torch.equal(hooks[0].grad_point_in_camera, sc.point_cloud.grad[ids])


@pytest.mark.parametrize("background", ["white", "random"])
def test_background_compositing_matches_dense_autograd(background):
    """A photometric loss on image + (1 - alpha) bg, the compositing of white- and random-background training."""
    scene = _scene(51)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    gen = torch.Generator().manual_seed(52)
    bg = torch.ones((H, W, 3)) if background == "white" else torch.rand((H, W, 3), generator=gen)
    target = torch.rand((H, W, 3), generator=gen)
    sc = cuda_scene(scene, requires_grad=True)
    image, _, _, alpha = run_forward(GPCR(Config(), differentiable_alpha=True), sc)
    composite = image + (1 - alpha)[..., None] * bg.cuda()
    ((composite - target.cuda()) ** 2).sum().backward()
    ex, ef = _dense(scene, n(sc.point_cloud_features),
                    lambda i, d, a: ((i + (1 - a)[..., None] * bg.double() - target.double()) ** 2).sum())
    _check(n(sc.point_cloud.grad), n(sc.point_cloud_features.grad), ex, ef)


def test_default_and_depth_operators_keep_three_outputs():
    sc = cuda_scene(_scene(5), requires_grad=True)
    for op in (GPCR(Config()), GPCR(Config(), differentiable_depth=True)):
        assert len(run_forward(op, sc)) == 3


def _run(op, sc, g_img, band=3):
    sc.point_cloud.grad = sc.point_cloud_features.grad = None
    image = run_forward(op, sc, band=band)[0]
    image.backward(g_img)
    return sc.point_cloud.grad.clone(), sc.point_cloud_features.grad.clone()


@pytest.mark.parametrize("exact_exp", [True, False])
def test_image_only_loss_in_alpha_mode_equals_the_default_operator(exact_exp):
    scene = make_scene(20000, 128, 192, 0.04, 9, sh_degree=3)
    sc = cuda_scene(scene, requires_grad=True)
    g_img = torch.randn((128, 192, 3), generator=torch.Generator().manual_seed(3)).cuda()
    ref_x, ref_f = _run(GPCR(Config(), exact_exp=exact_exp), sc, g_img)
    again_x, again_f = _run(GPCR(Config(), exact_exp=exact_exp), sc, g_img)  # the run-to-run noise of the float atomics
    noise_x, noise_f = float((again_x - ref_x).abs().max()), float((again_f - ref_f).abs().max())
    hooks = []
    op = GPCR(Config(), backward_valid_point_hook=hooks.append, exact_exp=exact_exp, differentiable_alpha=True)
    gx, gf = _run(op, sc, g_img)
    assert float((gx - ref_x).abs().max()) <= 4.0 * noise_x + 2e-6 * float(ref_x.abs().max())
    assert float((gf - ref_f).abs().max()) <= 4.0 * noise_f + 2e-6 * float(ref_f.abs().max())
    ids = hooks[0].point_id_in_camera_list.long()
    assert torch.equal(hooks[0].grad_point_in_camera, gx[ids])


class _LocalExchange:
    """A single-process stand-in for parallel.ViewParallelExchange (as in test_gpu_exchange): the first pass records every
    rank's compact buffers, the replay hands each rank the collectives' results (sum of the rows, gather of the blocks)."""

    def __init__(self, world, rank, store, replay):
        self.world, self.rank, self.store, self.replay = world, rank, store, replay

    def allocate(self, num_points, num_objects, device):
        stride = (3 * num_points + 3 * num_objects + 3) // 4 * 4
        return (torch.empty((num_points, 12), device=device), torch.empty((self.world, stride), device=device))

    def rows_written(self, grad_sum, blocks):
        pass

    def run_and_expand(self, grad_sum, blocks, expand):
        if not self.replay:
            self.store[self.rank] = (grad_sum.clone(), blocks[self.rank].clone())
            return expand(0)
        grad_sum.zero_()
        for r in range(self.world):  # rank order, like the expansion kernel's own sum
            grad_sum += self.store[r][0]
            blocks[r].copy_(self.store[r][1])
        expand(0)


def test_view_parallel_exchange_with_alpha_terms():
    R = 2
    views = [cuda_scene(make_scene(20000, 128, 192, 0.04, 9, sh_degree=3, yaw_degrees=6.0 * v - 3.0)) for v in range(R)]
    xyz = views[0].point_cloud.clone().requires_grad_(True)
    feat = views[0].point_cloud_features.clone().requires_grad_(True)
    gen = torch.Generator().manual_seed(61)
    g_img = [torch.randn((128, 192, 3), generator=gen).cuda() for _ in range(R)]
    g_alp = [torch.randn((128, 192), generator=gen).cuda() for _ in range(R)]

    def run(op, v):
        sc = views[v]
        sc.point_cloud, sc.point_cloud_features = xyz, feat
        xyz.grad = feat.grad = None
        image, _, _, alpha = run_forward(op, sc)
        ((image * g_img[v]).sum() + (alpha * g_alp[v]).sum()).backward()
        return xyz.grad.clone(), feat.grad.clone()

    dense_x, dense_f = torch.zeros_like(xyz), torch.zeros_like(feat)
    again_x, again_f = torch.zeros_like(xyz), torch.zeros_like(feat)
    for v in range(R):
        gx, gf = run(GPCR(Config(), differentiable_alpha=True), v)
        dense_x += gx
        dense_f += gf
        gx, gf = run(GPCR(Config(), differentiable_alpha=True), v)
        again_x += gx
        again_f += gf
    noise_x, noise_f = float((again_x - dense_x).abs().max()), float((again_f - dense_f).abs().max())
    store = {}
    for v in range(R):
        run(GPCR(Config(), differentiable_alpha=True, gradient_exchange=_LocalExchange(R, v, store, False)), v)
    for v in range(R):
        gx, gf = run(GPCR(Config(), differentiable_alpha=True, gradient_exchange=_LocalExchange(R, v, store, True)), v)
        assert float((gx - dense_x).abs().max()) <= 4.0 * noise_x + 2e-6 * float(dense_x.abs().max())
        assert float((gf - dense_f).abs().max()) <= 4.0 * noise_f + 2e-6 * float(dense_f.abs().max())
    # the alpha terms are really in there: the image-only sum is clearly different
    img_f = torch.zeros_like(feat)
    for v in range(R):
        sc = views[v]
        sc.point_cloud, sc.point_cloud_features = xyz, feat
        xyz.grad = feat.grad = None
        image, _, _ = run_forward(GPCR(Config()), sc)
        image.backward(g_img[v])
        img_f += feat.grad
    assert float((img_f - dense_f)[:, 7].abs().max()) > 0.1 * float(dense_f[:, 7].abs().max())


def test_mask_supervised_fit_lowers_the_mask_loss():
    """Make every splat more transparent (opacity logit - 2) and fit the features to the unperturbed scene's accumulated
    alpha (a soft object mask) with an L1 loss on alpha alone.  On an H100 the mean L1 went from 0.278 to 0.017 in 40 steps
    (ratio 0.061); the bound leaves four times that margin."""
    scene = make_scene(3000, 64, 96, 0.08, 17, sh_degree=0)
    sc = cuda_scene(scene)
    op = GPCR(Config(), differentiable_alpha=True)
    with torch.no_grad():
        *_, target = run_forward(op, sc)
        target = target.clone()
    feats = sc.point_cloud_features.clone()
    feats[:, 7] -= 2.0
    feats.requires_grad_(True)
    opt = torch.optim.Adam([feats], lr=0.05)
    losses = []
    for _ in range(40):
        sc.point_cloud_features = feats
        *_, alpha = run_forward(op, sc)
        loss = (alpha - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    print(f"mask L1: first {losses[0]:.4f}  last {losses[-1]:.4f}  min {min(losses):.4f}")
    assert np.isfinite(losses).all()
    assert losses[-1] < 0.25 * losses[0]
