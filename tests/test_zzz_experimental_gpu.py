"""The second implementation of the blend backward and the fused trainer-step kernels on the GPU: the transposed backward
(the default; ``backward_impl="butterfly"`` selects the other kernel) against the butterfly kernel and the oracle, and
``gsb200_image_loss`` / ``gsb200_adam_step`` / ``gsb200_controller_update`` against their torch counterparts.

Their logic is also verified on the CPU (tests/test_simt_blend_cpu.py, tests/test_simt_pipeline_cpu.py,
tests/test_simt_image_loss_cpu.py: the unmodified kernel sources under a lock-step SIMT emulator).  The module sorts after
every other test module."""
import numpy as np
import pytest
import torch

from gpu_helpers import Config, cuda_scene, n, run_forward
from helpers import grad_close, oracle_backward, oracle_forward
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H,W,lam", [(64, 96, 0.2), (37, 29, 0.2), (544, 976, 0.2), (32, 32, 1.0)])
def test_fused_image_loss_matches_the_torch_loss(H, W, lam):
    """gsb200_image_loss (csrc/image_loss.cu; logic verified on the CPU in tests/test_simt_image_loss_cpu.py) vs the
    torch restatement of the reference's loss with autograd, on the GPU."""
    from taichi_3d_gaussian_splatting_b200.loss import LossFunction, fused_image_loss
    g = torch.Generator().manual_seed(H + W)
    gt = torch.rand((3, H, W), generator=g).cuda()
    pred = (gt.permute(1, 2, 0) + 0.3 * torch.randn((H, W, 3), generator=g).cuda()).contiguous()
    fn = LossFunction(LossFunction.LossFunctionConfig(lambda_value=lam, enable_regularization=False))
    a = pred.clone().requires_grad_(True)
    # the torch restatement convolves with cuDNN, which may run float32 convolutions in TF32 (10-bit mantissa): the float32
    # parity target must not
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        loss_a, l1_a, ds_a = fn(torch.clamp(a, min=0, max=1).permute(2, 0, 1), gt)
        (3.0 * loss_a).backward()
    b = pred.clone().requires_grad_(True)
    loss_b, l1_b, ds_b = fused_image_loss(b, gt, lam)
    (3.0 * loss_b).backward()
    assert abs(float(loss_a) - float(loss_b)) <= 2e-6 * max(1.0, abs(float(loss_a)))
    assert abs(float(l1_a) - float(l1_b)) <= 2e-6 and abs(float(ds_a) - float(ds_b)) <= 1e-5
    scale = float(a.grad.abs().max())
    assert float((a.grad - b.grad).abs().max()) <= 5e-5 * scale
    loss_c, _, _ = fn.forward_rasterized(pred, gt)
    assert abs(float(loss_c) - float(loss_b)) <= 1e-7


@pytest.mark.parametrize("shape", [(1000, 56), (1000, 3), (7,)])
def test_fused_adam_follows_torch_adam(shape):
    """optim.FusedAdam (gsb200_adam_step) vs torch.optim.Adam as the reference trainer configures it, with the
    ExponentialLR schedule of the position optimiser (GaussianPointTrainer.py:126-132)."""
    from taichi_3d_gaussian_splatting_b200 import FusedAdam
    g = torch.Generator().manual_seed(3)
    w0 = torch.randn(shape, generator=g).cuda()
    a, b = w0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
    oa, ob = torch.optim.Adam([a], lr=5e-3, betas=(0.9, 0.999)), FusedAdam([b], lr=5e-3, betas=(0.9, 0.999))
    sa, sb = (torch.optim.lr_scheduler.ExponentialLR(o, gamma=0.97) for o in (oa, ob))
    for step in range(8):
        grad = (torch.randn(shape, generator=g) * 10.0 ** (step % 4 - 2)).cuda()
        a.grad, b.grad = grad.clone(), grad.clone()
        oa.step(); ob.step(); sa.step(); sb.step()
        assert float((a - b).abs().max()) <= 1e-6 * max(1.0, float(w0.abs().max()))
    assert torch.allclose(oa.state[a]["exp_avg_sq"], ob.state[b]["exp_avg_sq"], rtol=1e-5, atol=0)


def test_trainer_with_the_fused_step_follows_the_torch_step():
    """The trainer loop with the fused image loss, Adam and controller update vs the same loop with torch's ops."""
    from trainer_helpers import hidden_scene, initial_scene, render_views, train_config
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer
    hidden = hidden_scene(n=400)
    views = render_views(GPCR(Config()), hidden, device="cuda")
    histories, psnrs = [], []
    for fused in (False, True):
        tr = GaussianPointCloudTrainer(train_config(40), initial_scene(hidden, device="cuda"), views,
                                       fused_image_loss=fused, fused_adam=fused, fused_controller_update=fused)
        histories.append(tr.train(log_interval=1))
        psnrs.append(tr.validation())
    for ha, hb in zip(*histories):
        assert abs(ha["loss"] - hb["loss"]) <= 2e-3 * abs(ha["loss"]), (ha, hb)
    assert abs(psnrs[0] - psnrs[1]) < 0.1, psnrs


def test_fused_controller_update_matches_the_torch_update():
    """gsb200_controller_update vs GaussianPointAdaptiveController.update's torch ops (GaussianPointAdaptiveController.py:130-143)."""
    from taichi_3d_gaussian_splatting_b200 import GaussianPointAdaptiveController as C
    g = torch.Generator().manual_seed(2)
    N, M = 5000, 1800
    mp = lambda: C.GaussianPointAdaptiveControllerMaintainedParameters(  # noqa: E731
        pointcloud=torch.zeros((N, 3), device="cuda"), pointcloud_features=torch.zeros((N, 56), device="cuda"),
        point_invalid_mask=torch.zeros(N, dtype=torch.int8, device="cuda"), point_object_id=torch.zeros(N, dtype=torch.int32, device="cuda"))
    cfg = C.GaussianPointAdaptiveControllerConfig(num_iterations_warm_up=10 ** 9)
    a, b = C(cfg, mp()), C(cfg, mp(), fused_update=True)
    for it in range(3):
        ids = torch.randperm(N, generator=g)[:M].sort().values.to(torch.int32).cuda()
        npix = torch.randint(0, 50, (M,), generator=g, dtype=torch.int32).cuda()
        mag = (torch.rand(M, generator=g) * (npix.cpu() > 0)).cuda()
        h = GPCR.BackwardValidPointHookInput(
            point_id_in_camera_list=ids, grad_point_in_camera=torch.randn((M, 3), generator=g).cuda(),
            grad_pointfeatures_in_camera=torch.zeros((M, 56), device="cuda"), grad_viewspace=torch.zeros((M, 2), device="cuda"),
            magnitude_grad_viewspace=mag, magnitude_grad_viewspace_on_image=torch.zeros((16, 16, 2), device="cuda"),
            num_overlap_tiles=torch.ones(M, dtype=torch.int32, device="cuda"), num_affected_pixels=npix,
            point_depth=torch.ones(M, device="cuda"), point_uv_in_camera=torch.zeros((M, 2), device="cuda"))
        a.update(h)
        b.update(h)
    for name in ("accumulated_num_in_camera", "accumulated_num_pixels"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    for name in ("accumulated_view_space_position_gradients", "accumulated_view_space_position_gradients_avg",
                 "accumulated_position_gradients", "accumulated_position_gradients_norm"):
        assert torch.allclose(getattr(a, name), getattr(b, name), rtol=1e-6, atol=1e-7), name


# ---------------------------------------------------------------- the transposed blend backward (last)
def _run(scene, impl, exact, hook_store=None, band=3):
    sc = cuda_scene(scene, requires_grad=True)
    hook = (lambda h: hook_store.__setitem__("h", h)) if hook_store is not None else None
    op = GPCR(Config(), backward_valid_point_hook=hook, exact_exp=exact, backward_impl=impl)
    image, _, _ = run_forward(op, sc, band=band)
    g = torch.Generator().manual_seed(5)
    grad_image = torch.randn(image.shape, generator=g, dtype=torch.float32)
    image.backward(grad_image.cuda())
    return n(image), n(sc.point_cloud.grad), n(sc.point_cloud_features.grad), grad_image.numpy()


SCENES = [dict(num_points=4000, height=64, width=96, sigma_med=0.05, seed=11),
          dict(num_points=60000, height=128, width=128, sigma_med=0.04, seed=12),   # > 256-entry tile lists, saturation
          dict(num_points=1500, height=128, width=192, sigma_med=0.4, seed=13)]     # large splats


@pytest.mark.parametrize("scene_args", SCENES)
@pytest.mark.parametrize("exact", [True, False])
def test_transposed_backward_matches_the_default_backward(scene_args, exact):
    scene = make_scene(sh_degree=3, **scene_args)
    ref_store, got_store = {}, {}
    img_a, gx_a, gf_a, _ = _run(scene, "butterfly", exact, ref_store)
    img_b, gx_b, gf_b, _ = _run(scene, "transposed", exact, got_store)
    assert np.array_equal(img_a, img_b)
    assert grad_close(gx_b, gx_a, rtol=1e-4, floor_frac=2e-6)[0], grad_close(gx_b, gx_a, rtol=1e-4, floor_frac=2e-6)
    for sl in (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56)):
        assert grad_close(gf_b[:, sl], gf_a[:, sl], rtol=1e-4, floor_frac=2e-6)[0], sl
    a, b = ref_store["h"], got_store["h"]
    assert torch.equal(a.num_affected_pixels, b.num_affected_pixels)
    if exact:  # the per-pixel recursion is the same code in both kernels
        assert torch.equal(a.magnitude_grad_viewspace_on_image, b.magnitude_grad_viewspace_on_image)
    else:      # fast path: both take alpha from fast_alpha; the transposed kernel re-derives conic * d from the scaled conic
        assert torch.allclose(a.magnitude_grad_viewspace_on_image, b.magnitude_grad_viewspace_on_image, rtol=1e-5,
                              atol=1e-6 * float(a.magnitude_grad_viewspace_on_image.abs().max()))
    assert grad_close(n(b.magnitude_grad_viewspace), n(a.magnitude_grad_viewspace), rtol=1e-4, floor_frac=2e-6)[0]
    assert grad_close(n(b.grad_viewspace), n(a.grad_viewspace), rtol=1e-4, floor_frac=2e-6)[0]
    # without a hook the statistics are skipped; the gradients do not change
    _, gx_c, gf_c, _ = _run(scene, "transposed", exact, None)
    assert grad_close(gx_c, gx_b, rtol=1e-5, floor_frac=1e-6)[0] and grad_close(gf_c, gf_b, rtol=1e-5, floor_frac=1e-6)[0]


def test_default_backward_without_hook_statistics():
    """GSB_FLAG_NO_HOOK_STATS in the butterfly kernel: same gradients, no statistics work."""
    scene = make_scene(num_points=4000, height=64, width=96, sigma_med=0.05, seed=11, sh_degree=3)
    grads = []
    for skip in (False, True):
        sc = cuda_scene(scene, requires_grad=True)
        op = GPCR(Config(), skip_unused_hook_statistics=skip)
        image, _, _ = run_forward(op, sc)
        image.backward(torch.randn(image.shape, generator=torch.Generator().manual_seed(5)).cuda())
        grads.append((n(sc.point_cloud.grad), n(sc.point_cloud_features.grad)))
    assert grad_close(grads[1][0], grads[0][0], rtol=1e-5, floor_frac=1e-6)[0]
    assert grad_close(grads[1][1], grads[0][1], rtol=1e-5, floor_frac=1e-6)[0]


def test_transposed_backward_vs_oracle():
    scene = make_scene(num_points=4000, height=64, width=96, sigma_med=0.05, seed=11, sh_degree=3)
    o, fwd, feats_n = oracle_forward(scene)
    _, gx, gf, grad_image = _run(scene, "transposed", True, None)
    bwd = oracle_backward(o, fwd, scene, feats_n, grad_image, 3)
    assert grad_close(gx, bwd.grad_pointcloud)[0], grad_close(gx, bwd.grad_pointcloud)
    for sl in (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56)):
        assert grad_close(gf[:, sl], bwd.grad_pointcloud_features[:, sl])[0], sl
