"""-m gpu: the fused training iteration (``gsb200_train_step`` / ``fused_step.FusedTrainStep``: forward, image loss, backward
with the controller accumulators in its epilogue, both Adam updates in ONE library call, no autograd) against the same loop
driven through autograd (operator + ``LossFunction`` + ``torch.optim.Adam`` + the hook-fed controller) and against the CPU
oracle behind the same trainer (BASELINE config 5 in miniature)."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer

from oracle_module import OracleRasterisationModule
from test_gpu_trainer import _views_to
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config

pytestmark = pytest.mark.gpu


def test_fused_step_follows_the_autograd_loop_and_the_oracle():
    hidden = hidden_scene(n=400)
    views_cpu = render_views(OracleRasterisationModule(GPCR.GaussianPointCloudRasterisationConfig()), hidden)
    views = _views_to(views_cpu, "cuda")
    iters = 80
    t_ref = GaussianPointCloudTrainer(train_config(iters), initial_scene(hidden, device="cuda"), views)
    h_ref = t_ref.train(log_interval=1)
    t_fused = GaussianPointCloudTrainer(train_config(iters), initial_scene(hidden, device="cuda"), views, fused_step=True)
    h_fused = t_fused.train(log_interval=1)
    assert t_fused.fused_train_step.num_skipped_steps == 0
    l_ref, l_fused = np.array([h["loss"] for h in h_ref]), np.array([h["loss"] for h in h_fused])
    assert np.abs(l_ref - l_fused).max() < 2e-3 * l_ref.max(), np.abs(l_ref - l_fused).max()
    p_ref, p_fused = t_ref.validation(), t_fused.validation()
    assert p_ref > 26.0 and abs(p_ref - p_fused) < 0.15, (p_ref, p_fused)
    # the controller accumulators (never reset here: warm-up is infinite) were fed by the kernel epilogue resp. by the hook
    a, b = t_ref.adaptive_controller, t_fused.adaptive_controller
    assert a.iteration_counter == b.iteration_counter == iters - 1
    assert torch.equal(a.accumulated_num_in_camera, b.accumulated_num_in_camera)
    assert float((a.accumulated_num_pixels - b.accumulated_num_pixels).abs().float().mean()) < 0.05 * float(a.accumulated_num_pixels.float().mean() + 1)
    for x, y in ((a.accumulated_view_space_position_gradients, b.accumulated_view_space_position_gradients),
                 (a.accumulated_position_gradients_norm, b.accumulated_position_gradients_norm)):
        assert float((x - y).abs().sum()) < 0.05 * float(x.abs().sum())
    # and the oracle-backed trainer (CPU) on the same data: PSNR parity of the fused path with the reference arithmetic
    t_cpu = GaussianPointCloudTrainer(train_config(iters), initial_scene(hidden), views_cpu, rasterisation_factory=OracleRasterisationModule)
    t_cpu.train()
    p_cpu = t_cpu.validation()
    assert abs(p_cpu - p_fused) < 0.2, (p_cpu, p_fused)


def test_fused_step_first_iteration_is_the_autograd_iteration():
    """ONE iteration from identical state: same loss, same gradients (up to the float atomics), same updated parameters."""
    hidden = hidden_scene(n=400)
    views = render_views(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), hidden, device="cuda")
    t_ref = GaussianPointCloudTrainer(train_config(1), initial_scene(hidden, device="cuda"), views)
    # the autograd loss convolves with cuDNN, which may run float32 convolutions in TF32 (10-bit mantissa); the fused
    # step's loss kernel computes in float32, and so must the iteration it is compared with
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        h_ref = t_ref.train(log_interval=1)
    t_fused = GaussianPointCloudTrainer(train_config(1), initial_scene(hidden, device="cuda"), views, fused_step=True)
    h_fused = t_fused.train(log_interval=1)
    assert abs(h_ref[0]["loss"] - h_fused[0]["loss"]) <= 2e-6 * abs(h_ref[0]["loss"]) + 1e-7
    s = t_fused.fused_train_step
    gx_ref, gf_ref = t_ref.scene.point_cloud.grad, t_ref.scene.point_cloud_features.grad
    assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max())
    assert float((s.grad_pointcloud_features - gf_ref).abs().max()) <= 1e-4 * float(gf_ref.abs().max())
    # Adam's first step moves every entry with a non-zero gradient by lr * sign(g): compare where |g| is not noise
    for p_ref, p_fused, g, lr in ((t_ref.scene.point_cloud_features, t_fused.scene.point_cloud_features, gf_ref, 5e-3),
                                  (t_ref.scene.point_cloud, t_fused.scene.point_cloud, gx_ref, 2e-4)):
        solid = g.abs() > 1e-3 * g.abs().max()
        assert float((p_ref - p_fused)[solid].abs().max()) <= 0.02 * lr


def test_fused_step_with_densification():
    hidden = hidden_scene(n=400)
    views = render_views(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), hidden, device="cuda")
    trainer = GaussianPointCloudTrainer(train_config(120, densify=True), initial_scene(hidden, device="cuda"), views, fused_step=True,
                                        generator=torch.Generator(device="cuda").manual_seed(3))
    psnr0 = trainer.validation()
    hist = trainer.train(log_interval=1)
    psnr1 = trainer.validation()
    assert psnr1 > psnr0 + 2.0, (psnr0, psnr1)
    assert np.mean([h["loss"] for h in hist[-8:]]) < 0.8 * np.mean([h["loss"] for h in hist[:8]])
    assert hist[-1]["num_valid_points"] > hist[0]["num_valid_points"]
    assert trainer.fused_train_step.num_skipped_steps == 0


def test_fused_step_overflow_turns_the_iteration_into_a_no_op():
    """Key capacity too small: the device-side overflow counter must leave parameters, Adam state and controller accumulators
    untouched; the host notices one iteration later, grows the capacity and counts the skipped iteration."""
    from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
    from taichi_3d_gaussian_splatting_b200.densification import GaussianPointAdaptiveController as Controller
    hidden = hidden_scene(n=400)
    views = render_views(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), hidden, device="cuda")
    scene = initial_scene(hidden, device="cuda")
    cfg = train_config(1)
    ctl = Controller(cfg.adaptive_controller_config, Controller.GaussianPointAdaptiveControllerMaintainedParameters(
        pointcloud=scene.point_cloud, pointcloud_features=scene.point_cloud_features, point_invalid_mask=scene.point_invalid_mask,
        point_object_id=scene.point_object_id))
    step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, controller=ctl, key_capacity=64)
    xyz0, feat0 = scene.point_cloud.detach().clone(), scene.point_cloud_features.detach().clone()
    img, q, t, cam = views[0]
    with pytest.warns(UserWarning, match="no-op on the device"):
        step.run(img, q, t, cam, 3, 5e-3, 2e-4)
        torch.cuda.synchronize()
        # q of the in-frustum rows is normalised in place by the forward (GPCR:264-266) even in a skipped iteration
        assert torch.equal(scene.point_cloud.detach(), xyz0) and torch.equal(scene.point_cloud_features.detach()[:, 4:], feat0[:, 4:])
        assert float(step.feature_exp_avg.abs().max()) == 0.0 and int(ctl.accumulated_num_in_camera.max()) == 0
        step.run(img, q, t, cam, 3, 5e-3, 2e-4)  # notices the overflow of the first call (and overflows itself: 2 slots)
        step.run(img, q, t, cam, 3, 5e-3, 2e-4)
    torch.cuda.synchronize()
    assert step.num_skipped_steps >= 1 and step.key_capacity > 64
    step.run(img, q, t, cam, 3, 5e-3, 2e-4)
    torch.cuda.synchronize()
    assert not torch.equal(scene.point_cloud.detach(), xyz0) and int(ctl.accumulated_num_in_camera.max()) >= 1
