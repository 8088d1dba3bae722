"""-m gpu: the depth, mask and background terms in the fused train step (``gsb200_train_step_aux`` through
``FusedTrainStep`` / the trainer's ``fused_step=True``) against the autograd loop on ``loss.supervision_loss``, the
NULL / all-off supervision against ``gsb200_train_step``, a fit, and the overflow no-op.  Targets are rendered from the
hidden scene: its depth map, and its accumulated alpha as the mask."""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
from taichi_3d_gaussian_splatting_b200.densification import GaussianPointAdaptiveController as Controller
from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer

from trainer_helpers import H, W, hidden_scene, initial_scene, poses, train_config

pytestmark = pytest.mark.gpu


def _render(scene_pc, scene_feat, mask, obj, K, q, t):
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_alpha=True)
    from taichi_3d_gaussian_splatting_b200 import CameraInfo
    with torch.no_grad():
        img, depth, _, alpha = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene_pc, point_cloud_features=scene_feat.clone(), point_object_id=obj, point_invalid_mask=mask,
            camera_info=CameraInfo(K, H, W, 0), q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3))
    return img, depth, alpha


def supervised_views(hidden, sparse_depth=False, straight=False):
    """(image, q, t, camera, SupervisionTargets(depth, mask)) per pose, rendered from the hidden scene on the GPU.  The
    image is the render on black, or with ``straight`` the colour of an RGBA capture (not multiplied by the alpha,
    which is what ``gt * m + (1 - m) * bg`` composites)."""
    from taichi_3d_gaussian_splatting_b200 import CameraInfo
    dev = "cuda"
    K = hidden.camera_info.camera_intrinsics.to(dev)
    args = (hidden.point_cloud.to(dev), hidden.point_cloud_features.to(dev), hidden.point_invalid_mask.to(dev),
            hidden.point_object_id.to(dev), K)
    views = []
    for i, (q, t) in enumerate(poses()):
        q, t = q.to(dev), t.to(dev)
        img, depth, alpha = _render(*args, q, t)
        depth = depth.clone()
        if sparse_depth:  # a LiDAR-like target: most pixels without a measurement (0 or NaN)
            g = torch.Generator(device=dev).manual_seed(i)
            holes = torch.rand(depth.shape, generator=g, device=dev) < 0.6
            depth[holes] = float("nan")
            depth[::3] = 0.0
        if straight:
            img = torch.where(alpha[..., None] > 1e-3, img / alpha.clamp_min(1e-3)[..., None], torch.zeros_like(img))
        views.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q, t, CameraInfo(K, H, W, 0),
                      SupervisionTargets(depth=depth.contiguous(), mask=alpha.clone().contiguous())))
    return views


def _config(iters, depth=0.0, mask=0.0, background="black"):
    cfg = train_config(iters)
    return dataclasses.replace(cfg, depth_loss_weight=depth, mask_loss_weight=mask, background=background)


def _pair(cfg, views, seed=11):
    """The autograd trainer (TF32 off is the caller's business) and the fused one on identical state and colours."""
    mk = lambda **kw: GaussianPointCloudTrainer(  # noqa: E731
        cfg, initial_scene(hidden_scene(n=400), device="cuda"), views,
        background_generator=torch.Generator(device="cuda").manual_seed(seed), **kw)
    return mk(), mk(fused_step=True)


CASES = {"depth": dict(depth=0.5), "mask": dict(mask=0.5), "white": dict(background="white"),
         "random_mask": dict(mask=0.3, background="random"), "all": dict(depth=0.4, mask=0.4, background="random")}


@pytest.mark.parametrize("name", sorted(CASES))
def test_first_iteration_fused_equals_autograd(name):
    views = supervised_views(hidden_scene(n=400), sparse_depth=(name == "all"))
    t_ref, t_fused = _pair(_config(1, **CASES[name]), views)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        h_ref = t_ref.train(log_interval=1)
    h_fused = t_fused.train(log_interval=1)
    for key in ("loss", "mask_loss", "depth_loss"):
        assert (key in h_ref[0]) == (key in h_fused[0])
        if key in h_ref[0]:
            # a composited background makes flat regions where the float32 SSIM variances E[x^2] - mu^2 cancel: the total
            # then also allows lambda times the D-SSIM tolerance of the image-loss kernel's own test (5e-6)
            slack = 0.2 * 5e-6 if key == "loss" and CASES[name].get("background") else 0.0
            assert abs(h_ref[0][key] - h_fused[0][key]) <= 2e-6 * abs(h_ref[0][key]) + 1e-7 + slack, (key, h_ref[0], h_fused[0])
    s = t_fused.fused_train_step
    gx_ref, gf_ref = t_ref.scene.point_cloud.grad, t_ref.scene.point_cloud_features.grad
    assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max())
    assert float((s.grad_pointcloud_features - gf_ref).abs().max()) <= 1e-4 * float(gf_ref.abs().max())
    for p_ref, p_fused, g, lr in ((t_ref.scene.point_cloud_features, t_fused.scene.point_cloud_features, gf_ref, 5e-3),
                                  (t_ref.scene.point_cloud, t_fused.scene.point_cloud, gx_ref, 2e-4)):
        solid = g.abs() > 1e-3 * g.abs().max()
        assert float((p_ref - p_fused).detach()[solid].abs().max()) <= 0.02 * lr


def _step_state(step, scene, ctl):
    torch.cuda.synchronize()
    return dict(image=step.image.clone(), loss=step.loss.clone(), gx=step.grad_pointcloud.clone(),
                gf=step.grad_pointcloud_features.clone(), xyz=scene.point_cloud.detach().clone(),
                feat=scene.point_cloud_features.detach().clone(),
                ctl=[a.clone() for a in (ctl.accumulated_num_in_camera, ctl.accumulated_num_pixels,
                                         ctl.accumulated_view_space_position_gradients,
                                         ctl.accumulated_view_space_position_gradients_avg,
                                         ctl.accumulated_position_gradients, ctl.accumulated_position_gradients_norm)])


class _AuxLib:
    """Routes FusedTrainStep's gsb200_train_step call to gsb200_train_step_aux with the given supervision block."""
    def __init__(self, lib, sup):
        self._real, self._sup = lib, sup

    def __getattr__(self, name):
        return getattr(self._real, name)

    def gsb200_train_step(self, args):
        return self._real.gsb200_train_step_aux(args, None if self._sup is None else ctypes.byref(self._sup))


def test_null_or_all_off_supervision_is_the_plain_train_step():
    hidden = hidden_scene(n=400)
    views = supervised_views(hidden)
    img, q, t, cam, tg = views[1]
    cfg = train_config(1)
    lib = _lib.load()
    states = {}
    for name in ("plain", "plain_again", "null", "all_off"):
        scene = initial_scene(hidden, device="cuda")
        ctl = Controller(cfg.adaptive_controller_config, Controller.GaussianPointAdaptiveControllerMaintainedParameters(
            pointcloud=scene.point_cloud, pointcloud_features=scene.point_cloud_features,
            point_invalid_mask=scene.point_invalid_mask, point_object_id=scene.point_object_id))
        step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, controller=ctl)
        if name == "null":
            step._lib = _AuxLib(lib, None)
        elif name == "all_off":  # targets present, weights zero, no background: every term off
            step._lib = _AuxLib(lib, _lib.GsbSupervisionArgs(
                depth_target=tg.depth.data_ptr(), mask_target=tg.mask.data_ptr(), background=None, depth_weight=0.0,
                mask_weight=0.0, grad_depth=None, grad_pixel_accumulated_alpha=None, loss_out3=None, temp=None, temp_bytes=0))
        step.run(img, q, t, cam, 3, 5e-3, 2e-4)
        states[name] = _step_state(step, scene, ctl)
    ref, again = states["plain"], states["plain_again"]
    for name in ("null", "all_off"):
        st = states[name]
        assert torch.equal(st["image"], ref["image"]) and torch.equal(st["loss"], ref["loss"])
        for key in ("gx", "gf", "xyz", "feat"):
            spread = float((again[key] - ref[key]).abs().max())  # the float atomics of the backward blend
            err = float((st[key] - ref[key]).abs().max())
            assert err <= 4 * spread, (name, key, err, spread)
        for a, b, c in zip(st["ctl"], ref["ctl"], again["ctl"]):
            spread = float((c.double() - b.double()).abs().max())
            assert float((a.double() - b.double()).abs().max()) <= 4 * spread, name


def test_trajectories_with_depth_mask_and_random_background():
    views = supervised_views(hidden_scene(n=400), sparse_depth=True)
    iters = 80
    t_ref, t_fused = _pair(_config(iters, depth=0.3, mask=0.3, background="random"), views)
    h_ref = t_ref.train(log_interval=1)
    h_fused = t_fused.train(log_interval=1)
    assert t_fused.fused_train_step.num_skipped_steps == 0
    # the total as in the image-only trajectory test; a single term's share drifts faster relative to its own size
    for key, tol in (("loss", 2e-3), ("mask_loss", 1e-2), ("depth_loss", 1e-2)):
        a, b = np.array([h[key] for h in h_ref]), np.array([h[key] for h in h_fused])
        assert np.abs(a - b).max() < tol * a.max(), (key, np.abs(a - b).max(), a.max())
    a, b = t_ref.adaptive_controller, t_fused.adaptive_controller
    assert a.iteration_counter == b.iteration_counter == iters - 1
    assert torch.equal(a.accumulated_num_in_camera, b.accumulated_num_in_camera)
    assert float((a.accumulated_num_pixels - b.accumulated_num_pixels).abs().float().mean()) < 0.05 * float(a.accumulated_num_pixels.float().mean() + 1)
    for x, y in ((a.accumulated_view_space_position_gradients, b.accumulated_view_space_position_gradients),
                 (a.accumulated_position_gradients_norm, b.accumulated_position_gradients_norm)):
        assert float((x - y).abs().sum()) < 0.05 * float(x.abs().sum())


def _errors(scene, views):
    """Mean |D - d*| over the valid target pixels and mean |S - m|, over the views at full resolution."""
    pc, feat = scene.point_cloud.detach(), scene.point_cloud_features.detach()
    d_err, m_err = [], []
    for img, q, t, cam, tg in views:
        _, depth, alpha = _render(pc, feat, scene.point_invalid_mask, scene.point_object_id, cam.camera_intrinsics, q, t)
        valid = torch.isfinite(tg.depth) & (tg.depth > 0)
        d_err.append(float((depth - tg.depth)[valid].abs().mean()))
        m_err.append(float((alpha - tg.mask).abs().mean()))
    return float(np.mean(d_err)), float(np.mean(m_err))


def test_depth_and_mask_supervision_fit_better_than_the_image_alone():
    hidden = hidden_scene(n=400)
    views = supervised_views(hidden)  # on black, as a black-background run sees its images
    rgba_views = supervised_views(hidden, straight=True)  # RGBA captures: composited by their masks
    iters = 120
    runs = {}
    for name, kw in (("image", {}), ("depth", dict(depth=1.0)), ("random_mask", dict(background="random"))):
        trainer = GaussianPointCloudTrainer(_config(iters, **kw), initial_scene(hidden, device="cuda"),
                                            rgba_views if name == "random_mask" else views, fused_step=True,
                                            background_generator=torch.Generator(device="cuda").manual_seed(5))
        trainer.train()
        assert trainer.fused_train_step.num_skipped_steps == 0
        runs[name] = _errors(trainer.scene, views)
    start = _errors(initial_scene(hidden, device="cuda"), views)
    print(f"depth / mask error: start {start}, image only {runs['image']}, depth {runs['depth']}, "
          f"random background + mask {runs['random_mask']}")
    # measured on an H100 (120 iterations): depth error 0.081 vs 0.299 image only (0.339 at the start); mask error
    # 0.034 with a random background vs 0.049 on black (0.137 at the start)
    assert runs["depth"][0] < 0.5 * runs["image"][0], runs
    assert runs["random_mask"][1] < 0.85 * runs["image"][1], runs


def test_overflowing_frame_is_a_no_op_with_supervision_terms():
    hidden = hidden_scene(n=400)
    views = supervised_views(hidden)
    scene = initial_scene(hidden, device="cuda")
    cfg = train_config(1)
    ctl = Controller(cfg.adaptive_controller_config, Controller.GaussianPointAdaptiveControllerMaintainedParameters(
        pointcloud=scene.point_cloud, pointcloud_features=scene.point_cloud_features, point_invalid_mask=scene.point_invalid_mask,
        point_object_id=scene.point_object_id))
    step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, controller=ctl, key_capacity=64, depth_weight=0.5,
                          mask_weight=0.5)
    xyz0, feat0 = scene.point_cloud.detach().clone(), scene.point_cloud_features.detach().clone()
    img, q, t, cam, tg = views[0]
    bg = torch.tensor([0.2, 0.5, 0.9], device="cuda")
    with pytest.warns(UserWarning, match="no-op on the device"):
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg, background=bg)
        torch.cuda.synchronize()
        assert torch.equal(scene.point_cloud.detach(), xyz0) and torch.equal(scene.point_cloud_features.detach()[:, 4:], feat0[:, 4:])
        assert float(step.feature_exp_avg.abs().max()) == 0.0 and float(step.position_exp_avg.abs().max()) == 0.0
        assert int(ctl.accumulated_num_in_camera.max()) == 0
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg, background=bg)
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg, background=bg)
    torch.cuda.synchronize()
    assert step.num_skipped_steps >= 1 and step.key_capacity > 64
    step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg, background=bg)
    torch.cuda.synchronize()
    assert not torch.equal(scene.point_cloud.detach(), xyz0) and int(ctl.accumulated_num_in_camera.max()) >= 1
    assert torch.isfinite(step.supervision_loss).all() and float(step.supervision_loss[1]) > 0 and float(step.supervision_loss[2]) > 0
