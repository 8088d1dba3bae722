"""-m gpu: per-Gaussian feature training in the fused train step (``gsb200_train_step_ext`` through ``FusedTrainStep`` / the
trainer's ``fused_step=True``) against the autograd loop on ``loss.feature_loss``, with and without the depth, mask and
background terms, over 80 iterations with densification, the NULL feature block against ``gsb200_train_step_aux``, the
overflow no-op, and fits of rendered label and feature maps.  Targets are rendered from the hidden scene through the
operator: labels from one-hot class logits of its Gaussians, feature maps from random per-Gaussian vectors."""
import ctypes
import dataclasses
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib, CameraInfo
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.densification import GaussianPointAdaptiveController as Controller
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets, feature_loss
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from test_gpu_supervised_train_step import supervised_views
from trainer_helpers import H, W, hidden_scene, initial_scene, train_config

pytestmark = pytest.mark.gpu

C_LABELS, C_FEATURES = 8, 16


def hidden_features(hidden, kind, C):
    """(N, C) per-Gaussian values of the hidden scene: one-hot logits of a class given by the Gaussian's angular sector
    around the scene centre (coherent regions), or random vectors."""
    pc = hidden.point_cloud
    if kind == "cross_entropy":
        ang = torch.atan2(pc[:, 1] - pc[:, 1].mean(), pc[:, 0] - pc[:, 0].mean())
        cls = ((ang + math.pi) / (2 * math.pi) * C).long().clamp(0, C - 1)
        return torch.nn.functional.one_hot(cls, C).float(), cls
    g = torch.Generator().manual_seed(17)
    return torch.randn((pc.shape[0], C), generator=g), None


def render_features(pc, feat, mask, obj, K, q, t, F):
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_alpha=True)
    with torch.no_grad():
        _, _, _, alpha, fmap = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=pc, point_cloud_features=feat.clone(), point_object_id=obj, point_invalid_mask=mask,
            camera_info=CameraInfo(K, H, W, 0), q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3),
            point_extra_features=F)
    return alpha, fmap


def feature_views(hidden, kind):
    """supervised_views (image, depth, mask) with the labels (alpha > 0.5: argmax of the rendered one-hot logits, else -1)
    or the C = 16 feature map (NaN where alpha < 0.05) added to the targets."""
    C = C_LABELS if kind == "cross_entropy" else C_FEATURES
    Fh = hidden_features(hidden, kind, C)[0].cuda()
    args = [x.cuda() for x in (hidden.point_cloud, hidden.point_cloud_features, hidden.point_invalid_mask,
                               hidden.point_object_id)]
    out = []
    for img, q, t, cam, tg in supervised_views(hidden):
        alpha, fmap = render_features(*args, cam.camera_intrinsics, q, t, Fh)
        if kind == "cross_entropy":
            labels = torch.where(alpha > 0.5, fmap.argmax(-1), torch.full_like(alpha, -1, dtype=torch.int64))
            tg = dataclasses.replace(tg, labels=labels.to(torch.int32).contiguous())
        else:
            target = fmap.clone()
            target[alpha < 0.05] = float("nan")
            tg = dataclasses.replace(tg, features=target.contiguous())
        out.append((img, q, t, cam, tg))
    return out


def feature_scene(hidden, C, device="cuda"):
    sc = initial_scene(hidden, device=device)
    F = torch.zeros((sc.point_cloud.shape[0], C), device=device, requires_grad=True)
    return Scene(sc.point_cloud, sc.point_cloud_features, sc.point_invalid_mask, sc.point_object_id, point_extra_features=F)


def _config(iters, kind, densify=False, depth=0.0, mask=0.0, background="black", weight=0.5, lr=1e-2):
    cfg = train_config(iters, densify=densify)
    return dataclasses.replace(cfg, depth_loss_weight=depth, mask_loss_weight=mask, background=background, feature_loss=kind,
                               feature_loss_weight=weight, extra_feature_learning_rate=lr)


def _pair(cfg, views, hidden, C, densify=False):
    mk = lambda **kw: GaussianPointCloudTrainer(  # noqa: E731
        cfg, feature_scene(hidden, C), views, background_generator=torch.Generator(device="cuda").manual_seed(11),
        generator=torch.Generator(device="cuda").manual_seed(3) if densify else None, **kw)
    return mk(), mk(fused_step=True)


CASES = {"ce": ("cross_entropy", {}), "l2": ("l2", {}),
         "ce_all": ("cross_entropy", dict(depth=0.4, mask=0.4, background="random")),
         "l2_all": ("l2", dict(depth=0.4, mask=0.4, background="random"))}


@pytest.mark.parametrize("name", sorted(CASES))
def test_first_iteration_fused_equals_autograd(name):
    kind, kw = CASES[name]
    hidden = hidden_scene(n=400)
    C = C_LABELS if kind == "cross_entropy" else C_FEATURES
    t_ref, t_fused = _pair(_config(1, kind, **kw), feature_views(hidden, kind), hidden, C)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        h_ref = t_ref.train(log_interval=1)
    h_fused = t_fused.train(log_interval=1)
    a, b = h_ref[0], h_fused[0]
    assert set(a) == set(b) and "feature_loss" in a
    assert abs(a["feature_loss"] - b["feature_loss"]) <= 1e-5 * abs(a["feature_loss"]), (a, b)
    slack = 0.2 * 5e-6 if kw.get("background") else 0.0  # as in the supervised step's own test
    for key in ("loss", "mask_loss", "depth_loss"):
        if key in a:
            assert abs(a[key] - b[key]) <= 2e-6 * abs(a[key]) + 1e-7 + slack, (key, a, b)
    s = t_fused.fused_train_step
    assert int(s.feature_loss[1]) > 0
    gx_ref, gf_ref = t_ref.scene.point_cloud.grad, t_ref.scene.point_cloud_features.grad
    ge_ref = t_ref.scene.point_extra_features.grad
    assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max())
    assert float((s.grad_pointcloud_features - gf_ref).abs().max()) <= 1e-4 * float(gf_ref.abs().max())
    assert float((s.grad_extra_features - ge_ref).abs().max()) <= 1e-4 * float(ge_ref.abs().max())
    # Adam's first step moves every entry with a non-zero gradient by lr * sign(g): compare where |g| is not noise
    for p_ref, p_fused, g, lr in ((t_ref.scene.point_cloud_features, t_fused.scene.point_cloud_features, gf_ref, 5e-3),
                                  (t_ref.scene.point_cloud, t_fused.scene.point_cloud, gx_ref, 2e-4),
                                  (t_ref.scene.point_extra_features, t_fused.scene.point_extra_features, ge_ref, 1e-2)):
        solid = g.abs() > 1e-3 * g.abs().max()
        assert float((p_ref - p_fused).detach()[solid].abs().max()) <= 0.02 * lr


@pytest.mark.parametrize("kind", ["cross_entropy", "l2"])
def test_trajectories_with_densification(kind):
    hidden = hidden_scene(n=400)
    C = C_LABELS if kind == "cross_entropy" else C_FEATURES
    iters = 80
    t_ref, t_fused = _pair(_config(iters, kind, densify=True, mask=0.3, background="random"), feature_views(hidden, kind),
                           hidden, C, densify=True)
    h_ref = t_ref.train(log_interval=1)
    h_fused = t_fused.train(log_interval=1)
    assert t_fused.fused_train_step.num_skipped_steps == 0
    for h in (h_ref, h_fused):  # the controller densified within the run
        assert h[-1]["num_valid_points"] > h[0]["num_valid_points"], [x["num_valid_points"] for x in h[::10]]
    for key, tol in (("loss", 2e-3), ("feature_loss", 1e-2), ("mask_loss", 1e-2)):
        a, b = np.array([h[key] for h in h_ref]), np.array([h[key] for h in h_fused])
        print(key, np.abs(a - b).max(), a.max())
        assert np.abs(a - b).max() < tol * a.max(), (key, np.abs(a - b).max(), a.max())


class _ExtLib:
    """Routes FusedTrainStep's gsb200_train_step_aux call to gsb200_train_step_ext with a NULL feature block."""
    def __init__(self, lib):
        self._real = lib

    def __getattr__(self, name):
        return getattr(self._real, name)

    def gsb200_train_step_aux(self, args, sup):
        return self._real.gsb200_train_step_ext(args, sup, None)


def test_null_feature_block_is_the_supervised_train_step():
    hidden = hidden_scene(n=400)
    img, q, t, cam, tg = supervised_views(hidden)[1]
    cfg = train_config(1)
    states = {}
    for name in ("aux", "aux_again", "ext_null"):
        scene = initial_scene(hidden, device="cuda")
        ctl = Controller(cfg.adaptive_controller_config, Controller.GaussianPointAdaptiveControllerMaintainedParameters(
            pointcloud=scene.point_cloud, pointcloud_features=scene.point_cloud_features,
            point_invalid_mask=scene.point_invalid_mask, point_object_id=scene.point_object_id))
        step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, controller=ctl, depth_weight=0.4, mask_weight=0.4)
        if name == "ext_null":
            step._lib = _ExtLib(step._lib)
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg, background=torch.tensor([0.3, 0.6, 0.1], device="cuda"))
        torch.cuda.synchronize()
        states[name] = dict(image=step.image.clone(), loss=step.loss.clone(), sup=step.supervision_loss.clone(),
                            gx=step.grad_pointcloud.clone(), gf=step.grad_pointcloud_features.clone(),
                            xyz=scene.point_cloud.detach().clone(), feat=scene.point_cloud_features.detach().clone())
    ref, again, st = states["aux"], states["aux_again"], states["ext_null"]
    for key in ("image", "loss", "sup"):  # the forward and the loss kernels are deterministic: bit-identical
        assert torch.equal(st[key], ref[key]), key
    for key in ("gx", "gf", "xyz", "feat"):  # the float atomics of the backward blend: within the run-to-run spread
        spread = float((again[key] - ref[key]).abs().max())
        assert float((st[key] - ref[key]).abs().max()) <= 4 * spread, key


def test_overflowing_frame_leaves_the_features_and_their_moments_untouched():
    hidden = hidden_scene(n=400)
    img, q, t, cam, tg = feature_views(hidden, "cross_entropy")[0]
    scene = feature_scene(hidden, C_LABELS)
    with torch.no_grad():
        scene.point_extra_features.normal_()
    cfg = train_config(1)
    step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, key_capacity=64, extra_features=scene.point_extra_features,
                          feature_loss="cross_entropy", feature_weight=0.5)
    F0 = scene.point_extra_features.detach().clone()
    with pytest.warns(UserWarning, match="no-op on the device"):
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg)
        torch.cuda.synchronize()
        assert torch.equal(scene.point_extra_features.detach(), F0)
        assert float(step.extra_feature_exp_avg.abs().max()) == 0.0 and float(step.extra_feature_exp_avg_sq.abs().max()) == 0.0
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg)
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg)
    torch.cuda.synchronize()
    assert step.num_skipped_steps >= 1 and step.key_capacity > 64
    step.run(img, q, t, cam, 3, 5e-3, 2e-4, targets=tg)
    torch.cuda.synchronize()
    assert not torch.equal(scene.point_extra_features.detach(), F0) and float(step.extra_feature_exp_avg.abs().max()) > 0
    assert torch.isfinite(step.feature_loss).all() and float(step.feature_loss[0]) > 0


def _feature_terms(scene, views, kind):
    """Mean feature term over the views at full resolution, and the labelled-pixel accuracy (cross entropy)."""
    terms, hit, n = [], 0, 0
    pc, feat, F = scene.point_cloud.detach(), scene.point_cloud_features.detach(), scene.point_extra_features.detach()
    for img, q, t, cam, tg in views:
        _, fmap = render_features(pc, feat, scene.point_invalid_mask, scene.point_object_id, cam.camera_intrinsics, q, t, F)
        terms.append(float(feature_loss(fmap, tg, kind, 1.0)))
        if kind == "cross_entropy":
            lab = tg.labels.long()
            valid = lab >= 0
            hit += int((fmap.argmax(-1) == lab)[valid].sum())
            n += int(valid.sum())
    return float(np.mean(terms)), hit / max(n, 1)


@pytest.mark.parametrize("kind", ["cross_entropy", "l2"])
def test_fused_trainer_fits_rendered_labels_and_feature_maps(kind):
    hidden = hidden_scene(n=400)
    views = feature_views(hidden, kind)
    C = C_LABELS if kind == "cross_entropy" else C_FEATURES
    trainer = GaussianPointCloudTrainer(_config(150, kind, weight=1.0, lr=5e-2), feature_scene(hidden, C), views,
                                        fused_step=True)
    start = _feature_terms(trainer.scene, views, kind)
    trainer.train()
    assert trainer.fused_train_step.num_skipped_steps == 0
    end = _feature_terms(trainer.scene, views, kind)
    print(f"{kind}: feature term {start[0]:.4f} -> {end[0]:.4f}, labelled-pixel accuracy {start[1]:.3f} -> {end[1]:.3f}")
    # measured on an H100 80GB HBM3 (400 W power limit), 150 iterations: cross entropy 2.079 -> 0.048 with labelled-pixel
    # accuracy 0.166 -> 0.996; l2 (C = 16) 0.126 -> 0.004
    assert end[0] < 0.3 * start[0], (start, end)
    if kind == "cross_entropy":
        assert end[1] > 0.9, (start, end)
