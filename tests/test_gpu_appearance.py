"""-m gpu: the bilateral-grid kernels (``csrc/appearance.cu``) against ``grid_sample`` autograd in float64, the appearance
grids in the fused train step (``gsb200_train_step_appearance``) against the autograd trainer, the NULL / overflow
contracts, and recovery of known per-view colour transforms."""
import dataclasses
import math

import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.appearance import apply_bilateral_grid, identity_grids
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from appearance_reference import random_case
from trainer_helpers import H, W, hidden_scene, initial_scene, poses, train_config

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(16, 16, 8), (1, 1, 1)])
@pytest.mark.parametrize("size", [(1072, 1920), (77, 129)])
def test_kernels_match_grid_sample_autograd_in_float64(size, shape):
    Hs, Ws = size
    image, grid = random_case(Hs, Ws, shape, seed=Hs + sum(shape))
    image, grid = image.float(), grid.float()
    grad_out = torch.randn((Hs, Ws, 3), generator=torch.Generator().manual_seed(3)) * 1e-3
    ref_i, ref_g = image.double().requires_grad_(True), grid.double().requires_grad_(True)
    ref = apply_bilateral_grid(ref_i, ref_g)  # CPU: the grid_sample form
    gi_ref, gg_ref = torch.autograd.grad(ref, (ref_i, ref_g), grad_out.double())
    outs = []
    for _ in range(2):
        i, g = image.cuda().requires_grad_(True), grid.cuda().requires_grad_(True)
        out = apply_bilateral_grid(i, g)
        gi, gg = torch.autograd.grad(out, (i, g), grad_out.cuda())
        outs.append((out.detach(), gi, gg))
    out, gi, gg = outs[0]
    assert float((out.double().cpu() - ref.detach()).abs().max()) <= 1e-5
    assert float((gi.double().cpu() - gi_ref).abs().max()) <= 1e-4 * float(gi_ref.abs().max())
    assert float((gg.double().cpu() - gg_ref).abs().max()) <= 1e-4 * float(gg_ref.abs().max())
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)  # deterministic: no float atomics


def _views(hidden, transform=None):
    """(image, q, t, camera) per pose rendered from the hidden scene on the GPU; ``transform(v, img)`` alters view v's
    (H, W, 3) render before the clamp.  Also returns the unaltered renders."""
    from taichi_3d_gaussian_splatting_b200 import CameraInfo
    dev = "cuda"
    K = hidden.camera_info.camera_intrinsics.to(dev)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    pc, feat = hidden.point_cloud.to(dev), hidden.point_cloud_features.to(dev)
    mask, obj = hidden.point_invalid_mask.to(dev), hidden.point_object_id.to(dev)
    views, clean = [], []
    for v, (q, t) in enumerate(poses()):
        q, t = q.to(dev), t.to(dev)
        with torch.no_grad():
            img, _, _ = op(GPCR.GaussianPointCloudRasterisationInput(
                point_cloud=pc, point_cloud_features=feat.clone(), point_object_id=obj, point_invalid_mask=mask,
                camera_info=CameraInfo(K, H, W, 0), q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3))
        clean.append(img.clamp(0, 1).permute(2, 0, 1).contiguous())
        shown = transform(v, img) if transform else img
        views.append((shown.clamp(0, 1).permute(2, 0, 1).contiguous(), q, t, CameraInfo(K, H, W, 0)))
    return views, clean


def test_fused_step_with_appearance_matches_the_autograd_trainer():
    """The first iteration (loss, TV, scene and grid gradients, the Adam step) with the tolerances of the supervised-step
    test, then a short run whose grids must stay close."""
    views, _ = _views(hidden_scene(n=400))
    for iters in (1, 6):
        cfg = dataclasses.replace(train_config(iters), appearance_grid=(4, 3, 2), appearance_learning_rate=5e-3,
                                  appearance_tv_weight=1.0)
        mk = lambda **kw: GaussianPointCloudTrainer(cfg, initial_scene(hidden_scene(n=400), device="cuda"), views, **kw)  # noqa: E731
        t_ref, t_fused = mk(), mk(fused_step=True)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            h_ref = t_ref.train(log_interval=1)
        h_fused = t_fused.train(log_interval=1)
        for a, b in zip(h_ref, h_fused):
            assert abs(a["loss"] - b["loss"]) <= 2e-6 * abs(a["loss"]) + 1e-7 + (0 if iters == 1 else 1e-4), (a, b)
            assert abs(a["appearance_tv"] - b["appearance_tv"]) <= 1e-5 * abs(a["appearance_tv"]) + 1e-9
        G_ref, G_fused = t_ref.appearance_grids(), t_fused.appearance_grids()
        lr = cfg.appearance_learning_rate
        if iters == 1:
            s = t_fused.fused_train_step
            g_ref = t_ref._appearance_leaves[0].grad
            assert float((s.grad_appearance_grid - g_ref).abs().max()) <= 1e-4 * float(g_ref.abs().max())
            gx_ref = t_ref.scene.point_cloud.grad
            assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max())
            solid = g_ref.abs() > 1e-3 * g_ref.abs().max()
            assert float((G_ref[0] - G_fused[0])[solid].abs().max()) <= 0.02 * lr
            assert torch.equal(G_ref[1:], G_fused[1:])  # views not visited: untouched
        else:
            assert float((G_ref - G_fused).abs().max()) <= 0.2 * lr * iters


class _NullAppearance:
    """Routes every train-step call of a FusedTrainStep through gsb200_train_step_appearance with NULL appearance."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def gsb200_train_step(self, args):
        return self._lib.gsb200_train_step_appearance(args, None, None, None)


def test_null_appearance_is_the_plain_train_step():
    """One step through gsb200_train_step_appearance(args, NULL, NULL, NULL) against gsb200_train_step on the same state:
    the image and the loss bit for bit; the gradients and updated tensors within the spread of two plain steps (the
    backward blend's float atomics)."""
    views, _ = _views(hidden_scene(n=400))
    img, q, t, cam = views[1]
    states = {}
    for name in ("plain", "plain_again", "null"):
        sc = initial_scene(hidden_scene(n=400), device="cuda")
        scene = Scene(sc.point_cloud.detach().contiguous(), sc.point_cloud_features.detach().contiguous(),
                      sc.point_invalid_mask, sc.point_object_id)
        step = FusedTrainStep(scene, GPCR.GaussianPointCloudRasterisationConfig())
        if name == "null":
            step._lib = _NullAppearance(step._lib)
        step.run(img, q, t, cam, 1, 5e-3, 2e-4)
        torch.cuda.synchronize()
        states[name] = dict(image=step.image.clone(), loss=step.loss.clone(), gx=step.grad_pointcloud.clone(),
                            gf=step.grad_pointcloud_features.clone(), xyz=scene.point_cloud.clone(),
                            feat=scene.point_cloud_features.clone())
    ref, again, st = states["plain"], states["plain_again"], states["null"]
    assert torch.equal(st["image"], ref["image"]) and torch.equal(st["loss"], ref["loss"])
    for key in ("gx", "gf", "xyz", "feat"):
        spread = float((again[key] - ref[key]).abs().max())
        assert float((st[key] - ref[key]).abs().max()) <= 4 * spread, key


def test_key_capacity_overflow_leaves_the_grid_and_its_moments_untouched():
    views, _ = _views(hidden_scene(n=400))
    sc = initial_scene(hidden_scene(n=400), device="cuda")
    scene = Scene(sc.point_cloud.detach().contiguous(), sc.point_cloud_features.detach().contiguous(),
                  sc.point_invalid_mask, sc.point_object_id)
    grids = identity_grids(len(views), (4, 4, 2), device="cuda")
    grids += 0.01 * torch.randn(grids.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    before = grids.clone()
    step = FusedTrainStep(scene, GPCR.GaussianPointCloudRasterisationConfig(), key_capacity=64, appearance_grids=grids)
    img, q, t, cam = views[0]
    step.run(img, q, t, cam, 1, 5e-3, 2e-4, appearance_view=0)
    torch.cuda.synchronize()
    assert torch.equal(grids, before)
    assert not step.appearance_exp_avg.any() and not step.appearance_exp_avg_sq.any()
    with pytest.warns(UserWarning, match="no-op"):
        step.run(img, q, t, cam, 1, 5e-3, 2e-4, appearance_view=1)
    assert step.num_skipped_steps == 1


def _affine(v):
    """A known gain, white balance and offset of view v."""
    gain = (0.85, 1.0, 0.9, 0.8)[v]
    wb = ((1.0, 0.95, 0.85), (0.9, 1.0, 1.05), (1.05, 0.9, 1.0), (0.95, 1.05, 0.9))[v]
    off = ((0.02, 0.0, 0.03), (0.0, 0.03, 0.0), (0.03, 0.02, 0.0), (0.0, 0.0, 0.04))[v]
    M = torch.zeros(3, 4)
    for i in range(3):
        M[i, i] = gain * wb[i]
        M[i, 3] = off[i]
    return M


def test_recovery_of_per_view_affines_with_one_node_grids():
    """Views of the hidden scene through a known per-view affine; the scene stays the hidden scene and only the (1, 1, 1)
    grids train.  Each recovered affine must match the known one.  Measured on an H100 80GB HBM3 at a 700 W power limit:
    largest entry error 0.0025, mean colour error 0.00065 on the worst view."""
    hidden = hidden_scene(n=400)
    Ms = [_affine(v).cuda() for v in range(4)]
    views, clean = _views(hidden, lambda v, img: img @ Ms[v][:, :3].T + Ms[v][:, 3])
    cfg = dataclasses.replace(train_config(2400), feature_learning_rate=0.0, position_learning_rate=0.0,
                              initial_downsample_factor=1, appearance_grid=(1, 1, 1), appearance_learning_rate=2e-3,
                              appearance_tv_weight=0.0)
    scene = initial_scene(hidden, capacity_ratio=1.0, device="cuda")
    with torch.no_grad():
        scene.point_cloud.copy_(hidden.point_cloud.cuda())
        scene.point_cloud_features.copy_(hidden.point_cloud_features.cuda())
    trainer = GaussianPointCloudTrainer(cfg, scene, views, fused_step=True)
    trainer.train()
    G = trainer.appearance_grids().reshape(4, 3, 4).cpu()
    err = max(float((G[v] - Ms[v].cpu()).abs().max()) for v in range(4))
    # the recovered affine applied to the views' colours: what the grid has to explain
    col = max(float((torch.einsum("ij,jhw->ihw", G[v][:, :3].cuda() - Ms[v][:, :3], clean[v]) +
                     (G[v][:, 3].cuda() - Ms[v][:, 3])[:, None, None]).abs().mean()) for v in range(4))
    print(f"max |recovered - known| affine entry: {err:.4f}; mean |colour error| (worst view): {col:.5f}")
    assert err <= 0.01 and col <= 0.003, (G, Ms)


def test_recovery_with_vignetting_beats_training_without_appearance():
    """Per-view gains with a radial vignette, scene and (16, 16, 8) grids trained together from initial_scene: the raw
    render's PSNR against the unaltered renders must beat the same run without appearance grids.  Measured on an H100 80GB
    HBM3 at a 700 W power limit: 25.57 dB without and 30.97 dB with the grids (+5.4 dB); the margin is 2.5 dB."""
    hidden = hidden_scene(n=400)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H, device="cuda"), torch.linspace(-1, 1, W, device="cuda"), indexing="ij")
    vignette = 1.0 - 0.35 * (xs ** 2 + ys ** 2) / 2
    gains = (0.7, 1.0, 0.85, 1.15)
    views, clean = _views(hidden, lambda v, img: img * (gains[v] * vignette)[..., None])
    results = {}
    for name, grid in (("off", None), ("on", (16, 16, 8))):
        cfg = dataclasses.replace(train_config(600), initial_downsample_factor=1, appearance_grid=grid)
        trainer = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views, fused_step=True)
        trainer.train()
        clean_views = [(c,) + tuple(v[1:]) for c, v in zip(clean, views)]
        results[name] = trainer.validation(clean_views)
    print(f"PSNR of the raw render against the unaltered views: without appearance {results['off']:.2f} dB, "
          f"with (16, 16, 8) grids {results['on']:.2f} dB")
    assert math.isfinite(results["on"])
    assert results["on"] > results["off"] + 2.5
