"""Appearance grids in the trainer's autograd loop (``TrainConfig.appearance_grid``), on the CPU: configuration checks,
identity grids at learning rate 0 leave the training trajectory unchanged (with the oracle as rasteriser), and the slice is
applied to whatever image the operator returns (a stub rasteriser and a lens view)."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.appearance import apply_bilateral_grid, bilateral_grid_tv, identity_grids
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.loss import LossFunction
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene

from oracle_module import OracleRasterisationModule
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config


def _stub_trainer(lens=None, **kw):
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    g = torch.Generator().manual_seed(0)
    gts = [torch.rand((3, 32, 48), generator=g) for _ in range(2)]
    ci = sc.camera_info
    views = [(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, CameraInfo(ci.camera_intrinsics, 32, 48, 0, lens))
             for gt in gts]
    rendered = torch.rand((32, 48, 3), generator=g) * 1.2 - 0.1
    seen = []

    class Stub:
        """Returns a fixed image that depends on the scene's features (so the scene gets a gradient too)."""

        def __init__(self, **kwargs):
            pass

        def __call__(self, inp, **kw):
            seen.append(inp.camera_info)
            image = rendered + 0.0 * inp.point_cloud_features.sum()
            return image, torch.zeros(32, 48), torch.zeros(32, 48, dtype=torch.int32)

    cfg = T.TrainConfig(num_iterations=1, initial_downsample_factor=1, **kw)
    cfg.loss_function_config.enable_regularization = False
    return T(cfg, scene, views, rasterisation_factory=Stub), views, rendered, seen


@pytest.mark.parametrize("kw,match", [
    (dict(appearance_grid=(0, 1, 1)), "grid shape"), (dict(appearance_grid=(65, 1, 1)), "grid shape"),
    (dict(appearance_grid=(1, 1, 17)), "grid shape"), (dict(appearance_grid=(4, 4)), "grid shape"),
    (dict(appearance_grid=(1, 1, 1), appearance_learning_rate=-1e-3), "appearance_learning_rate"),
    (dict(appearance_grid=(1, 1, 1), appearance_learning_rate=math.nan), "appearance_learning_rate"),
    (dict(appearance_grid=(1, 1, 1), appearance_tv_weight=math.inf), "appearance_tv_weight"),
    (dict(appearance_grid=(1, 1, 1), appearance_tv_weight=-1.0), "appearance_tv_weight"),
])
def test_configuration_errors(kw, match):
    with pytest.raises(ValueError, match=match):
        _stub_trainer(**kw)


def test_each_view_gets_an_identity_leaf_and_off_means_none():
    trainer, views, _, _ = _stub_trainer(appearance_grid=(4, 3, 2))
    G = trainer.appearance_grids()
    assert G.shape == (2, 12, 2, 3, 4)
    ident = torch.zeros(3, 4)
    ident[:3, :3] = torch.eye(3)
    assert torch.equal(G, ident.reshape(12, 1, 1, 1).expand(2, 12, 2, 3, 4))
    assert all(g.is_leaf and g.requires_grad for g in trainer._appearance_leaves)
    assert _stub_trainer()[0].appearance_grids() is None


def test_slice_is_applied_to_whatever_image_the_operator_returns():
    """A lens view through a stub rasteriser: one iteration's loss is the image loss of the stub's image sliced through view
    0's grid, plus the TV term; only view 0's grid moves."""
    lens = LensDistortion("opencv", (-0.05, 0.01, 0, 0, 0))
    trainer, views, rendered, seen = _stub_trainer(lens=lens, appearance_grid=(3, 2, 2), appearance_learning_rate=1e-2,
                                                   appearance_tv_weight=0.5)
    with torch.no_grad():  # a grid that is not the identity, so that the slice shows in the loss
        trainer._appearance_leaves[0].mul_(1.1).add_(0.02)
    grid0 = trainer._appearance_leaves[0].detach().clone()
    hist = trainer.train(log_interval=1)
    assert seen and seen[0].distortion == lens
    lf = LossFunction(trainer.config.loss_function_config)
    want, l1, _ = lf(apply_bilateral_grid(rendered, grid0).clamp(0, 1).permute(2, 0, 1), views[0][0])
    tv = 0.5 * bilateral_grid_tv(grid0)
    assert hist[0]["appearance_tv"] == pytest.approx(float(tv), rel=1e-6)
    assert hist[0]["loss"] == pytest.approx(float(want + tv), rel=1e-6)
    assert hist[0]["l1"] == pytest.approx(float(l1), rel=1e-6)
    G = trainer.appearance_grids()
    assert not torch.equal(G[0], grid0)
    assert torch.equal(G[1], identity_grids(1, (3, 2, 2))[0])  # view 1 was not visited: no gradient, no step


def test_identity_grids_at_learning_rate_zero_match_appearance_off():
    hidden = hidden_scene(n=120)
    views = render_views(OracleRasterisationModule(GPCR.GaussianPointCloudRasterisationConfig()), hidden)
    hists = []
    for kw in ({}, dict(appearance_grid=(4, 4, 2), appearance_learning_rate=0.0)):
        cfg = train_config(12)
        for k, v in kw.items():
            setattr(cfg, k, v)
        trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)
        hists.append(trainer.train(log_interval=1))
        if kw:
            assert all(h["appearance_tv"] == 0.0 for h in hists[-1])
            G = trainer.appearance_grids()
            assert torch.equal(G, identity_grids(len(views), (4, 4, 2)))
    off, on = hists
    assert len(off) == len(on) == 12
    for a, b in zip(off, on):
        assert b["loss"] == pytest.approx(a["loss"], rel=1e-5, abs=1e-7)
        assert b["psnr"] == pytest.approx(a["psnr"], rel=1e-5)
        assert b["num_valid_points"] == a["num_valid_points"]
    assert np.isfinite([h["loss"] for h in on]).all()
