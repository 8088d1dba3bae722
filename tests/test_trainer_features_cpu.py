"""CPU checks of per-Gaussian feature training around the operator: the trainer's configuration errors and the options it
passes on, the down-sampled label and feature targets, and the densification controller keeping ``point_extra_features``
in step with the scene when it clones and splits Gaussians."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.densification import GaussianPointAdaptiveController as Controller
from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene, downsample_targets

from trainer_helpers import H, W, hidden_scene, initial_scene, poses, train_config

C = 6


def _views(labels=True, features=True, top=C - 1):
    hidden = hidden_scene(n=50)
    g = torch.Generator().manual_seed(1)
    views = []
    for q, t in poses():
        lab = torch.randint(-1, top + 1, (H, W), generator=g, dtype=torch.int32) if labels else None
        feat = torch.randn((H, W, C), generator=g) if features else None
        views.append((torch.rand(3, H, W, generator=g), q, t, hidden.camera_info, SupervisionTargets(labels=lab, features=feat)))
    return hidden, views


def _scene(hidden, channels=C):
    sc = initial_scene(hidden)
    n = sc.point_cloud.shape[0]
    return Scene(sc.point_cloud, sc.point_cloud_features, sc.point_invalid_mask, sc.point_object_id,
                 point_extra_features=None if channels is None else torch.zeros((n, channels), requires_grad=True))


class _Factory:
    def __init__(self):
        self.kwargs = None

    def __call__(self, config, backward_valid_point_hook=None, **kwargs):
        self.kwargs = kwargs
        return torch.nn.Identity()


def _cfg(**kw):
    return dataclasses.replace(train_config(1), **kw)


def _make(cfg, scene, views):
    return GaussianPointCloudTrainer(cfg, scene, views, rasterisation_factory=_Factory())


@pytest.mark.parametrize("kind", ["cross_entropy", "l2"])
def test_a_valid_configuration_passes_the_features_to_the_controller(kind):
    hidden, views = _views()
    scene = _scene(hidden)
    tr = _make(_cfg(feature_loss=kind, feature_loss_weight=0.5), scene, views)
    assert tr.adaptive_controller.maintained_parameters.point_extra_features is scene.point_extra_features
    assert tr.rasterisation is not None
    # without a feature loss the controller does not touch the features
    tr = _make(_cfg(), scene, views)
    assert tr.adaptive_controller.maintained_parameters.point_extra_features is None
    assert GaussianPointCloudTrainer.TrainConfig().feature_loss == "none"


@pytest.mark.parametrize("kw,views_kw,channels,match", [
    (dict(feature_loss="cross_entropy", feature_loss_weight=1.0), {}, None, "point_extra_features"),
    (dict(feature_loss="l2", feature_loss_weight=1.0), {}, None, "point_extra_features"),
    (dict(feature_loss="cross_entropy", feature_loss_weight=1.0), dict(labels=False), C, "labels on every view"),
    (dict(feature_loss="l2", feature_loss_weight=1.0), dict(features=False), C, "feature map on every view"),
    (dict(feature_loss="cross_entropy", feature_loss_weight=1.0), {}, 1, "C >= 2"),
    (dict(feature_loss="cross_entropy", feature_loss_weight=1.0), dict(top=C), C, "labels must be < C"),
    (dict(feature_loss="l2", feature_loss_weight=1.0), {}, C + 1, "C = 7 channels"),
    (dict(feature_loss="l2", feature_loss_weight=1.0), {}, 17, "1 <= C <= 16"),
    (dict(feature_loss="l1", feature_loss_weight=1.0), {}, C, "feature_loss must be one of"),
    (dict(feature_loss="l2", feature_loss_weight=0.0), {}, C, "feature_loss_weight"),
    (dict(feature_loss="l2", feature_loss_weight=math.nan), {}, C, "feature_loss_weight"),
])
def test_configuration_errors(kw, views_kw, channels, match):
    hidden, views = _views(**views_kw)
    with pytest.raises(ValueError, match=match):
        _make(_cfg(**kw), _scene(hidden, channels), views)


def test_downsampled_labels_and_features_are_nearest_neighbour_and_cropped():
    hidden = hidden_scene(n=50)
    cam = hidden.camera_info
    g = torch.Generator().manual_seed(0)
    labels = torch.randint(-5, 9, (H, W), generator=g, dtype=torch.int32)
    labels[0, 0] = 2147483647
    feats = torch.randn((H, W, C), generator=g)
    feats[::4, ::3, 1] = math.nan
    depth = torch.rand((H, W), generator=g) + 1
    tg = downsample_targets(SupervisionTargets(depth=depth, labels=labels, features=feats), cam, 2)
    h, w = tg.depth.shape
    assert tg.labels.shape == (h, w) and tg.labels.dtype == torch.int32 and tg.features.shape == (h, w, C)
    assert torch.equal(tg.labels, labels[0::2, 0::2][:h, :w]) and int(tg.labels[0, 0]) == 2147483647
    assert torch.equal(tg.features.isnan(), feats[0::2, 0::2][:h, :w].isnan())
    assert torch.equal(tg.features.nan_to_num(), feats[0::2, 0::2][:h, :w].nan_to_num())
    # the same pixels as the depth's nearest-neighbour resize, at a factor where rows are skipped unevenly
    index = torch.arange(H * W, dtype=torch.float32).reshape(H, W)
    tg3 = downsample_targets(SupervisionTargets(depth=index, labels=index.to(torch.int32)), cam, 3)
    assert torch.equal(tg3.labels, tg3.depth.to(torch.int32))


def _controller(n_alive=10, cap=16, channels=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    pc = torch.randn((cap, 3), generator=g)
    feat = torch.randn((cap, 56), generator=g)
    feat[:, 0:4] = torch.tensor([0.0, 0.0, 0.0, 1.0])
    feat[:, 4:7] = -2.0
    invalid = torch.ones(cap, dtype=torch.int8)
    invalid[:n_alive] = 0
    extra = torch.randn((cap, channels), generator=g)
    cfg = Controller.GaussianPointAdaptiveControllerConfig()
    mp = Controller.GaussianPointAdaptiveControllerMaintainedParameters(
        pointcloud=pc, pointcloud_features=feat, point_invalid_mask=invalid,
        point_object_id=torch.zeros(cap, dtype=torch.int32), point_extra_features=extra)
    return Controller(cfg, mp, generator=torch.Generator().manual_seed(1)), extra


def test_densification_copies_the_source_feature_rows_into_the_filled_slots():
    ctl, extra = _controller()
    before = extra.clone()
    src = torch.tensor([1, 4, 6, 7, 2, 9, 3, 8, 1])  # more candidates than free rows after the removals: 8 are placed
    shrink = torch.tensor([0.0, math.log(1.6), 0.0, math.log(1.6), 0.0, 0.0, math.log(1.6), 0.0, 0.0])[:, None]  # clones and splits
    ctl.densify_point_info = Controller.GaussianPointAdaptiveControllerDensifyPointInfo(
        floater_point_id=torch.tensor([0], dtype=torch.int64), transparent_point_id=torch.tensor([5], dtype=torch.int64),
        densify_point_id=src, densify_point_position_before_optimization=ctl.maintained_parameters.pointcloud[src].clone(),
        densify_size_reduction_factor=shrink, densify_point_grad_position=torch.zeros((src.shape[0], 3)))
    ctl._add_densify_points()
    slots = torch.tensor([0, 5, 10, 11, 12, 13, 14, 15])  # the removed rows first, then the spare ones, lowest ids first
    assert (ctl.maintained_parameters.point_invalid_mask[slots] == 0).all()
    assert torch.equal(extra[slots], before[src[:8]])
    untouched = np.setdiff1d(np.arange(16), slots.numpy())
    assert torch.equal(extra[untouched], before[untouched])  # the sources included: a split shrinks s, not the features


def test_densification_without_feature_rows_is_unchanged():
    ctl, _ = _controller()
    ctl.maintained_parameters.point_extra_features = None
    src = torch.tensor([1, 2])
    ctl.densify_point_info = Controller.GaussianPointAdaptiveControllerDensifyPointInfo(
        floater_point_id=torch.empty(0, dtype=torch.int64), transparent_point_id=torch.empty(0, dtype=torch.int64),
        densify_point_id=src, densify_point_position_before_optimization=ctl.maintained_parameters.pointcloud[src].clone(),
        densify_size_reduction_factor=torch.zeros((2, 1)), densify_point_grad_position=torch.zeros((2, 3)))
    ctl._add_densify_points()
    assert int((ctl.maintained_parameters.point_invalid_mask == 0).sum()) == 12
