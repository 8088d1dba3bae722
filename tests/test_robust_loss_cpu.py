"""Per-pixel weights of the image loss on the CPU: ``RobustLossConfig``'s validation, properties of the torch statement
(``loss.robust_weight`` / ``robust_composite``), ``downsample_targets`` of ``loss_weight``, the dataset's
``loss_weight_path`` key, and the trainer's autograd loop (oracle-backed): the weights reach the loss, the history reports
the inlier fraction, and the view-parallel exchange is refused."""
import json
import math
import os

import numpy as np
import PIL.Image
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo
from taichi_3d_gaussian_splatting_b200.image_pose_dataset import MAX_RESOLUTION_TRAIN, ImagePoseDataset
from taichi_3d_gaussian_splatting_b200.loss import (RobustLossConfig, SupervisionTargets, _torch_image_loss,
                                                    robust_composite, robust_weight)
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, downsample_targets

from oracle_module import OracleRasterisationModule
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR


@pytest.mark.parametrize("kw", [dict(inlier_quantile=0.0), dict(inlier_quantile=1.5), dict(inlier_quantile=math.nan),
                                dict(box_threshold=-0.1), dict(box_threshold=1.1), dict(patch_threshold=2.0),
                                dict(patch_threshold=math.nan), dict(start_iteration=-1), dict(start_iteration=1.5)])
def test_config_rejects_values_outside_their_ranges(kw):
    with pytest.raises(ValueError):
        RobustLossConfig(**kw)


def test_config_defaults_and_limits():
    c = RobustLossConfig()
    assert (c.inlier_quantile, c.box_threshold, c.patch_threshold, c.start_iteration) == (0.9, 0.5, 0.6, 0)
    RobustLossConfig(inlier_quantile=1.0, box_threshold=0.0, patch_threshold=1.0)


def test_statement_properties():
    g = torch.Generator().manual_seed(1)
    H, W = 32, 48
    gt = torch.rand(3, H, W, generator=g)
    x = gt.permute(1, 2, 0) + 0.02 * torch.randn(H, W, 3, generator=g)
    x[8:24, 16:32] = torch.tensor([1.0, 0.0, 1.0])  # a distractor covering one tile
    w, stats = robust_weight(x, gt, None, RobustLossConfig(inlier_quantile=1.0))
    assert (w == 1).all() and stats[0] == 1.0
    w, stats = robust_weight(x, gt, None, RobustLossConfig(inlier_quantile=0.5))
    assert (w[8:24, 16:32] == 0).float().mean() > 0.9 and 0.4 < float(stats[0]) < 0.9
    s = torch.ones(H, W)
    s[:, :16] = 0.0
    ws, _ = robust_weight(x, gt, s, None)
    assert torch.equal(ws, s)
    xr = x.clone().requires_grad_(True)
    loss, _, _ = _torch_image_loss(robust_composite(xr, gt, ws), gt, 0.2)
    loss.backward()
    assert (xr.grad[:, :16] == 0).all() and (xr.grad[:, 16:] != 0).any()
    with pytest.raises(ValueError, match="multiples of 16"):
        robust_weight(x[:20], gt[:, :20], None, RobustLossConfig())


def test_downsample_targets_resizes_the_loss_weight_like_the_mask():
    H, W = 70, 100
    g = torch.Generator().manual_seed(2)
    m = torch.rand(H, W, generator=g)
    cam = CameraInfo(torch.eye(3), H, W, 0)
    out = downsample_targets(SupervisionTargets(mask=m, loss_weight=m.clone()), cam, 2)
    assert out.loss_weight.shape == (32, 48) and torch.equal(out.loss_weight, out.mask)
    assert downsample_targets(SupervisionTargets(), cam, 2).loss_weight is None


def _dataset(root, weight_files):
    rng = np.random.default_rng(4)
    records = []
    for i, (h, w, kind) in enumerate(weight_files):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        PIL.Image.fromarray(rgb, mode="RGB").save(os.path.join(root, f"img{i}.png"))
        rec = dict(image_path=f"img{i}.png", T_pointcloud_camera=np.eye(4).tolist(),
                   camera_intrinsics=[[100.0, 0, w / 2], [0, 100.0, h / 2], [0, 0, 1]], camera_height=h, camera_width=w,
                   camera_id=i)
        if kind == "png":
            PIL.Image.fromarray(rgb[:, :, 1], mode="L").save(os.path.join(root, f"weight{i}.png"))
            rec["loss_weight_path"] = f"weight{i}.png"
        elif kind in ("npy", "bad"):
            arr = (np.arange(h * w, dtype=np.float32).reshape(h, w) / (h * w)).astype(np.float32)
            if kind == "bad":
                arr[0, 0] = 1.5
            np.save(os.path.join(root, f"weight{i}.npy"), arr)
            rec["loss_weight_path"] = f"weight{i}.npy"
        records.append(rec)
    path = os.path.join(root, "train.json")
    with open(path, "w") as f:
        json.dump(records, f)
    return path, rng


def test_dataset_reads_loss_weight_path(tmp_path):
    path, _ = _dataset(str(tmp_path), [(40, 72, "png"), (37, 50, "npy"), (70, MAX_RESOLUTION_TRAIN + 41, "npy"),
                                       (32, 32, None)])
    ds = ImagePoseDataset(path, with_targets=True)
    img, _, _, info, tg = ds[0]
    expect = torch.from_numpy(np.array(PIL.Image.open(os.path.join(str(tmp_path), "weight0.png")))).float() / 255.0
    assert torch.equal(tg.loss_weight, expect[:32, :64]) and tg.mask is None
    _, _, _, info, tg = ds[1]
    arr = torch.from_numpy(np.load(os.path.join(str(tmp_path), "weight1.npy")))
    assert torch.equal(tg.loss_weight, arr[:32, :48])
    img, _, _, info, tg = ds[2]  # autoscaled like the mask
    assert tg.loss_weight.shape == (info.camera_height, info.camera_width) == tuple(img.shape[1:])
    assert float(tg.loss_weight.min()) >= 0.0 and float(tg.loss_weight.max()) <= 1.0
    assert ds[3][4].loss_weight is None
    assert len(ImagePoseDataset(path)[0]) == 4


def test_dataset_rejects_weights_outside_0_1(tmp_path):
    path, _ = _dataset(str(tmp_path), [(32, 32, "bad")])
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        ImagePoseDataset(path, with_targets=True)[0]


@pytest.fixture(scope="module")
def problem():
    hidden = hidden_scene(n=200)
    return hidden, render_views(OracleRasterisationModule(GPCR.GaussianPointCloudRasterisationConfig()), hidden)


def test_trainer_applies_the_weights_and_reports_the_inlier_fraction(problem):
    hidden, views = problem
    cfg = train_config(6)
    cfg.robust_loss = RobustLossConfig(inlier_quantile=0.5, start_iteration=3)
    trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)
    trainer.train(log_interval=1)
    fr = [e["robust_inlier_fraction"] for e in trainer.history]
    assert fr[:3] == [1.0, 1.0, 1.0] and all(0.0 < f < 1.0 for f in fr[3:]), fr
    # a static zero weight everywhere: the image loss is 0 and nothing moves
    zero = [(v[0], v[1], v[2], v[3], SupervisionTargets(loss_weight=torch.zeros(v[3].camera_height, v[3].camera_width)))
            for v in views]
    cfg = train_config(2)
    scene = initial_scene(hidden)
    before = scene.point_cloud.detach().clone()
    trainer = T(cfg, scene, zero, rasterisation_factory=OracleRasterisationModule)
    trainer.train(log_interval=1)
    assert all(e["loss"] == 0.0 and e["robust_inlier_fraction"] == 0.0 for e in trainer.history)
    assert torch.equal(scene.point_cloud.detach(), before)


def test_trainer_refusals(problem):
    hidden, views = problem
    cfg = train_config(2)
    cfg.robust_loss = 0.5
    with pytest.raises(ValueError, match="RobustLossConfig"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)

    class Exchanging(OracleRasterisationModule):
        gradient_exchange = object()
    cfg = train_config(2)
    cfg.robust_loss = RobustLossConfig()
    with pytest.raises(ValueError, match="view-parallel"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=Exchanging)
    weighted = [(v[0], v[1], v[2], v[3], SupervisionTargets(loss_weight=torch.ones(v[3].camera_height, v[3].camera_width)))
                for v in views]
    with pytest.raises(ValueError, match="view-parallel"):
        T(train_config(2), initial_scene(hidden), weighted, rasterisation_factory=Exchanging)
