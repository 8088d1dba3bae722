"""CPU checks of the trainer's supervision options: configuration errors, the operator options it asks for, and the
down-sampled targets (the mask resized like the image, the depth by nearest neighbour)."""
import dataclasses
import math

import pytest
import torch

from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets
from taichi_3d_gaussian_splatting_b200.trainer import (GaussianPointCloudTrainer, downsample_image_and_camera_info,
                                                       downsample_targets)

from trainer_helpers import H, W, hidden_scene, initial_scene, poses, train_config


def _views(with_mask=True, with_depth=True):
    hidden = hidden_scene(n=50)
    views = []
    for q, t in poses():
        image = torch.rand(3, H, W)
        tg = SupervisionTargets(depth=torch.rand(H, W) + 1 if with_depth else None, mask=torch.rand(H, W) if with_mask else None)
        views.append((image, q, t, hidden.camera_info, tg))
    return hidden, views


class _Factory:
    """Records the keyword arguments the trainer builds its rasteriser with."""
    def __init__(self):
        self.kwargs = None

    def __call__(self, config, backward_valid_point_hook=None, **kwargs):
        self.kwargs = kwargs
        return torch.nn.Identity()


def _cfg(**kw):
    return dataclasses.replace(train_config(1), **kw)


@pytest.mark.parametrize("kw,needs", [(dict(background="random"), (False, True)), (dict(mask_loss_weight=0.5), (False, True)),
                                      (dict(depth_loss_weight=0.5), (True, False)), (dict(background="white"), (False, True)),
                                      (dict(), (False, False))])
def test_operator_options_follow_the_terms(kw, needs):
    hidden, views = _views()
    f = _Factory()
    GaussianPointCloudTrainer(_cfg(**kw), initial_scene(hidden), views, rasterisation_factory=f)
    expect = {**({"differentiable_depth": True} if needs[0] else {}), **({"differentiable_alpha": True} if needs[1] else {})}
    assert f.kwargs == expect  # nothing extra without a term: injected factories such as the oracle module keep working


@pytest.mark.parametrize("kw,match", [(dict(background="random"), "random"), (dict(mask_loss_weight=1.0), "mask"),
                                      (dict(background="grey"), "background"), (dict(depth_loss_weight=-1.0), "depth_loss_weight"),
                                      (dict(mask_loss_weight=math.nan), "mask_loss_weight")])
def test_configuration_errors(kw, match):
    hidden, views = _views(with_mask=False)
    with pytest.raises(ValueError, match=match):
        GaussianPointCloudTrainer(_cfg(**kw), initial_scene(hidden), views, rasterisation_factory=_Factory())
    hidden, views = _views(with_depth=False)
    with pytest.raises(ValueError, match="depth"):
        GaussianPointCloudTrainer(_cfg(depth_loss_weight=1.0), initial_scene(hidden), views, rasterisation_factory=_Factory())


def test_downsampled_targets_match_the_image_schedule():
    hidden = hidden_scene(n=50)
    cam = hidden.camera_info
    g = torch.Generator().manual_seed(0)
    image = torch.rand((3, H, W), generator=g)
    depth = torch.rand((H, W), generator=g) + 1
    depth[1::2] = 0.0  # odd rows: no measurement (not sampled at factor 2)
    depth[::4, ::3] = math.nan  # holes on sampled pixels stay holes
    tg = downsample_targets(SupervisionTargets(depth=depth, mask=image[0].clone()), cam, 2)
    img2, cam2 = downsample_image_and_camera_info(image, cam, 2)
    assert tg.mask.shape == tg.depth.shape == (cam2.camera_height, cam2.camera_width)
    assert torch.allclose(tg.mask, img2[0], atol=1e-6)  # the image's own antialiased resize
    # nearest neighbour at factor 2: pixel (i, j) <- (2i, 2j); the zero rows stay zero, values are never blended
    src = depth[0::2, 0::2][:tg.depth.shape[0], :tg.depth.shape[1]]
    same = (tg.depth == src) | (tg.depth.isnan() & src.isnan())
    assert bool(same.all())
