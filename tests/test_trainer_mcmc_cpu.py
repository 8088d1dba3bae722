"""MCMC densification on the CPU: the controller's bookkeeping on constructed scenes, and the trainer's autograd loop with
the oracle as rasteriser (``TrainConfig.densification="mcmc"``)."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.mcmc import GaussianPointMCMCController, MCMCConfig, MCMCMoments
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T

from oracle_module import OracleRasterisationModule
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config


def _scene(n_rows, opacities, seed=0, channels=0):
    """``len(opacities)`` valid rows with the given opacities, then invalid rows up to ``n_rows``."""
    g = torch.Generator().manual_seed(seed)
    n = len(opacities)
    xyz = torch.randn((n_rows, 3), generator=g)
    feat = torch.randn((n_rows, 56), generator=g) * 0.3
    o = torch.tensor(opacities, dtype=torch.float64)
    feat[:n, 7] = torch.log(o / (1 - o)).float()
    mask = torch.ones(n_rows, dtype=torch.int8)
    mask[:n] = 0
    obj = torch.randint(0, 4, (n_rows,), generator=g, dtype=torch.int32)
    extra = torch.randn((n_rows, channels), generator=g) if channels else None
    return GaussianPointMCMCController.MaintainedParameters(xyz, feat, mask, obj, extra)


def _controller(mp, cap_max, seed=1, **kw):
    cfg = MCMCConfig(cap_max=cap_max, refine_start=0, refine_every=1, **kw)
    return GaussianPointMCMCController(cfg, mp, generator=torch.Generator().manual_seed(seed))


def _dead(mp, tau=0.005):
    o = torch.sigmoid(mp.pointcloud_features[:, 7])
    return (mp.point_invalid_mask == 0) & ((o <= tau) | ~torch.isfinite(mp.pointcloud_features).all(1))


def test_growth_follows_the_budget_and_no_row_stays_dead():
    mp = _scene(400, [0.5] * 90 + [0.001] * 10)
    mp.pointcloud_features[3, 20] = math.nan  # a broken row is dead too
    ctl = _controller(mp, cap_max=150)
    n_v = 100
    assert ctl.num_valid == n_v
    for _ in range(12):
        ctl.refinement()
        n_v = min(150, math.floor(1.05 * n_v))
        assert ctl.num_valid == n_v == int((mp.point_invalid_mask == 0).sum())
        assert not _dead(mp).any()
        assert (mp.point_invalid_mask[:n_v] == 0).all()  # the lowest invalid rows were filled
    assert ctl.num_valid == 150
    assert ctl.last_refinement == (0, 0)


def test_a_full_scene_only_relocates_and_moments_are_zeroed():
    mp = _scene(60, [0.6] * 50 + [0.002] * 10, channels=3)
    before = mp.pointcloud_features.clone()
    moments = MCMCMoments(*[(torch.ones(60, c), torch.ones(60, c)) for c in (56, 3, 3)])
    ctl = _controller(mp, cap_max=1000)
    ctl.refinement(moments)
    assert ctl.last_refinement == (10, 0) and ctl.num_valid == 60
    changed = (mp.pointcloud_features != before).any(1)
    assert changed[50:].all()  # every dead row was overwritten ...
    for d in range(50, 60):  # ... by a whole copy of an alive row
        src = [s for s in range(50) if torch.equal(mp.pointcloud_features[s], mp.pointcloud_features[d])]
        assert len(src) == 1
        s = src[0]
        assert torch.equal(mp.pointcloud[s], mp.pointcloud[d]) and mp.point_object_id[s] == mp.point_object_id[d]
        assert torch.equal(mp.point_extra_features[s], mp.point_extra_features[d])
        assert changed[s]  # the source was updated before it was copied
    touched = changed
    for pair in (moments.features, moments.positions, moments.extra_features):
        for m in pair:
            assert not m[touched].any() and (m[~touched] == 1).all()
    # the copies keep the rendered opacity: n copies of o_new compose to the source's o
    for s in torch.nonzero(changed[:50]).reshape(-1).tolist():
        n = int((mp.pointcloud_features[:, 8:] == mp.pointcloud_features[s, 8:]).all(1).sum())
        o_new = torch.sigmoid(mp.pointcloud_features[s, 7].double())
        assert float(1 - (1 - o_new) ** n) == pytest.approx(0.6, abs=1e-5)


def test_no_alive_row_is_a_no_op():
    mp = _scene(30, [0.001] * 20)
    before = [t.clone() for t in (mp.pointcloud, mp.pointcloud_features, mp.point_invalid_mask)]
    ctl = _controller(mp, cap_max=30)
    ctl.refinement()
    assert all(torch.equal(a, b) for a, b in zip(before, (mp.pointcloud, mp.pointcloud_features, mp.point_invalid_mask)))
    assert ctl.num_valid == 20 and ctl.last_refinement is None


def test_the_refinement_window():
    mp = _scene(100, [0.5] * 40)
    ctl = GaussianPointMCMCController(MCMCConfig(cap_max=100, refine_start=4, refine_stop=9, refine_every=2), mp,
                                      generator=torch.Generator().manual_seed(0))
    counts = []
    for _ in range(12):
        ctl.refinement()
        counts.append(ctl.num_valid)
    assert counts == [40, 40, 40, 40, 42, 42, 44, 44, 46, 46, 46, 46]  # t = 4, 6, 8 refine; t = 10 is past the stop


def test_sources_are_alive_and_follow_the_opacities():
    opac = [0.05, 0.1, 0.2, 0.4, 0.8, 0.003, 0.0001]
    mp = _scene(8, opac)
    ctl = _controller(mp, cap_max=8)
    draws = 40_000
    _, _, picked = ctl._draw(draws)
    counts = torch.bincount(picked, minlength=8).double()
    assert counts[5:].sum() == 0  # dead and invalid rows are never drawn
    o = torch.sigmoid(mp.pointcloud_features[:5, 7].double())
    expected = o / o.sum() * draws
    chi2 = float(((counts[:5] - expected) ** 2 / expected).sum())
    assert chi2 < 18.47  # the 0.999 quantile of chi-squared with 4 degrees of freedom
    ids, k, _ = ctl._draw(3)
    assert ids.numel() == k.numel() and int(k.sum()) == 3 and (k > 0).all()


def test_equal_seeds_give_identical_scenes():
    outs = []
    for _ in range(2):
        mp = _scene(300, [0.3, 0.7, 0.002, 0.5] * 25, seed=5)
        ctl = _controller(mp, cap_max=200, seed=11)
        for _ in range(5):
            ctl.refinement()
        outs.append((mp.pointcloud.clone(), mp.pointcloud_features.clone(), mp.point_invalid_mask.clone()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    mp = _scene(300, [0.3, 0.7, 0.002, 0.5] * 25, seed=5)
    ctl = _controller(mp, cap_max=200, seed=12)
    for _ in range(5):
        ctl.refinement()
    assert not torch.equal(mp.pointcloud_features, outs[0][1])


@pytest.mark.parametrize("kw,match", [
    (dict(cap_max=0), "cap_max"), (dict(cap_max=10.5), "cap_max"), (dict(cap_max=10, refine_every=0), "refinement window"),
    (dict(cap_max=10, refine_start=10, refine_stop=5), "refinement window"), (dict(cap_max=10, grow_factor=0.9), "grow_factor"),
    (dict(cap_max=10, min_opacity=0.0), "min_opacity"), (dict(cap_max=10, min_opacity=1.0), "min_opacity"),
    (dict(cap_max=10, noise_lr=-1.0), "noise_lr"), (dict(cap_max=10, opacity_reg=math.nan), "opacity_reg"),
    (dict(cap_max=10, scale_reg=math.inf), "scale_reg"), (dict(cap_max=10, seed=-1), "seed"),
])
def test_mcmc_config_errors(kw, match):
    with pytest.raises(ValueError, match=match):
        MCMCConfig(**kw).check()


# ---------------------------------------------------------------------------------------------- the trainer's autograd loop
@pytest.fixture(scope="module")
def problem():
    hidden = hidden_scene(n=120)
    return hidden, render_views(OracleRasterisationModule(GPCR.GaussianPointCloudRasterisationConfig()), hidden)


def _mcmc_trainer(problem, iterations, cap_max, seed=0, **kw):
    hidden, views = problem
    cfg = train_config(iterations)
    cfg.densification = "mcmc"
    cfg.mcmc_config = MCMCConfig(cap_max=cap_max, refine_start=4, refine_every=4, noise_lr=50.0, seed=seed, **kw)
    return T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule,
             generator=torch.Generator().manual_seed(3))


def test_trainer_configuration_errors(problem):
    hidden, views = problem
    cfg = train_config(1)
    cfg.densification = "mcmc"
    with pytest.raises(ValueError, match="mcmc_config"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)
    cfg.mcmc_config = MCMCConfig(cap_max=100)
    cfg.loss_function_config.enable_regularization = True
    with pytest.raises(ValueError, match="enable_regularization"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)
    cfg = train_config(1)
    cfg.densification = "sometimes"
    with pytest.raises(ValueError, match="densification"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=OracleRasterisationModule)
    cfg = train_config(1)
    cfg.densification = "mcmc"
    cfg.mcmc_config = MCMCConfig(cap_max=100)

    class Exchanging(OracleRasterisationModule):
        gradient_exchange = object()

    with pytest.raises(ValueError, match="view-parallel"):
        T(cfg, initial_scene(hidden), views, rasterisation_factory=Exchanging)


def test_mcmc_builds_the_operator_without_a_backward_hook(problem):
    hidden, views = problem
    seen = {}

    def factory(config, backward_valid_point_hook=None, **kw):
        seen["hook"] = backward_valid_point_hook
        return OracleRasterisationModule(config, backward_valid_point_hook=backward_valid_point_hook, **kw)

    cfg = train_config(1)
    cfg.densification = "mcmc"
    cfg.mcmc_config = MCMCConfig(cap_max=100)
    trainer = T(cfg, initial_scene(hidden), views, rasterisation_factory=factory)
    assert seen["hook"] is None and trainer.adaptive_controller is None and trainer.mcmc_controller is not None
    T(train_config(1), initial_scene(hidden), views, rasterisation_factory=factory)
    assert seen["hook"] is not None


def test_trainer_grows_to_the_budget_and_the_loss_falls(problem):
    trainer = _mcmc_trainer(problem, 40, cap_max=150)
    hist = trainer.train(log_interval=1)
    n_v, want = 120, []
    for it in range(40):
        if it >= 4 and it % 4 == 0:
            n_v = min(150, math.floor(1.05 * n_v))
        want.append(n_v)
    assert [h["num_valid_points"] for h in hist] == want and want[-1] == 150
    assert all(math.isfinite(h["loss"]) and h["mcmc_opacity_reg"] > 0 and h["mcmc_scale_reg"] > 0 for h in hist)
    assert torch.isfinite(trainer.scene.point_cloud).all() and torch.isfinite(trainer.scene.point_cloud_features).all()
    first, last = np.mean([h["loss"] for h in hist[:4]]), np.mean([h["loss"] for h in hist[-4:]])
    assert last < first
    o = torch.sigmoid(trainer.scene.point_cloud_features.detach()[:, 7])
    valid = trainer.scene.point_invalid_mask == 0
    assert float(hist[-1]["mcmc_opacity_reg"]) == pytest.approx(0.01 * float(o[valid].mean()), rel=0.05)


def test_trainer_runs_are_reproducible_and_the_noise_seed_matters(problem):
    a = _mcmc_trainer(problem, 10, cap_max=140)
    b = _mcmc_trainer(problem, 10, cap_max=140)
    c = _mcmc_trainer(problem, 10, cap_max=140, seed=1)
    for t in (a, b, c):
        with torch.no_grad():  # nearly transparent rows: the only ones the gate lets the noise move
            t.scene.point_cloud_features[:10, 7] = -5.2
        t.train()
    assert torch.equal(a.scene.point_cloud, b.scene.point_cloud)
    assert torch.equal(a.scene.point_cloud_features, b.scene.point_cloud_features)
    assert torch.equal(a.scene.point_invalid_mask, b.scene.point_invalid_mask)
    assert not torch.equal(a.scene.point_cloud, c.scene.point_cloud)
