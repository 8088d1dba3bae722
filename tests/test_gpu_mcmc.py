"""-m gpu: MCMC densification on the device -- each kernel of ``csrc/mcmc.cu`` against the torch form of ``mcmc.py`` /
``loss.mcmc_regulariser``, one fused MCMC iteration against one iteration of the autograd loop, the overflow no-op, and a fit
from a sparse initialisation that grows to its budget."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.loss import mcmc_regulariser
from taichi_3d_gaussian_splatting_b200.mcmc import (GaussianPointMCMCController, MCMCConfig, MCMCMoments, add_position_noise,
                                                    relocation_opacity_scale)
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from trainer_helpers import hidden_scene, initial_scene, render_views, train_config

pytestmark = pytest.mark.gpu
N = 100_000


def _rows(n, seed, logit_range=(-7.0, -4.0)):
    g = torch.Generator().manual_seed(seed)
    f = torch.zeros((n, 56))
    f[:, :4] = torch.randn((n, 4), generator=g) * (0.3 + 2.7 * torch.rand((n, 1), generator=g))
    f[:, 4:7] = torch.rand((n, 3), generator=g) * 3.5 - 3.0
    f[:, 7] = torch.rand(n, generator=g) * (logit_range[1] - logit_range[0]) + logit_range[0]
    f[:, 8:] = torch.randn((n, 48), generator=g)
    xyz = torch.randn((n, 3), generator=g)
    mask = (torch.rand(n, generator=g) < 0.2).to(torch.int8)
    return xyz, f, mask


def test_regulariser_kernel_matches_the_torch_form():
    _, f, mask = _rows(N, 1, logit_range=(-4.0, 4.0))
    ref = f.double().requires_grad_(True)
    want = mcmc_regulariser(ref, mask, 0.01, 0.03)
    want.sum().backward()
    dev = f.cuda().requires_grad_(True)
    got = mcmc_regulariser(dev, mask.cuda(), 0.01, 0.03)
    got.sum().backward()
    assert torch.allclose(got.detach().cpu().double(), want.detach(), rtol=1e-6)
    assert torch.allclose(dev.grad.cpu().double(), ref.grad, rtol=1e-5, atol=0)
    assert float(ref.grad[mask == 0][:, 4:8].abs().min()) > 0
    assert not dev.grad[mask.cuda() != 0].any()
    again = mcmc_regulariser(f.cuda(), mask.cuda(), 0.01, 0.03)
    assert torch.equal(again, got.detach())  # fixed summation order


def test_noise_kernel_matches_the_torch_form():
    xyz, f, mask = _rows(N, 2)
    seed, step, scale = 0xFEDCBA9876543210, 2 ** 33 + 5, 0.37
    want = xyz.clone()
    add_position_noise(want, f, mask, scale, seed, step)
    got = xyz.cuda()
    add_position_noise(got, f.cuda(), mask.cuda(), scale, seed, step)
    again = xyz.cuda()
    add_position_noise(again, f.cuda(), mask.cuda(), scale, seed, step)
    assert torch.equal(got, again)
    got = got.cpu()
    valid = mask == 0
    assert torch.equal(got[~valid], xyz[~valid])
    size = scale * torch.exp(2 * f[:, 4:7]).max(1).values * 6.0  # |Sigma| |eps| noise_scale, |eps| < 6
    tol = 3e-6 * size[:, None] + 2.4e-7 * xyz.abs() + 1e-12
    assert bool(((got - want).abs() <= tol)[valid].all())
    assert float((want - xyz)[valid].abs().max()) > 1e-3
    other = xyz.cuda()
    add_position_noise(other, f.cuda(), mask.cuda(), scale, seed, step + 1)
    assert not torch.equal(other.cpu()[valid], got[valid])


def test_relocation_kernels_match_the_torch_form():
    xyz, f, mask = _rows(N, 3, logit_range=(-3.0, 5.0))
    g = torch.Generator().manual_seed(4)
    obj = torch.randint(0, 7, (N,), generator=g, dtype=torch.int32)
    extra = torch.randn((N, 5), generator=g)
    perm = torch.randperm(N, generator=g)
    sources, destinations = perm[:3000], perm[3000:8000]
    dest_sources = sources[torch.randint(0, 3000, (5000,), generator=g)]
    counts = torch.bincount(dest_sources, minlength=N)[sources]
    counts[:4] = torch.tensor([60, 50, 49, 0])  # beyond N_MAX, at it, below it, and a source that was not drawn
    mp = GaussianPointMCMCController.MaintainedParameters(xyz.cuda(), f.cuda(), mask.cuda(), obj.cuda(), extra.cuda())
    ctl = GaussianPointMCMCController(MCMCConfig(cap_max=N), mp)
    moments = MCMCMoments(*[(torch.ones((N, c), device="cuda"), torch.ones((N, c), device="cuda")) for c in (56, 3, 5)])
    ctl._apply_cuda(sources.cuda(), counts.cuda(), destinations.cuda(), dest_sources.cuda(), mp.pointcloud,
                    mp.pointcloud_features, mp.point_extra_features, moments)
    torch.cuda.synchronize()
    want = f.clone()
    logit, log_scale = relocation_opacity_scale(f[sources, 7], f[sources, 4:7], counts + 1)
    want[sources, 7], want[sources, 4:7] = logit, log_scale
    want[destinations] = want[dest_sources]
    got = mp.pointcloud_features.cpu()
    assert torch.allclose(got[:, 4:7], want[:, 4:7], rtol=0, atol=5e-7)
    assert torch.allclose(got[:, 7], want[:, 7], rtol=2e-6, atol=2e-6)
    assert torch.equal(got[:, :4], want[:, :4]) and torch.equal(got[:, 8:], want[:, 8:])
    assert torch.equal(got[destinations], got[dest_sources])  # whole, bit-exact copies of the updated rows
    want_xyz, want_obj, want_extra, want_mask = xyz.clone(), obj.clone(), extra.clone(), mask.clone()
    want_xyz[destinations], want_obj[destinations] = xyz[dest_sources], obj[dest_sources]
    want_extra[destinations], want_mask[destinations] = extra[dest_sources], 0
    assert torch.equal(mp.pointcloud.cpu(), want_xyz) and torch.equal(mp.point_object_id.cpu(), want_obj)
    assert torch.equal(mp.point_extra_features.cpu(), want_extra) and torch.equal(mp.point_invalid_mask.cpu(), want_mask)
    touched = torch.zeros(N, dtype=torch.bool)
    touched[sources], touched[destinations] = True, True
    for pair in (moments.features, moments.positions, moments.extra_features):
        for m in pair:
            m = m.cpu()
            assert not m[touched].any() and bool((m[~touched] == 1).all())


# ---------------------------------------------------------------------------------------------- the two training loops
def _problem():
    hidden = hidden_scene(n=400)
    return hidden, render_views(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), hidden, device="cuda")


def _trainer(hidden, views, iterations, fused, noise_lr=50.0, cap_max=500, **kw):
    cfg = train_config(iterations)
    cfg.densification = "mcmc"
    cfg.mcmc_config = MCMCConfig(cap_max=cap_max, refine_start=4, refine_every=4, noise_lr=noise_lr, seed=17, **kw)
    scene = initial_scene(hidden, device="cuda")
    with torch.no_grad():  # nearly transparent rows: the ones the gate lets the noise move
        scene.point_cloud_features[:40, 7] = -5.2
    return GaussianPointCloudTrainer(cfg, scene, views, fused_step=fused,
                                     generator=torch.Generator(device="cuda").manual_seed(3))


def test_one_fused_mcmc_iteration_is_the_autograd_iteration():
    hidden, views = _problem()
    t_ref = _trainer(hidden, views, 1, fused=False)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        h_ref = t_ref.train(log_interval=1)
    t_fused = _trainer(hidden, views, 1, fused=True)
    h_fused = t_fused.train(log_interval=1)
    for key in ("loss", "mcmc_opacity_reg", "mcmc_scale_reg"):
        assert abs(h_ref[0][key] - h_fused[0][key]) <= 2e-6 * abs(h_ref[0][key]) + 1e-7, key
    assert h_fused[0]["mcmc_opacity_reg"] > 0 and h_fused[0]["mcmc_scale_reg"] > 0
    s = t_fused.fused_train_step
    gx_ref, gf_ref = t_ref.scene.point_cloud.grad, t_ref.scene.point_cloud_features.grad
    assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max())
    assert float((s.grad_pointcloud_features - gf_ref).abs().max()) <= 1e-4 * float(gf_ref.abs().max())
    # the regulariser's share is in both gradients; an invalid row gets none
    invalid = t_fused.scene.point_invalid_mask != 0
    assert not s.grad_pointcloud_features[invalid].any()
    for p_ref, p_fused, g, lr in ((t_ref.scene.point_cloud_features, t_fused.scene.point_cloud_features, gf_ref, 5e-3),
                                  (t_ref.scene.point_cloud, t_fused.scene.point_cloud, gx_ref, 2e-4)):
        solid = g.abs() > 1e-3 * g.abs().max()
        assert float((p_ref - p_fused)[solid].abs().max()) <= 0.02 * lr
    # the noise: the fused call draws what gsb200_mcmc_noise draws for the same (seed, step)
    t_quiet = _trainer(hidden, views, 1, fused=True, noise_lr=0.0)
    t_quiet.train()
    quiet = t_quiet.scene.point_cloud.detach().clone()
    add_position_noise(t_quiet.scene.point_cloud, t_quiet.scene.point_cloud_features, t_quiet.scene.point_invalid_mask,
                       50.0 * 2e-4, 17, 0)
    moved = (t_quiet.scene.point_cloud.detach() - quiet).abs().max(1).values
    assert float(moved[:40].min()) > 1e-7 and float(moved.max()) > 1e-5
    # rows whose Adam step does not depend on the order of the backward's float atomics (no gradient, or a solid one)
    g = s.grad_pointcloud
    steady = ((g == 0) | (g.abs() > 1e-3 * g.abs().max())).all(1)
    assert int((steady & (moved > 1e-6)).sum()) >= 10
    diff = (t_quiet.scene.point_cloud - t_fused.scene.point_cloud).detach().abs().max(1).values
    assert bool((diff <= 0.02 * 2e-4 + 0.05 * moved)[steady].all())


def test_both_loops_end_with_the_same_valid_set():
    hidden, views = _problem()
    t_ref = _trainer(hidden, views, 10, fused=False)
    t_fused = _trainer(hidden, views, 10, fused=True)
    h_ref, h_fused = t_ref.train(log_interval=1), t_fused.train(log_interval=1)
    assert t_fused.fused_train_step.num_skipped_steps == 0
    assert [h["num_valid_points"] for h in h_ref] == [h["num_valid_points"] for h in h_fused]
    assert h_fused[-1]["num_valid_points"] == math.floor(1.05 * math.floor(1.05 * 400)) == t_fused.mcmc_controller.num_valid
    assert torch.equal(t_ref.scene.point_invalid_mask, t_fused.scene.point_invalid_mask)
    l_ref, l_fused = np.array([h["loss"] for h in h_ref]), np.array([h["loss"] for h in h_fused])
    assert np.abs(l_ref - l_fused).max() < 5e-3 * l_ref.max()
    o = torch.sigmoid(t_fused.scene.point_cloud_features.detach()[:, 7])
    assert bool((o[t_fused.scene.point_invalid_mask == 0] > 0.004).all())  # the dead rows were relocated


def test_overflow_iteration_leaves_the_scene_and_the_moments_untouched():
    from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
    hidden, views = _problem()
    scene = initial_scene(hidden, device="cuda")
    with torch.no_grad():
        scene.point_cloud_features[:40, 7] = -5.2
    cfg = train_config(1)
    step = FusedTrainStep(scene, cfg.rasterisation_config, 0.2, key_capacity=64, mcmc=MCMCConfig(cap_max=800))
    xyz0, feat0 = scene.point_cloud.detach().clone(), scene.point_cloud_features.detach().clone()
    img, q, t, cam = views[0]
    with pytest.warns(UserWarning, match="no-op on the device"):
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, mcmc_num_valid=400)
        torch.cuda.synchronize()
        # q of the in-frustum rows is normalised in place by the forward even in a skipped iteration
        assert torch.equal(scene.point_cloud.detach(), xyz0)
        assert torch.equal(scene.point_cloud_features.detach()[:, 4:], feat0[:, 4:])
        for m in (step.feature_exp_avg, step.feature_exp_avg_sq, step.position_exp_avg, step.position_exp_avg_sq):
            assert not m.any()
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, mcmc_num_valid=400)  # notices the overflow of the first call
        step.run(img, q, t, cam, 3, 5e-3, 2e-4, mcmc_num_valid=400)
    torch.cuda.synchronize()
    assert step.num_skipped_steps >= 1 and step.key_capacity > 64
    step.run(img, q, t, cam, 3, 5e-3, 2e-4, mcmc_num_valid=400)
    torch.cuda.synchronize()
    assert not torch.equal(scene.point_cloud.detach(), xyz0) and float(step.mcmc_terms.min()) > 0


def _sparse_scene(hidden, count, capacity, seed=21):
    """``count`` Gaussians at random places in the hidden scene's bounding box, the other rows invalid."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = hidden.point_cloud.min(0).values, hidden.point_cloud.max(0).values
    pc = torch.zeros((capacity, 3))
    pc[:count] = lo + (hi - lo) * torch.rand((count, 3), generator=g)
    feat = torch.zeros((capacity, 56))
    feat[:, 3] = 1.0
    feat[:count, 4:7] = hidden.point_cloud_features[:, 4:7].median() + 0.5
    feat[:count, 7] = 0.5
    feat[:count, 8], feat[:count, 24], feat[:count, 40] = 0.5, 0.5, 0.5
    mask = torch.ones(capacity, dtype=torch.int8)
    mask[:count] = 0
    return Scene(pc.cuda().requires_grad_(True), feat.cuda().requires_grad_(True), mask.cuda(),
                 torch.zeros(capacity, dtype=torch.int32, device="cuda"))


def test_fit_from_a_sparse_initialisation_grows_to_the_budget():
    hidden, views = _problem()
    count, result = 60, {}
    for cap_max in (4 * count, count):
        cfg = train_config(450)
        cfg.densification = "mcmc"
        cfg.mcmc_config = MCMCConfig(cap_max=cap_max, refine_start=20, refine_every=10)
        trainer = GaussianPointCloudTrainer(cfg, _sparse_scene(hidden, count, 512), views, fused_step=True,
                                            generator=torch.Generator(device="cuda").manual_seed(5))
        trainer.train()
        assert trainer.mcmc_controller.num_valid == cap_max == int((trainer.scene.point_invalid_mask == 0).sum())
        valid = trainer.scene.point_invalid_mask == 0
        assert bool(torch.isfinite(trainer.scene.point_cloud[valid]).all())
        assert bool(torch.isfinite(trainer.scene.point_cloud_features[valid]).all())
        result[cap_max] = trainer.validation()
    print(f"validation PSNR: cap_max={4 * count}: {result[4 * count]:.2f} dB, cap_max={count}: {result[count]:.2f} dB")
    assert result[4 * count] > result[count], result
