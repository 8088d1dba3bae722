"""-m gpu: the 3D smoothing filter (``mip_filter``, ``point_filter_3d``, ``gsb200_forward_filter3d`` /
``gsb200_backward_filter3d`` / ``gsb200_train_step_filter3d`` / ``gsb200_filter3d_from_views``).

The views kernel bit for bit against the emulated kernel and the host rule; the filtered forward against the unfiltered forward on
the baked rows at C2 full size; the filtered gradients against torch autograd through the bake and the unfiltered operator,
for a pinhole, an opencv lens and a rolling shutter with image, depth, alpha and feature-map losses; the fused step with the
filter against the autograd loop; and an MCMC run with the filter."""
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion, RollingShutter
from taichi_3d_gaussian_splatting_b200.mcmc import MCMCConfig
from taichi_3d_gaussian_splatting_b200.mip_filter import bake_filter_3d, compute_filter_3d
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer

from mip_filter_reference import bake_torch, random_views
from simt_filter3d_helpers import build_filter3d_emulator, emulated_filter
from oracle_module import OracleRasterisationModule
from test_gpu_trainer import _views_to
from trainer_helpers import hidden_scene, initial_scene, render_views, train_config

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput


def _input(sc, camera_info, features=None, q=None, t=None):
    return Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features if features is None else features,
                 point_object_id=sc.point_object_id, point_invalid_mask=sc.point_invalid_mask, camera_info=camera_info,
                 q_pointcloud_camera=sc.q_pointcloud_camera if q is None else q,
                 t_pointcloud_camera=sc.t_pointcloud_camera if t is None else t, color_max_sh_band=3)


def test_views_kernel_is_the_rule():
    g = torch.Generator().manual_seed(5)
    N, V, n_obj = 200_000, 120, 2
    xyz = (torch.rand((N, 3), generator=g) * torch.tensor([12.0, 8.0, 14.0]) - torch.tensor([6.0, 4.0, 2.0])).contiguous()
    mask = (torch.rand(N, generator=g) < 0.05).to(torch.int8)
    obj = torch.randint(0, n_obj, (N,), generator=g, dtype=torch.int32)
    views = random_views(V, n_obj, g)
    cpu = compute_filter_3d(xyz, mask, obj, views, 0.5, 0.2)
    dev = compute_filter_3d(xyz.cuda(), mask.cuda(), obj.cuda(),
                            [(q.cuda(), t.cuda(), CameraInfo(ci.camera_intrinsics.cuda(), ci.camera_height, ci.camera_width, 0))
                             for q, t, ci in views], 0.5, 0.2).cpu()
    assert torch.equal(cpu.view(torch.int32), dev.view(torch.int32))
    emulated = emulated_filter(build_filter3d_emulator(), xyz.numpy(), mask.numpy(), obj.numpy(), views, 0.5, 0.2)
    assert torch.equal(torch.from_numpy(emulated).view(torch.int32), dev.view(torch.int32))
    assert (dev[mask == 1] == 0).all() and (dev[mask == 0] > 0).all()
    # twice: bit-identical
    again = compute_filter_3d(xyz.cuda(), mask.cuda(), obj.cuda(),
                              [(q.cuda(), t.cuda(), CameraInfo(ci.camera_intrinsics.cuda(), ci.camera_height, ci.camera_width, 0))
                               for q, t, ci in views], 0.5, 0.2).cpu()
    assert torch.equal(again.view(torch.int32), dev.view(torch.int32))


def test_filtered_forward_is_the_unfiltered_forward_of_the_baked_rows_at_c2():
    sc = make_scene(**CONFIGS["C2"]).to("cuda")
    ci = sc.camera_info
    views = []
    for yaw in (0.0, 8.0, -8.0):
        half = math.radians(yaw) / 2
        views.append((torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device="cuda"),
                      torch.zeros((1, 3), device="cuda"), ci))
    f3d = compute_filter_3d(sc.point_cloud, sc.point_invalid_mask, sc.point_object_id, views, 0.8, 0.2)
    assert float(f3d.min()) > 0
    op = GPCR(Config(), differentiable_alpha=True, keep_all_tile_pairs=False)
    baked = bake_filter_3d(sc.point_cloud_features, f3d).contiguous()
    with torch.no_grad():
        a = op(_input(sc, ci), point_filter_3d=f3d)
        fa = op.last_frame
        ranges_a = (fa.tile_points_end - fa.tile_points_start).cpu()
        b = op(_input(sc, ci, features=baked))
        fb = op.last_frame
        ranges_b = (fb.tile_points_end - fb.tile_points_start).cpu()
    HW = ci.camera_height * ci.camera_width
    for name, x, y in (("image", a[0], b[0]), ("depth", a[1], b[1]), ("alpha", a[3], b[3])):
        over = int(((x - y).abs() > 1e-4).sum())
        assert over <= 1e-4 * HW, (name, over, float((x - y).abs().max()))
    assert fa.num_points_in_camera == fb.num_points_in_camera
    assert int((ranges_a != ranges_b).sum()) <= 2, int((ranges_a != ranges_b).sum())
    # the filter widened every visible splat: the records differ from the unfiltered render of the raw rows
    with torch.no_grad():
        c = op(_input(sc, ci))
    assert float((c[0] - a[0]).abs().mean()) > 1e-4


CASES = [("pinhole", None), ("opencv", None), ("pinhole", (0.06, -0.09, 0.04, 0.05, -0.08, 0.06))]


@pytest.mark.parametrize("lens,motion", CASES)
@pytest.mark.parametrize("terms", ["image", "all"])
def test_gradients_are_autograd_through_the_bake(lens, motion, terms):
    sc = make_scene(500, 48, 64, 0.1, 11).to("cuda")
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.0
    sc.point_cloud_features[3, 7] = 30.0  # fl(1 - o) = 0: only the compensation term is dropped
    sc.point_cloud[3] = torch.tensor([0.1, -0.1, 2.5], device="cuda")  # in the middle of the frame
    sc.point_invalid_mask[3] = 0
    sc.point_invalid_mask[::9] = 1
    g = torch.Generator().manual_seed(3)
    f3d = (torch.rand(500, generator=g) * 0.06).cuda()
    f3d[::5] = 0.0
    f3d[7] = float("nan")
    f3d[8] = -1.0
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0,
                    LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)) if lens == "opencv" else None,
                    RollingShutter(motion[:3], motion[3:]) if motion else None)
    both = terms == "all"
    cfg = Config()
    for k in ("grad_color_factor", "grad_high_order_color_factor", "grad_s_factor", "grad_q_factor", "grad_alpha_factor"):
        setattr(cfg, k, 1.0)
    op = GPCR(cfg, differentiable_depth=both, differentiable_alpha=both)
    gen = torch.Generator(device="cuda").manual_seed(1)
    H, W = ci.camera_height, ci.camera_width
    w_img = torch.randn((H, W, 3), device="cuda", generator=gen)
    w_d, w_a = torch.randn((H, W), device="cuda", generator=gen), torch.randn((H, W), device="cuda", generator=gen)
    w_f = torch.randn((H, W, 3), device="cuda", generator=gen)

    def loss(outs):
        total = (outs[0] * w_img).sum()
        if both:
            total = total + 0.1 * (outs[1] * w_d).sum() + (outs[3] * w_a).sum() + (outs[-1] * w_f).sum()
        return total

    extra = torch.randn((500, 3), device="cuda", generator=gen)
    feats = sc.point_cloud_features.clone()
    xyz = sc.point_cloud.clone().requires_grad_(True)
    feats_a = feats.clone().requires_grad_(True)
    ex_a = extra.clone().requires_grad_(True)
    sc_a = sc
    sc_a.point_cloud = xyz
    kw = dict(point_extra_features=ex_a) if both else {}
    outs = op(_input(sc_a, ci, features=feats_a), point_filter_3d=f3d, **kw)
    loss(outs).backward()
    # the unfiltered operator on the baked rows, with autograd through the bake
    xyz_b = sc.point_cloud.detach().clone().requires_grad_(True)
    feats_b = feats.clone().requires_grad_(True)
    ex_b = extra.clone().requires_grad_(True)
    sc_a.point_cloud = xyz_b
    kw = dict(point_extra_features=ex_b) if both else {}
    baked = bake_torch(feats_b, f3d)
    baked.retain_grad()
    outs_b = op(_input(sc_a, ci, features=baked), **kw)
    loss(outs_b).backward()
    for name, x, y in (("image", outs[0], outs_b[0]),):
        assert float((x - y).abs().max()) < 1e-4, (name, float((x - y).abs().max()))
    gx, gx_b = xyz.grad, xyz_b.grad
    gf, gf_b = feats_a.grad, feats_b.grad
    scale_x, scale_f = float(gx_b.abs().max()), float(gf_b[:, 4:8].abs().max())
    assert float((gx - gx_b).abs().max()) <= 2e-3 * scale_x, float((gx - gx_b).abs().max()) / scale_x
    rows = torch.arange(500, device="cuda") != 3  # row 3 is checked below: the bake keeps its compensation term
    for cols in (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56)):
        d = float((gf[rows, cols] - gf_b[rows, cols]).abs().max())
        assert d <= 2e-3 * max(float(gf_b[:, cols].abs().max()), 1e-6 * scale_f), (cols, d)
    if both:
        assert float((ex_a.grad - ex_b.grad).abs().max()) <= 1e-4 * float(ex_b.grad.abs().max())
    # the saturated row: o = 1.0f exactly, so fl(1 - o) = 0 and the kernel drops its compensation term: its scale gradient is
    # the bake's minus G_a sigma^2 / e^, with G_a = dL/dlogit of the baked row / (1 - o^) (o^ = c < 1 there)
    assert torch.isfinite(gf[3]).all() and float(gf[3, 7]) == 0.0
    s3 = float(f3d[3])
    e = torch.exp(feats[3, 4:7].double()) ** 2
    o_hat = torch.sigmoid(baked[3, 7].detach().double())
    g_alpha = baked.grad[3, 7].double() / (1 - o_hat)
    assert float(g_alpha.abs()) > 0 and float(gf_b[3, 4:7].abs().max()) > 0  # row 3 is rendered
    expected = gf_b[3, 4:7].double() - g_alpha * s3 * s3 / (e + s3 * s3)
    assert torch.allclose(gf[3, 4:7].double(), expected, rtol=2e-3, atol=2e-3 * scale_f), (gf[3, 4:7], expected)


def test_fused_step_with_the_filter_follows_the_autograd_loop():
    hidden = hidden_scene(n=400)
    views = _views_to(render_views(OracleRasterisationModule(Config()), hidden), "cuda")
    iters = 80
    cfg = train_config(iters)
    cfg.mip_filter_3d = True
    cfg.mip_filter_interval = 30
    t_ref = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views)
    h_ref = t_ref.train(log_interval=1)
    t_fused = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views, fused_step=True)
    h_fused = t_fused.train(log_interval=1)
    assert t_fused.fused_train_step.num_skipped_steps == 0
    l_ref, l_fused = np.array([h["loss"] for h in h_ref]), np.array([h["loss"] for h in h_fused])
    assert np.abs(l_ref - l_fused).max() < 2e-3 * l_ref.max(), np.abs(l_ref - l_fused).max()
    p_ref, p_fused = t_ref.validation(), t_fused.validation()
    assert p_ref > 24.0 and abs(p_ref - p_fused) < 0.15, (p_ref, p_fused)
    f_ref, f_fused = t_ref.filter_3d(), t_fused.filter_3d()
    assert f_ref is not None and float(f_ref.max()) > 0
    assert float((f_ref - f_fused).abs().max()) <= 1e-3 * float(f_ref.max())


def test_mcmc_with_the_filter_stays_finite_and_in_step():
    hidden = hidden_scene(n=300)
    views = _views_to(render_views(OracleRasterisationModule(Config()), hidden), "cuda")
    for fused in (False, True):
        cfg = train_config(60)
        cfg.densification = "mcmc"
        cfg.mcmc_config = MCMCConfig(cap_max=450, refine_start=10, refine_every=10)
        cfg.mip_filter_3d = True
        cfg.mip_filter_interval = 1000
        trainer = GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views, fused_step=fused)
        hist = trainer.train(log_interval=5)
        assert all(math.isfinite(h["loss"]) for h in hist)
        s = trainer.scene
        assert torch.isfinite(s.point_cloud).all() and torch.isfinite(s.point_cloud_features).all()
        f = trainer.filter_3d()
        valid = s.point_invalid_mask == 0
        assert int(valid.sum()) > 300
        assert (f[~valid] == 0).all() and (f[valid] > 0).all()
        # the filter was recomputed after the last refinement: it is the filter of the current rows
        now = compute_filter_3d(s.point_cloud, s.point_invalid_mask, s.point_object_id,
                                [(v[1], v[2], v[3]) for v in views], cfg.rasterisation_config.near_plane, 0.2)
        assert float((now[valid] - f[valid]).abs().max()) <= 0.05 * float(now.max())
        assert trainer.validation() > 15.0
