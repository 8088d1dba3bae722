"""-m gpu: per-pixel weights of the image loss on the device -- the kernels of ``csrc/robust_loss.cu`` against the torch
statement (``loss.robust_weight``), the fused step against the plain step and against the autograd trainer, the static
weight, the key-capacity overflow, and a fit through transient distractors."""
import dataclasses
import json
import math

import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import CameraInfo
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep
from taichi_3d_gaussian_splatting_b200.loss import (RobustLossConfig, SupervisionTargets, _torch_image_loss,
                                                    fused_image_loss_with_grad, fused_robust_image_loss_with_grad,
                                                    robust_composite, robust_weight)
from taichi_3d_gaussian_splatting_b200.mcmc import MCMCConfig
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from trainer_helpers import hidden_scene, initial_scene, render_views, train_config

pytestmark = pytest.mark.gpu


def _frame(H, W, seed, static_kind):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gt = torch.rand((3, H, W), device="cuda", generator=g)
    x = gt.permute(1, 2, 0) + 0.05 * torch.randn((H, W, 3), device="cuda", generator=g)
    for k in range(4):  # distractor boxes
        h, w = H // (3 + k), W // (4 + k)
        r, c = (H * (k + 1)) // 6, (W * (2 * k + 1)) // 9
        x[r:r + h, c:c + w] = torch.rand(3, device="cuda", generator=g)
    x[::7, ::3, 0] = 1.0
    x[1::7, ::3, 1] = 0.0
    x[2::9, ::4, 2] = 1.3
    s = None
    if static_kind:
        s = torch.rand((H, W), device="cuda", generator=g)
        s[s < 0.2] = 0.0
        s[s > 0.8] = 1.0
    return x.contiguous(), gt.contiguous(), s


@pytest.mark.parametrize("H,W", [(64, 96), (1072, 1920)])
@pytest.mark.parametrize("static_kind", [None, "soft"])
@pytest.mark.parametrize("q", [0.3, 0.5, 0.9, 1.0])
def test_kernels_match_the_torch_statement(H, W, static_kind, q):
    x, gt, s = _frame(H, W, seed=H + int(100 * q), static_kind=static_kind)
    cfg = RobustLossConfig(inlier_quantile=q)
    losses, grad, w, stats = fused_robust_image_loss_with_grad(x, gt, 0.2, s, cfg)
    w_ref, stats_ref = robust_weight(x, gt, s, cfg)
    assert torch.equal(w, w_ref) and torch.equal(stats, stats_ref)
    if q == 1.0 and s is None:
        assert bool((w == 1).all())
    # dL/dx from the image loss's own dL/dx' on the same composite, bit for bit
    comp = robust_composite(x, gt, w_ref).contiguous()
    losses_c, grad_c = fused_image_loss_with_grad(comp, gt, 0.2)
    assert torch.equal(losses, losses_c)
    gate = (x >= 0) & (x <= 1)
    assert torch.equal(grad, torch.where(gate, w[..., None] * grad_c, torch.zeros_like(grad_c)))
    # the loss and dL/dx against torch autograd
    xr = x.clone().requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        loss, l1, dssim = _torch_image_loss(robust_composite(xr, gt, w_ref), gt, 0.2)
        loss.backward()
    for a, b in zip(losses.tolist(), (loss, l1, dssim)):
        b = float(b.detach())
        assert abs(a - b) <= 2e-6 * max(1.0, abs(b))
    assert float((grad - xr.grad).abs().max()) <= 1e-4 * float(xr.grad.abs().max())
    if s is not None:
        assert not grad[s == 0].any()
    again = fused_robust_image_loss_with_grad(x, gt, 0.2, s, cfg)
    for a, b in zip((losses, grad, w, stats), again):
        assert torch.equal(a, b)


def _plain_scene():
    sc = initial_scene(hidden_scene(n=400), device="cuda")
    return Scene(sc.point_cloud.detach().contiguous(), sc.point_cloud_features.detach().contiguous(), sc.point_invalid_mask,
                 sc.point_object_id)


class _NullRobust:
    """Routes every plain train-step call of a FusedTrainStep through gsb200_train_step_robust with NULL blocks."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def gsb200_train_step(self, args):
        return self._lib.gsb200_train_step_robust(args, None, None, None, None, None, None)


def _views():
    hidden = hidden_scene(n=400)
    return render_views(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), hidden, device="cuda")


def test_q_1_and_null_robust_are_the_plain_train_step():
    """q = 1 without a static weight, and a NULL robust block, against gsb200_train_step on the same state.  Everything up to
    the hand-off to the backward is deterministic, so the image, the loss and dL/dI are compared bit for bit.  The backward
    sums with float atomics, so the gradients and the updated tensors are compared against the spread of three plain steps,
    with a floor that does not depend on two plain steps happening to agree: 1e-5 of the gradient's largest entry, and for
    the parameters 2 % of the learning rate where the gradient is solid (Adam's first step moves an entry by lr g / |g|, so
    the atomics' rounding cannot flip it there) and twice the learning rate anywhere (the most a first step can move)."""
    img, q, t, cam = _views()[1]
    lrs = dict(xyz=2e-4, feat=5e-3)
    states = {}
    for name in ("plain", "plain_again", "plain_third", "null", "q1"):
        scene = _plain_scene()
        step = FusedTrainStep(scene, GPCR.GaussianPointCloudRasterisationConfig(),
                              robust=RobustLossConfig(inlier_quantile=1.0) if name == "q1" else None)
        if name == "null":
            step._lib = _NullRobust(step._lib)
        step.run(img, q, t, cam, 1, lrs["feat"], lrs["xyz"])
        torch.cuda.synchronize()
        states[name] = dict(image=step.image.clone(), loss=step.loss.clone(), dI=step._last.buffers.grad_image.clone(),
                            gx=step.grad_pointcloud.clone(), gf=step.grad_pointcloud_features.clone(),
                            xyz=scene.point_cloud.clone(), feat=scene.point_cloud_features.clone())
        if name == "q1":
            assert bool((step.loss_weight == 1).all()) and float(step.robust_stats[0]) == 1.0
    plains = [states[k] for k in ("plain", "plain_again", "plain_third")]
    ref = plains[0]

    def spread(key):
        return max(float((a[key] - b[key]).abs().max()) for i, a in enumerate(plains) for b in plains[i + 1:])
    for name in ("null", "q1"):
        st = states[name]
        for key in ("image", "loss", "dI"):
            assert torch.equal(st[key], ref[key]), (name, key)
        for key in ("gx", "gf"):
            bound = max(4 * spread(key), 1e-5 * float(ref[key].abs().max()))
            assert float((st[key] - ref[key]).abs().max()) <= bound, (name, key)
        for key, grad in (("xyz", "gx"), ("feat", "gf")):
            diff = (st[key] - ref[key]).abs()
            solid = ref[grad].abs() > 1e-3 * ref[grad].abs().max()
            assert float(diff[solid].max()) <= max(4 * spread(key), 0.02 * lrs[key]), (name, key)
            assert float(diff.max()) <= 2.01 * lrs[key], (name, key)


def test_static_zero_weight_gets_exactly_zero_gradient():
    img, q, t, cam = _views()[2]
    s = torch.ones((cam.camera_height, cam.camera_width), device="cuda")
    s[10:40, 20:70] = 0.0
    s[:, :8] = 0.25
    step = FusedTrainStep(_plain_scene(), GPCR.GaussianPointCloudRasterisationConfig(), robust=RobustLossConfig())
    step.run(img, q, t, cam, 1, 5e-3, 2e-4, targets=SupervisionTargets(loss_weight=s))
    torch.cuda.synchronize()
    g = step._last.buffers.grad_image
    assert not g[s == 0].any() and g[s > 0].abs().sum() > 0
    w_ref, stats_ref = robust_weight(step.image, img, s, RobustLossConfig())
    assert torch.equal(step.loss_weight, w_ref) and torch.equal(step.robust_stats, stats_ref)
    step.run(img, q, t, cam, 1, 5e-3, 2e-4, targets=SupervisionTargets(loss_weight=s), robust_active=False)
    torch.cuda.synchronize()
    assert torch.equal(step.loss_weight, s) and float(step.robust_stats[1]) == 1.0


def test_key_capacity_overflow_stays_a_no_op():
    """An overflow iteration with the loss weights leaves the scene and the Adam moments exactly as the plain step's overflow
    iteration does, and is counted as skipped."""
    img, q, t, cam = _views()[0]
    s = torch.ones((cam.camera_height, cam.camera_width), device="cuda")
    s[:16] = 0.0
    out = {}
    for name in ("plain", "robust"):
        scene = _plain_scene()
        xyz0 = scene.point_cloud.clone()
        step = FusedTrainStep(scene, GPCR.GaussianPointCloudRasterisationConfig(), key_capacity=64,
                              robust=RobustLossConfig() if name == "robust" else None)
        kw = dict(targets=SupervisionTargets(loss_weight=s)) if name == "robust" else {}
        step.run(img, q, t, cam, 1, 5e-3, 2e-4, **kw)
        torch.cuda.synchronize()
        assert torch.equal(scene.point_cloud, xyz0)
        assert not step.position_exp_avg.any() and not step.feature_exp_avg.any()
        out[name] = (scene.point_cloud.clone(), scene.point_cloud_features.clone())
        with pytest.warns(UserWarning, match="no-op"):
            step.run(img, q, t, cam, 1, 5e-3, 2e-4, **kw)
        assert step.num_skipped_steps == 1
    assert all(torch.equal(a, b) for a, b in zip(out["plain"], out["robust"]))


def _masked_views(views):
    return [(v[0], v[1], v[2], v[3], SupervisionTargets(mask=(v[0].mean(0) > 0.05).float().contiguous())) for v in views]


CASES = {
    "robust": dict(),
    "background_mask": dict(background="random", mask_loss_weight=0.3),
    "appearance": dict(appearance_grid=(4, 3, 2), appearance_learning_rate=5e-3, appearance_tv_weight=1.0),
    "mcmc": dict(densification="mcmc", mcmc_config=MCMCConfig(cap_max=500, refine_start=4, refine_every=4, seed=17)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_fused_step_matches_the_autograd_trainer(case):
    hidden = hidden_scene(n=400)
    views = _views()
    if case == "background_mask":
        views = _masked_views(views)
    for iters in (1, 6):
        cfg = dataclasses.replace(train_config(iters), robust_loss=RobustLossConfig(inlier_quantile=0.5),
                                  **CASES[case])
        if case == "mcmc":
            cfg.loss_function_config.enable_regularization = False

        def mk(**kw):
            return GaussianPointCloudTrainer(cfg, initial_scene(hidden, device="cuda"), views,
                                             background_generator=torch.Generator(device="cuda").manual_seed(5),
                                             generator=torch.Generator(device="cuda").manual_seed(3), **kw)
        t_ref, t_fused = mk(), mk(fused_step=True)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            h_ref = t_ref.train(log_interval=1)
        h_fused = t_fused.train(log_interval=1)
        for a, b in zip(h_ref, h_fused):
            assert abs(a["loss"] - b["loss"]) <= 2e-6 * abs(a["loss"]) + 1e-7 + (0 if iters == 1 else 1e-4), (case, a, b)
            tol = 2e-3 if iters == 1 else 0.02
            assert abs(a["robust_inlier_fraction"] - b["robust_inlier_fraction"]) <= tol, (case, a, b)
        assert 0.0 < h_fused[0]["robust_inlier_fraction"] < 1.0
        if iters == 1:
            s = t_fused.fused_train_step
            gx_ref = t_ref.scene.point_cloud.grad
            assert float((s.grad_pointcloud - gx_ref).abs().max()) <= 1e-4 * float(gx_ref.abs().max()), case
            gf_ref = t_ref.scene.point_cloud_features.grad
            assert float((s.grad_pointcloud_features - gf_ref).abs().max()) <= 1e-4 * float(gf_ref.abs().max()), case


# ---------------------------------------------------------------------------------------------- distractor fit
FH, FW = 128, 192
FIT_YAWS = [-11.0 + 2.0 * i for i in range(14)]
HELD_OUT = (3, 10)
FIT_ITERS = 600


def _fit_problem():
    hidden = make_scene(1500, FH, FW, 0.08, 21, sh_degree=1)
    hidden.point_cloud[:, 2] = hidden.point_cloud[:, 2] * 0.5 + 1.0
    hidden.point_cloud_features[:, 7] += 1.0
    dev = "cuda"
    K = hidden.camera_info.camera_intrinsics.to(dev)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    pc, feat = hidden.point_cloud.to(dev), hidden.point_cloud_features.to(dev)
    mask, obj = hidden.point_invalid_mask.to(dev), hidden.point_object_id.to(dev)
    g = torch.Generator().manual_seed(8)
    train, clean_train, held = [], [], []
    for i, yaw in enumerate(FIT_YAWS):
        half = math.radians(yaw) / 2
        q = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device=dev)
        t = torch.zeros((1, 3), device=dev)
        cam = CameraInfo(K, FH, FW, 0)
        with torch.no_grad():
            img, _, _ = op(GPCR.GaussianPointCloudRasterisationInput(
                point_cloud=pc, point_cloud_features=feat.clone(), point_object_id=obj, point_invalid_mask=mask,
                camera_info=cam, q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3))
        clean = img.clamp(0, 1).permute(2, 0, 1).contiguous()
        if i in HELD_OUT:
            held.append((clean, q, t, cam))
            continue
        shown = clean.clone()
        weight = torch.ones((FH, FW), device=dev)
        for _ in range(2):  # opaque rectangles of a random colour at view-specific places
            h, w = int(torch.randint(20, 45, (1,), generator=g)), int(torch.randint(25, 60, (1,), generator=g))
            r, c = int(torch.randint(0, FH - h, (1,), generator=g)), int(torch.randint(0, FW - w, (1,), generator=g))
            shown[:, r:r + h, c:c + w] = torch.rand(3, 1, 1, generator=g).to(dev)
            weight[r:r + h, c:c + w] = 0.0
        train.append((shown.contiguous(), q, t, cam, SupervisionTargets(loss_weight=weight.contiguous())))
        clean_train.append((clean, q, t, cam))
    return hidden, train, clean_train, held


def _fit(hidden, views, robust, static):
    cfg = train_config(FIT_ITERS)
    cfg.robust_loss = robust
    scene = initial_scene(hidden, device="cuda")
    if not static:
        views = [v[:4] for v in views]
    trainer = GaussianPointCloudTrainer(cfg, scene, views, fused_step=True)
    trainer.train()
    return trainer


@pytest.fixture(scope="module")
def fit_results():
    hidden, train, clean_train, held = _fit_problem()
    out = {}
    for name, robust, static in (("plain", None, False), ("q0.5", RobustLossConfig(0.5, start_iteration=100), False),
                                 ("q0.7", RobustLossConfig(0.7, start_iteration=100), False),
                                 ("q0.9", RobustLossConfig(0.9, start_iteration=100), False), ("static", None, True)):
        trainer = _fit(hidden, train, robust, static)
        out[name] = (trainer.validation(clean_train), trainer.validation(held))
    print(json.dumps(dict(card=torch.cuda.get_device_properties(0).name, psnr_train_clean_and_held_out=out)))
    return out


def test_distractor_fit_with_the_robust_mask_beats_the_plain_fit(fit_results):
    """Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, PSNR against clean renders of the training / the 2
    held-out poses: plain 41.80 / 42.00 dB; q = 0.5: 33.66 / 33.94 dB; q = 0.7: 37.30 / 37.82 dB; q = 0.9: 42.54 / 42.84 dB;
    static weights over the boxes: 42.80 / 42.92 dB.  The default q (0.9) must keep about half of its measured gain (0.74 /
    0.84 dB); the smaller quantiles are recorded, not asserted."""
    plain, robust = fit_results["plain"], fit_results["q0.9"]
    assert robust[0] > plain[0] + 0.35 and robust[1] > plain[1] + 0.4, fit_results
    assert RobustLossConfig().inlier_quantile == 0.9


def test_distractor_fit_with_static_weights_fits_at_least_as_well(fit_results):
    """The static weights must beat the plain fit by the margin asked of the robust mask, and stay within 0.2 dB of the
    robust fit.  The slack is run-to-run noise of the backward's float atomics over 600 iterations, not a loss of fit: on
    the card of the measurement above three runs gave static 42.80 / 42.92 dB against q = 0.9's 42.54 / 42.84 dB, then
    42.62 / 42.74 against 42.59 / 42.88 and 42.54 / 42.66 against 42.51 / 42.80 (the held-out pair reversed by up to
    0.14 dB)."""
    static, robust, plain = fit_results["static"], fit_results["q0.9"], fit_results["plain"]
    assert static[0] > plain[0] + 0.35 and static[1] > plain[1] + 0.4, fit_results
    assert static[0] >= robust[0] - 0.2 and static[1] >= robust[1] - 0.2, fit_results
