"""The per-pixel loss weights (``csrc/robust_loss.cu``: histogram and mask pre-passes -> the image loss of
``csrc/image_loss.cu`` on the composite -> post-pass) executed on the CPU under the SIMT emulator from the unmodified kernel
sources, against the torch statement ``loss.robust_weight`` / ``loss.robust_composite``: the weight map, the threshold bin
and the composite bit for bit, dL/dx bit for bit from the kernel's own dL/dx', and the loss and dL/dx against torch
autograd."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.loss import RobustLossConfig, _torch_image_loss, robust_composite, robust_weight
from simt_robust_helpers import build_robust_emulator, emulated_robust_step, new_temps


@pytest.fixture(scope="module")
def emu():
    return build_robust_emulator()


def _frame(H, W, seed, distractors=True):
    rng = np.random.default_rng(seed)
    gt = rng.random((3, H, W)).astype(np.float32)
    image = (gt.transpose(1, 2, 0) + 0.05 * rng.standard_normal((H, W, 3))).astype(np.float32)
    if distractors:  # opaque boxes of random colour: residuals far above the rest
        for _ in range(3):
            h, w = rng.integers(3, max(4, H // 2)), rng.integers(3, max(4, W // 2))
            r, c = rng.integers(0, H - h + 1), rng.integers(0, W - w + 1)
            image[r:r + h, c:c + w] = rng.random(3).astype(np.float32)
    image[::7, ::3, 0] = 1.0   # clamp boundaries: the gradient passes there
    image[1::7, ::3, 1] = 0.0
    image[2::9, ::4, 2] = 1.3  # outside [0, 1]: no gradient
    return image, gt


def _static(H, W, seed, kind):
    if kind is None:
        return None
    rng = np.random.default_rng(seed + 100)
    s = rng.random((H, W)).astype(np.float32)
    if kind == "binary":
        s = (s > 0.3).astype(np.float32)
    else:
        s[rng.random((H, W)) < 0.25] = 0.0
        s[rng.random((H, W)) < 0.25] = 1.0
    return s


def _check(emu, image, gt, static, config, lam=0.2):
    H, W = image.shape[:2]
    out = emulated_robust_step(emu, image, gt, static, config, lam)
    xt, gtt = torch.tensor(image), torch.tensor(gt)
    st = None if static is None else torch.tensor(static)
    w, stats = robust_weight(xt, gtt, st, config)
    np.testing.assert_array_equal(out.weight, w.numpy())
    np.testing.assert_array_equal(out.stats, stats.numpy())
    comp = robust_composite(xt, gtt, w)
    np.testing.assert_array_equal(out.composite, comp.numpy())
    # dL/dx from the kernel's own dL/dx': the chain through an unweighted call on x' (in [0, 1], so w = 1, x'' = x')
    plain = emulated_robust_step(emu, out.composite, gt, None, None, lam)
    np.testing.assert_array_equal(plain.composite, out.composite)
    np.testing.assert_array_equal(plain.image_loss, out.image_loss)
    gate = (image >= 0) & (image <= 1)
    expect = np.where(gate, out.weight[..., None] * plain.grad, np.float32(0.0)).astype(np.float32)
    np.testing.assert_array_equal(out.grad, expect)
    # against torch autograd through the composite
    xr = xt.clone().requires_grad_(True)
    loss, l1, dssim = _torch_image_loss(robust_composite(xr, gtt, w), gtt, lam)
    loss.backward()
    np.testing.assert_allclose(out.image_loss, [float(v.detach()) for v in (loss, l1, dssim)], rtol=2e-5, atol=2e-6)
    scale = float(np.abs(xr.grad.numpy()).max()) + 1e-12
    np.testing.assert_allclose(out.grad, xr.grad.numpy(), rtol=0, atol=2e-4 * scale)
    assert np.isfinite(out.grad).all() and np.isfinite(out.image_loss).all()
    return out, w, stats


@pytest.mark.parametrize("H,W", [(16, 16), (48, 64), (64, 96)])
@pytest.mark.parametrize("q", [0.3, 0.5, 0.9, 1.0])
def test_random_frames_match_the_torch_statement(emu, H, W, q):
    image, gt = _frame(H, W, seed=H * 7 + W + int(q * 10))
    out, w, _ = _check(emu, image, gt, None, RobustLossConfig(inlier_quantile=q))
    if q == 1.0:
        assert (out.weight == 1.0).all()


@pytest.mark.parametrize("kind", ["binary", "soft"])
@pytest.mark.parametrize("q", [0.5, 0.9])
def test_static_weights_with_and_without_the_robust_mask(emu, kind, q):
    H, W = 48, 64
    image, gt = _frame(H, W, seed=5)
    static = _static(H, W, 5, kind)
    _check(emu, image, gt, static, RobustLossConfig(inlier_quantile=q))
    out, _, stats = _check(emu, image, gt, static, None)
    np.testing.assert_array_equal(out.weight, static)
    assert stats[1] == 1.0
    zero = static == 0
    assert (out.grad[zero] == 0).all()


def test_all_residuals_equal(emu):
    H, W = 32, 48
    gt = np.full((3, H, W), 0.25, np.float32)
    image = np.full((H, W, 3), 0.5, np.float32)
    out, _, stats = _check(emu, image, gt, None, RobustLossConfig(inlier_quantile=0.3))
    assert (out.weight == 1.0).all()
    assert stats[0] == 1.0 and stats[1] == np.float32((1024 + 1) / 4096)


def test_residuals_on_bin_edges_and_ties_at_the_quantile(emu):
    H, W = 48, 64
    rng = np.random.default_rng(11)
    k = rng.integers(0, 8, (H, W))  # residual exactly k / 4096: bin k, many ties per bin
    k[:16, :16] = 4000  # one tile of outliers
    gt = np.zeros((3, H, W), np.float32)
    image = np.repeat((k / 4096.0).astype(np.float32)[..., None], 3, axis=2)
    for q in (0.25, 0.5, float(np.float32(np.mean(k <= 3))), 1.0):
        cfg = RobustLossConfig(inlier_quantile=q)
        _, w, stats = _check(emu, image, gt, None, cfg)
        b = int(round(float(stats[1]) * 4096)) - 1
        counts = np.bincount(k.ravel(), minlength=4096).cumsum()
        assert b == int(np.nonzero(counts.astype(np.float32) >= np.float32(q) * np.float32(H * W))[0][0])
    assert (w[:16, :16] == 1.0).all()  # q = 1: everything is an inlier


def test_all_zero_static_weight(emu):
    H, W = 32, 32
    image, gt = _frame(H, W, seed=3)
    static = np.zeros((H, W), np.float32)
    out, _, stats = _check(emu, image, gt, static, RobustLossConfig())
    assert (out.weight == 0).all() and (out.grad == 0).all()
    np.testing.assert_array_equal(out.composite, gt.transpose(1, 2, 0))
    assert stats[0] == 0.0
    assert abs(float(out.image_loss[0])) < 1e-6 and np.isfinite(out.image_loss).all()


def test_a_single_tile_of_distractors_is_dropped(emu):
    H, W = 64, 96
    rng = np.random.default_rng(2)
    gt = rng.random((3, H, W)).astype(np.float32)
    image = (gt.transpose(1, 2, 0) + 0.01 * rng.standard_normal((H, W, 3))).astype(np.float32)
    image[16:32, 32:48] = (1.0 - gt.transpose(1, 2, 0)[16:32, 32:48])  # a distractor covering one tile
    out, _, _ = _check(emu, image, gt, None, RobustLossConfig())
    assert (out.weight[16:32, 32:48] == 0).mean() > 0.9
    assert (out.weight[:16] > 0).mean() > 0.45


def test_two_calls_on_one_temp_are_bit_identical(emu):
    H, W = 48, 64
    image, gt = _frame(H, W, seed=9)
    static = _static(H, W, 9, "soft")
    temps = new_temps(emu, H, W)
    a = emulated_robust_step(emu, image, gt, static, RobustLossConfig(), temps=temps)
    b = emulated_robust_step(emu, image, gt, static, RobustLossConfig(), temps=temps)
    for x, y in ((a.weight, b.weight), (a.grad, b.grad), (a.stats, b.stats), (a.image_loss, b.image_loss)):
        np.testing.assert_array_equal(x, y)
    t = temps[0]  # the ticket and the histogram are left zero for the next call; bytes 16..31 hold b, 32..47 the counts
    assert (t[:16] == 0).all() and (t[48:] == 0).all()
