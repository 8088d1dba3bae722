"""The depth, mask and background terms of the fused train step (``csrc/supervision_loss.cu`` pre-pass -> the image loss of
``csrc/image_loss.cu`` on the composited images -> post-pass) executed on the CPU under the SIMT emulator from the unmodified
kernel sources, against ``loss.supervision_loss`` and torch autograd: the three losses and dL/dI, dL/dS, dL/dD."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets, supervision_loss
from simt_supervision_helpers import build_supervision_emulator, emulated_supervision_step, new_temps


@pytest.fixture(scope="module")
def emu():
    return build_supervision_emulator()


def _frame(H, W, seed, depth_kind="dense"):
    rng = np.random.default_rng(seed)
    gt = rng.random((3, H, W)).astype(np.float32)
    image = (gt.transpose(1, 2, 0) + 0.3 * rng.standard_normal((H, W, 3))).astype(np.float32)
    alpha = rng.random((H, W)).astype(np.float32)
    alpha[::4, ::3] = 1.0
    alpha[1::7, ::5] = 0.0
    depth = (1.0 + 2.0 * rng.random((H, W))).astype(np.float32)
    mask = rng.random((H, W)).astype(np.float32)
    mask[::3] = (mask[::3] > 0.5).astype(np.float32)
    mask[2::9, 1::4] = alpha[2::9, 1::4]  # |S - m| = 0: subgradient 0
    d_target = (depth + 0.3 * rng.standard_normal((H, W))).astype(np.float32)
    d_target[::6, ::5] = depth[::6, ::5]  # |D - d*| = 0
    if depth_kind == "sparse":
        holes = rng.random((H, W)) < 0.7
        d_target[holes] = np.where(rng.random(int(holes.sum())) < 0.5, 0.0, np.nan).astype(np.float32)
        d_target[0, 0] = np.inf
        d_target[0, 1] = -1.0
    elif depth_kind == "none":
        d_target[:] = 0.0
        d_target[::2] = np.nan
    # pixels on the clamp boundaries: I' exactly 0 or 1 must pass the gradient (torch.clamp does)
    image[::5, ::2, 0] = 1.0
    image[1::5, ::2, 1] = 0.0
    alpha[::5, ::2] = 1.0  # I' = I there whatever the background
    alpha[1::5, ::2] = 1.0
    return image, gt, alpha, depth, d_target, mask


def _reference(image, gt, alpha, depth, d_target, mask, bg, lam, w_d, w_m):
    I = torch.tensor(image, dtype=torch.float32, requires_grad=True)
    S = torch.tensor(alpha, dtype=torch.float32, requires_grad=True)
    D = torch.tensor(depth, dtype=torch.float32, requires_grad=True)
    targets = SupervisionTargets(depth=None if d_target is None else torch.tensor(d_target),
                                 mask=None if mask is None else torch.tensor(mask))
    bgt = None if bg is None else torch.tensor(bg, dtype=torch.float32)
    total, l1, dssim, mterm, dterm = supervision_loss(I, D, S, torch.tensor(gt), targets, bgt, lam, w_d, w_m)
    total.backward()
    grad = lambda t: np.zeros(t.shape, np.float32) if t.grad is None else t.grad.numpy()  # noqa: E731
    return tuple(float(x.detach()) for x in (total, l1, dssim, mterm, dterm)), grad(I), grad(S), grad(D)


CASES = {  # name: (depth weight, mask weight, background, mask given, depth kind)
    "depth": (0.5, 0.0, None, False, "dense"),
    "mask": (0.0, 0.7, None, True, "dense"),
    "white": (0.0, 0.0, (1.0, 1.0, 1.0), False, "dense"),
    "white_mask": (0.0, 0.0, (1.0, 1.0, 1.0), True, "dense"),
    "random_mask": (0.0, 0.3, (0.21, 0.83, 0.47), True, "dense"),
    "random_nomask": (0.0, 0.0, (0.6, 0.1, 0.9), False, "dense"),
    "sparse_depth": (1.3, 0.0, None, False, "sparse"),
    "no_valid_depth": (0.8, 0.0, None, False, "none"),
    "all": (0.4, 0.6, (0.3, 0.7, 0.2), True, "sparse"),
}


# 37 x 29: not a multiple of the 16-pixel tile, nor of 256 pixels.  272 x 976 = 265,472 pixels: more than the 1024 CTAs x 256
# threads of the capped grid, so both kernels run their grid-stride loop twice, as on every real frame (one emulated call
# takes about 30 s on a CPU, so the repeated-call check stays on the small frames)
@pytest.mark.parametrize("H,W", [(32, 48), (37, 29), (272, 976)])
@pytest.mark.parametrize("name", sorted(CASES))
def test_supervision_source_matches_the_torch_loss(emu, name, H, W):
    w_d, w_m, bg, with_mask, depth_kind = CASES[name]
    image, gt, alpha, depth, d_target, mask = _frame(H, W, H * 31 + W + len(name), depth_kind)
    mask = mask if with_mask else None
    d_target = d_target if w_d > 0 else None
    bg_arr = None if bg is None else np.array(bg, np.float32)
    temps = new_temps(emu, H, W)
    runs = [emulated_supervision_step(emu, image, gt, alpha, depth, d_target, mask, bg_arr, 0.2, w_d, w_m, temps=temps)
            for _ in range(2 if H * W <= 256 * 1024 else 1)]
    for again in runs[1:]:  # second call on the same temps: bit-identical
        for a, b in zip(runs[0].__dict__.values(), again.__dict__.values()):
            assert np.array_equal(a, b, equal_nan=True)
    out = runs[0]
    (total, l1, dssim, mterm, dterm), gI, gS, gD = _reference(image, gt, alpha, depth, d_target, mask, bg_arr, 0.2, w_d, w_m)
    assert abs(out.loss[0] - total) <= 2e-6 * max(1.0, abs(total)), (out.loss, total)
    assert abs(out.loss[1] - mterm) <= 1e-6 * max(1.0, abs(mterm))
    assert abs(out.loss[2] - dterm) <= 1e-6 * max(1.0, abs(dterm))
    assert abs(out.image_loss[1] - l1) <= 2e-6 and abs(out.image_loss[2] - dssim) <= 5e-6
    assert np.abs(out.grad_image - gI).max() <= 2e-5 * np.abs(gI).max()
    if w_m > 0 or bg is not None:
        assert np.isfinite(out.grad_alpha).all()
        assert np.abs(out.grad_alpha - gS).max() <= 1e-5 * max(np.abs(gS).max(), 1e-30), np.abs(out.grad_alpha - gS).max()
    else:
        assert np.isnan(out.grad_alpha).all()  # the term is off: not written
    if w_d > 0:
        assert np.isfinite(out.grad_depth).all()
        assert np.abs(out.grad_depth - gD).max() <= 1e-6 * max(np.abs(gD).max(), 1e-30)
        if depth_kind == "none":
            assert out.loss[2] == 0.0 and (out.grad_depth == 0).all()
    else:
        assert np.isnan(out.grad_depth).all()


def test_mask_and_depth_gradients_have_the_exact_torch_values(emu):
    """The subgradient at |.| = 0 is 0, and off-zero the value is exactly w / count, as torch's autograd forms it."""
    H, W = 24, 40
    image, gt, alpha, depth, d_target, mask = _frame(H, W, 5, "sparse")
    out = emulated_supervision_step(emu, image, gt, alpha, depth, d_target, mask, None, 0.2, 0.9, 0.4)
    _, _, gS, gD = _reference(image, gt, alpha, depth, d_target, mask, None, 0.2, 0.9, 0.4)
    assert np.array_equal(out.grad_alpha, gS)
    assert np.array_equal(out.grad_depth, gD)
    assert (out.grad_alpha[alpha == mask] == 0).all()
