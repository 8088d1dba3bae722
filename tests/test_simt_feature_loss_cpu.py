"""The feature term of the fused train step (``csrc/feature_loss.cu``: sum pass -> gradient pass) executed on the CPU under
the SIMT emulator from the unmodified kernel source, against ``loss.feature_loss`` and torch autograd: the term, the
supervised-pixel count and dL/dF, for both kinds."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.loss import SupervisionTargets, feature_loss
from simt_feature_loss_helpers import build_feature_loss_emulator, emulated_feature_loss, new_temp


@pytest.fixture(scope="module")
def emu():
    return build_feature_loss_emulator()


def _reference(fmap, labels, target, kind, weight):
    F = torch.tensor(fmap, dtype=torch.float32, requires_grad=True)
    targets = SupervisionTargets(labels=None if labels is None else torch.tensor(labels),
                                 features=None if target is None else torch.tensor(target))
    term = feature_loss(F, targets, kind, weight)
    term.backward()
    return float(term.detach()), F.grad.numpy()


def _frame(H, W, C, seed, kind, scale=3.0):
    rng = np.random.default_rng(seed)
    fmap = (scale * rng.standard_normal((H, W, C))).astype(np.float32)
    labels = target = None
    if kind == "cross_entropy":
        labels = rng.integers(-2, C + 3, size=(H, W)).astype(np.int32)  # negatives and labels >= C: no label
        labels[0, 0], labels[-1, -1] = -1, C  # at least one of each
        labels[1::5, ::3] = 2147483647
    else:
        target = (fmap + rng.standard_normal((H, W, C))).astype(np.float32)
        nan_rows = rng.random((H, W)) < 0.3
        target[nan_rows, rng.integers(0, C)] = np.nan  # one NaN makes the whole pixel unsupervised
        target[0, 0, :] = np.inf
        target[1, 1, :] = fmap[1, 1, :]  # zero error
    return fmap, labels, target


def _check(out, term, grad, n_sup):
    assert abs(float(out.loss[0]) - term) <= 1e-5 * max(abs(term), 1e-30), (out.loss, term)
    assert float(out.loss[1]) == n_sup
    assert np.isfinite(out.grad).all()
    assert np.abs(out.grad - grad).max() <= 1e-5 * max(np.abs(grad).max(), 1e-30), np.abs(out.grad - grad).max()


KINDS_AND_CHANNELS = [("l2", 1)] + [(k, c) for k in ("cross_entropy", "l2") for c in (2, 3, 5, 8, 16)]


# 37 x 29: odd, and not a multiple of the 256-thread CTA.  272 x 976 = 265,472 pixels: more than the 1024 CTAs x 256 threads
# of the capped grid, so both passes run their grid-stride loop twice, as on every real frame
@pytest.mark.parametrize("H,W", [(32, 48), (37, 29), (272, 976)])
@pytest.mark.parametrize("kind,C", KINDS_AND_CHANNELS)
def test_feature_loss_source_matches_the_torch_loss(emu, kind, C, H, W):
    fmap, labels, target = _frame(H, W, C, H * 131 + W * 7 + C, kind)
    weight = 0.7
    temp = new_temp(emu)
    runs = [emulated_feature_loss(emu, fmap, labels, target, weight, temp=temp) for _ in range(2)]
    assert np.array_equal(runs[0].loss, runs[1].loss) and np.array_equal(runs[0].grad, runs[1].grad)  # same temp: bit-identical
    term, grad = _reference(fmap, labels, target, kind, weight)
    if kind == "cross_entropy":
        n_sup = int(((labels >= 0) & (labels < C)).sum())
        assert (runs[0].grad[(labels < 0) | (labels >= C)] == 0).all()
    else:
        n_sup = int(np.isfinite(target).all(axis=-1).sum())
        assert (runs[0].grad[~np.isfinite(target).all(axis=-1)] == 0).all()
    assert 0 < n_sup < H * W
    _check(runs[0], term, grad, n_sup)


@pytest.mark.parametrize("kind,C", [("cross_entropy", 2), ("cross_entropy", 7), ("l2", 1), ("l2", 12)])
def test_all_unsupervised_frame_gives_zero_term_and_zero_gradient(emu, kind, C):
    H, W = 21, 19
    fmap, labels, target = _frame(H, W, C, 3, kind)
    if labels is not None:
        labels[:] = np.where(np.arange(W) % 2 == 0, -1, C)[None, :]
    else:
        target[:, :, 0] = np.nan
    out = emulated_feature_loss(emu, fmap, labels, target, 1.3)
    assert out.loss[0] == 0.0 and out.loss[1] == 0.0
    assert (out.grad == 0).all()
    term, grad = _reference(fmap, labels, target, kind, 1.3)
    assert term == 0.0 and (grad == 0).all()


@pytest.mark.parametrize("C", [2, 5, 16])
def test_cross_entropy_is_stable_for_large_logits(emu, C):
    """Logits of +-80 overflow exp in float32 without the max subtraction; the term and the gradient stay finite."""
    H, W = 17, 23
    rng = np.random.default_rng(C)
    fmap = np.where(rng.random((H, W, C)) < 0.5, 80.0, -80.0).astype(np.float32)
    fmap[::2, ::2, 0] = 80.0
    fmap[1::3, :, :] = 80.0  # ties
    labels = rng.integers(0, C, size=(H, W)).astype(np.int32)
    out = emulated_feature_loss(emu, fmap, labels, None, 0.9)
    assert np.isfinite(out.loss).all() and np.isfinite(out.grad).all()
    term, grad = _reference(fmap, labels, None, "cross_entropy", 0.9)
    _check(out, term, grad, H * W)


def test_l2_gradient_has_the_exact_torch_value_on_a_small_frame(emu):
    H, W, C = 5, 7, 3
    fmap, _, target = _frame(H, W, C, 11, "l2", scale=1.0)
    out = emulated_feature_loss(emu, fmap, None, target, 1.0)
    term, grad = _reference(fmap, None, target, "l2", 1.0)
    _check(out, term, grad, int(np.isfinite(target).all(axis=-1).sum()))


def test_feature_loss_refuses_bad_arguments():
    F = torch.zeros(4, 4, 1)
    with pytest.raises(ValueError, match="C >= 2"):
        feature_loss(F, SupervisionTargets(labels=torch.zeros(4, 4, dtype=torch.int32)), "cross_entropy", 1.0)
    with pytest.raises(ValueError, match="targets.labels"):
        feature_loss(torch.zeros(4, 4, 3), SupervisionTargets(), "cross_entropy", 1.0)
    with pytest.raises(ValueError, match="targets.features"):
        feature_loss(F, SupervisionTargets(), "l2", 1.0)
    with pytest.raises(ValueError, match="must be one of"):
        feature_loss(F, SupervisionTargets(features=F), "l1", 1.0)
    # positional (depth, mask) keeps working
    tg = SupervisionTargets(torch.ones(2, 2), torch.zeros(2, 2))
    assert tg.labels is None and tg.features is None and float(tg.depth[0, 0]) == 1.0
