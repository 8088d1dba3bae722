"""The bilateral-grid kernels of ``csrc/appearance.cu`` (slice forward, slice backward with its finishing kernel, TV), run
unmodified under the SIMT emulator, against the explicit float64 trilinear formula and its autograd gradients."""
import numpy as np
import pytest
import torch

from appearance_reference import explicit_slice, explicit_tv, random_case
from simt_appearance_helpers import build_appearance_emulator, emulated_slice, emulated_slice_backward

FRAMES = [(37, 53), (64, 48), (1, 17), (17, 1)]
GRIDS = [(1, 1, 1), (16, 16, 8), (5, 7, 4)]  # (Gx, Gy, Gz); 16 nodes exceed the pixels of the 1- and 17-pixel axes


@pytest.fixture(scope="module")
def emu():
    return build_appearance_emulator()


def _reference(image, grid, grad_out):
    image = image.clone().requires_grad_(True)
    grid = grid.clone().requires_grad_(True)
    out = explicit_slice(image, grid)
    gi, gg = torch.autograd.grad(out, (image, grid), grad_out)
    return out.detach().numpy(), gi.numpy(), gg.numpy()


def _close(got, want, rel):
    scale = max(float(np.abs(want).max()), 1e-30)
    return float(np.abs(got.astype(np.float64) - want).max()) <= rel * scale


@pytest.mark.parametrize("shape", GRIDS)
@pytest.mark.parametrize("H,W", FRAMES)
def test_slice_and_gradients_match_the_float64_formula(emu, H, W, shape):
    image, grid = random_case(H, W, shape, seed=H * 7 + W + sum(shape))
    # float32 inputs, evaluated in float64 by the reference
    image = image.float().double()
    grid = grid.float().double()
    assert (image < 0).any() and (image > 1).any()
    grad_out = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(1), dtype=torch.float64).float().double()
    out_ref, gi_ref, gg_ref = _reference(image, grid, grad_out)
    out = emulated_slice(emu, image.numpy(), grid.numpy())
    assert float(np.abs(out - out_ref).max()) <= 1e-5
    b = emulated_slice_backward(emu, image.numpy(), grid.numpy(), grad_out.numpy())
    assert _close(b.grad_image, gi_ref, 1e-4)
    assert _close(b.grad_grid, gg_ref, 1e-4)
    again = emulated_slice_backward(emu, image.numpy(), grid.numpy(), grad_out.numpy())
    assert np.array_equal(again.grad_image, b.grad_image) and np.array_equal(again.grad_grid, b.grad_grid)
    assert np.array_equal(emulated_slice(emu, image.numpy(), grid.numpy()), out)


@pytest.mark.parametrize("shape", GRIDS)
def test_tv_term_and_its_gradient(emu, shape):
    H, W = 37, 53
    image, grid = random_case(H, W, shape, seed=11)
    image, grid = image.float().double(), grid.float().double()
    grad_out = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(2), dtype=torch.float64).float().double()
    w = 10.0
    g = grid.clone().requires_grad_(True)
    loss = (explicit_slice(image, g) * grad_out).sum() + w * explicit_tv(g)
    want, = torch.autograd.grad(loss, g)
    b = emulated_slice_backward(emu, image.numpy(), grid.numpy(), grad_out.numpy(), tv_weight=w)
    assert abs(b.tv - w * float(explicit_tv(grid))) <= 1e-5 * max(abs(b.tv), 1e-30) + 1e-12
    assert _close(b.grad_grid, want.numpy(), 1e-4)
    if shape == (1, 1, 1):
        assert b.tv == 0.0


def test_identity_grid_reproduces_the_image(emu):
    image, _ = random_case(17, 23, (16, 16, 8), seed=4)
    grid = torch.zeros((3, 4, 8, 16, 16), dtype=torch.float64)
    for i in range(3):
        grid[i, i] = 1.0
    out = emulated_slice(emu, image.float().numpy(), grid.reshape(12, 8, 16, 16).numpy())
    assert np.array_equal(out, image.float().numpy())
