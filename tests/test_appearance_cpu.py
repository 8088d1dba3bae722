"""The torch path of the bilateral-grid slice (``appearance.apply_bilateral_grid`` on CPU tensors, the ``grid_sample`` form)
against the explicit float64 trilinear formula, its gradients by ``gradcheck``, and the TV prior."""
import pytest
import torch

from appearance_reference import explicit_slice, random_case
from taichi_3d_gaussian_splatting_b200.appearance import (apply_bilateral_grid, bilateral_grid_tv, check_grid_shape,
                                                          identity_grids)


@pytest.mark.parametrize("shape", [(16, 16, 8), (1, 1, 1), (7, 5, 4), (64, 3, 16)])
@pytest.mark.parametrize("H,W", [(37, 53), (1, 17), (17, 1)])
def test_torch_path_matches_the_explicit_formula(shape, H, W):
    image, grid = random_case(H, W, shape, seed=H * 100 + W)
    out = apply_bilateral_grid(image, grid)
    assert out.shape == (H, W, 3) and out.dtype == torch.float64
    assert torch.allclose(out, explicit_slice(image, grid), atol=1e-12, rtol=0)


@pytest.mark.parametrize("shape", [(16, 16, 8), (1, 1, 1), (5, 7, 4)])
def test_identity_grid_returns_the_image(shape):
    image, _ = random_case(37, 53, shape)
    grids = identity_grids(2, shape, dtype=torch.float64)
    assert grids.shape == (2, 12, shape[2], shape[1], shape[0])
    assert torch.allclose(apply_bilateral_grid(image, grids[1]), image, atol=1e-14, rtol=0)


def test_one_node_grid_is_a_plain_affine():
    image, _ = random_case(20, 30, (1, 1, 1), seed=3)
    M = torch.tensor([[1.2, 0.1, -0.05, 0.02], [0.0, 0.9, 0.1, -0.03], [0.05, -0.1, 1.1, 0.04]], dtype=torch.float64)
    grid = M.reshape(12, 1, 1, 1)
    want = image @ M[:, :3].T + M[:, 3]
    assert torch.allclose(apply_bilateral_grid(image, grid), want, atol=1e-14, rtol=0)


def test_gradcheck_including_the_luminance_term():
    """Colours keep 0 < lum < 1 and stay away from the z nodes, so the finite differences see one trilinear piece along z
    (the pixel positions are not differentiated)."""
    g = torch.Generator().manual_seed(5)
    H, W, shape = 6, 7, (4, 3, 5)
    gx, gy, gz = shape
    base = torch.rand((H, W), generator=g, dtype=torch.float64)
    # lum = 0.1 + 0.8 * base, nudged off the z nodes (multiples of 1 / (Gz - 1) = 0.25)
    lum = 0.1 + 0.8 * base
    lum = torch.where(((lum * (gz - 1)) % 1 - 0.5).abs() > 0.45, lum + 0.04, lum)
    tint = torch.tensor([0.02, -0.01, 0.0], dtype=torch.float64)
    image = (lum[..., None] + tint).clone().requires_grad_(True)
    _, grid = random_case(H, W, shape, seed=6, spread=0.2)
    grid.requires_grad_(True)
    assert torch.autograd.gradcheck(apply_bilateral_grid, (image, grid), eps=1e-6, atol=1e-6)


def test_luminance_gradient_is_zero_where_the_clamp_is_active():
    """lum = 1.5 is clamped: dL/dc is A^T dL/dout alone, which the explicit formula (its clamp passes no gradient outside
    [0, 1]) gives as well; inside the range the two paths agree with the luminance term included."""
    _, grid = random_case(3, 4, (2, 2, 3), seed=2)
    for value in (1.5, 0.4):
        image = torch.full((3, 4, 3), value, dtype=torch.float64, requires_grad=True)
        gimg, = torch.autograd.grad(apply_bilateral_grid(image, grid).sum(), image)
        want, = torch.autograd.grad(explicit_slice(image, grid).sum(), image)
        assert torch.allclose(gimg, want, atol=1e-12, rtol=0)


def test_tv_against_a_hand_computed_value():
    grid = torch.zeros((12, 2, 1, 3), dtype=torch.float64)
    grid[0, 0, 0] = torch.tensor([0.0, 1.0, 3.0])  # x differences 1, 2 on channel 0, z = 0
    grid[5, 1, 0, 2] = 2.0                         # one node of channel 5 at z = 1
    # x axis: differences (12, 2, 1, 2) = 48 values; squares 1 + 4 (channel 0) + 4 (channel 5, x = 1 -> 2) = 9
    # y axis: one node, 0.  z axis: (12, 1, 1, 3) = 36 values; channel 0: (0 - 0)^2 + (0 - 1)^2 + (0 - 3)^2 = 10,
    # channel 5: 4
    want = 9 / 48 + 14 / 36
    assert abs(float(bilateral_grid_tv(grid)) - want) < 1e-15
    assert float(bilateral_grid_tv(identity_grids(1, (5, 4, 3), dtype=torch.float64)[0])) == 0.0
    assert float(bilateral_grid_tv(torch.randn(12, 1, 1, 1, dtype=torch.float64))) == 0.0


@pytest.mark.parametrize("shape", [(0, 1, 1), (65, 1, 1), (1, 65, 1), (1, 1, 17), (1, 1, 0), (2, 2)])
def test_grid_shape_limits(shape):
    with pytest.raises(ValueError):
        check_grid_shape(shape)
    with pytest.raises(ValueError):
        identity_grids(1, shape)
