"""The bilateral-grid slice written out as its explicit trilinear formula (include/gsb200.h), in float64 torch: the reference
the torch path, the emulated kernels and the GPU kernels are held to.  Test infrastructure."""
import torch


def _split(g, n):
    i0 = g.floor().clamp(0, max(n - 2, 0)).long()
    return i0, (i0 + 1).clamp(max=n - 1), g - i0


def explicit_slice(image: torch.Tensor, grid: torch.Tensor) -> torch.Tensor:
    """image (H, W, 3), grid (12, Gz, Gy, Gx) -> (H, W, 3), in the inputs' dtype (differentiable)."""
    H, W, _ = image.shape
    _, gz, gy, gx = grid.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=image.dtype), torch.arange(W, dtype=image.dtype), indexing="ij")
    cx = xs * (gx - 1) / max(W - 1, 1)
    cy = ys * (gy - 1) / max(H - 1, 1)
    lum = (image @ torch.tensor([0.299, 0.587, 0.114], dtype=image.dtype)).clamp(0, 1)
    cz = lum * (gz - 1)
    x0, x1, fx = _split(cx, gx)
    y0, y1, fy = _split(cy, gy)
    z0, z1, fz = _split(cz, gz)
    coef = 0
    for zi, wz in ((z0, 1 - fz), (z1, fz)):
        for yi, wy in ((y0, 1 - fy), (y1, fy)):
            for xi, wx in ((x0, 1 - fx), (x1, fx)):
                coef = coef + (wz * wy * wx)[..., None] * grid[:, zi, yi, xi].permute(1, 2, 0)
    A = coef.reshape(H, W, 3, 4)
    return (A[..., :3] @ image[..., None])[..., 0] + A[..., 3]


def explicit_tv(grid: torch.Tensor) -> torch.Tensor:
    return sum((torch.diff(grid, dim=d) ** 2).mean() for d in (1, 2, 3) if grid.shape[d] > 1) if max(grid.shape[1:]) > 1 \
        else torch.zeros((), dtype=grid.dtype)


def random_case(H, W, shape, seed=0, spread=0.3):
    """A float64 image with colours in [-0.1, 1.1] and a grid = identity + noise; shape is (Gx, Gy, Gz)."""
    g = torch.Generator().manual_seed(seed)
    gx, gy, gz = shape
    image = torch.rand((H, W, 3), generator=g, dtype=torch.float64) * 1.2 - 0.1
    grid = torch.zeros((3, 4, gz, gy, gx), dtype=torch.float64)
    for i in range(3):
        grid[i, i] = 1.0
    grid = grid.reshape(12, gz, gy, gx) + spread * torch.randn((12, gz, gy, gx), generator=g, dtype=torch.float64)
    return image, grid
