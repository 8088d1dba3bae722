"""Per-view appearance compensation: a bilateral grid per training image (Wang et al., "Bilateral Guided Radiance Field
Processing", SIGGRAPH 2024), trained with the scene and dropped at test time, so that per-view exposure, white balance and
vignetting end up in the grids instead of the scene.

A grid ``G`` of one view is a (12, Gz, Gy, Gx) float32 tensor: a 3x4 affine ``[A | b]`` (row-major) per node over (x, y,
luminance).  At pixel (px, py) of an (H, W, 3) image with colour c::

    gx = px (Gx-1) / max(W-1, 1),  gy = py (Gy-1) / max(H-1, 1),  gz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) (Gz-1)
    [A | b] = trilinear interpolation of G at (gx, gy, gz),  out = A c + b

which is ``F.grid_sample(G[None], (x, y, 2 lum - 1), align_corners=True, padding_mode="border")``.  A (1, 1, 1) grid is a
plain per-view affine colour transform (exposure and white balance).  On CUDA tensors the slice and its gradient run in the
library's kernels (``gsb200_bilateral_grid_forward`` / ``_backward``: deterministic, no float atomics); on CPU tensors the
``grid_sample`` form above is used.
"""
import ctypes
from typing import Tuple

import torch
import torch.nn.functional as F

__all__ = ["identity_grids", "apply_bilateral_grid", "bilateral_grid_tv", "check_grid_shape", "DEFAULT_GRID_SHAPE"]

DEFAULT_GRID_SHAPE = (16, 16, 8)  # (Gx, Gy, Gz)
MAX_XY, MAX_Z = 64, 16  # GSB_BILATERAL_GRID_MAX_XY / _MAX_Z of include/gsb200.h
_LUMA = (0.299, 0.587, 0.114)


def check_grid_shape(shape) -> Tuple[int, int, int]:
    """(Gx, Gy, Gz) as ints, or ``ValueError`` outside 1 <= Gx, Gy <= 64 and 1 <= Gz <= 16."""
    try:
        gx, gy, gz = (int(v) for v in shape)
    except (TypeError, ValueError):
        raise ValueError(f"a grid shape is (Gx, Gy, Gz), got {shape!r}") from None
    if not (1 <= gx <= MAX_XY and 1 <= gy <= MAX_XY and 1 <= gz <= MAX_Z) or tuple(shape) != (gx, gy, gz):
        raise ValueError(f"a grid shape needs 1 <= Gx, Gy <= {MAX_XY} and 1 <= Gz <= {MAX_Z}, got {tuple(shape)}")
    return gx, gy, gz


def identity_grids(num_views: int, shape=DEFAULT_GRID_SHAPE, device=None, dtype=torch.float32) -> torch.Tensor:
    """(num_views, 12, Gz, Gy, Gx) grids that reproduce the image (A = I, b = 0 at every node); ``shape`` is (Gx, Gy, Gz)."""
    gx, gy, gz = check_grid_shape(shape)
    g = torch.zeros((num_views, 3, 4, gz, gy, gx), dtype=dtype, device=device)
    for i in range(3):
        g[:, i, i] = 1.0
    return g.reshape(num_views, 12, gz, gy, gx).contiguous()


def _check(image: torch.Tensor, grid: torch.Tensor):
    if image.dim() != 3 or image.shape[-1] != 3:
        raise ValueError(f"image must be (H, W, 3), got {tuple(image.shape)}")
    if grid.dim() != 4 or grid.shape[0] != 12:
        raise ValueError(f"grid must be (12, Gz, Gy, Gx), got {tuple(grid.shape)}")
    check_grid_shape((grid.shape[3], grid.shape[2], grid.shape[1]))
    if image.device != grid.device or image.dtype != grid.dtype:
        raise ValueError("image and grid must share device and dtype")


def _slice_torch(image: torch.Tensor, grid: torch.Tensor) -> torch.Tensor:
    """The grid_sample formulation (CPU path, and the tests' reference)."""
    H, W, _ = image.shape
    ys = torch.linspace(-1, 1, H, dtype=image.dtype, device=image.device)  # [-1] when H == 1
    xs = torch.linspace(-1, 1, W, dtype=image.dtype, device=image.device)
    yy, xx = torch.meshgrid(ys, xs, indexing="ij")
    lum = image @ torch.tensor(_LUMA, dtype=image.dtype, device=image.device)
    coords = torch.stack([xx, yy, lum * 2 - 1], -1)[None, None]  # (1, 1, H, W, 3): x, y, z
    coef = F.grid_sample(grid[None], coords, mode="bilinear", align_corners=True, padding_mode="border")[0, :, 0]
    A = coef.permute(1, 2, 0).reshape(H, W, 3, 4)
    return (A[..., :3] @ image[..., None])[..., 0] + A[..., 3]


def _ptr(t: torch.Tensor):
    return ctypes.c_void_p(t.data_ptr())


class _BilateralGridSlice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, grid):
        from . import _lib
        lib = _lib.load()
        image, grid = image.contiguous(), grid.contiguous()
        H, W = image.shape[:2]
        gz, gy, gx = grid.shape[1:]
        out = torch.empty_like(image)
        stream = torch.cuda.current_stream(image.device).cuda_stream
        with torch.cuda.device(image.device):
            _lib.check(lib.gsb200_bilateral_grid_forward(_ptr(image), _ptr(grid), H, W, gx, gy, gz, _ptr(out),
                                                         ctypes.c_void_p(stream)), "gsb200_bilateral_grid_forward")
        ctx.save_for_backward(image, grid)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from . import _lib
        lib = _lib.load()
        image, grid = ctx.saved_tensors
        H, W = image.shape[:2]
        gz, gy, gx = grid.shape[1:]
        grad_out = grad_out.contiguous()
        grad_image = torch.empty_like(image)
        grad_grid = torch.empty_like(grid)
        temp_bytes = int(lib.gsb200_bilateral_grid_temp_bytes(H, W, gx, gy, gz))
        temp = torch.empty((temp_bytes + 15) // 16 * 16, dtype=torch.uint8, device=image.device)
        stream = torch.cuda.current_stream(image.device).cuda_stream
        with torch.cuda.device(image.device):
            _lib.check(lib.gsb200_bilateral_grid_backward(_ptr(image), _ptr(grid), H, W, gx, gy, gz, _ptr(grad_out),
                                                          _ptr(grad_image), _ptr(grad_grid), _ptr(temp), temp_bytes,
                                                          ctypes.c_void_p(stream)), "gsb200_bilateral_grid_backward")
        return grad_image, grad_grid


def apply_bilateral_grid(image: torch.Tensor, grid: torch.Tensor) -> torch.Tensor:
    """The (H, W, 3) image sliced through the (12, Gz, Gy, Gx) grid, differentiable in both.  CUDA tensors (float32) run
    the library's kernels; CPU tensors (any float dtype) the ``grid_sample`` form."""
    _check(image, grid)
    if image.is_cuda:
        if image.dtype != torch.float32:
            raise ValueError("the CUDA slice takes float32 tensors")
        return _BilateralGridSlice.apply(image, grid)
    return _slice_torch(image, grid)


def bilateral_grid_tv(grid: torch.Tensor) -> torch.Tensor:
    """tv(G) = sum over the x, y and z axes of mean((G[i+1] - G[i])^2) of one (12, Gz, Gy, Gx) grid; an axis with one node
    contributes 0.  A 0-dim tensor."""
    total = torch.zeros((), dtype=grid.dtype, device=grid.device)
    for dim in (3, 2, 1):
        if grid.shape[dim] > 1:
            total = total + torch.diff(grid, dim=dim).pow(2).mean()
    return total
