"""Large splats (17..96 tiles each) through the CUDA operator vs the oracle -- the more-than-64-tiles branch of the
cooperative reach filter and ~1000-entry tile lists.  Kept in its own module, after the other GPU parity modules."""
import numpy as np
import pytest
import torch

from gpu_helpers import count_above, cuda_scene, make_op, n, run_forward
from helpers import grad_close, oracle_backward, oracle_forward
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from test_gpu_parity import _check_stages

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("keep_all", [False, True])
@pytest.mark.parametrize("sigma", [0.3, 0.6])
def test_large_splats_vs_oracle(sigma, keep_all):
    """Splats whose 3-sigma square spans 17..96 tiles of a 12 x 8 tile image (several hundred of them cover more
    than 64 tiles): the cooperative reach filter tests only the first 64 tiles of a splat and keeps the rest, and
    the per-tile lists run to ~1000 entries before the pixels saturate."""
    scene = make_scene(1500, 128, 192, sigma, 31, sh_degree=3, yaw_degrees=4.0)
    scene.point_cloud_features[:, 7] -= 2.0  # low opacity: long lists before saturation
    o, fwd, feats_n = oracle_forward(scene)
    assert int((fwd.num_overlap_tiles > 64).sum()) >= 20 and int(fwd.num_overlap_tiles.max()) == 96
    sc = cuda_scene(scene, requires_grad=True)
    op = make_op(exact_exp=True, keep_all_tile_pairs=keep_all)
    image, depth, count = run_forward(op, sc, band=3)
    _check_stages(op.last_frame, fwd)
    # up to 1.7e7 (pixel, splat) evaluations: allow the odd pair that sits within an ulp of the alpha = 1/255 cut-off
    # to fall on the other side of it (CUDA expf vs libm expf), as in the full-size test
    d = np.abs(n(image) - fwd.image)
    assert (d > 1e-4).sum() <= 3 and d.max() <= 5e-3
    assert count_above(n(count), fwd.pixel_valid_point_count, 0) <= 3
    g = torch.Generator().manual_seed(9)
    grad_image = torch.randn(image.shape, generator=g, dtype=torch.float32)
    image.backward(grad_image.cuda())
    bwd = oracle_backward(o, fwd, scene, feats_n, grad_image.numpy(), 3)
    gx, gf = n(sc.point_cloud.grad), n(sc.point_cloud_features.grad)
    # lists are ~10x deeper than in the small scenes: f32 accumulation over up to ~150 blended splats per pixel, so a
    # few entries in a thousand may leave the per-entry tolerance; none may be off by more than 1e-3 of the largest
    for got, exp in ((gx, bwd.grad_pointcloud), (gf[:, :4], bwd.grad_pointcloud_features[:, :4]),
                     (gf[:, 4:7], bwd.grad_pointcloud_features[:, 4:7]), (gf[:, 7:8], bwd.grad_pointcloud_features[:, 7:8]),
                     (gf[:, 8:], bwd.grad_pointcloud_features[:, 8:])):
        ok, worst, nviol = grad_close(got, exp)
        assert nviol <= 2e-3 * exp.size, (worst, nviol, exp.size)
        assert np.abs(got - exp).max() <= 1e-3 * np.abs(exp).max()
