"""The depth-map gradient (``differentiable_depth=True``, ``gsb200_backward_with_depth``) without a GPU.

The DEPTH instantiations of the transposed loop A and of the per-point kernel run under the SIMT emulator of
``tests/simt`` (the unmodified CUDA sources), chained with the emulated preprocess, sort, tile ranges and forward blend,
and are compared with torch autograd through the float64 dense evaluator (``dense_render`` with the depth map of
``torch_reference_depth``, differentiable in z as well).
Also: a zero depth gradient changes nothing, the gradient is linear in (image, depth) gradients, the C entry point's
argument rules, and the operator's constructor checks."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.utils import inverse_SE3_qt_torch

from helpers import grad_close
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth, emulated_points
from simt_helpers import build_emulator, emulated_forward
from torch_reference import dense_render, postprocess_feature_grads
from torch_reference_depth import differentiable_depth

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))


@pytest.fixture(scope="module")
def emu():
    return build_emulator()


@pytest.fixture(scope="module")
def demu():
    return build_depth_emulator()


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, sh_degree=3):
    """As in test_oracle_dense_crosscheck: dense coverage, points behind near, saturation and early stop, invalid slots."""
    sc = make_scene(n, h, w, sigma, seed, sh_degree=sh_degree, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    return sc


def _grads(seed, H, W, image_grad):
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g, dtype=torch.float32)
    g_dep = torch.randn((H, W), generator=g, dtype=torch.float32)
    return (g_img if image_grad else torch.zeros_like(g_img)), g_dep


def _dense_grads(sc, feats_n, g_img, g_dep, band):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    q_cp, t_cp = inverse_SE3_qt_torch(sc.q_pointcloud_camera, sc.t_pointcloud_camera)
    xyz = sc.point_cloud.clone().double().requires_grad_(True)
    feats = torch.from_numpy(feats_n).double().requires_grad_(True)
    image, aux = dense_render(xyz, feats, sc.point_invalid_mask, sc.camera_info.camera_intrinsics, q_cp, t_cp, H, W)
    depth, count = differentiable_depth(aux, H, W)
    assert torch.equal(count, aux["count"]) and torch.equal(depth.detach(), aux["depth"].detach())  # the same compositing
    ((image * g_img.double()).sum() + (depth * g_dep.double()).sum()).backward()
    return xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), aux


@pytest.mark.parametrize("image_grad", [False, True])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_emulated_depth_gradient_matches_dense_autograd(emu, demu, seed, band, exact, image_grad):
    sc = _scene(seed)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, g_dep = _grads(seed, H, W, image_grad)
    gx, gf, _, _ = emulated_backward_depth(emu, demu, st, g_img.numpy(), g_dep.numpy(), band)
    ex, ef, aux = _dense_grads(sc, st.pre.feats, g_img, g_dep, band)
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()  # multi-splat blending and saturated pixels
    assert np.abs(aux["depth"].detach().numpy() - st.depth).max() < 1e-3
    ok = grad_close(gx, ex)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], ok
    for sl in GROUPS:
        ok = grad_close(gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    # the depth term really moved xyz: without it the gradient is clearly different
    ex0, _, _ = _dense_grads(sc, st.pre.feats, g_img, torch.zeros_like(g_dep), band)
    assert not grad_close(ex0, ex)[0]


@pytest.mark.parametrize("stats", [True, False])
@pytest.mark.parametrize("exact", [True, False])
def test_zero_depth_gradient_matches_the_default_kernels(emu, demu, exact, stats):
    sc = _scene(21)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, _ = _grads(21, H, W, True)
    gx0, gf0, acc0, mag0 = emulated_backward_depth(emu, demu, st, g_img.numpy(), None, stats=stats)
    gx1, gf1, acc1, mag1 = emulated_backward_depth(emu, demu, st, g_img.numpy(), np.zeros((H, W), np.float32), stats=stats)
    assert (acc1[:, 11] == 0).all() and (acc0[:, 11] == 0).all()
    # per pixel the arithmetic is bit-identical: the per-pixel magnitude image is a sum over the pixel's own splats
    assert np.array_equal(mag1, mag0)
    # a row collects float atomics from several warps of a CTA.  The emulator switches warps at collectives only, and
    # the DEPTH kernel has one more shuffle per chunk, so the warps interleave differently and the adds of one row
    # land in another order (as between the STATS and lean instantiations, test_simt_blend_cpu): equal up to that
    assert (acc1[:, 10] == acc0[:, 10]).all()  # affected-pixel counts: exact in any order
    for cols in (slice(0, 2), slice(2, 5), slice(5, 8), slice(8, 9), slice(9, 10)):
        ok = grad_close(acc1[:, cols], acc0[:, cols], 1e-6, 1e-7)
        assert ok[0], (cols, ok)
    for a, b in ((gx1, gx0), (gf1, gf0)):
        ok = grad_close(a, b, 1e-6, 1e-7)
        assert ok[0], ok
    # the per-point DEPTH kernel on the same accumulator rows with word 11 = 0: bit-identical to the default one
    gx2, gf2 = emulated_points(emu, demu, st, acc0, depth=True)
    assert (gx2 == gx0).all() and (gf2 == gf0).all()


@pytest.mark.parametrize("exact", [True, False])
def test_gradient_is_linear_in_image_and_depth_gradients(emu, demu, exact):
    sc = _scene(31)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, g_dep = _grads(31, H, W, True)
    zero_img, zero_dep = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32)
    both = emulated_backward_depth(emu, demu, st, g_img.numpy(), g_dep.numpy())
    img = emulated_backward_depth(emu, demu, st, g_img.numpy(), zero_dep)
    dep = emulated_backward_depth(emu, demu, st, zero_img, g_dep.numpy())
    for k in (0, 1):
        total = both[k].astype(np.float64)
        parts = img[k].astype(np.float64) + dep[k].astype(np.float64)
        # float32 rounding of the recursions and of the per-pixel sums: a few ulp of the largest terms
        assert np.abs(total - parts).max() <= 2e-5 * np.abs(total).max(), np.abs(total - parts).max() / np.abs(total).max()
    assert np.abs(dep[0]).max() > 0 and np.abs(img[0]).max() > 0


def _args(flags):
    return _lib.GsbBackwardArgs(flags=flags)


def test_c_entry_point_checks_its_arguments_without_a_gpu():
    lib = _lib.load()
    assert hasattr(lib, "gsb200_backward_with_depth") and "gsb200_backward_with_depth" in _lib.EXPORTS
    fake = ctypes.c_void_p(256)  # never dereferenced: the checks come before any CUDA call
    T = _lib.GSB_FLAG_BACKWARD_TRANSPOSED
    for one in ((fake, None), (None, fake)):
        assert lib.gsb200_backward_with_depth(ctypes.byref(_args(T)), *one) == -1  # GSB_EINVAL
        assert b"both NULL or both set" in lib.gsb200_last_error()
    assert lib.gsb200_backward_with_depth(ctypes.byref(_args(0)), fake, fake) == -4  # GSB_EUNSUPPORTED
    assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    # both NULL: exactly gsb200_backward (here: its own null-pointer check)
    assert lib.gsb200_backward_with_depth(ctypes.byref(_args(T)), None, None) == lib.gsb200_backward(ctypes.byref(_args(T))) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()
    assert lib.gsb200_backward_with_depth(None, None, None) == -1


def test_operator_option_and_its_constructor_checks():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    param = inspect.signature(G.__init__).parameters["differentiable_depth"]
    assert param.kind is inspect.Parameter.KEYWORD_ONLY and param.default is False
    assert G(Config()).differentiable_depth is False
    assert G(Config(), differentiable_depth=True).differentiable_depth is True
    with pytest.raises(ValueError, match="transposed"):
        G(Config(), backward_impl="butterfly", differentiable_depth=True)
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_depth=True)
    G(Config(rgb_only=True))  # unchanged without the option
    G(Config(), backward_impl="butterfly")
