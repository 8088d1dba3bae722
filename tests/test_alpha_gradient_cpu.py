"""The accumulated-alpha gradient (``differentiable_alpha=True``, ``gsb200_backward_aux``) without a GPU.

The ALPHA and ALPHA + DEPTH instantiations of the transposed loop A run under the SIMT emulator of ``tests/simt`` (the
unmodified CUDA sources), chained with the emulated preprocess, sort, tile ranges and forward blend and with the emulated
per-point kernel, and are compared with torch autograd through the float64 dense evaluator (``dense_render``'s
``acc_alpha = 1 - T``, and the depth map of ``torch_reference_depth`` for the combined loss).
Also: a zero alpha gradient changes nothing, the gradient is linear in (image, depth, alpha) gradients, the C entry
point's argument rules, and the operator's constructor checks."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.utils import inverse_SE3_qt_torch

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_helpers import build_emulator, emulated_forward
from torch_reference import dense_render, postprocess_feature_grads
from torch_reference_depth import differentiable_depth

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LOSSES = ("alpha", "alpha+image", "alpha+image+depth")


@pytest.fixture(scope="module")
def emu():
    return build_emulator()


@pytest.fixture(scope="module")
def demu():
    return build_depth_emulator()


@pytest.fixture(scope="module")
def aemu():
    return build_alpha_emulator()


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, sh_degree=3):
    """As in test_oracle_dense_crosscheck: dense coverage, points behind near, saturation and early stop, invalid slots."""
    sc = make_scene(n, h, w, sigma, seed, sh_degree=sh_degree, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    return sc


def _grads(seed, H, W, loss):
    """(dL/dimage, dL/ddepth or None, dL/dalpha) for one of LOSSES; the image gradient is zero for an alpha-only loss."""
    g = torch.Generator().manual_seed(seed + 200)
    g_img = torch.randn((H, W, 3), generator=g, dtype=torch.float32)
    g_dep = torch.randn((H, W), generator=g, dtype=torch.float32)
    g_alp = torch.randn((H, W), generator=g, dtype=torch.float32)
    return (g_img if "image" in loss else torch.zeros_like(g_img)), (g_dep if "depth" in loss else None), g_alp


def _dense_grads(sc, feats_n, g_img, g_dep, g_alp, band):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    q_cp, t_cp = inverse_SE3_qt_torch(sc.q_pointcloud_camera, sc.t_pointcloud_camera)
    xyz = sc.point_cloud.clone().double().requires_grad_(True)
    feats = torch.from_numpy(feats_n).double().requires_grad_(True)
    image, aux = dense_render(xyz, feats, sc.point_invalid_mask, sc.camera_info.camera_intrinsics, q_cp, t_cp, H, W)
    loss = (image * g_img.double()).sum() + (aux["acc_alpha"] * g_alp.double()).sum()
    if g_dep is not None:
        depth, _ = differentiable_depth(aux, H, W)
        loss = loss + (depth * g_dep.double()).sum()
    loss.backward()
    return xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), aux


@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("seed,band", [(11, 3), (12, 1), (13, 0)])
def test_emulated_alpha_gradient_matches_dense_autograd(emu, demu, aemu, seed, band, exact, loss):
    sc = _scene(seed)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, g_dep, g_alp = _grads(seed, H, W, loss)
    gx, gf, _, _ = emulated_backward_alpha(emu, demu, aemu, st, g_img.numpy(), g_alp.numpy(),
                                           None if g_dep is None else g_dep.numpy(), band)
    ex, ef, aux = _dense_grads(sc, st.pre.feats, g_img, g_dep, g_alp, band)
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()  # multi-splat blending and saturated pixels
    assert np.abs(aux["acc_alpha"].detach().numpy() - st.acc_alpha).max() < 1e-4
    ok = grad_close(gx, ex)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], ok
    for sl in GROUPS:
        ok = grad_close(gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    # the alpha term really moved xyz: without it the gradient is clearly different (or zero, for an alpha-only loss)
    ex0, _, _ = _dense_grads(sc, st.pre.feats, g_img, g_dep, torch.zeros_like(g_alp), band)
    assert not grad_close(ex0, ex)[0]


@pytest.mark.parametrize("stats", [True, False])
@pytest.mark.parametrize("exact", [True, False])
def test_zero_alpha_gradient_matches_the_default_kernels(emu, demu, aemu, exact, stats):
    sc = _scene(21)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, _, _ = _grads(21, H, W, "alpha+image")
    gx0, gf0, acc0, mag0 = emulated_backward_depth(emu, demu, st, g_img.numpy(), None, stats=stats)
    gx1, gf1, acc1, mag1 = emulated_backward_alpha(emu, demu, aemu, st, g_img.numpy(), np.zeros((H, W), np.float32),
                                                   stats=stats)
    assert (acc1[:, 11] == 0).all()
    # per pixel the arithmetic is bit-identical: the per-pixel magnitude image is a sum over the pixel's own splats
    assert np.array_equal(mag1, mag0)
    # a row collects float atomics from several warps of a CTA, in an order the emulator's warp interleaving decides:
    # equal up to that order
    assert (acc1[:, 10] == acc0[:, 10]).all()  # affected-pixel counts: exact in any order
    for cols in (slice(0, 2), slice(2, 5), slice(5, 8), slice(8, 9), slice(9, 10)):
        ok = grad_close(acc1[:, cols], acc0[:, cols], 1e-6, 1e-7)
        assert ok[0], (cols, ok)
    for a, b in ((gx1, gx0), (gf1, gf0)):
        ok = grad_close(a, b, 1e-6, 1e-7)
        assert ok[0], ok


@pytest.mark.parametrize("exact", [True, False])
def test_gradient_is_linear_in_image_depth_and_alpha_gradients(emu, demu, aemu, exact):
    sc = _scene(31)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    g_img, g_dep, g_alp = (t.numpy() for t in _grads(31, H, W, "alpha+image+depth"))
    z3, z = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32)
    total = emulated_backward_alpha(emu, demu, aemu, st, g_img, g_alp, g_dep)
    parts = [emulated_backward_alpha(emu, demu, aemu, st, g_img, z, z),
             emulated_backward_alpha(emu, demu, aemu, st, z3, z, g_dep),
             emulated_backward_alpha(emu, demu, aemu, st, z3, g_alp, z)]
    for k in (0, 1):
        t = total[k].astype(np.float64)
        s = sum(p[k].astype(np.float64) for p in parts)
        # float32 rounding of the recursions and of the per-pixel sums: a few ulp of the largest terms
        assert np.abs(t - s).max() <= 2e-5 * np.abs(t).max(), np.abs(t - s).max() / np.abs(t).max()
    assert all(np.abs(p[0]).max() > 0 for p in parts)


def _args(flags):
    return _lib.GsbBackwardArgs(flags=flags)


def test_c_entry_point_checks_its_arguments_without_a_gpu():
    lib = _lib.load()
    assert "gsb200_backward_aux" in _lib.EXPORTS and lib.gsb200_backward_aux.argtypes is not None
    fake = ctypes.c_void_p(256)  # never dereferenced: the checks come before any CUDA call
    T = _lib.GSB_FLAG_BACKWARD_TRANSPOSED
    for alpha in (None, fake):
        for one in ((fake, None), (None, fake)):
            assert lib.gsb200_backward_aux(ctypes.byref(_args(T)), *one, alpha) == -1  # GSB_EINVAL
            assert b"both NULL or both set" in lib.gsb200_last_error()
    for terms in ((None, None, fake), (fake, fake, None), (fake, fake, fake)):
        assert lib.gsb200_backward_aux(ctypes.byref(_args(0)), *terms) == -4  # GSB_EUNSUPPORTED
        assert b"GSB_FLAG_BACKWARD_TRANSPOSED" in lib.gsb200_last_error()
    # a valid set of terms reaches gsb200_backward's own checks (here: its null-pointer check)
    for terms in ((None, None, fake), (fake, fake, fake)):
        assert lib.gsb200_backward_aux(ctypes.byref(_args(T)), *terms) == -1
        assert b"backward: null pointer argument" in lib.gsb200_last_error()
    # all three NULL: exactly gsb200_backward, with or without the transposed flag
    for flags in (0, T):
        assert lib.gsb200_backward_aux(ctypes.byref(_args(flags)), None, None, None) == \
            lib.gsb200_backward(ctypes.byref(_args(flags))) == -1
        assert b"backward: null pointer argument" in lib.gsb200_last_error()
    assert lib.gsb200_backward_aux(None, None, None, fake) == -1
    assert b"args is null" in lib.gsb200_last_error()


def test_operator_option_and_its_constructor_checks():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    param = inspect.signature(G.__init__).parameters["differentiable_alpha"]
    assert param.kind is inspect.Parameter.KEYWORD_ONLY and param.default is False
    assert G(Config()).differentiable_alpha is False
    op = G(Config(), differentiable_alpha=True, differentiable_depth=True)
    assert op.differentiable_alpha is True and op.differentiable_depth is True
    for depth in (False, True):
        with pytest.raises(ValueError, match="transposed"):
            G(Config(), backward_impl="butterfly", differentiable_alpha=True, differentiable_depth=depth)
        with pytest.raises(ValueError, match="rgb_only"):
            G(Config(rgb_only=True), differentiable_alpha=True, differentiable_depth=depth)
    G(Config(rgb_only=True))  # unchanged without the option
    G(Config(), backward_impl="butterfly")
