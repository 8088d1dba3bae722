"""Per-Gaussian feature channels (``point_extra_features``, ``gsb200_forward_ext`` / ``gsb200_backward_ext``) without a GPU.

The CF instantiations of the forward blend and of the transposed loop A run under the SIMT emulator of ``tests/simt`` (the
unmodified CUDA sources), on the emulated preprocess, sort and tile ranges and followed by the emulated per-point kernel.
They are compared with torch autograd through the float64 dense evaluator (``torch_reference_features``; the depth map of
``torch_reference_depth`` and ``dense_render``'s accumulated alpha for the combined loss), for C = 1, 3, 4, 5, 8 and 16 --
every compile-time width and its padding -- on both arithmetic paths.  Also: the other forward outputs do not move, a zero
feature gradient changes nothing, and features equal to the splats' colours reproduce the image and its colour sums."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from taichi_3d_gaussian_splatting_b200.utils import inverse_SE3_qt_torch

from helpers import grad_close
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features, emulated_forward_features
from simt_helpers import build_emulator, emulated_forward
from torch_reference import dense_render, postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LOSSES = ("features", "features+image", "features+image+depth+alpha")


@pytest.fixture(scope="module")
def emu():
    return build_emulator()


@pytest.fixture(scope="module")
def demu():
    return build_depth_emulator()


@pytest.fixture(scope="module")
def femu():
    return build_feature_emulator()


def _scene(seed, n=400, h=32, w=48, sigma=0.12, yaw=4.0, sh_degree=3):
    """As in test_oracle_dense_crosscheck: dense coverage, points behind near, saturation and early stop, invalid slots."""
    sc = make_scene(n, h, w, sigma, seed, sh_degree=sh_degree, yaw_degrees=yaw)
    sc.point_cloud[:, 2] = sc.point_cloud[:, 2] * 0.5
    sc.point_cloud_features[:, 7] += 1.5
    sc.point_invalid_mask[::7] = 1
    return sc


def _features(seed, N, C):
    """Normal draws: unbounded, signed, not limited to [0, 1]."""
    return torch.randn((N, C), generator=torch.Generator().manual_seed(seed + 300), dtype=torch.float32)


def _grads(seed, H, W, C, loss):
    g = torch.Generator().manual_seed(seed + 200)
    g_img, g_dep, g_alp = (torch.randn(s, generator=g) for s in ((H, W, 3), (H, W), (H, W)))
    g_feat = torch.randn((H, W, C), generator=g)
    return (g_feat, g_img if "image" in loss else torch.zeros_like(g_img), g_dep if "depth" in loss else None,
            g_alp if "alpha" in loss else None)


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("C", [1, 3, 4, 5, 8, 16])
def test_emulated_features_match_dense_autograd(emu, demu, femu, C, exact):
    seed = 11 + C
    sc = _scene(seed)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    N = sc.point_cloud.shape[0]
    st = emulated_forward(emu, sc, exact=exact)
    F = _features(seed, N, C)
    image, depth, acc, last, cnt, fmap = emulated_forward_features(femu, st, F.numpy())
    # the frame's other outputs are those of the feature-off forward, bit for bit
    for a, b in ((image, st.image), (depth, st.depth), (acc, st.acc_alpha), (last, st.last_effective), (cnt, st.count)):
        assert np.array_equal(a, b)
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()  # multi-splat blending and saturated pixels

    q_cp, t_cp = inverse_SE3_qt_torch(sc.q_pointcloud_camera, sc.t_pointcloud_camera)
    xyz = sc.point_cloud.clone().double().requires_grad_(True)
    feats = torch.from_numpy(st.pre.feats).double().requires_grad_(True)
    Fd = F.double().requires_grad_(True)
    ref_image, aux = dense_render(xyz, feats, sc.point_invalid_mask, sc.camera_info.camera_intrinsics, q_cp, t_cp, H, W)
    ref_fmap = feature_map(aux, Fd, H, W)
    ref_depth, _ = differentiable_depth(aux, H, W)
    # the feature map within the image's bounds, relative to the largest feature value
    tol = (2e-6 if exact else 1e-4) * float(F.abs().max())
    assert np.abs(fmap - ref_fmap.detach().numpy()).max() <= tol, np.abs(fmap - ref_fmap.detach().numpy()).max() / tol

    for k, loss_name in enumerate(LOSSES):
        stats = k % 2 == 0  # with and without the hook statistics
        g_feat, g_img, g_dep, g_alp = _grads(seed, H, W, C, loss_name)
        gx, gf, gF, _, _ = emulated_backward_features(
            emu, demu, femu, st, F.numpy(), g_feat.numpy(), g_img.numpy(), None if g_dep is None else g_dep.numpy(),
            None if g_alp is None else g_alp.numpy(), band=3, stats=stats)
        loss = (ref_fmap * g_feat.double()).sum() + (ref_image * g_img.double()).sum()
        if g_dep is not None:
            loss = loss + (ref_depth * g_dep.double()).sum() + (aux["acc_alpha"] * g_alp.double()).sum()
        ex, ef, eF = torch.autograd.grad(loss, (xyz, feats, Fd), retain_graph=True)
        ef = postprocess_feature_grads(ef, 3)
        ok = grad_close(gF, eF.numpy())
        assert ok[0], (loss_name, "dL/dF", ok)
        ok = grad_close(gx, ex.numpy())
        assert ok[0], (loss_name, "xyz", ok)
        for sl in GROUPS:
            ok = grad_close(gf[:, sl], ef[:, sl].numpy())
            assert ok[0], (loss_name, sl, ok)
        # rows of points outside the frustum (and invalid slots) get exactly zero
        outside = np.ones(N, bool)
        outside[st.pre.point_id[:st.M]] = False
        assert (gF[outside] == 0).all()


@pytest.mark.parametrize("stats", [True, False])
@pytest.mark.parametrize("exact", [True, False])
def test_zero_feature_gradient_changes_nothing(emu, demu, femu, exact, stats):
    sc = _scene(21)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward(emu, sc, exact=exact)
    F = _features(21, sc.point_cloud.shape[0], 5)
    _, g_img, _, _ = _grads(21, H, W, 5, "features+image")
    gx0, gf0, acc0, mag0 = emulated_backward_depth(emu, demu, st, g_img.numpy(), None, stats=stats)
    gx1, gf1, gF, acc1, mag1 = emulated_backward_features(emu, demu, femu, st, F.numpy(), np.zeros((H, W, 5), np.float32),
                                                          g_img.numpy(), stats=stats)
    assert (gF == 0).all()
    # per pixel the arithmetic is bit-identical: the magnitude image is a sum over the pixel's own splats
    assert (mag1 == mag0).all()
    # a row collects float atomics from several warps of a CTA, in an order the emulator's warp interleaving decides (the
    # feature kernel's extra shuffles move it): equal up to that order
    assert (acc1[:, 10] == acc0[:, 10]).all()  # affected-pixel counts: exact in any order
    for cols in (slice(0, 2), slice(2, 5), slice(5, 8), slice(8, 9), slice(9, 10)):
        ok = grad_close(acc1[:, cols], acc0[:, cols], 1e-6, 1e-7)
        assert ok[0], (cols, ok)
    for a, b in ((gx1, gx0), (gf1, gf0)):
        ok = grad_close(a, b, 1e-6, 1e-7)
        assert ok[0], ok


def test_colour_features_reproduce_the_image_and_its_colour_sums(emu, demu, femu):
    """Features set to every splat's rendered colour (records to scene rows): on the fast path the feature map IS the image
    (same weights, same FMAs, same order), and dL/dF equals the accumulator's per-splat sums alpha T g (columns 5-7, before
    the colour factor) for a feature-map gradient equal to the image gradient."""
    sc = _scene(31)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    N = sc.point_cloud.shape[0]
    st = emulated_forward(emu, sc, exact=False)
    ids = st.pre.point_id[:st.M]
    F = _features(31, N, 3).numpy()  # rows outside the frustum never contribute
    F[ids] = st.pre.records[:st.M, 8:11]
    *_, fmap = emulated_forward_features(femu, st, F)
    assert np.array_equal(fmap, st.image)
    g = _grads(31, H, W, 3, "features+image")[1].numpy()
    _, _, gF, acc, _ = emulated_backward_features(emu, demu, femu, st, F, g, g)
    ok = grad_close(gF[ids], acc[:, 5:8], 1e-6, 1e-7)
    assert ok[0], ok
    assert np.abs(acc[:, 5:8]).max() > 0
