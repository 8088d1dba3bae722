"""The 3D smoothing filter's kernels under the SIMT emulator (``tests/simt/emu_filter3d.cpp``): the views kernels against the
loop reference of ``tests/mip_filter_reference.py`` -- margins, the near plane, points behind the camera, several objects
and focal lengths, unseen rows, no row seen, invalid rows, more entries than one shared-memory chunk -- and the FILTER
instantiation of the per-point forward against the unfiltered kernel on the baked rows."""
import ctypes

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo
from taichi_3d_gaussian_splatting_b200.mip_filter import _pose_matrices, bake_filter_3d, compute_filter_3d
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from mip_filter_reference import filter_reference, random_views
from simt_filter3d_helpers import build_filter3d_emulator, emulated_backward, emulated_filter
from simt_helpers import _bit_width, c


@pytest.fixture(scope="module")
def emu():
    return build_filter3d_emulator()


def _reference(xyz, mask, obj, views, near, variance):
    V, n_obj = len(views), views[0][0].shape[0]
    poses = _pose_matrices(torch.cat([v[0] for v in views]), torch.cat([v[1] for v in views])).view(V, n_obj, 3, 4).numpy()
    K = np.stack([v[2].camera_intrinsics.numpy() for v in views])
    return filter_reference(xyz, mask, obj, poses, K, [(v[2].camera_width, v[2].camera_height) for v in views], near, variance)


@pytest.mark.parametrize("V,n_obj", [(5, 1), (9, 3), (150, 1), (50, 3)])  # 150 and 3 x 50 entries: more than one chunk
def test_views_kernel_is_the_reference(emu, V, n_obj):
    g = torch.Generator().manual_seed(V + n_obj)
    N = 600
    xyz = (torch.rand((N, 3), generator=g) * torch.tensor([12.0, 8.0, 14.0]) - torch.tensor([6.0, 4.0, 3.0])).numpy()
    mask = (torch.rand(N, generator=g) < 0.1).to(torch.int8).numpy()
    obj = torch.randint(0, n_obj, (N,), generator=g, dtype=torch.int32).numpy()
    views = random_views(V, n_obj, g)
    got = emulated_filter(emu, xyz, mask, obj, views, 0.5, 0.2)
    ref = _reference(xyz, mask, obj, views, 0.5, 0.2)
    np.testing.assert_array_equal(got.view(np.int32), ref.view(np.int32))
    host_rule = compute_filter_3d(torch.from_numpy(xyz), torch.from_numpy(mask), torch.from_numpy(obj), views, 0.5, 0.2)
    np.testing.assert_array_equal(host_rule.numpy().view(np.int32), got.view(np.int32))


def test_views_kernel_edges(emu):
    W, H = 64, 48
    K = torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.5, 0.0], [0.0, 0.0, 1.0]])
    view = (torch.tensor([[0.0, 0.0, 0.0, 1.0]]), torch.zeros((1, 3)), CameraInfo(K, H, W, 0))
    lo_w, hi_w = np.float32(-0.15) * np.float32(W), np.float32(1.15) * np.float32(W)
    pts = np.array([(lo_w, 0, 1), (np.nextafter(lo_w, np.float32(-1e9)), 0, 1), (hi_w, 0, 1),
                    (np.nextafter(hi_w, np.float32(1e9)), 0, 1), (0, 0, 0.5), (0, 0, np.nextafter(np.float32(0.5), 1)),
                    (0, 0, -2), (1, 1, 4), (5, 5, 3)], np.float32)
    mask = np.array([0, 0, 0, 0, 0, 0, 0, 0, 1], np.int8)
    obj = np.zeros(len(pts), np.int32)
    got = emulated_filter(emu, pts, mask, obj, [view], 0.5, 0.2)
    ref = _reference(pts, mask, obj, [view], 0.5, 0.2)
    np.testing.assert_array_equal(got.view(np.int32), ref.view(np.int32))
    sv = np.sqrt(np.float32(0.2))
    assert got[0] == sv * np.float32(1) and got[1] == sv * np.float32(4) and got[8] == 0  # unseen: the largest seen d
    none_seen = emulated_filter(emu, pts[[1, 3, 4, 6]], mask[:4], obj[:4], [view], 0.5, 0.2)
    assert (none_seen == 0).all()
    # a view with a NaN K00 or K11 sees nothing; an object id outside [0, objects) matches no view
    K_nan = K.clone()
    K_nan[0, 0] = float("nan")
    K_both = K_nan.clone()
    K_both[1, 1] = float("nan")
    near_view = (view[0], view[1], CameraInfo(K_nan, H, W, 0))
    K_far = K.clone()
    K_far[0, 0] = K_far[1, 1] = 0.25  # sees (1, 1, 4) with d = 16
    views = [near_view, (view[0], view[1], CameraInfo(K_both, H, W, 0)), (view[0], view[1], CameraInfo(K_far, H, W, 0))]
    pts2 = np.array([(0, 0, 2), (1, 1, 4), (0, 0, 3)], np.float32)
    obj2 = np.array([0, 0, 5], np.int32)
    got = emulated_filter(emu, pts2, np.zeros(3, np.int8), obj2, views, 0.5, 0.2)
    ref = _reference(pts2, np.zeros(3, np.int8), obj2, views, 0.5, 0.2)
    np.testing.assert_array_equal(got.view(np.int32), ref.view(np.int32))
    host = compute_filter_3d(torch.from_numpy(pts2), torch.zeros(3, dtype=torch.int8), torch.from_numpy(obj2), views, 0.5, 0.2)
    np.testing.assert_array_equal(host.numpy().view(np.int32), got.view(np.int32))
    # a NaN K00 makes u NaN, so that view sees nothing although fmaxf(K00, K11) = 0.5 > 0; row 2 has no object and gets the
    # largest seen d
    assert got[0] == sv * np.float32(8) and got[1] == sv * np.float32(16) and got[2] == sv * np.float32(16)


def _preprocess(emu, sc, features, filter3d):
    xyz = sc.point_cloud.numpy().astype(np.float32).copy()
    feats = features.numpy().astype(np.float32).copy()
    N = xyz.shape[0]
    ci = sc.camera_info
    H, W = ci.camera_height, ci.camera_width
    depth_bits = max(_bit_width(int(np.float32(1000.0) * np.float32(100.0))), 1)
    cap = 64 * N + 4096
    counters = np.zeros(8, np.int64)
    point_id, point_offset, num_tiles = (np.full(N, -9, np.int32) for _ in range(3))
    records, pic = np.zeros((N, 12), np.float32), np.zeros((N, 3), np.float32)
    keys, vals = np.zeros(cap, np.uint32), np.zeros(cap, np.int32)
    q, t = sc.q_pointcloud_camera.numpy().copy(), sc.t_pointcloud_camera.numpy().copy()
    K = ci.camera_intrinsics.numpy().copy()
    inv, obj = sc.point_invalid_mask.numpy().copy(), sc.point_object_id.numpy().copy()
    f3 = None if filter3d is None else np.ascontiguousarray(filter3d.numpy(), np.float32)
    sw = emu.emu_preprocess_filter(
        ctypes.c_longlong(N), c(xyz), c(feats), c(inv), c(obj), q.shape[0], c(q), c(t), c(K), W, H, ctypes.c_float(0.8),
        ctypes.c_float(1000.0), ctypes.c_float(100.0), depth_bits, ctypes.c_longlong(cap), c(counters), c(point_id),
        c(point_offset), c(num_tiles), c(records), c(pic), c(keys), c(vals), c(f3) if f3 is not None else None)
    assert sw > 0
    M = int(counters[0])
    return records[:M], point_id[:M], num_tiles[:M], counters


def test_filtered_preprocess_is_the_unfiltered_one_on_baked_rows(emu):
    sc = make_scene(700, 64, 96, 0.05, 12)
    sc.point_invalid_mask[::11] = 1
    g = torch.Generator().manual_seed(1)
    sigma = torch.rand(700, generator=g) * 0.03
    sigma[::4] = 0.0
    sigma[5] = float("nan")
    sigma[6] = -1.0
    rf, idf, ntf, cf = _preprocess(emu, sc, sc.point_cloud_features, sigma)
    rb, idb, ntb, cb = _preprocess(emu, sc, bake_filter_3d(sc.point_cloud_features, sigma), None)
    np.testing.assert_array_equal(idf, idb)
    np.testing.assert_array_equal(ntf, ntb)
    # record = u v a b | c rescale*c_comp o depth | r g b radius; the opacity slot keeps the raw o, the rescale slot carries
    # the compensation, so their product is the baked row's rescale * o^
    raw_o = 1 / (1 + np.exp(-sc.point_cloud_features.numpy()[idf, 7].astype(np.float64)))
    np.testing.assert_allclose(rf[:, 6], raw_o, rtol=1e-6)
    np.testing.assert_allclose(rf[:, 5] * rf[:, 6], rb[:, 5] * rb[:, 6], rtol=2e-5, atol=1e-7)
    for col in (0, 1, 2, 3, 4, 7, 8, 9, 10, 11):
        np.testing.assert_allclose(rf[:, col], rb[:, col], rtol=2e-5, atol=1e-6 * np.abs(rb[:, col]).max(), err_msg=str(col))
    # sigma = 0 everywhere: exactly the unfiltered kernel
    r0, id0, nt0, c0 = _preprocess(emu, sc, sc.point_cloud_features, torch.zeros(700))
    ru, idu, ntu, cu = _preprocess(emu, sc, sc.point_cloud_features, None)
    np.testing.assert_array_equal(r0.view(np.int32), ru.view(np.int32))
    np.testing.assert_array_equal(nt0, ntu)
    np.testing.assert_array_equal(c0[:3], cu[:3])


# ---- the FILTER per-point backward, on constructed frame state: the chain rule of the filter against the unfiltered kernel on
# the baked rows composed with torch autograd through the bake (float64)
def _frame_state(N=300, seed=0):
    from types import SimpleNamespace
    from taichi_3d_gaussian_splatting_b200.synthetic import make_scene as ms
    sc = ms(N, 48, 64, 0.08, seed, yaw_degrees=3.0)
    g = torch.Generator().manual_seed(seed)
    xyz = sc.point_cloud.numpy().astype(np.float32)
    T = _pose_matrices(sc.q_pointcloud_camera, sc.t_pointcloud_camera).numpy()[0]
    poses = np.zeros((1, 20), np.float32)
    poses[0, :12] = T.reshape(-1)
    pic = (((T[:, 0] * xyz[:, :1] + T[:, 1] * xyz[:, 1:2]) + T[:, 2] * xyz[:, 2:3]) + T[:, 3]).astype(np.float32)
    offset = np.where((pic[:, 2] > 0.5) & (np.arange(N) % 13 != 5), np.arange(N), -1).astype(np.int32)
    feats = sc.point_cloud_features.clone()
    feats[:, 4:7] -= 1.0
    feats[3, 7] = 30.0  # o = 1.0f: fl(1 - o) = 0
    accum = (torch.randn((N, 12), generator=g) * 0.05).numpy().astype(np.float32)
    colours = (torch.rand((N, 3), generator=g) * 0.8 + 0.1).numpy().astype(np.float32)
    g_alpha = (torch.randn(N, generator=g) * 0.1).numpy().astype(np.float32)
    sigma = (torch.rand(N, generator=g) * 0.05).numpy().astype(np.float32)
    sigma[::7] = 0.0
    sigma[5], sigma[6] = np.nan, -1.0
    row_time = ((torch.rand(N, generator=g) - 0.5)).numpy().astype(np.float32)
    return SimpleNamespace(xyz=xyz, poses=poses, pic=np.ascontiguousarray(pic), point_offset=offset, feats=feats, accum=accum,
                           colours=colours, g_alpha=g_alpha, sigma=sigma, obj=np.zeros(N, np.int32),
                           t_pc=sc.t_pointcloud_camera.numpy().astype(np.float32), K=sc.camera_info.camera_intrinsics.numpy(),
                           row_time=row_time, motion=np.array([0.05, -0.08, 0.03, 0.04, -0.06, 0.05], np.float32))


def _records_and_accum(st, features):
    """Records whose opacity slot is the rows' float32 sigmoid, and accumulator rows whose glogit is G_a (1 - o)."""
    N = features.shape[0]
    o = (1.0 / (1.0 + np.exp(-features[:, 7].numpy().astype(np.float64)))).astype(np.float32)
    rec = np.zeros((N, 12), np.float32)
    rec[:, 6] = o
    rec[:, 8:11] = st.colours
    acc = st.accum.copy()
    acc[:, 8] = st.g_alpha * (np.float32(1) - o)
    return rec, acc


@pytest.mark.parametrize("rolling", [False, True])
@pytest.mark.parametrize("depth", [False, True])
def test_filtered_backward_is_the_chain_rule_through_the_bake(emu, rolling, depth):
    from mip_filter_reference import bake_torch
    st = _frame_state()
    sigma = torch.from_numpy(st.sigma)
    rec, acc = _records_and_accum(st, st.feats)
    gx, gf = emulated_backward(emu, st, st.feats.numpy(), rec, acc, st.sigma, depth, rolling)
    baked = bake_torch(st.feats.double(), sigma.double()).float()
    rec_b, acc_b = _records_and_accum(st, baked)
    gx_b, gf_b = emulated_backward(emu, st, baked.numpy(), rec_b, acc_b, None, depth, rolling)
    np.testing.assert_array_equal(gx, gx_b)  # the position gradient does not see the scales or the opacity
    f64 = st.feats.double().requires_grad_(True)
    (expected,) = torch.autograd.grad(bake_torch(f64, sigma.double()), f64, torch.from_numpy(gf_b).double())
    expected = expected.numpy()
    # the saturated row: fl(1 - o) = 0, so the kernel drops its compensation term G_a sigma^2 / e^ (and its logit gradient is 0)
    s3 = float(st.sigma[3])
    e = np.exp(st.feats[3, 4:7].numpy().astype(np.float64)) ** 2
    c3 = np.sqrt(np.prod(e / (e + s3 * s3)))
    expected[3, 4:7] -= float(st.g_alpha[3]) * s3 * s3 / (e + s3 * s3)
    assert c3 < 1 and st.point_offset[3] >= 0 and np.isfinite(gf[3]).all() and gf[3, 7] == 0.0
    live = st.point_offset >= 0
    for cols in (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56)):
        scale = np.abs(expected[live, cols]).max()
        np.testing.assert_allclose(gf[live, cols], expected[live, cols], rtol=0, atol=2e-5 * scale, err_msg=str(cols))
    np.testing.assert_allclose(gf[3, 4:7], expected[3, 4:7], rtol=1e-4, atol=1e-6 * np.abs(expected[:, 4:7]).max())
    assert (gf[~live] == 0).all()


@pytest.mark.parametrize("rolling", [False, True])
def test_filtered_backward_with_zero_sigma_is_the_unfiltered_kernel(emu, rolling):
    st = _frame_state(seed=2)
    rec, acc = _records_and_accum(st, st.feats)
    sigma = np.zeros_like(st.sigma)
    sigma[5], sigma[6] = np.nan, -1.0  # read as 0
    a = emulated_backward(emu, st, st.feats.numpy(), rec, acc, sigma, True, rolling)
    b = emulated_backward(emu, st, st.feats.numpy(), rec, acc, None, True, rolling)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x.view(np.int32), y.view(np.int32))
