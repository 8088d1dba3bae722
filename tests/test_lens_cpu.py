"""Lens distortion (``CameraInfo.distortion``, ``gsb200_forward_lens`` / ``gsb200_backward_lens``) without a GPU.

* Known answers of OpenCV (``golden/lens_vectors.json``, written by ``golden/make_lens_golden.py`` with cv2): the float64
  reference ``torch_reference_lens`` and its autograd Jacobian, the float32 device helper and the records of the emulated
  lens per-point kernel.
* The validity bound r_max (host, double) against numpy's polynomial roots, and points just inside / outside it.
* The emulated lens forward (the unmodified CUDA sources under the SIMT emulator of ``tests/simt``) against the dense float64
  evaluator, and with zero coefficients against the pinhole path.
* The emulated LENS per-point kernel on emulated loop-A rows against torch autograd of the evaluator, for image, depth,
  alpha and feature-map losses, under both loop-A kernels; determinism.
* The C entry points' argument rules, the ABI size, ``LensDistortion`` / ``from_colmap``, and the operator's, dataset's and
  trainer's configuration."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator, emulated_forward
from simt_lens_helpers import (build_lens_emulator, emulated_forward_lens, emulated_points_lens, lens_distort, r2_bound,
                               run_preprocess_lens)
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference import postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_lens import dense_render_lens, project
from torch_reference_lens import r2_bound as r2_bound_ref

HERE = os.path.dirname(os.path.abspath(__file__))
GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator())


def _golden():
    with open(os.path.join(HERE, "golden", "lens_vectors.json")) as f:
        return json.load(f)


# ------------------------------------------------------------------ known answers of OpenCV
def test_golden_vectors_cover_the_listed_cases():
    d = _golden()
    assert d["cv2_version"]
    names = {c["name"] for c in d["cases"]}
    assert {"simple_radial_k1", "radial_k1_k2", "opencv_full", "strong_barrel", "fisheye"} <= names
    for c in d["cases"]:
        pts = np.array(c["points"])
        assert (pts[0, :2] == 0).all() and np.hypot(*(pts[1, :2] / pts[1, 2])) < 1e-6  # on and next to the axis


@pytest.mark.parametrize("case", range(6))
def test_float64_reference_matches_opencv(case):
    c = _golden()["cases"][case]
    K = torch.tensor(c["K"], dtype=torch.float64)
    pts = torch.tensor(c["points"], dtype=torch.float64)
    uv = project(pts, K, c["model"], c["coefficients"])
    assert np.abs(uv.numpy() - np.array(c["uv"])).max() <= 1e-9
    jac = torch.stack([torch.autograd.functional.jacobian(
        lambda p: project(p[None], K, c["model"], c["coefficients"])[0], p) for p in pts])
    assert np.abs(jac.numpy() - np.array(c["duv_dpc"])).max() <= 1e-7


@pytest.mark.parametrize("case", range(6))
def test_device_helper_and_emulated_records_match_opencv(emus, case):
    c = _golden()["cases"][case]
    K = np.array(c["K"], np.float32)
    pts = np.array(c["points"], np.float64)
    want = np.array(c["uv"])
    # the float32 helper itself
    xn32, yn32 = (pts[:, 0] / pts[:, 2]).astype(np.float32), (pts[:, 1] / pts[:, 2]).astype(np.float32)
    ox, oy, D = lens_distort(emus["lemu"], c["model"], c["coefficients"], xn32, yn32)
    xd, yd = xn32 + ox, yn32 + oy
    u = K[0, 0] * xd + K[0, 1] * yd + K[0, 2]
    v = K[1, 0] * xd + K[1, 1] * yd + K[1, 2]
    assert np.abs(np.stack([u, v], -1) - want).max() <= 1e-3
    # D P K: the helper's Jacobian against OpenCV's (relative, float32)
    z = pts[:, 2]
    xn, yn = pts[:, 0] / z, pts[:, 1] / z
    P = np.zeros((len(z), 2, 3))
    P[:, 0, 0] = P[:, 1, 1] = 1 / z
    P[:, 0, 2], P[:, 1, 2] = -xn / z, -yn / z
    duv = K[:2, :2].astype(np.float64) @ D.astype(np.float64) @ P
    ok = grad_close(duv, np.array(c["duv_dpc"]), rtol=1e-4)
    assert ok[0], ok
    # the per-point kernel: points given in the camera frame (identity pose), records in point_offset order
    sc = make_scene(len(pts), 480, 640, 0.05, 1)
    sc.point_cloud = torch.from_numpy(pts.astype(np.float32)).contiguous()
    sc.q_pointcloud_camera = torch.tensor([[0.0, 0.0, 0.0, 1.0]])
    sc.camera_info = CameraInfo(torch.from_numpy(K), 480, 640, 0)
    pre = run_preprocess_lens(emus["lemu"], sc, c["model"], c["coefficients"])
    kept = pre.point_offset >= 0
    r2 = xn ** 2 + yn ** 2
    expect = (r2 <= r2_bound_ref(c["model"], c["coefficients"])) & (want[:, 0] >= -48) & (want[:, 0] < 688) & \
        (want[:, 1] >= -48) & (want[:, 1] < 528)
    assert np.array_equal(kept, expect) and kept.sum() >= 8
    got = pre.records[pre.point_offset[kept], 0:2]
    assert np.abs(got - want[kept]).max() <= 1e-3


# ------------------------------------------------------------------ validity
@pytest.mark.parametrize("model,k", [("opencv", (-0.3, 0.0, 0.0, 0.0, 0.0)), ("opencv", (-0.35, 0.12, 0.0, 0.0, -0.02)),
                                     ("opencv", (0.1, -0.05, 0.0, 0.0, 0.0)), ("fisheye", (-0.3, 0.0, 0.0, 0.0)),
                                     ("fisheye", (0.05, -0.06, 0.0, 0.0))])
def test_validity_bound_and_points_on_either_side(emus, model, k):
    want = r2_bound_ref(model, [float(np.float32(v)) for v in k])  # the library reads float32 coefficients
    got = r2_bound(emus["lemu"], model, k)
    assert math.isfinite(want) and abs(got - want) <= 1e-9 * want
    # x = 0, y = z r: points at r_max (1 -+ 2e-3), placed to land inside a wide image; the fold maps the outer one back
    r_max = math.sqrt(want)
    K = torch.tensor([[40.0, 0.0, 320.0], [0.0, 40.0, 240.0], [0.0, 0.0, 1.0]])
    rs = [r_max * (1 - 2e-3), r_max * (1 + 2e-3), r_max * 1.3, 0.2]
    pts = torch.tensor([[0.0, 2.0 * r, 2.0] for r in rs] + [[2.0 * r / math.sqrt(2), -2.0 * r / math.sqrt(2), 2.0] for r in rs])
    sc = make_scene(len(pts), 480, 640, 0.05, 1)
    sc.point_cloud = pts.float().contiguous()
    sc.q_pointcloud_camera = torch.tensor([[0.0, 0.0, 0.0, 1.0]])
    sc.camera_info = CameraInfo(K, 480, 640, 0)
    pre = run_preprocess_lens(emus["lemu"], sc, model, k)
    uv = project(pts.double(), K.double(), model, k)
    assert ((uv[:, 0] > 0) & (uv[:, 0] < 640) & (uv[:, 1] > 0) & (uv[:, 1] < 480)).all()  # every one would land inside
    assert (pre.point_offset >= 0).tolist() == [True, False, False, True] * 2


def test_unbounded_models():
    assert r2_bound_ref("opencv", (0.1, 0.01, 0.0, 0.0, 0.0)) == math.inf
    assert r2_bound_ref("fisheye", (0.05, -0.01, 0.003, -0.0005)) == math.inf
    lemu = build_lens_emulator()
    assert r2_bound(lemu, "opencv", (0.1, 0.01, 0.0, 0.0, 0.0)) == math.inf
    assert r2_bound(lemu, "opencv", (0.0, 0.0, 0.5, 0.5, 0.0)) == math.inf  # tangential terms do not enter the bound
    assert r2_bound(lemu, "fisheye", (0.05, -0.01, 0.003, -0.0005)) == math.inf


# ------------------------------------------------------------------ forward
def _dense(sc, feats_n, model, k, requires_grad=False):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = torch.from_numpy(feats_n).double().requires_grad_(requires_grad)
    image, aux = dense_render_lens(xyz, feats, sc.point_invalid_mask, sc.point_object_id, sc.camera_info.camera_intrinsics,
                                   sc.q_pointcloud_camera, sc.t_pointcloud_camera, H, W, model, k)
    return xyz, feats, image, aux


@pytest.mark.parametrize("objects", [1, 3])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_lens_forward_matches_dense_evaluator(emus, lens, objects):
    model, k = LENSES[lens]
    sc = _scene(31 + objects, objects=objects)
    st = emulated_forward_lens(emus["emu"], emus["lemu"], sc, model, k, exact=True)
    _, _, image, aux = _dense(sc, st.pre.feats, model, k)
    H, W = st.pre.H, st.pre.W
    assert st.count.max() >= 5 and (st.acc_alpha > 0.9).any()
    assert np.array_equal(aux["count"].numpy(), st.count)  # the same (pixel, splat) pairs
    assert np.abs(image.detach().numpy() - st.image).max() < 1e-4
    assert np.abs(aux["acc_alpha"].detach().numpy() - st.acc_alpha).max() < 1e-4
    depth, _ = differentiable_depth(aux, H, W)
    assert np.abs(depth.detach().numpy() - st.depth).max() < 1e-3
    ids = st.pre.point_id[:st.M]
    assert np.array_equal(np.sort(ids), np.sort(aux["ids"].numpy()))
    # the lens moved the splats: the pinhole forward of the same scene renders a different image
    assert np.abs(emulated_forward(emus["emu"], sc, exact=True).image - st.image).max() > 0.05


def test_zero_coefficients_agree_with_the_pinhole_path(emus):
    """opencv with k = 0 is the pinhole (fisheye with k = 0 is the equidistant lens theta_d = theta, not a pinhole)."""
    model, k = "opencv", (0.0,) * 5
    sc = _scene(35, objects=2)
    st = emulated_forward_lens(emus["emu"], emus["lemu"], sc, model, k)
    ref = emulated_forward(emus["emu"], sc)
    assert st.M == ref.M and np.array_equal(st.pre.point_offset, ref.pre.point_offset)
    # every op of the lens path is exact for zero coefficients (x + z 0, K D = K, ...): the same records, image and keys
    assert np.array_equal(st.pre.records, ref.pre.records) and np.array_equal(st.pre.pic, ref.pre.pic)
    assert np.array_equal(st.sorted_vals, ref.sorted_vals) and np.array_equal(st.image, ref.image)
    # and the LENS per-point backward gives the default kernel's gradients
    from simt_depth_helpers import emulated_points
    H, W = st.pre.H, st.pre.W
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(3)).numpy()
    accum = _loop_a_image(emus["emu"], st, g_img, True)
    gx, gf = emulated_points_lens(emus["emu"], emus["lemu"], st, accum)
    gx0, gf0 = emulated_points(emus["emu"], emus["demu"], ref, accum)
    assert np.array_equal(gx, gx0) and np.array_equal(gf, gf0)


# ------------------------------------------------------------------ backward
def _case(emus, lens, kind, seed, objects=1, transposed=True, band=3):
    model, k = LENSES[lens]
    emu, demu = emus["emu"], emus["demu"]
    sc = _scene(seed, objects=objects)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward_lens(emu, emus["lemu"], sc, model, k, exact=False)
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g, dtype=torch.float32)
    g_dep = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "depth" else None
    g_alpha = torch.randn((H, W), generator=g, dtype=torch.float32) if kind == "alpha" else None
    extra = g_map = None
    if kind == "image":
        accum = _loop_a_image(emu, st, g_img.numpy(), transposed)
    elif kind == "depth":
        _, _, accum, _ = emulated_backward_depth(emu, demu, st, g_img.numpy(), g_dep.numpy(), band)
    elif kind == "alpha":
        _, _, accum, _ = emulated_backward_alpha(emu, demu, emus["aemu"], st, g_img.numpy(), g_alpha.numpy(), band=band)
    else:
        N = sc.point_cloud.shape[0]
        extra = torch.randn((N, 5), generator=g, dtype=torch.float32).numpy()
        g_map = torch.randn((H, W, 5), generator=g, dtype=torch.float32)
        _, _, _, accum, _ = emulated_backward_features(emu, demu, emus["femu"], st, extra, g_map.numpy(), g_img.numpy(),
                                                       band=band)
    gx, gf = emulated_points_lens(emu, emus["lemu"], st, accum, band, depth=kind == "depth")
    xyz, feats, image, aux = _dense(sc, st.pre.feats, model, k, requires_grad=True)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)
    return st, accum, gx, gf, xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy()


def _check(gx, gf, ex, ef):
    ok = grad_close(gx, ex)  # the path's gradient criterion: 1e-3 relative + 1e-5 of the group's largest entry
    assert ok[0], ok
    for sl in GROUPS:
        ok = grad_close(gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_lens_gradient_matches_dense_autograd(emus, lens, kind):
    # one object: the SH view direction of the per-point backward takes t_pc as the camera centre, which is the evaluator's
    # only for a unit q (the multi-object scenes of test_pose_gradient_cpu give the other objects non-unit ones)
    _, _, gx, gf, ex, ef = _case(emus, lens, kind, 41)
    _check(gx, gf, ex, ef)


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_lens_gradient_under_the_butterfly_loop_a(emus, lens):
    _, _, gx, gf, ex, ef = _case(emus, lens, "image", 43, transposed=False, band=1)
    _check(gx, gf, ex, ef)


def test_lens_gradient_is_deterministic_and_differs_from_the_pinhole_chain_rule(emus):
    st, accum, gx, gf, ex, _ = _case(emus, "opencv", "image", 45)
    gx2, gf2 = emulated_points_lens(emus["emu"], emus["lemu"], st, accum)
    assert np.array_equal(gx, gx2) and np.array_equal(gf, gf2)
    # the default per-point kernel on the same rows (pinhole Jacobians) is clearly wrong here
    from simt_depth_helpers import emulated_points
    gx0, _ = emulated_points(emus["emu"], emus["demu"], st, accum)
    assert not grad_close(gx0, ex)[0]


# ------------------------------------------------------------------ C ABI
def _fwd_args():
    return _lib.GsbForwardArgs()


def _lens(model, *co):
    return _lib.GsbLensArgs(model=model, coefficients=(ctypes.c_float * 5)(*(list(co) + [0.0] * (5 - len(co)))))


def test_c_entry_points_check_the_lens_before_any_cuda_call():
    lib = _lib.load()
    for name in ("gsb200_forward_lens", "gsb200_backward_lens"):
        assert hasattr(lib, name) and name in _lib.EXPORTS
    bad = [(_lens(3), b"unknown lens model"), (_lens(-1), b"unknown lens model"),
           (_lens(1, 0.1, float("nan")), b"not finite"), (_lens(2, 0.1, float("inf")), b"not finite"),
           (_lens(2, 0.1, 0.0, 0.0, 0.0, 0.5), b"must be 0"), (_lens(0, 0.1), b"must be 0")]
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    for lens, msg in bad:
        # args point at nothing the call could use: the lens is checked first
        assert lib.gsb200_forward_lens(ctypes.byref(_fwd_args()), None, ctypes.byref(lens)) == -1
        assert msg in lib.gsb200_last_error()
        assert lib.gsb200_backward_lens(ctypes.byref(bargs), None, None, None, None, ctypes.byref(lens)) == -1
        assert msg in lib.gsb200_last_error()
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for model in (1, 2):
        assert lib.gsb200_backward_lens(ctypes.byref(compact), None, None, None, None, ctypes.byref(_lens(model, 0.1))) == -4
        assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # a valid lens reaches the usual argument checks
    assert lib.gsb200_backward_lens(ctypes.byref(bargs), None, None, None, None, ctypes.byref(_lens(1, 0.1))) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_and_pinhole_lens_are_exactly_the_ext_calls():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ext = _lib.GsbExtraFeatureArgs(channels=0, features=fake, grad_rasterized=fake, grad_features=fake)
    for lens in (None, ctypes.byref(_lens(0))):
        for e in (None, ctypes.byref(ext)):
            want = lib.gsb200_forward_ext(ctypes.byref(_fwd_args()), e)
            want_msg = lib.gsb200_last_error()
            assert lib.gsb200_forward_lens(ctypes.byref(_fwd_args()), e, lens) == want != 0
            assert lib.gsb200_last_error() == want_msg
        cases = [(_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                 (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (fake, None, None, None)),
                 (_lib.GsbBackwardArgs(), (fake, fake, None, None)),
                 (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_COMPACT_GRADS), (None, None, None, ctypes.byref(ext)))]
        for args, extra in cases:
            want = lib.gsb200_backward_ext(ctypes.byref(args), *extra)
            want_msg = lib.gsb200_last_error()
            assert lib.gsb200_backward_lens(ctypes.byref(args), *extra, lens) == want != 0
            assert lib.gsb200_last_error() == want_msg


def test_abi_size_of_the_lens_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 11)()
    lib.gsb200_abi_sizes_ext(sizes, 11)
    assert sizes[10] == ctypes.sizeof(_lib.GsbLensArgs) == 24
    first10 = (ctypes.c_int64 * 10)()
    lib.gsb200_abi_sizes_ext(first10, 10)
    assert list(first10) == list(sizes)[:10]


# ------------------------------------------------------------------ Python surface
def test_lens_distortion_dataclass_and_from_colmap():
    d = LensDistortion("opencv", [0.1, 0, 0, 0, 0])
    assert d.coefficients == (0.1, 0.0, 0.0, 0.0, 0.0) and hash(d) == hash(LensDistortion("opencv", (0.1, 0, 0, 0, 0)))
    with pytest.raises(Exception):
        d.model = "fisheye"  # frozen
    for bad in (("pinhole", ()), ("opencv", (0.1,)), ("fisheye", (0.1, 0, 0, 0, 0)), ("opencv", (math.nan, 0, 0, 0, 0))):
        with pytest.raises(ValueError):
            LensDistortion(*bad)
    assert CameraInfo(torch.eye(3), 16, 16, 0).distortion is None
    cases = {
        "SIMPLE_PINHOLE": ([500, 320, 240], [[500, 0, 320], [0, 500, 240]], None),
        "PINHOLE": ([500, 510, 320, 240], [[500, 0, 320], [0, 510, 240]], None),
        "SIMPLE_RADIAL": ([500, 320, 240, -0.1], [[500, 0, 320], [0, 500, 240]], ("opencv", (-0.1, 0, 0, 0, 0))),
        "RADIAL": ([500, 320, 240, -0.1, 0.02], [[500, 0, 320], [0, 500, 240]], ("opencv", (-0.1, 0.02, 0, 0, 0))),
        "OPENCV": ([500, 510, 320, 240, -0.1, 0.02, 1e-3, -2e-3], [[500, 0, 320], [0, 510, 240]],
                   ("opencv", (-0.1, 0.02, 1e-3, -2e-3, 0))),
        "OPENCV_FISHEYE": ([300, 310, 320, 240, 0.05, -0.01, 0.003, -0.0005], [[300, 0, 320], [0, 310, 240]],
                           ("fisheye", (0.05, -0.01, 0.003, -0.0005))),
    }
    for name, (params, rows, lens) in cases.items():
        K, dist = LensDistortion.from_colmap(name, params)
        assert K.dtype == torch.float32 and torch.allclose(K, torch.tensor(rows + [[0, 0, 1]], dtype=torch.float32))
        assert dist == (None if lens is None else LensDistortion(*lens)), name
    for name, params in (("FOV", [500, 500, 320, 240, 0.9]), ("THIN_PRISM_FISHEYE", [0] * 12), ("FULL_OPENCV", [0] * 12),
                         ("OPENCV", [500, 510, 320, 240])):
        with pytest.raises(ValueError):
            LensDistortion.from_colmap(name, params)


def test_operator_refuses_a_lens_with_pose_intrinsics_or_exchange():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, LensDistortion("fisheye", (0.1, 0, 0, 0)))
    inp = G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)
    for kw, msg in ((dict(differentiable_pose=True), "differentiable_pose"),
                    (dict(differentiable_intrinsics=True), "differentiable_intrinsics"),
                    (dict(gradient_exchange=object()), "gradient_exchange")):
        with pytest.raises(ValueError, match=msg):
            G(Config(), **kw)(inp)
    lens = G(Config())._lens_args(ci)
    assert lens.model == _lib.GSB_LENS_FISHEYE and list(lens.coefficients) == pytest.approx([0.1, 0, 0, 0, 0])
    assert G(Config())._lens_args(sc.camera_info) is None


def _trainer(distorted, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    lens = LensDistortion("opencv", (-0.1, 0.01, 0, 0, 0))
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, 0, lens if distorted else None))]
    cfg = T.TrainConfig(**{k: v for k, v in kw.items() if k.endswith("learning_rate")})
    return T(cfg, scene, views, rasterisation_factory=lambda **kwargs: (lambda *a, **k: None),
             fused_step=kw.get("fused_step", False))


def test_trainer_configuration_and_downsampling_carry_the_lens():
    from taichi_3d_gaussian_splatting_b200.trainer import downsample_image_and_camera_info
    trainer = _trainer(True)
    image, q, t, ci, _ = trainer._view(0, 2)
    assert ci.distortion == LensDistortion("opencv", (-0.1, 0.01, 0, 0, 0)) and ci.camera_width == 48
    _, ci4 = downsample_image_and_camera_info(torch.zeros((3, 64, 96)), trainer.train_views[0][3], 4)
    assert ci4.distortion is trainer.train_views[0][3].distortion
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(pose_learning_rate=1e-3), "pose"),
                    (dict(intrinsics_learning_rate=1e-3), "intrinsics")):
        with pytest.raises(ValueError, match=msg):
            _trainer(True, **kw)
        if "fused_step" not in kw:
            _trainer(False, **kw)  # unchanged without a lens


def test_dataset_reads_the_distortion_key_and_keeps_it_through_autoscale_and_crop(tmp_path):
    import PIL.Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    recs = []
    for i, (h, w, dist) in enumerate(((40, 50, {"model": "fisheye", "coefficients": [0.05, -0.01, 0.003, -0.0005]}),
                                      (1700, 1800, {"model": "opencv", "coefficients": [-0.1, 0.02, 1e-3, -2e-3, 0.0]}),
                                      (40, 50, None))):
        path = tmp_path / f"im{i}.png"
        PIL.Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(path)
        rec = dict(image_path=str(path), T_pointcloud_camera=np.eye(4).tolist(),
                   camera_intrinsics=[[0.6 * w, 0, w / 2], [0, 0.6 * w, h / 2], [0, 0, 1]], camera_height=h, camera_width=w,
                   camera_id=i)
        if dist is not None:
            rec["distortion"] = dist
        recs.append(rec)
    path = tmp_path / "ds.json"
    path.write_text(json.dumps(recs))
    ds = ImagePoseDataset(str(path))
    ci0, ci1, ci2 = ds[0][3], ds[1][3], ds[2][3]
    assert (ci0.camera_height, ci0.camera_width) == (32, 48)  # cropped to tiles
    assert ci0.distortion == LensDistortion("fisheye", (0.05, -0.01, 0.003, -0.0005))
    assert max(ci1.camera_height, ci1.camera_width) <= 1600  # autoscaled
    assert ci1.distortion == LensDistortion("opencv", (-0.1, 0.02, 1e-3, -2e-3, 0.0))
    assert ci2.distortion is None
    recs[0]["distortion"] = {"model": "kannala"}
    path.write_text(json.dumps(recs))
    with pytest.raises(ValueError):
        ImagePoseDataset(str(path))[0]
