"""Lens-coefficient gradients (``gsb200_backward_lens_grad``, ``differentiable_distortion``,
``TrainConfig.distortion_learning_rate``) without a GPU.

* Known answers of OpenCV (``golden/lens_coefficient_vectors.json``, written by ``golden/make_lens_coefficient_golden.py``
  with cv2): the distCoeffs columns d uv / dk against the float64 reference ``torch_reference_lens_grad`` and the float32
  device helper ``lens_coefficient_grad``.
* The emulated LGRAD per-point kernel (the unmodified CUDA sources under the SIMT emulator of ``tests/simt``) on emulated
  loop-A rows against torch autograd of the dense float64 evaluator with k as a leaf, for image, depth, alpha and feature-map
  losses, both lenses, three objects sharing warps and both loop-A kernels; determinism; every other output bit-identical to
  the LENS kernel's.
* The C entry point's argument rules and ABI size, and the operator's and trainer's configuration."""
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

from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator
from simt_lens_grad_helpers import build_lens_grad_emulator, coefficient_jacobian, emulated_points_lens_grad
from simt_lens_helpers import build_lens_emulator, emulated_forward_lens, emulated_points_lens
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_lens_grad import dense_render_lens_k, project_k

HERE = os.path.dirname(os.path.abspath(__file__))
LENSES = {
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator(), gemu=build_lens_grad_emulator())


def _golden():
    with open(os.path.join(HERE, "golden", "lens_coefficient_vectors.json")) as f:
        return json.load(f)


def _used(model):
    return 5 if model == "opencv" else 4


# ------------------------------------------------------------------ known answers of OpenCV
def test_golden_vectors_cover_both_models_and_the_axis():
    d = _golden()
    assert d["cv2_version"]
    assert {c["model"] for c in d["cases"]} == {"opencv", "fisheye"}
    for c in d["cases"]:
        pts = np.array(c["points"])
        r2 = (pts[:, 0] / pts[:, 2]) ** 2 + (pts[:, 1] / pts[:, 2]) ** 2
        assert r2[0] == 0 and r2[1] < 1e-12 and (r2 < 0.04).sum() >= 4 and (r2 > 0.04).sum() >= 10
        assert np.array(c["duv_dk"]).shape == (len(pts), 2, _used(c["model"]))


@pytest.mark.parametrize("case", range(5))
def test_float64_reference_matches_opencv(case):
    c = _golden()["cases"][case]
    K = torch.tensor(c["K"], dtype=torch.float64)
    pts = torch.tensor(c["points"], dtype=torch.float64)
    k0 = torch.tensor(c["coefficients"][:_used(c["model"])], dtype=torch.float64)
    assert np.abs(project_k(pts, K, c["model"], k0).numpy() - np.array(c["uv"])).max() <= 1e-9
    jac = torch.autograd.functional.jacobian(lambda k: project_k(pts, K, c["model"], k), k0)
    assert np.abs(jac.numpy() - np.array(c["duv_dk"])).max() <= 1e-10


@pytest.mark.parametrize("case", range(5))
def test_device_helper_matches_opencv(emus, case):
    c = _golden()["cases"][case]
    K = np.array(c["K"], np.float64)
    pts = np.array(c["points"], np.float64)
    xn, yn = (pts[:, 0] / pts[:, 2]).astype(np.float32), (pts[:, 1] / pts[:, 2]).astype(np.float32)
    dxy = coefficient_jacobian(emus["gemu"], c["model"], xn, yn).astype(np.float64)  # (n, 2, 5)
    duv = K[:2, :2] @ dxy
    n = _used(c["model"])
    want = np.array(c["duv_dk"])
    assert np.abs(duv[:, :, :n] - want).max() <= 1e-5 * np.abs(want).max()
    if n == 4:
        assert (dxy[:, :, 4] == 0).all()


# ------------------------------------------------------------------ the per-point kernel
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
    res = emulated_points_lens_grad(emu, emus["gemu"], st, accum, band, depth=kind == "depth")
    kk = torch.tensor(k, dtype=torch.float64, requires_grad=True)
    ci = sc.camera_info
    image, aux = dense_render_lens_k(sc.point_cloud.double(), torch.from_numpy(st.pre.feats).double(), sc.point_invalid_mask,
                                     sc.point_object_id, ci.camera_intrinsics, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
                                     H, W, model, kk)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)
    return st, accum, res, kk.grad.numpy()


def _check(gk, ek, model):
    n = _used(model)
    scale = np.abs(ek).max()
    assert scale > 0
    err = np.abs(gk[:n] - ek)
    assert (err <= 2e-3 * np.abs(ek) + 2e-4 * scale).all(), (gk, ek)
    assert (gk[n:] == 0).all()


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_coefficient_gradient_matches_dense_autograd(emus, lens, kind):
    _, _, res, ek = _case(emus, lens, kind, 41)
    _check(res.gk, ek, LENSES[lens][0])


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_coefficient_gradient_with_three_objects_sharing_warps(emus, lens):
    st, _, res, ek = _case(emus, lens, "image", 47, objects=3)
    obj = st.scene.point_object_id.numpy()
    kept = st.pre.point_offset >= 0
    assert len(set(obj[:32][kept[:32]].tolist())) == 3  # one warp holds in-camera points of all three objects
    _check(res.gk, ek, LENSES[lens][0])


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_emulated_coefficient_gradient_under_the_butterfly_loop_a(emus, lens):
    _, _, res, ek = _case(emus, lens, "image", 43, transposed=False, band=1)
    _check(res.gk, ek, LENSES[lens][0])


@pytest.mark.parametrize("kind", ["image", "depth"])
def test_coefficient_gradient_is_deterministic_and_leaves_every_other_output_unchanged(emus, kind):
    st, accum, res, _ = _case(emus, "opencv", kind, 45)
    again = emulated_points_lens_grad(emus["emu"], emus["gemu"], st, accum, depth=kind == "depth")
    assert np.array_equal(res.gk, again.gk) and np.array_equal(res.partials, again.partials)
    assert res.blocks == min(math.ceil(st.pre.point_offset.shape[0] / 128), 2048)
    # the finishing kernel's sum of the per-CTA rows
    assert np.allclose(res.partials.astype(np.float64).sum(0), res.gk, rtol=1e-5, atol=1e-6 * np.abs(res.gk).max())
    gx, gf = emulated_points_lens(emus["emu"], emus["lemu"], st, accum, depth=kind == "depth")
    assert np.array_equal(res.gx, gx) and np.array_equal(res.gf, gf)


def test_zero_opencv_coefficients_get_a_gradient(emus):
    """Refining k1, k2 from zero: the pinhole-identical lens still has a non-zero coefficient gradient."""
    sc = _scene(49)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward_lens(emus["emu"], emus["lemu"], sc, "opencv", (0.0,) * 5, exact=False)
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(5)).numpy()
    res = emulated_points_lens_grad(emus["emu"], emus["gemu"], st, _loop_a_image(emus["emu"], st, g_img, True))
    assert (np.abs(res.gk) > 0).all()


# ------------------------------------------------------------------ C ABI
def _lens(model, *co):
    return _lib.GsbLensArgs(model=model, coefficients=(ctypes.c_float * 5)(*(list(co) + [0.0] * (5 - len(co)))))


def test_c_entry_point_checks_its_arguments_before_any_cuda_call():
    lib = _lib.load()
    for name in ("gsb200_backward_lens_grad", "gsb200_lens_grad_temp_bytes"):
        assert hasattr(lib, name) and name in _lib.EXPORTS
    assert lib.gsb200_lens_grad_temp_bytes() == 2048 * 5 * 4
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    ok = ctypes.c_void_p(256)
    good = _lib.GsbLensGradArgs(grad_coefficients=ok, temp=ok)
    bad = [(_lens(1, 0.1), _lib.GsbLensGradArgs(grad_coefficients=None, temp=ok), b"null grad_coefficients"),
           (_lens(1, 0.1), _lib.GsbLensGradArgs(grad_coefficients=ok, temp=None), b"null grad_coefficients"),
           (_lens(2, 0.1), _lib.GsbLensGradArgs(grad_coefficients=ctypes.c_void_p(258), temp=ok), b"4-byte aligned"),
           (_lens(2, 0.1), _lib.GsbLensGradArgs(grad_coefficients=ok, temp=ctypes.c_void_p(260)), b"16-byte aligned"),
           (None, good, b"needs an opencv or fisheye lens"), (_lens(0), good, b"needs an opencv or fisheye lens"),
           (_lens(1, float("nan")), good, b"not finite"), (_lens(7), good, b"unknown lens model")]
    for lens, lg, msg in bad:
        # args point at nothing the call could use: these checks come first
        assert lib.gsb200_backward_lens_grad(ctypes.byref(bargs), None, None, None, None,
                                             ctypes.byref(lens) if lens is not None else None, ctypes.byref(lg)) == -1
        assert msg in lib.gsb200_last_error()
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for model in (1, 2):
        assert lib.gsb200_backward_lens_grad(ctypes.byref(compact), None, None, None, None, ctypes.byref(_lens(model, 0.1)),
                                             ctypes.byref(good)) == -4
        assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # valid arguments reach the usual argument checks
    assert lib.gsb200_backward_lens_grad(ctypes.byref(bargs), None, None, None, None, ctypes.byref(_lens(1, 0.1)),
                                         ctypes.byref(good)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_lens_grad_is_exactly_backward_lens():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ext = _lib.GsbExtraFeatureArgs(channels=0, features=fake, grad_rasterized=fake, grad_features=fake)
    for lens in (None, ctypes.byref(_lens(0)), ctypes.byref(_lens(1, 0.1)), ctypes.byref(_lens(3))):
        for args, extra in ((_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                            (_lib.GsbBackwardArgs(), (fake, fake, None, None)),
                            (_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_COMPACT_GRADS), (None, None, None, ctypes.byref(ext)))):
            want = lib.gsb200_backward_lens(ctypes.byref(args), *extra, lens)
            want_msg = lib.gsb200_last_error()
            assert lib.gsb200_backward_lens_grad(ctypes.byref(args), *extra, lens, None) == want != 0
            assert lib.gsb200_last_error() == want_msg


def test_abi_size_of_the_lens_gradient_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 12)()
    lib.gsb200_abi_sizes_ext(sizes, 12)
    assert sizes[11] == ctypes.sizeof(_lib.GsbLensGradArgs) == 16
    first11 = (ctypes.c_int64 * 11)()
    lib.gsb200_abi_sizes_ext(first11, 11)
    assert list(first11) == list(sizes)[:11]


# ------------------------------------------------------------------ Python surface
def _input(distorted=True):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0,
                    LensDistortion("fisheye", (0.1, 0, 0, 0)) if distorted else None)
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_configuration_of_differentiable_distortion():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_distortion=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_distortion=True, gradient_exchange=object())
    op = G(Config(), differentiable_distortion=True)
    inp = _input()
    for k, msg in ((torch.zeros(5), "4"), (torch.zeros(4, dtype=torch.float64), "float32"), (torch.zeros(2, 2), "4"),
                   ([0.1, 0, 0, 0], "torch.Tensor")):
        with pytest.raises(ValueError, match=msg):
            op(inp, lens_coefficients=k)
    with pytest.raises(ValueError, match="no lens"):
        op(_input(distorted=False), lens_coefficients=torch.zeros(5))
    with pytest.raises(ValueError, match="differentiable_distortion"):
        G(Config())(inp, lens_coefficients=torch.zeros(4))
    # the values rendered are the tensor's; the model is the camera's
    lens = op._lens_args(inp.camera_info, torch.tensor([0.2, -0.01, 0.0, 0.0]))
    assert lens.model == _lib.GSB_LENS_FISHEYE and list(lens.coefficients) == pytest.approx([0.2, -0.01, 0, 0, 0])
    # the existing refusals stay
    with pytest.raises(ValueError, match="differentiable_pose"):
        G(Config(), differentiable_pose=True, differentiable_distortion=True)(inp, lens_coefficients=torch.zeros(4))


def _trainer(lenses, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, cam, lens))
             for cam, lens in lenses]
    seen = {}
    factory = lambda **kwargs: seen.update(kwargs) or (lambda *a, **k: None)  # noqa: E731
    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=factory), seen


def test_trainer_configuration_of_distortion_learning_rate():
    a = LensDistortion("opencv", (-0.1, 0.01, 0, 0, 0))
    b = LensDistortion("opencv", (-0.2, 0.01, 0, 0, 0))
    for rate in (-1e-3, math.nan, math.inf):
        with pytest.raises(ValueError, match="distortion_learning_rate"):
            _trainer([(0, a)], distortion_learning_rate=rate)
    with pytest.raises(ValueError, match="distorted"):
        _trainer([(0, None), (1, None)], distortion_learning_rate=1e-3)
    with pytest.raises(ValueError, match="camera_id 0"):
        _trainer([(0, a), (0, b)], distortion_learning_rate=1e-3)
    for kw in (dict(pose_learning_rate=1e-3), dict(intrinsics_learning_rate=1e-3)):  # the existing rules stay
        with pytest.raises(ValueError):
            _trainer([(0, a)], distortion_learning_rate=1e-3, **kw)
    trainer, seen = _trainer([(0, a), (1, b), (0, a), (2, None)], distortion_learning_rate=1e-3)
    assert seen.get("differentiable_distortion") is True
    assert sorted(trainer._distortion) == [0, 1]
    leaf = trainer._distortion[0]
    assert leaf.is_leaf and leaf.requires_grad and leaf.device.type == "cpu" and leaf.dtype == torch.float32
    f32 = lambda lens: LensDistortion(lens.model, [float(np.float32(v)) for v in lens.coefficients])  # noqa: E731
    assert trainer.refined_distortion() == [f32(a), f32(b), f32(a), None]  # float32 leaves
    with torch.no_grad():
        leaf[0] = -0.15
    assert trainer.refined_distortion()[0] == f32(LensDistortion("opencv", (-0.15, 0.01, 0, 0, 0)))
    # off: the views' own lenses and no extra operator option
    trainer, seen = _trainer([(0, a)])
    assert "differentiable_distortion" not in seen and trainer.refined_distortion() == [a]
