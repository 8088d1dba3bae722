"""Depth of field (``gsb200_forward_defocus`` / ``gsb200_backward_defocus``) on the CPU: the unmodified DEFOCUS kernels under the
SIMT emulator against the float64 dense evaluator (``torch_reference_defocus``) and autograd on it, a closed-form splat, the
mean of pinhole renders over the aperture, zero aperture against the motion-blur kernels bit for bit, the determinism of the
(a, rho) gradient, the C ABI's argument checks, and the Python surface (``Camera.Defocus``, the dataset key, the operator's and
the trainer's refusals)."""
import ctypes
import json
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, Defocus, LensDistortion, MotionBlur, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene

from helpers import grad_close
from simt_alpha_helpers import build_alpha_emulator, emulated_backward_alpha
from simt_defocus_helpers import build_defocus_emulator, emulated_forward_defocus, emulated_points_defocus, \
    run_preprocess_defocus
from simt_depth_helpers import build_depth_emulator, emulated_backward_depth
from simt_feature_helpers import build_feature_emulator, emulated_backward_features
from simt_helpers import build_emulator
from simt_lens_helpers import build_lens_emulator
from simt_motion_blur_helpers import build_motion_blur_emulator, emulated_forward_blur, emulated_points_blur
from simt_rolling_shutter_helpers import build_rolling_shutter_emulator
from test_pose_gradient_cpu import _loop_a_image, _scene
from torch_reference import postprocess_feature_grads
from torch_reference_defocus import dense_render_defocus
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map

GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "pinhole": ("pinhole", ()),
    "opencv": ("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": ("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
RS_MOTION = (0.06, -0.09, 0.04, 0.05, -0.08, 0.06)  # v, w over one readout
BLUR = (0.05, 0.03, -0.02, -0.02, 0.03, 0.01)  # v, w over the exposure
NO_BLUR = (0.0,) * 6
# a = 0.2, focus at 2.2: disks of up to ~4 px near the camera and ~1.5 px at the back of the 48 x 32 scenes (f = 28.8 px)
DEFOCUS = (0.2, 1 / 2.2)


@pytest.fixture(scope="module")
def emus():
    return dict(emu=build_emulator(), demu=build_depth_emulator(), aemu=build_alpha_emulator(), femu=build_feature_emulator(),
                lemu=build_lens_emulator(), remu=build_rolling_shutter_emulator(), bemu=build_motion_blur_emulator(),
                dfemu=build_defocus_emulator())


def _dense(sc, feats_n, model, k, motion, blur, defocus, requires_grad=False):
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    xyz = sc.point_cloud.clone().double().requires_grad_(requires_grad)
    feats = torch.from_numpy(feats_n).double().requires_grad_(requires_grad)
    df = torch.tensor(defocus, dtype=torch.float64, requires_grad=requires_grad)
    image, aux = dense_render_defocus(xyz, feats, sc.point_invalid_mask, sc.point_object_id, sc.camera_info.camera_intrinsics,
                                      sc.q_pointcloud_camera, sc.t_pointcloud_camera, H, W, model, k, motion, blur, df)
    return xyz, feats, df, image, aux


# ------------------------------------------------------------------ forward against the float64 evaluator
@pytest.mark.parametrize("blurred", [False, True])
@pytest.mark.parametrize("rolling", [False, True])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_forward_matches_dense_evaluator(emus, lens, rolling, blurred):
    model, k = LENSES[lens]
    motion = RS_MOTION if rolling else NO_BLUR
    blur = BLUR if blurred else NO_BLUR
    sc = _scene(61, objects=2)
    st = emulated_forward_defocus(emus["emu"], emus["dfemu"], sc, model, k, motion, blur, DEFOCUS, rolling, exact=True)
    _, _, _, image, aux = _dense(sc, st.pre.feats, model, k, motion, blur, DEFOCUS)
    ids = st.pre.point_id[:st.M]
    assert np.array_equal(np.sort(ids), np.sort(aux["ids"].numpy()))
    assert aux["blur_px"].max() > 3.0  # the defocus is visible
    order = np.argsort(ids)
    rec = st.pre.records[:st.M][order]
    assert np.allclose(rec[:, 0:2], aux["uv"].detach().numpy(), rtol=1e-5, atol=1e-4)
    conic = aux["conic"].detach().numpy()
    assert np.allclose(rec[:, 2:5], conic[:, 0:3], rtol=1e-4, atol=1e-5 * np.abs(conic[:, 0:3]).max())
    slot = (aux["conic"][:, 3] * aux["comp"]).detach().numpy()  # rescale c_b
    assert np.allclose(rec[:, 5], slot, rtol=1e-4, atol=1e-6)
    assert (aux["comp"].detach().numpy() < 0.9).any()
    assert np.allclose(rec[:, 11], aux["radius"].numpy(), rtol=1e-4, atol=1e-4)  # from Sigma' + B
    assert np.array_equal(aux["count"].numpy(), st.count)
    assert np.abs(image.detach().numpy() - st.image).max() < 1e-4
    depth, _ = differentiable_depth(aux, st.pre.H, st.pre.W)
    assert np.abs(depth.detach().numpy() - st.depth).max() < 1e-3
    # the defocus changed the render
    sharp = emulated_forward_blur(emus["emu"], emus["bemu"], sc, model, k, motion, blur, rolling)
    assert np.abs(sharp.image - st.image).max() > 0.02


def _single_splat(K, H, W, z=2.0, log_scale=-3.0, logit=2.2, t=(0.0, 0.0, 0.0)):
    row = [0.0] * 56
    row[3] = 1.0
    row[4] = row[5] = row[6] = log_scale
    row[7] = logit
    return SimpleNamespace(point_cloud=torch.tensor([[0.0, 0.0, z]]), point_cloud_features=torch.tensor([row]),
                           point_invalid_mask=torch.zeros(1, dtype=torch.int8), point_object_id=torch.zeros(1, dtype=torch.int32),
                           q_pointcloud_camera=torch.tensor([[0.0, 0.0, 0.0, 1.0]]), t_pointcloud_camera=torch.tensor([t]),
                           camera_info=CameraInfo(torch.tensor(K), H, W, 0))


def test_closed_form_fronto_parallel_splat(emus):
    """An isotropic splat of std s facing the camera: the footprint variance is s^2 f^2 / z^2 + 0.3 + a^2 (rho - 1/z)^2 f^2 / 16
    on both axes, the rescale slot carries the matching peak sqrt(det Sigma_d / det(Sigma_d + B)), and the radius grows."""
    f, z, a, rho = 50.0, 2.0, 0.4, 0.25
    K = [[f, 0, 48.0], [0, f, 32.0], [0, 0, 1]]
    sc = _single_splat(K, 64, 96, z=z)
    pre = run_preprocess_defocus(emus["dfemu"], sc, "pinhole", (), NO_BLUR, NO_BLUR, (a, rho), False)
    base = run_preprocess_defocus(emus["dfemu"], sc, "pinhole", (), NO_BLUR, NO_BLUR, (0.0, rho), False)
    s = math.exp(-3.0) * f / z
    bd = a * a * (rho - 1 / z) ** 2 * f * f / 16
    var = s * s + 0.3 + bd
    r, r0 = pre.records[0], base.records[0]
    assert [r[2], r[3], r[4]] == pytest.approx([1 / var, 0.0, 1 / var], rel=1e-5, abs=1e-7)
    assert r[5] == pytest.approx(r0[5] * (s * s + 0.3) / var, rel=1e-5)  # sqrt of the determinant ratio, isotropic
    assert r[11] == pytest.approx(3 * math.sqrt(s * s + bd), rel=1e-5) and r[11] > r0[11]
    # the disk diameter in pixels is a f |rho - 1/z| = 5 px; its per-axis variance is (diameter / 4)^2
    assert bd == pytest.approx((a * f * abs(rho - 1 / z) / 4) ** 2)


def _image_covariance(img):
    w = img[..., 0].astype(np.float64)
    ys, xs = np.mgrid[0:w.shape[0], 0:w.shape[1]] + 0.5
    m = w.sum()
    mx, my = (w * xs).sum() / m, (w * ys).sum() / m
    return np.array([[(w * (xs - mx) ** 2).sum(), (w * (xs - mx) * (ys - my)).sum()],
                     [(w * (xs - mx) * (ys - my)).sum(), (w * (ys - my) ** 2).sum()]]) / m


def test_mean_of_pinhole_renders_over_the_aperture_has_the_covariance_of_the_model(emus):
    """A stratified disk of camera offsets s (the aperture), each with the principal point moved by K[:2,:2] s rho so that the
    focal plane stays fixed: the mean of these pinhole renders of a faint splat has the footprint covariance of the defocus
    render, Sigma_d + B_d.  Moving the principal point the other way gives a much wider mean: this pins the sign."""
    f, z, a, rho, H, W = 50.0, 2.0, 0.4, 0.25, 64, 96
    K = np.array([[f, 0, 48.0], [0, f, 32.0], [0, 0, 1]])

    def render(t, Kv, defocus=(0.0, 0.0)):
        sc = _single_splat(Kv.tolist(), H, W, z=z, t=t)
        return emulated_forward_defocus(emus["emu"], emus["dfemu"], sc, "pinhole", (), NO_BLUR, NO_BLUR, defocus,
                                        False).image

    n_r, n_t = 8, 8
    means = {+1: np.zeros((H, W, 3)), -1: np.zeros((H, W, 3))}
    for i in range(n_r):
        for j in range(n_t):
            rad = a / 2 * math.sqrt((i + 0.5) / n_r)
            th = 2 * math.pi * (j + 0.5) / n_t + 0.37 * i
            sx, sy = rad * math.cos(th), rad * math.sin(th)
            for sign in (+1, -1):
                Ks = K.copy()
                Ks[0, 2] += sign * f * sx * rho
                Ks[1, 2] += sign * f * sy * rho
                means[sign] += render((sx, sy, 0.0), Ks) / (n_r * n_t)
    model = render((0.0, 0.0, 0.0), K, (a, rho))
    cm, cp, cw = _image_covariance(model), _image_covariance(means[+1]), _image_covariance(means[-1])
    sharp = _image_covariance(render((0.0, 0.0, 0.0), K))
    bd = a * a * (rho - 1 / z) ** 2 * f * f / 16
    assert cm[0, 0] - sharp[0, 0] == pytest.approx(bd, rel=0.12)  # the model adds B_d (up to the 1/255 cut of the tails)
    assert np.allclose(cp, cm, rtol=0.06, atol=0.05)
    assert cw[0, 0] > cm[0, 0] + 3 * bd
    assert means[+1][..., 0].sum() == pytest.approx(model[..., 0].sum(), rel=0.03)  # c_b keeps the integrated weight


def test_zero_aperture_is_bit_identical_to_the_motion_blur_kernels(emus):
    g_img = torch.randn((32, 48, 3), generator=torch.Generator().manual_seed(3)).numpy()
    for lens in ("pinhole", "opencv", "fisheye"):
        model, k = LENSES[lens]
        for rolling, blur in ((False, BLUR), (True, NO_BLUR), (True, BLUR)):
            motion = RS_MOTION if rolling else NO_BLUR
            sc = _scene(63, objects=3)
            st = emulated_forward_defocus(emus["emu"], emus["dfemu"], sc, model, k, motion, blur, (0.0, DEFOCUS[1]), rolling)
            ref = emulated_forward_blur(emus["emu"], emus["bemu"], sc, model, k, motion, blur, rolling)
            assert st.M == ref.M and st.K == ref.K and np.array_equal(st.pre.point_offset, ref.pre.point_offset)
            assert np.array_equal(st.pre.records, ref.pre.records) and np.array_equal(st.pre.pic, ref.pre.pic)
            assert np.array_equal(st.pre.keys[:st.K], ref.pre.keys[:ref.K])
            assert np.array_equal(st.sorted_vals, ref.sorted_vals) and np.array_equal(st.image, ref.image)
            if rolling:
                assert np.array_equal(st.pre.row_time, ref.pre.row_time)
            for depth in (False, True):
                if depth:
                    g_dep = torch.randn((32, 48), generator=torch.Generator().manual_seed(4)).numpy()
                    _, _, accum, _ = emulated_backward_depth(emus["emu"], emus["demu"], st, g_img, g_dep)
                else:
                    accum = _loop_a_image(emus["emu"], st, g_img, True)
                res = emulated_points_defocus(emus["emu"], emus["dfemu"], st, accum, depth=depth, dgrad=True)
                want = emulated_points_blur(emus["emu"], emus["bemu"], ref, accum, depth=depth, bgrad=False)
                assert np.array_equal(res.gx, want.gx) and np.array_equal(res.gf, want.gf), (lens, rolling, depth)
                assert (res.gd == 0).all()  # both gradients vanish at a = 0: refinement cannot start from zero


# ------------------------------------------------------------------ backward against float64 autograd
def _case(emus, lens, kind, seed, objects=1, transposed=True, band=3, rolling=False, blur=NO_BLUR, defocus=DEFOCUS):
    model, k = LENSES[lens]
    motion = RS_MOTION if rolling else NO_BLUR
    emu, demu = emus["emu"], emus["demu"]
    sc = _scene(seed, objects=objects)
    H, W = sc.camera_info.camera_height, sc.camera_info.camera_width
    st = emulated_forward_defocus(emu, emus["dfemu"], sc, model, k, motion, blur, defocus, rolling, exact=False)
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
    res = emulated_points_defocus(emu, emus["dfemu"], st, accum, band, depth=kind == "depth")
    xyz, feats, df, image, aux = _dense(sc, st.pre.feats, model, k, motion, blur, defocus, requires_grad=True)
    loss = (image * g_img.double()).sum()
    if g_dep is not None:
        loss = loss + (differentiable_depth(aux, H, W)[0] * g_dep.double()).sum()
    if g_alpha is not None:
        loss = loss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        loss = loss + (feature_map(aux, torch.from_numpy(extra).double(), H, W) * g_map.double()).sum()
    loss.backward()
    assert np.array_equal(aux["count"].numpy(), st.count)
    return st, accum, res, xyz.grad.numpy(), postprocess_feature_grads(feats.grad, band).numpy(), df.grad.numpy()


def _check(res, ex, ef, ed, groups=GROUPS):
    ok = grad_close(res.gx, ex)
    assert ok[0], ok
    for sl in groups:
        ok = grad_close(res.gf[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    scale = np.abs(ed).max()
    assert scale > 0
    assert (np.abs(res.gd - ed) <= 2e-3 * np.abs(ed) + 2e-4 * scale).all(), (res.gd, ed)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_gradients_match_dense_autograd(emus, lens, kind):
    _, _, res, ex, ef, ed = _case(emus, lens, kind, 71)
    _check(res, ex, ef, ed)


@pytest.mark.parametrize("blurred", [False, True])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_emulated_gradients_through_a_rolling_shutter(emus, lens, blurred):
    _, _, res, ex, ef, ed = _case(emus, lens, "image", 72, rolling=True, blur=BLUR if blurred else NO_BLUR)
    _check(res, ex, ef, ed)


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_emulated_gradients_with_motion_blur(emus, lens):
    _, _, res, ex, ef, ed = _case(emus, lens, "depth", 74, blur=BLUR)
    _check(res, ex, ef, ed)


def test_emulated_gradients_with_three_objects_and_the_butterfly_loop_a(emus):
    st, _, res, ex, ef, ed = _case(emus, "opencv", "image", 73, objects=3, transposed=False, band=1)
    _check(res, ex, ef, ed, groups=GROUPS[:3])  # SH columns: see the rolling-shutter test of the same name


def test_reference_defocus_gradient_matches_finite_differences():
    """The evaluator's dL/d(a, rho) by autograd against central differences (tile membership and the blend order are piecewise
    constant in (a, rho); the step is small enough to keep them)."""
    sc = _scene(79)
    feats = sc.point_cloud_features.numpy().astype(np.float32)
    g = torch.randn((32, 48, 3), generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    lens = LENSES["opencv"]
    _, _, df, image, _ = _dense(sc, feats, *lens, NO_BLUR, BLUR, DEFOCUS, requires_grad=True)
    (image * g).sum().backward()
    want = df.grad.numpy()
    h = 1e-6
    for i in range(2):
        e = np.zeros(2)
        e[i] = h
        lp = float((_dense(sc, feats, *lens, NO_BLUR, BLUR, tuple(np.add(DEFOCUS, e)))[3] * g).sum())
        lm = float((_dense(sc, feats, *lens, NO_BLUR, BLUR, tuple(np.subtract(DEFOCUS, e)))[3] * g).sum())
        assert (lp - lm) / (2 * h) == pytest.approx(want[i], rel=1e-4, abs=1e-6 * np.abs(want).max())


def test_sign_of_the_aperture_is_not_observable(emus):
    sc = _scene(81)
    a = emulated_forward_defocus(emus["emu"], emus["dfemu"], sc, "pinhole", (), NO_BLUR, NO_BLUR, DEFOCUS, False)
    b = emulated_forward_defocus(emus["emu"], emus["dfemu"], sc, "pinhole", (), NO_BLUR, NO_BLUR, (-DEFOCUS[0], DEFOCUS[1]),
                                 False)
    assert np.array_equal(a.pre.records, b.pre.records) and np.array_equal(a.image, b.image)


@pytest.mark.parametrize("kind", ["image", "depth"])
def test_defocus_gradient_is_deterministic_and_leaves_every_other_output_unchanged(emus, kind):
    st, accum, res, _, _, _ = _case(emus, "opencv", kind, 77, blur=BLUR)
    again = emulated_points_defocus(emus["emu"], emus["dfemu"], st, accum, depth=kind == "depth")
    assert np.array_equal(res.gd, again.gd) and np.array_equal(res.partials, again.partials)
    assert res.blocks == min(math.ceil(st.pre.point_offset.shape[0] / 128), 2048)
    assert np.allclose(res.partials.astype(np.float64).sum(0)[:2], res.gd, rtol=1e-5, atol=1e-6 * np.abs(res.gd).max())
    assert (res.partials[:, 2:] == 0).all()
    off = emulated_points_defocus(emus["emu"], emus["dfemu"], st, accum, depth=kind == "depth", dgrad=False)
    assert off.gd is None and np.array_equal(res.gx, off.gx) and np.array_equal(res.gf, off.gf)


# ------------------------------------------------------------------ C ABI
def _df(a=0.1, rho=0.5):
    return _lib.GsbDefocusArgs(aperture=a, inverse_focus=rho)


def test_abi_sizes_of_the_defocus_arguments():
    lib = _lib.load()
    sizes = (ctypes.c_int64 * 3)(*([-7] * 3))
    lib.gsb200_abi_sizes_defocus(sizes)
    assert sizes[0] == ctypes.sizeof(_lib.GsbDefocusArgs) == 8
    assert sizes[1] == ctypes.sizeof(_lib.GsbDefocusGradArgs) == 16
    assert sizes[2] == -7
    ext = (ctypes.c_int64 * 17)(*([-7] * 17))
    lib.gsb200_abi_sizes_ext(ext, 17)  # the extension table still ends at GsbAppearanceArgs
    assert ext[15] == ext[16] == -7
    assert lib.gsb200_defocus_grad_temp_bytes() == 2049 * 6 * 4
    for name in ("gsb200_forward_defocus", "gsb200_backward_defocus", "gsb200_defocus_grad_temp_bytes",
                 "gsb200_abi_sizes_defocus"):
        assert hasattr(lib, name) and name in _lib.EXPORTS


def test_c_entry_points_check_their_arguments_before_any_cuda_call():
    lib = _lib.load()
    fargs = _lib.GsbForwardArgs()
    bargs = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED, num_objects=1)
    ok = ctypes.c_void_p(256)
    good = _lib.GsbDefocusGradArgs(grad=ok, temp=ok)
    for d in (_df(math.nan), _df(0.1, math.inf), _df(-math.inf, 0.0)):
        assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, None, None, None, ctypes.byref(d)) == -1
        assert b"not finite" in lib.gsb200_last_error()
        assert lib.gsb200_backward_defocus(ctypes.byref(bargs), None, None, None, None, None, None, None, ctypes.byref(d),
                                           ctypes.byref(good)) == -1
        assert b"not finite" in lib.gsb200_last_error()
    blur = _lib.GsbMotionBlurArgs(motion=(ctypes.c_float * 6)(math.nan, 0, 0, 0, 0, 0))
    assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, None, None, ctypes.byref(blur), ctypes.byref(_df())) == -1
    assert b"exposure motion 0 is not finite" in lib.gsb200_last_error()
    lens = _lib.GsbLensArgs(model=7)
    assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, ctypes.byref(lens), None, None, ctypes.byref(_df())) == -1
    assert b"unknown lens model" in lib.gsb200_last_error()
    rs = _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(0.1, 0, 0, 0, 0, 0), row_time=None)
    assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, None, ctypes.byref(rs), None, ctypes.byref(_df())) == -1
    assert b"null row_time" in lib.gsb200_last_error()
    bad_grad = [(_lib.GsbDefocusGradArgs(grad=None, temp=ok), b"null grad"),
                (_lib.GsbDefocusGradArgs(grad=ok, temp=None), b"null grad"),
                (_lib.GsbDefocusGradArgs(grad=ctypes.c_void_p(258), temp=ok), b"4-byte aligned"),
                (_lib.GsbDefocusGradArgs(grad=ok, temp=ctypes.c_void_p(260)), b"16-byte aligned")]
    for g, msg in bad_grad:
        assert lib.gsb200_backward_defocus(ctypes.byref(bargs), None, None, None, None, None, None, None,
                                           ctypes.byref(_df()), ctypes.byref(g)) == -1
        assert msg in lib.gsb200_last_error()
    assert lib.gsb200_backward_defocus(ctypes.byref(bargs), None, None, None, None, None, None, None, None,
                                       ctypes.byref(good)) == -1
    assert b"needs a defocus" in lib.gsb200_last_error()
    compact = _lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED | _lib.GSB_FLAG_COMPACT_GRADS, num_objects=1)
    for g in (None, ctypes.byref(good)):
        assert lib.gsb200_backward_defocus(ctypes.byref(compact), None, None, None, None, None, None, None,
                                           ctypes.byref(_df()), g) == -4
        assert b"GSB_FLAG_COMPACT_GRADS" in lib.gsb200_last_error()
    # valid arguments reach the usual argument checks
    assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, None, None, None, ctypes.byref(_df())) == -1
    assert b"forward: null camera_intrinsics" in lib.gsb200_last_error()
    assert lib.gsb200_backward_defocus(ctypes.byref(bargs), None, None, None, None, None, None, None, ctypes.byref(_df()),
                                       ctypes.byref(good)) == -1
    assert b"backward: null pointer argument" in lib.gsb200_last_error()


def test_null_defocus_is_exactly_the_motion_blur_calls():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    rs = _lib.GsbRollingShutterArgs(motion=(ctypes.c_float * 6)(0.1, 0, 0, 0, 0, 0), row_time=fake)
    blur = _lib.GsbMotionBlurArgs(motion=(ctypes.c_float * 6)(0.1, 0, 0, 0, 0, 0))
    for lens in (None, ctypes.byref(_lib.GsbLensArgs(model=0)), ctypes.byref(_lib.GsbLensArgs(model=3))):
        for r in (None, ctypes.byref(rs)):
            for b in (None, ctypes.byref(blur)):
                fargs = _lib.GsbForwardArgs()
                want = lib.gsb200_forward_motion_blur(ctypes.byref(fargs), None, lens, r, b)
                want_msg = lib.gsb200_last_error()
                assert lib.gsb200_forward_defocus(ctypes.byref(fargs), None, lens, r, b, None) == want != 0
                assert lib.gsb200_last_error() == want_msg
                for args, extra in ((_lib.GsbBackwardArgs(flags=_lib.GSB_FLAG_BACKWARD_TRANSPOSED), (None, None, None, None)),
                                    (_lib.GsbBackwardArgs(), (fake, fake, None, None))):
                    want = lib.gsb200_backward_motion_blur(ctypes.byref(args), *extra, lens, r, b, None)
                    want_msg = lib.gsb200_last_error()
                    assert lib.gsb200_backward_defocus(ctypes.byref(args), *extra, lens, r, b, None, None) == want != 0
                    assert lib.gsb200_last_error() == want_msg


# ------------------------------------------------------------------ Python surface
def test_defocus_record_and_lens_conversion():
    d = Defocus(0.01, 2.0)
    assert d.parameters == (0.01, 0.5)
    assert Defocus(0.02).focus_distance == math.inf and Defocus(0.02).parameters == (0.02, 0.0)
    for bad in ((-0.1, 1.0), (math.nan, 1.0), (math.inf, 1.0), (0.1, 0.0), (0.1, -2.0), (0.1, math.nan)):
        with pytest.raises(ValueError):
            Defocus(*bad)
    # 50 mm at f/2, focused at 3 m, in a scene of 10 units to the metre: a 25 mm pupil = 0.25 units, focus at 30 units
    e = Defocus.from_lens(50.0, 2.0, 3.0, 10.0)
    assert e.aperture == pytest.approx(0.25) and e.focus_distance == pytest.approx(30.0)
    assert Defocus.from_lens(24.0, 8.0, math.inf, 1.0).parameters == pytest.approx((0.003, 0.0))
    for bad in ((0.0, 2.0, 1.0, 1.0), (50.0, -2.0, 1.0, 1.0), (50.0, 2.0, 1.0, math.nan), (50.0, 2.0, 0.0, 1.0)):
        with pytest.raises(ValueError):
            Defocus.from_lens(*bad)
    assert CameraInfo(torch.eye(3), 16, 16, 0).defocus is None


def _input(defocus=True, blur=False, lens=None, rolling=False):
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    sc = make_scene(64, 32, 48, 0.12, 3)
    ci = sc.camera_info
    ci = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, lens,
                    RollingShutter((0.1, 0, 0), (0, 0.02, 0)) if rolling else None,
                    MotionBlur((0.1, 0, 0), (0, 0.02, 0)) if blur else None, Defocus(0.05, 2.0) if defocus else None)
    return G.GaussianPointCloudRasterisationInput(
        point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
        point_invalid_mask=sc.point_invalid_mask, camera_info=ci, q_pointcloud_camera=sc.q_pointcloud_camera,
        t_pointcloud_camera=sc.t_pointcloud_camera)


def test_operator_configuration_of_the_defocus():
    from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as G
    Config = G.GaussianPointCloudRasterisationConfig
    with pytest.raises(ValueError, match="rgb_only"):
        G(Config(rgb_only=True), differentiable_defocus=True)
    with pytest.raises(ValueError, match="gradient_exchange"):
        G(Config(), differentiable_defocus=True, gradient_exchange=object())
    inp = _input()
    for option in ("differentiable_pose", "differentiable_intrinsics", "differentiable_distortion"):
        with pytest.raises(ValueError, match=option):
            G(Config(), **{option: True})(inp)
    op = G(Config(), differentiable_defocus=True)
    op.gradient_exchange = object()
    with pytest.raises(ValueError, match="gradient_exchange"):
        op(inp)
    op = G(Config(), differentiable_defocus=True, differentiable_rolling_shutter=True, differentiable_motion_blur=True)
    with pytest.raises(ValueError, match="point_filter_3d"):
        op(inp, point_filter_3d=torch.zeros(64))
    with pytest.raises(ValueError, match="rolling_shutter_motion"):
        op(_input(rolling=True), rolling_shutter_motion=torch.zeros(6), defocus_parameters=torch.zeros(2))
    with pytest.raises(ValueError, match="exposure_motion"):
        op(_input(blur=True), exposure_motion=torch.zeros(6))
    with pytest.raises(ValueError, match="lens_coefficients"):
        op(_input(lens=LensDistortion("opencv", (0.1, 0, 0, 0, 0))), lens_coefficients=torch.zeros(5))
    for p, msg in ((torch.zeros(3), r"\(2,\)"), (torch.zeros(2, dtype=torch.float64), "float32"),
                   ([0.0] * 2, "torch.Tensor"), (torch.tensor([math.nan, 0.0]), "finite")):
        with pytest.raises(ValueError, match=msg):
            op(inp, defocus_parameters=p)
    with pytest.raises(ValueError, match="without defocus"):
        op(_input(defocus=False), defocus_parameters=torch.zeros(2))
    with pytest.raises(ValueError, match="differentiable_defocus"):
        G(Config())(inp, defocus_parameters=torch.zeros(2))
    d = op._defocus_args(inp.camera_info, torch.tensor([-0.2, 0.25]))
    assert (d.aperture, d.inverse_focus) == pytest.approx((-0.2, 0.25))
    d = G(Config())._defocus_args(inp.camera_info)
    assert (d.aperture, d.inverse_focus) == pytest.approx((0.05, 0.5))
    assert G(Config())._defocus_args(_input(defocus=False).camera_info) is None


def _trainer(cams, fused_step=False, **kw):
    from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer as T, Scene
    sc = make_scene(64, 32, 48, 0.12, 3)
    scene = Scene(sc.point_cloud.clone().requires_grad_(True), sc.point_cloud_features.clone().requires_grad_(True),
                  sc.point_invalid_mask, sc.point_object_id)
    img = torch.zeros((3, 64, 96))
    ci = sc.camera_info
    views = [(img, sc.q_pointcloud_camera, sc.t_pointcloud_camera,
              CameraInfo(ci.camera_intrinsics * torch.tensor([[2.0], [2.0], [1.0]]), 64, 96, cam, lens, rs, mb, df))
             for cam, lens, rs, mb, df in cams]
    seen = {}

    class Factory:
        gradient_exchange = kw.pop("_exchange", None)

        def __init__(self, **kwargs):
            seen.update(kwargs)

    return T(T.TrainConfig(**kw), scene, views, rasterisation_factory=Factory, fused_step=fused_step), seen


def test_trainer_configuration_of_the_defocus():
    a = Defocus(0.05, 2.0)
    b = Defocus(0.1, math.inf)
    rs = RollingShutter((0.05, 0, 0), (0, 0, 0))
    mb = MotionBlur((0.1, 0, 0), (0, 0.02, 0))
    for rate in (-1e-3, math.nan, math.inf):
        with pytest.raises(ValueError, match="defocus_learning_rate"):
            _trainer([(0, None, None, None, a)], defocus_learning_rate=rate)
    with pytest.raises(ValueError, match="defocused"):
        _trainer([(0, None, None, None, None)], defocus_learning_rate=1e-3)
    for kw, msg in ((dict(fused_step=True), "fused_step"), (dict(pose_learning_rate=1e-3), "pose"),
                    (dict(intrinsics_learning_rate=1e-3), "intrinsics"), (dict(distortion_learning_rate=1e-3), "distortion"),
                    (dict(rolling_shutter_learning_rate=1e-3), "rolling_shutter_learning_rate"),
                    (dict(motion_blur_learning_rate=1e-3, defocus_learning_rate=1e-3), "motion_blur_learning_rate"),
                    (dict(mip_filter_3d=True), "mip_filter_3d"), (dict(_exchange=object()), "gradient exchange")):
        lens = LensDistortion("opencv", (-0.1, 0, 0, 0, 0)) if "distortion" in kw else None
        with pytest.raises(ValueError, match=msg):
            _trainer([(0, lens, rs, mb, a)], **kw)
    trainer, seen = _trainer([(0, None, None, None, a), (1, None, rs, mb, b), (0, None, None, None, None)],
                             defocus_learning_rate=1e-3)
    assert seen.get("differentiable_defocus") is True and "differentiable_motion_blur" not in seen
    assert sorted(trainer._defocus) == [0, 1]
    leaf = trainer._defocus[0]
    assert leaf.is_leaf and leaf.requires_grad and leaf.device.type == "cpu" and leaf.dtype == torch.float32
    f32 = lambda d: Defocus(float(np.float32(d.aperture)), 1 / float(np.float32(1 / d.focus_distance)))  # noqa: E731
    assert trainer.refined_defocus() == [f32(a), Defocus(float(np.float32(0.1)), math.inf), None]
    with torch.no_grad():
        leaf[0] = -0.25  # only |a| is observable
        leaf[1] = -0.1  # beyond infinity: reported at infinity
    assert trainer.refined_defocus()[0] == Defocus(0.25, math.inf)
    trainer, seen = _trainer([(0, None, None, None, a)])
    assert "differentiable_defocus" not in seen and trainer.refined_defocus() == [a]


def test_dataset_reads_the_defocus_record_key_and_downsampling_keeps_it(tmp_path):
    from PIL import Image
    from taichi_3d_gaussian_splatting_b200.image_pose_dataset import ImagePoseDataset
    from taichi_3d_gaussian_splatting_b200.trainer import downsample_image_and_camera_info
    img = tmp_path / "a.png"
    Image.fromarray(np.zeros((32, 48, 3), np.uint8)).save(img)
    base = {"image_path": str(img), "T_pointcloud_camera": np.eye(4).tolist(),
            "camera_intrinsics": [[40.0, 0, 24.0], [0, 40.0, 16.0], [0, 0, 1]], "camera_height": 32, "camera_width": 48,
            "camera_id": 0}
    records = [dict(base), dict(base, defocus={"aperture": 0.02, "focus_distance": 1.5},
                                motion_blur={"linear_velocity": [1.0, 0, 0], "angular_velocity": [0, 0.5, 0],
                                             "exposure_time": 1 / 30})]
    path = tmp_path / "poses.json"
    path.write_text(json.dumps(records))
    ds = ImagePoseDataset(str(path))
    assert ds[0][3].defocus is None
    d = ds[1][3].defocus
    assert d == Defocus(0.02, 1.5) and ds[1][3].motion_blur is not None
    for broken in ({"aperture": 0.02}, {"aperture": -1.0, "focus_distance": 1.0}, [0.02, 1.5]):
        bad = tmp_path / "bad.json"
        bad.write_text(json.dumps([dict(base, defocus=broken)]))
        with pytest.raises(ValueError, match="defocus"):
            ImagePoseDataset(str(bad))[0]
    _, ci = downsample_image_and_camera_info(torch.zeros((3, 32, 48)), ds[1][3], 2)
    assert ci.defocus == d and ci.defocus.parameters == d.parameters and ci.motion_blur == ds[1][3].motion_blur
    from taichi_3d_gaussian_splatting_b200.synthetic import SyntheticScene
    sc = make_scene(16, 32, 48, 0.12, 3)
    sc.camera_info.defocus = d
    assert SyntheticScene.to(sc, "cpu").camera_info.defocus == d
