"""-m gpu: motion blur in the CUDA operator (``CameraInfo.motion_blur``, ``gsb200_forward_motion_blur`` /
``gsb200_backward_motion_blur``, ``differentiable_motion_blur``, ``TrainConfig.motion_blur_learning_rate``).

Forward outputs, point gradients and dL/dm_b against the float64 dense evaluator (``torch_reference_motion_blur``) on the small
scenes of ``test_gpu_rolling_shutter``, for every lens and loss, with and without a rolling shutter, under both loop-A kernels;
at C3 full size zero exposure motion against the call without blur and bit-identical repeats with a real motion; the blurred
render against the mean of 64 sharp renders over the exposure (the physics the model approximates); and training on averaged
sharp renders with and without the model, and the trainer refining a rough motion."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion, MotionBlur, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from gpu_helpers import cuda_scene, n
from helpers import grad_close
from test_gpu_pose_gradient import _scene
from torch_reference import postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_motion_blur import dense_render_blur
from torch_reference_rolling_shutter import rodrigues

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput
GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "pinhole": None,
    "opencv": LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": LensDistortion("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
RS_MOTION = (0.06, -0.09, 0.04, 0.05, -0.08, 0.06)
BLUR = (0.05, 0.03, -0.02, -0.02, 0.03, 0.01)


def _input(sc, lens, rs, mb, band=3, q=None, t=None):
    ci = sc.camera_info
    return Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                 point_invalid_mask=sc.point_invalid_mask,
                 camera_info=CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, lens, rs, mb),
                 q_pointcloud_camera=sc.q_pointcloud_camera if q is None else q,
                 t_pointcloud_camera=sc.t_pointcloud_camera if t is None else t, color_max_sh_band=band)


@pytest.mark.parametrize("rolling", [False, True])
@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_cuda_motion_blur_matches_dense_evaluator(lens, kind, rolling, backward_impl="transposed", seed=81):
    scene = _scene(seed)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    dist = LENSES[lens]
    rs = RollingShutter(RS_MOTION[:3], RS_MOTION[3:]) if rolling else None
    mb = MotionBlur(BLUR[:3], BLUR[3:])
    op = GPCR(Config(), exact_exp=True, backward_impl=backward_impl, differentiable_depth=kind == "depth",
              differentiable_alpha=kind == "alpha", differentiable_motion_blur=True)
    m = torch.tensor(BLUR, dtype=torch.float32, requires_grad=True)
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    extra = g_map = None
    if kind == "features":
        extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g)
        g_map = torch.randn((H, W, 5), generator=g)
    inp = _input(sc, dist, rs, mb)
    outs = op(inp, exposure_motion=m) if extra is None else op(inp, point_extra_features=extra.cuda(), exposure_motion=m)
    image, depth = outs[0], outs[1]
    loss = (image * g_img.cuda()).sum()
    g_dep = g_alpha = None
    if kind == "depth":
        g_dep = torch.randn((H, W), generator=g)
        loss = loss + (depth * g_dep.cuda()).sum()
    if kind == "alpha":
        g_alpha = torch.randn((H, W), generator=g)
        loss = loss + (outs[3] * g_alpha.cuda()).sum()
    if kind == "features":
        loss = loss + (outs[-1] * g_map.cuda()).sum()
    loss.backward()
    assert m.grad is not None and m.grad.device.type == "cpu"
    feats_n = sc.point_cloud_features.detach().cpu()
    xyz = scene.point_cloud.clone().double().requires_grad_(True)
    feats = feats_n.double().requires_grad_(True)
    mr = torch.tensor(BLUR, dtype=torch.float64, requires_grad=True)
    ref, aux = dense_render_blur(xyz, feats, scene.point_invalid_mask, scene.point_object_id,
                                 scene.camera_info.camera_intrinsics, scene.q_pointcloud_camera, scene.t_pointcloud_camera, H, W,
                                 dist.model if dist else "pinhole", dist.coefficients if dist else (),
                                 RS_MOTION if rolling else (0.0,) * 6, mr)
    assert float(aux["streak"].detach().max()) > 2.0
    ref_depth, _ = differentiable_depth(aux, H, W)
    assert np.abs(n(image) - ref.detach().numpy()).max() < 1e-4
    assert np.abs(n(depth) - ref_depth.detach().numpy()).max() < 1e-3
    assert op.last_frame.num_points_in_camera == aux["ids"].shape[0]
    rloss = (ref * g_img.double()).sum()
    if g_dep is not None:
        rloss = rloss + (ref_depth * g_dep.double()).sum()
    if g_alpha is not None:
        assert np.abs(n(outs[3]) - aux["acc_alpha"].detach().numpy()).max() < 1e-4
        rloss = rloss + (aux["acc_alpha"] * g_alpha.double()).sum()
    if g_map is not None:
        fm = feature_map(aux, extra.double(), H, W)
        assert np.abs(n(outs[-1]) - fm.detach().numpy()).max() < 1e-4
        rloss = rloss + (fm * g_map.double()).sum()
    rloss.backward()
    ok = grad_close(n(sc.point_cloud.grad), xyz.grad.numpy())
    assert ok[0], ok
    ef = postprocess_feature_grads(feats.grad, 3).numpy()
    for sl in GROUPS:
        ok = grad_close(n(sc.point_cloud_features.grad)[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    ok = grad_close(m.grad.numpy(), mr.grad.numpy(), floor_frac=1e-3)
    assert ok[0], (m.grad, mr.grad, ok)


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_image_loss_motion_blur_gradient_under_the_butterfly_loop_a(lens):
    test_cuda_motion_blur_matches_dense_evaluator(lens, "image", False, backward_impl="butterfly", seed=83)


def _full_size(cameras, blur_grad=False):
    scene = make_scene(**CONFIGS["C3"]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    feats0 = scene.point_cloud_features.detach().clone()
    op = GPCR(Config(), differentiable_depth=True, differentiable_motion_blur=blur_grad)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    gen = torch.Generator().manual_seed(3)
    g_img, g_dep = torch.randn((H, W, 3), generator=gen).cuda(), torch.randn((H, W), generator=gen).cuda()
    out = []
    for lens, mb in cameras:
        with torch.no_grad():
            scene.point_cloud_features.copy_(feats0)
        kw = {"exposure_motion": torch.tensor(mb.motion, requires_grad=True)} if blur_grad else {}
        image, depth, _ = op(_input(scene, lens, None, mb), **kw)
        leaves = [scene.point_cloud, scene.point_cloud_features] + ([kw["exposure_motion"]] if blur_grad else [])
        loss = (image * g_img).sum() + (depth * g_dep).sum()
        grads = torch.autograd.grad([loss], leaves)
        fr = op.last_frame
        out.append(dict(image=n(image), depth=n(depth), gx=n(grads[0]), gf=n(grads[1]), records=n(fr.records),
                        offsets=n(fr.point_id_in_camera_list), pic=n(fr.point_in_camera), keys=n(fr.sorted_keys),
                        gm=n(grads[2]) if blur_grad else None))
    return out


def test_full_size_zero_motion_matches_the_call_without_blur_and_real_motion_repeats_bit_for_bit():
    zero = MotionBlur((0.0,) * 3, (0.0,) * 3)
    for lens in (None, LENSES["fisheye"]):
        sharp, bz = _full_size([(lens, None), (lens, zero)])
        for k in ("records", "offsets", "pic", "keys", "image", "depth"):
            assert np.array_equal(sharp[k], bz[k]), k
        for k in ("gx", "gf"):  # loop A adds with float atomics: the accumulator rows repeat up to rounding
            ok = grad_close(bz[k], sharp[k])
            assert ok[0], (k, ok)
    real = MotionBlur((0.03, -0.05, 0.02), (0.01, 0.02, -0.01))
    a, b = _full_size([(None, real), (None, real)], blur_grad=True)
    for k in ("records", "offsets", "pic", "keys", "image", "depth"):
        assert np.array_equal(a[k], b[k]), k
    assert np.isfinite(a["gm"]).all() and (a["gm"] != 0).all()
    ok = grad_close(a["gm"], b["gm"], rtol=1e-4)
    assert ok[0], ok


# ------------------------------------------------------------------ the physics: the mean of sharp renders over the exposure
def _pose_at(q, t, m, s):
    """(q, t) (camera -> scene, xyzw) of the sharp camera at exposure time s in [-1/2, 1/2]: W(s) = Rd(s) W,
    tw(s) = Rd(s) tw + s v with (W, tw) the scene -> camera map of (q, t) and Rd(s) = exp(s [w]x)."""
    R = Rotation.from_quat(q / np.linalg.norm(q)).as_matrix()
    Wm, tw = R.T, -R.T @ t
    Rd = rodrigues(torch.tensor(s * np.asarray(m[3:]))[None, :]).numpy()[0]
    W1, t1 = Rd @ Wm, Rd @ tw + s * np.asarray(m[:3])
    return Rotation.from_matrix(W1.T).as_quat(), -W1.T @ t1


def _sharp_mean(op, sc, q, t, m, samples=64):
    acc = None
    for k in range(samples):
        s = (k + 0.5) / samples - 0.5
        qk, tk = _pose_at(q, t, m, s)
        with torch.no_grad():
            img = op(_input(sc, None, None, None, q=torch.tensor(qk[None], dtype=torch.float32, device="cuda"),
                            t=torch.tensor(tk[None], dtype=torch.float32, device="cuda")))[0].double()
        acc = img if acc is None else acc + img
    return acc / samples


def _streak_motion(sc, op, length):
    """A sideways pan with a little rotation whose median splat streak is about ``length`` pixels."""
    with torch.no_grad():
        op(_input(sc, None, None, None))
    z = float(op.last_frame.point_in_camera[:, 2].median())
    fx = float(sc.camera_info.camera_intrinsics[0, 0])
    v = length * z / fx
    return (0.8 * v, 0.5 * v, 0.1 * v, 0.2 * v / z, -0.3 * v / z, 0.05)


def test_blurred_render_is_close_to_the_mean_of_sharp_renders_over_the_exposure():
    from trainer_helpers import hidden_scene
    sc = cuda_scene(hidden_scene(n=600))
    op = GPCR(Config())
    q, t = sc.q_pointcloud_camera[0].double().cpu().numpy(), sc.t_pointcloud_camera[0].double().cpu().numpy()
    ratios = {}
    for length in (2, 8, 16):
        m = _streak_motion(sc, op, length)
        truth = _sharp_mean(op, sc, q, t, m)
        with torch.no_grad():
            blurred = op(_input(sc, None, None, MotionBlur(m[:3], m[3:])))[0].double()
            sharp = op(_input(sc, None, None, None))[0].double()
        e_blur = float((blurred - truth).abs().mean())
        e_sharp = float((sharp - truth).abs().mean())
        ratios[length] = e_blur / e_sharp
        print(f"streak ~{length} px: mean |blurred - truth| {e_blur:.5f}, mean |sharp - truth| {e_sharp:.5f}, "
              f"ratio {ratios[length]:.3f}")
    # measured on an H100 80GB HBM3 at 700 W: 0.303 / 0.262 / 0.246 for 2 / 8 / 16 px (DESIGN section 3)
    for length, r in ratios.items():
        assert r < 0.45, (length, ratios)


# ------------------------------------------------------------------ training on averaged sharp renders
def _motions():
    from trainer_helpers import YAWS
    out = []
    for i in range(len(YAWS)):
        s = 1.0 if i % 2 == 0 else -1.0
        out.append((0.10 * s, -0.05, 0.02, 0.01, 0.04 * s, -0.02 * s))
    return out


def _blurred_targets(hidden, motions, samples=32):
    from trainer_helpers import poses
    sc = cuda_scene(hidden)
    op = GPCR(Config())
    out = []
    for (q, t), m in zip(poses(), motions):
        img = _sharp_mean(op, sc, q[0].double().numpy(), t[0].double().numpy(), m, samples).float()
        out.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q.cuda(), t.cuda()))
    return sc.camera_info.camera_intrinsics, out


def _held_out_psnr(trainer, hidden):
    """PSNR of sharp renders of the trained scene against sharp renders of the hidden scene at poses between the training
    views."""
    from trainer_helpers import H, W
    op = GPCR(Config())
    sc = cuda_scene(hidden)
    K = sc.camera_info.camera_intrinsics
    psnrs = []
    for yaw in (-4.0, 0.0, 4.0):
        half = math.radians(yaw) / 2
        q = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device="cuda")
        tt = torch.zeros((1, 3), device="cuda")
        with torch.no_grad():
            want = op(_input(sc, None, None, None, q=q, t=tt))[0].clamp(0, 1)
            s = trainer.scene
            got = op(Input(point_cloud=s.point_cloud, point_cloud_features=s.point_cloud_features,
                           point_object_id=s.point_object_id, point_invalid_mask=s.point_invalid_mask,
                           camera_info=CameraInfo(K, H, W, 0), q_pointcloud_camera=q, t_pointcloud_camera=tt,
                           color_max_sh_band=3))[0].clamp(0, 1)
        psnrs.append(float(-10 * torch.log10(((got - want) ** 2).mean())))
    return float(np.mean(psnrs))


def test_training_with_the_blur_model_beats_training_without_it():
    from trainer_helpers import H, W, hidden_scene, initial_scene, train_config
    hidden = hidden_scene(n=600)
    motions = _motions()
    K, targets = _blurred_targets(hidden, motions)
    blurred = [(img, q, t, CameraInfo(K, H, W, 0, motion_blur=MotionBlur(m[:3], m[3:]))) for (img, q, t), m in
               zip(targets, motions)]
    sharp = [(img, q, t, CameraInfo(K, H, W, 0)) for img, q, t in targets]
    psnrs = {}
    for name, views in (("blur", blurred), ("sharp", sharp)):
        trainer = GaussianPointCloudTrainer(train_config(300), initial_scene(hidden, device="cuda"), views)
        trainer.train()
        psnrs[name] = _held_out_psnr(trainer, hidden)
    print(f"held-out sharp PSNR: trained with the blur model {psnrs['blur']:.2f} dB, without {psnrs['sharp']:.2f} dB")
    assert psnrs["blur"] > psnrs["sharp"] + 2.5  # measured: 36.41 against 31.28 dB (DESIGN section 3)


def _dd(m):
    """The observable part of an exposure motion: the outer product of its 6 values (blind to the sign)."""
    m = np.asarray(m, np.float64)
    return np.outer(m, m)


def test_trainer_refines_a_rough_exposure_motion():
    """A frozen scene and views of averaged sharp renders; the trainer starts from the true motion scaled by 0.5 and rotated
    by about 20 degrees in the 6-space; the error of m m^T (sign-blind) must fall."""
    from trainer_helpers import H, W, hidden_scene, train_config
    hidden = hidden_scene(n=600)
    motions = _motions()
    K, targets = _blurred_targets(hidden, motions)
    rng = np.random.default_rng(0)
    starts = []
    for m in motions:
        m = np.asarray(m)
        u = rng.normal(size=6)
        u -= u.dot(m) / m.dot(m) * m
        u *= np.linalg.norm(m) / np.linalg.norm(u)
        a = math.radians(20.0)
        starts.append(0.5 * (math.cos(a) * m + math.sin(a) * u))
    cfg = train_config(300)
    cfg.feature_learning_rate = cfg.position_learning_rate = 0.0
    cfg.initial_downsample_factor = 1
    cfg.motion_blur_learning_rate = 2e-3
    pc, feat = hidden.point_cloud.cuda(), hidden.point_cloud_features.clone().cuda()
    mask, obj = hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda()
    scene = Scene(pc.clone().requires_grad_(True), feat.clone().requires_grad_(True), mask.clone(), obj.clone())
    views = [(img, q, t, CameraInfo(K, H, W, 0, motion_blur=MotionBlur(tuple(s[:3]), tuple(s[3:]))))
             for (img, q, t), s in zip(targets, starts)]
    trainer = GaussianPointCloudTrainer(cfg, scene, views)
    trainer.train()
    refined = trainer.refined_motion_blur()
    before = [np.linalg.norm(_dd(s) - _dd(m)) / np.linalg.norm(_dd(m)) for s, m in zip(starts, motions)]
    after = [np.linalg.norm(_dd(r.motion) - _dd(m)) / np.linalg.norm(_dd(m)) for r, m in zip(refined, motions)]
    cos = [abs(np.dot(r.motion, m)) / (np.linalg.norm(r.motion) * np.linalg.norm(m)) for r, m in zip(refined, motions)]
    print(f"exposure-motion refinement: |m m^T - m* m*^T| / |m* m*^T| per view before {[f'{e:.3f}' for e in before]}, after "
          f"{[f'{e:.3f}' for e in after]}; |cos| after {[f'{c:.3f}' for c in cos]}")
    # measured: 0.788 before, 0.18-0.29 after, |cos| >= 0.985 (DESIGN section 3)
    assert np.mean(after) < 0.5 * np.mean(before)
    assert min(cos) > 0.95
