"""-m gpu: rolling-shutter cameras in the CUDA operator (``CameraInfo.rolling_shutter``, ``gsb200_forward_rolling_shutter`` /
``gsb200_backward_rolling_shutter``, ``differentiable_rolling_shutter``, ``TrainConfig.rolling_shutter_learning_rate``).

Forward outputs, point gradients and dL/dm against the float64 dense evaluator (``torch_reference_rolling_shutter``) on small
scenes, for a pinhole, an opencv and a fisheye camera and image, depth, alpha and feature-map losses, and an image loss under
both loop-A kernels; at C3 full size zero motion against the global-shutter call and bit-identical repeats with a real motion;
training through the rolling shutter against training as a global shutter; and the trainer refining the motion from zero."""
import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion, RollingShutter
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene

from gpu_helpers import cuda_scene, n
from helpers import grad_close
from test_gpu_pose_gradient import _scene
from torch_reference import postprocess_feature_grads
from torch_reference_depth import differentiable_depth
from torch_reference_features import feature_map
from torch_reference_rolling_shutter import dense_render_rs

pytestmark = pytest.mark.gpu

Config = GPCR.GaussianPointCloudRasterisationConfig
Input = GPCR.GaussianPointCloudRasterisationInput
GROUPS = (slice(0, 4), slice(4, 7), slice(7, 8), slice(8, 56))
LENSES = {
    "pinhole": None,
    "opencv": LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": LensDistortion("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}
MOTION = (0.06, -0.09, 0.04, 0.05, -0.08, 0.06)


def _input(sc, lens, rs, band=3):
    ci = sc.camera_info
    return Input(point_cloud=sc.point_cloud, point_cloud_features=sc.point_cloud_features, point_object_id=sc.point_object_id,
                 point_invalid_mask=sc.point_invalid_mask,
                 camera_info=CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, lens, rs),
                 q_pointcloud_camera=sc.q_pointcloud_camera, t_pointcloud_camera=sc.t_pointcloud_camera,
                 color_max_sh_band=band)


@pytest.mark.parametrize("kind", ["image", "depth", "alpha", "features"])
@pytest.mark.parametrize("lens", ["pinhole", "opencv", "fisheye"])
def test_cuda_rolling_shutter_matches_dense_evaluator(lens, kind, backward_impl="transposed", seed=81):
    scene = _scene(seed)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    sc = cuda_scene(scene, requires_grad=True)
    dist = LENSES[lens]
    rs = RollingShutter(MOTION[:3], MOTION[3:])
    op = GPCR(Config(), exact_exp=True, backward_impl=backward_impl, differentiable_depth=kind == "depth",
              differentiable_alpha=kind == "alpha", differentiable_rolling_shutter=True)
    m = torch.tensor(MOTION, dtype=torch.float32, requires_grad=True)
    g = torch.Generator().manual_seed(seed + 100)
    g_img = torch.randn((H, W, 3), generator=g)
    extra = g_map = None
    if kind == "features":
        extra = torch.randn((scene.point_cloud.shape[0], 5), generator=g)
        g_map = torch.randn((H, W, 5), generator=g)
    inp = _input(sc, dist, rs)
    outs = op(inp, rolling_shutter_motion=m) if extra is None else \
        op(inp, point_extra_features=extra.cuda(), rolling_shutter_motion=m)
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
    feats_n = sc.point_cloud_features.detach().cpu()  # q normalised in place by the forward, as the evaluator assumes
    xyz = scene.point_cloud.clone().double().requires_grad_(True)
    feats = feats_n.double().requires_grad_(True)
    mr = torch.tensor(MOTION, dtype=torch.float64, requires_grad=True)
    ref, aux = dense_render_rs(xyz, feats, scene.point_invalid_mask, scene.point_object_id, scene.camera_info.camera_intrinsics,
                               scene.q_pointcloud_camera, scene.t_pointcloud_camera, H, W,
                               dist.model if dist else "pinhole", dist.coefficients if dist else (), mr)
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
    ok = grad_close(n(sc.point_cloud.grad), xyz.grad.numpy())  # the path's criterion: 1e-3 rel + 1e-5 of the max
    assert ok[0], ok
    ef = postprocess_feature_grads(feats.grad, 3).numpy()
    for sl in GROUPS:
        ok = grad_close(n(sc.point_cloud_features.grad)[:, sl], ef[:, sl])
        assert ok[0], (sl, ok)
    em = mr.grad.numpy()
    ok = grad_close(m.grad.numpy(), em, floor_frac=1e-3)  # the same bar for dL/dm: 1e-3 of its largest entry
    assert ok[0], (m.grad, em, ok)


@pytest.mark.parametrize("lens", ["pinhole", "fisheye"])
def test_image_loss_rolling_shutter_gradient_under_the_butterfly_loop_a(lens):
    test_cuda_rolling_shutter_matches_dense_evaluator(lens, "image", backward_impl="butterfly", seed=83)


def _full_size(cameras, motion_grad=False):
    scene = make_scene(**CONFIGS["C3"]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    feats0 = scene.point_cloud_features.detach().clone()
    op = GPCR(Config(), differentiable_depth=True, differentiable_rolling_shutter=motion_grad)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    gen = torch.Generator().manual_seed(3)
    g_img, g_dep = torch.randn((H, W, 3), generator=gen).cuda(), torch.randn((H, W), generator=gen).cuda()
    out = []
    for lens, rs in cameras:
        with torch.no_grad():
            scene.point_cloud_features.copy_(feats0)
        kw = {"rolling_shutter_motion": torch.tensor(rs.motion, requires_grad=True)} if motion_grad else {}
        image, depth, _ = op(_input(scene, lens, rs), **kw)
        leaves = [scene.point_cloud, scene.point_cloud_features] + ([kw["rolling_shutter_motion"]] if motion_grad else [])
        loss = (image * g_img).sum() + (depth * g_dep).sum()
        grads = torch.autograd.grad([loss], leaves)
        fr = op.last_frame
        out.append(dict(image=n(image), depth=n(depth), gx=n(grads[0]), gf=n(grads[1]), records=n(fr.records),
                        offsets=n(fr.point_id_in_camera_list), pic=n(fr.point_in_camera),
                        gm=n(grads[2]) if motion_grad else None))
    return out


def test_full_size_zero_motion_matches_the_global_shutter_and_real_motion_repeats_bit_for_bit():
    zero = RollingShutter((0.0,) * 3, (0.0,) * 3)
    for lens in (None, LENSES["fisheye"]):
        gs, rz = _full_size([(lens, None), (lens, zero)])
        # every op of the rolling-shutter path is exact for zero motion: the per-point stage, the sort and the blend
        for k in ("records", "offsets", "pic", "image", "depth"):
            assert np.array_equal(gs[k], rz[k]), k
        for k in ("gx", "gf"):  # loop A adds with float atomics: the accumulator rows repeat up to rounding
            ok = grad_close(rz[k], gs[k])
            assert ok[0], (k, ok)
    real = RollingShutter(MOTION[:3], MOTION[3:])
    a, b = _full_size([(None, real), (None, real)], motion_grad=True)
    for k in ("records", "offsets", "pic", "image", "depth"):
        assert np.array_equal(a[k], b[k]), k
    assert np.isfinite(a["gm"]).all() and (a["gm"] != 0).all()
    ok = grad_close(a["gm"], b["gm"], rtol=1e-4)
    assert ok[0], ok


# ------------------------------------------------------------------ training through a rolling shutter
def _motions():
    """A different motion per training view (a hand-held walk-through: the camera pans and drifts one way, then the other)."""
    from trainer_helpers import YAWS
    out = []
    for i in range(len(YAWS)):
        s = 1.0 if i % 2 == 0 else -1.0
        out.append(RollingShutter((0.12 * s, -0.06, 0.03), (0.02, 0.08 * s, -0.03 * s)))
    return out


def _targets(hidden, motions):
    from trainer_helpers import H, W, poses
    op = GPCR(Config())
    K = hidden.camera_info.camera_intrinsics.cuda()
    pc, feat = hidden.point_cloud.cuda(), hidden.point_cloud_features.clone().cuda()
    mask, obj = hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda()
    out = []
    for (q, t), rs in zip(poses(), motions):
        with torch.no_grad():
            img = op(Input(point_cloud=pc, point_cloud_features=feat, point_object_id=obj, point_invalid_mask=mask,
                           camera_info=CameraInfo(K, H, W, 0, None, rs), q_pointcloud_camera=q.cuda(),
                           t_pointcloud_camera=t.cuda(), color_max_sh_band=3))[0]
        out.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q.cuda(), t.cuda()))
    return K, out


def test_training_through_the_rolling_shutter_beats_training_as_a_global_shutter():
    """Ground truth rendered through a different rolling-shutter motion per view; a perturbed copy of the scene trained on it
    with the views' rolling shutter and with rolling_shutter=None, the validation PSNR of each on its own views."""
    from trainer_helpers import H, W, hidden_scene, initial_scene, train_config
    hidden = hidden_scene(n=600)
    motions = _motions()
    K, targets = _targets(hidden, motions)
    rs_views = [(img, q, t, CameraInfo(K, H, W, 0, None, rs)) for (img, q, t), rs in zip(targets, motions)]
    gs_views = [(img, q, t, CameraInfo(K, H, W, 0)) for img, q, t in targets]
    psnrs = {}
    for name, views in (("rolling", rs_views), ("global", gs_views)):
        trainer = GaussianPointCloudTrainer(train_config(200), initial_scene(hidden, device="cuda"), views)
        trainer.train()
        psnrs[name] = trainer.validation(views)
    print(f"training through a rolling shutter: validation PSNR {psnrs['rolling']:.2f} dB, as a global shutter "
          f"{psnrs['global']:.2f} dB")
    assert psnrs["rolling"] > psnrs["global"] + 3.0


def test_trainer_refines_the_motion_from_zero():
    """A frozen scene (learning rates 0) and views rendered through a rolling shutter; the trainer starts every view from zero
    motion.  |m - m*| must fall below a quarter of its starting value |m*|, and the validation PSNR through the refined
    motions must beat the zero motion's (the loss falls)."""
    from trainer_helpers import H, W, hidden_scene, train_config
    hidden = hidden_scene(n=600)
    motions = _motions()
    K, targets = _targets(hidden, motions)
    zero = RollingShutter((0.0,) * 3, (0.0,) * 3)

    def views(rss):
        return [(img, q, t, CameraInfo(K, H, W, 0, None, rs)) for (img, q, t), rs in zip(targets, rss)]

    cfg = train_config(400)
    cfg.feature_learning_rate = cfg.position_learning_rate = 0.0
    cfg.initial_downsample_factor = 1
    cfg.rolling_shutter_learning_rate = 4e-3
    pc, feat = hidden.point_cloud.cuda(), hidden.point_cloud_features.clone().cuda()
    mask, obj = hidden.point_invalid_mask.cuda(), hidden.point_object_id.cuda()
    scene = Scene(pc.clone().requires_grad_(True), feat.clone().requires_grad_(True), mask.clone(), obj.clone())
    trainer = GaussianPointCloudTrainer(cfg, scene, views([zero] * len(motions)))
    trainer.train()
    refined = trainer.refined_rolling_shutter()
    err = [np.linalg.norm(np.subtract(r.motion, m.motion)) / np.linalg.norm(m.motion) for r, m in zip(refined, motions)]
    psnr_refined, psnr_zero = trainer.validation(views(refined)), trainer.validation(views([zero] * len(motions)))
    print(f"trainer: |m - m*| / |m*| per view {[f'{e:.3f}' for e in err]}, validation PSNR {psnr_refined:.2f} dB through the "
          f"refined motions, {psnr_zero:.2f} dB through zero motion")
    assert max(err) < 0.25
    assert psnr_refined > psnr_zero
