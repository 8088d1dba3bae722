"""Cost and effect of the 3D smoothing filter (``mip_filter``, ``point_filter_3d``, ``gsb200_train_step_filter3d``).

1. The views kernel (``gsb200_filter3d_from_views``) at N = 1e6 rows (C3's points) with V in {50, 300} views (CUDA events
   around --launches calls, median of --regions regions; 3e8 row-view tests at V = 300).
2. The fused train step at a bench configuration (default C3) without and with the filter, alternating in one process
   (--regions regions of --steps timed steps each after --warmup untimed ones; CUDA events around each call).
3. Effect: a synthetic scene (``synthetic.make_scene``, 4 training views) fitted at 1/4 resolution, then rendered at full
   resolution and at 2x focal length (the full-resolution image of a camera with twice the focal length), with and without the
   filter; PSNR against the ground-truth scene rendered with the same camera.
Prints the card name and power limit read in the same run, as one JSON object.

    python scripts/bench_mip_filter.py [C3] [--regions 5] [--steps 20] [--warmup 3] [--fit-iterations 300]
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_appearance import _stats, _timed, card  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo  # noqa: E402
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep  # noqa: E402
from taichi_3d_gaussian_splatting_b200.mip_filter import compute_filter_3d  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene, psnr  # noqa: E402

Input = GPCR.GaussianPointCloudRasterisationInput


def _yaw_views(ci, yaws, device="cuda"):
    out = []
    for yaw in yaws:
        half = math.radians(yaw) / 2
        out.append((torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device=device),
                    torch.zeros((1, 3), device=device), ci))
    return out


def bench_views(args):
    sc = make_scene(**CONFIGS["C3"]).to("cuda")
    res = {}
    for V in (50, 300):
        views = _yaw_views(sc.camera_info, [-20.0 + 40.0 * k / (V - 1) for k in range(V)])
        run = lambda: compute_filter_3d(sc.point_cloud, sc.point_invalid_mask, sc.point_object_id, views, 0.8)  # noqa: E731
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.regions):
            ts += [t / args.launches for t in _timed(lambda: [run() for _ in range(args.launches)], 1)]
        res[f"views_kernel_V{V}"] = _stats(ts)
    return res


def bench_step(args):
    cfg = CONFIGS[args.config]
    base = make_scene(**cfg).to("cuda")
    ci = base.camera_info
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        image, _, _ = op(Input(point_cloud=base.point_cloud, point_cloud_features=base.point_cloud_features.clone(),
                               point_object_id=base.point_object_id, point_invalid_mask=base.point_invalid_mask,
                               camera_info=ci, q_pointcloud_camera=base.q_pointcloud_camera,
                               t_pointcloud_camera=base.t_pointcloud_camera, color_max_sh_band=3))
    gt = (image.clamp(0, 1) * 0.9 + 0.05).permute(2, 0, 1).contiguous()
    f3d = compute_filter_3d(base.point_cloud, base.point_invalid_mask, base.point_object_id, _yaw_views(ci, (0.0, 5.0, -5.0)),
                            0.8)
    steps = {}
    for name in ("none", "filter"):
        sc = make_scene(**cfg).to("cuda")
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2))

    def run(name):
        sc, step = steps[name]
        kw = {"filter_3d": f3d} if name == "filter" else {}
        step.run(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5, **kw)

    for name in steps:
        for _ in range(args.warmup):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in steps}
    order = list(steps)
    for region in range(args.regions):
        for name in (order if region % 2 == 0 else order[::-1]):
            times[name] += _timed(lambda: run(name), args.steps)
    out = {"step_" + k: _stats(v) for k, v in times.items()}
    out["step_filter_minus_none_ms"] = round(out["step_filter"]["median_ms"] - out["step_none"]["median_ms"], 4)
    out["skipped_steps"] = {n: s[1].num_skipped_steps for n, s in steps.items()}
    return out


def bench_psnr(args):
    H, W = 256, 384
    truth = make_scene(30_000, H, W, 0.004, 21, sh_degree=1)
    truth.point_cloud[:, 2] = truth.point_cloud[:, 2] * 0.5 + 1.0
    truth = truth.to("cuda")
    K = truth.camera_info.camera_intrinsics
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())

    def render(features, xyz, mask, q, t, ci, f3d=None):
        with torch.no_grad():
            kw = {"point_filter_3d": f3d} if f3d is not None else {}
            return op(Input(point_cloud=xyz, point_cloud_features=features.clone(), point_object_id=truth.point_object_id[:1]
                            .expand(xyz.shape[0]).contiguous(), point_invalid_mask=mask, camera_info=ci,
                            q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3), **kw)[0]

    yaws = (-6.0, -2.0, 2.0, 6.0)
    views = []
    for q, t, ci in _yaw_views(CameraInfo(K, H, W, 0), yaws):
        img = render(truth.point_cloud_features, truth.point_cloud, truth.point_invalid_mask, q, t, ci)
        views.append((img.clamp(0, 1).permute(2, 0, 1).contiguous(), q, t, ci))
    K2 = K.clone()
    K2[0, 0] *= 2
    K2[1, 1] *= 2
    tests = {"full": CameraInfo(K, H, W, 0), "focal_2x": CameraInfo(K2, H, W, 0)}
    out = {}
    for mip in (False, True):
        g = torch.Generator().manual_seed(4)
        n = truth.point_cloud.shape[0]
        xyz = truth.point_cloud.cpu() + 0.02 * torch.randn((n, 3), generator=g)
        feat = truth.point_cloud_features.cpu().clone()
        feat[:, 4:7] += 0.3 * torch.randn((n, 3), generator=g)
        feat[:, 7] = 0.5
        scene = Scene(point_cloud=xyz.cuda().requires_grad_(True), point_cloud_features=feat.cuda().requires_grad_(True),
                      point_invalid_mask=torch.zeros(n, dtype=torch.int8, device="cuda"),
                      point_object_id=torch.zeros(n, dtype=torch.int32, device="cuda"))
        cfg = GaussianPointCloudTrainer.TrainConfig(
            num_iterations=args.fit_iterations, feature_learning_rate=5e-3, position_learning_rate=1e-4,
            initial_downsample_factor=4, half_downsample_factor_interval=10 ** 9, increase_color_max_sh_band_interval=100.0,
            mip_filter_3d=mip)
        cfg.adaptive_controller_config.num_iterations_warm_up = 10 ** 9
        cfg.loss_function_config.enable_regularization = False
        trainer = GaussianPointCloudTrainer(cfg, scene, views, fused_step=True)
        trainer.train()
        f3d = trainer.filter_3d()
        for name, ci in tests.items():
            q, t = views[1][1], views[1][2]
            gt = render(truth.point_cloud_features, truth.point_cloud, truth.point_invalid_mask, q, t, ci)
            pred = render(scene.point_cloud_features.detach(), scene.point_cloud.detach(), scene.point_invalid_mask, q, t, ci,
                          f3d)
            out[f"psnr_{name}_{'filter' if mip else 'none'}"] = round(
                psnr(pred.clamp(0, 1).permute(2, 0, 1), gt.clamp(0, 1).permute(2, 0, 1)), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--fit-iterations", type=int, default=300)
    args = ap.parse_args()
    name, power = card()
    out = dict(config=args.config, card=name, power_limit=power)
    out.update(bench_views(args))
    out.update(bench_step(args))
    out.update(bench_psnr(args))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
