"""Cost of the pose and intrinsics gradients through a lens (``differentiable_pose`` / ``differentiable_intrinsics`` on an
OpenCV or fisheye view, ``gsb200_backward_lens_calib``) at a bench configuration (default C3), for the lenses of
``bench_lens.py``.

1. Backward: one forward of the scene per variant, then the backward of an image loss is timed repeatedly
   (``torch.autograd.grad`` with ``retain_graph``) in five variants that alternate within the process:
     lens:              dL/dxyz and dL/dfeatures through the lens -> gsb200_backward_lens, the LENS per-point kernel;
     lens_pose:         the same plus dL/dq, dL/dt -> gsb200_backward_lens_calib (POSE);
     lens_intrinsics:   the same plus dL/dK -> gsb200_backward_lens_calib (INTR);
     lens_joint:        dL/dq, dL/dt, dL/dK and dL/dk -> gsb200_backward_lens_calib (POSE, INTR, LGRAD);
     pinhole_calib:     the pinhole view with dL/dq, dL/dt, dL/dK -> gsb200_backward_calib, for comparison.
   Each of --regions regions runs --steps timed steps of every variant (CUDA events; the order reverses every region) after
   --warmup untimed ones.  A torch.profiler pass then reports the device time per kernel.
2. Training: the autograd loop (``GaussianPointCloudTrainer.train``) on two views rendered through the lens, without camera
   refinement and with pose + intrinsics + lens refinement, --steps iterations per region after --warmup, alternating; wall
   time per iteration.
Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_lens_calib.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_intrinsics_grad import card  # noqa: E402
from bench_lens import LENSES  # noqa: E402
from bench_lens_grad import _alternate, _event_time, _stats  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene  # noqa: E402


def _kernels(fn, steps):
    """Device time per step of the per-point and finishing kernels, by torch.profiler over `steps` calls."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t and ("backward_points" in e.key or "_finish" in e.key):
            per[e.key.split("(")[0][:120]] = round(t / 1e3 / steps, 4)  # ms per step
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lens_calib.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=torch.Generator().manual_seed(1)).cuda()
    Config = GPCR.GaussianPointCloudRasterisationConfig

    def render(op, lens, q, t, K, **kw):
        camera = CameraInfo(K, ci.camera_height, ci.camera_width, ci.camera_id, lens)
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=q, t_pointcloud_camera=t, color_max_sh_band=3), **kw)[0]

    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps}
    for lens in ("opencv", "fisheye"):
        dist = LENSES[lens]
        q = scene.q_pointcloud_camera.clone().requires_grad_(True)
        t = scene.t_pointcloud_camera.clone().requires_grad_(True)
        K = ci.camera_intrinsics.clone().requires_grad_(True)
        k = torch.tensor(dist.coefficients, dtype=torch.float32, requires_grad=True)
        through = dict(camera_gradients_through_lens=True)
        ops = {"lens": GPCR(Config()), "lens_pose": GPCR(Config(), differentiable_pose=True, **through),
               "lens_intrinsics": GPCR(Config(), differentiable_intrinsics=True, **through),
               "lens_joint": GPCR(Config(), differentiable_pose=True, differentiable_intrinsics=True,
                                  differentiable_distortion=True, **through),
               "pinhole_calib": GPCR(Config(), differentiable_pose=True, differentiable_intrinsics=True)}
        images = {"lens": render(ops["lens"], dist, q.detach(), t.detach(), K.detach()),
                  "lens_pose": render(ops["lens_pose"], dist, q, t, K.detach()),
                  "lens_intrinsics": render(ops["lens_intrinsics"], dist, q.detach(), t.detach(), K),
                  "lens_joint": render(ops["lens_joint"], dist, q, t, K, lens_coefficients=k),
                  "pinhole_calib": render(ops["pinhole_calib"], None, q, t, K)}
        wrt = {"lens": inputs, "lens_pose": inputs + [q, t], "lens_intrinsics": inputs + [K],
               "lens_joint": inputs + [q, t, K, k], "pinhole_calib": inputs + [q, t, K]}
        variants = {v: (lambda v=v: torch.autograd.grad([images[v]], wrt[v], [g_img], retain_graph=True)) for v in images}
        times = _alternate(variants, args.regions, args.steps, args.warmup, _event_time)
        out = {"M": ops["lens"].last_frame.num_points_in_camera, "K": ops["lens"].last_frame.num_keys,
               "M_pinhole": ops["pinhole_calib"].last_frame.num_points_in_camera}
        for v, tm in times.items():
            out[v] = _stats(tm, args.regions, args.steps)
        out["kernels_ms_per_step"] = {v: _kernels(fn, args.steps) for v, fn in variants.items()}

        # the autograd training loop on two views through the lens, without and with joint camera refinement
        views = []
        for yaw in (0.0, 2.0):
            half = math.radians(yaw) / 2
            dq = torch.tensor([[0.0, math.sin(half), 0.0, math.cos(half)]], device="cuda")
            w0, v0, w1, v1 = dq[:, 3], dq[:, :3], scene.q_pointcloud_camera[:, 3], scene.q_pointcloud_camera[:, :3]
            qv = torch.cat([w0[:, None] * v1 + w1[:, None] * v0 + torch.linalg.cross(v0, v1),
                            (w0 * w1 - (v0 * v1).sum(-1))[:, None]], -1).contiguous()
            with torch.no_grad():
                target = render(GPCR(Config()), dist, qv, scene.t_pointcloud_camera, ci.camera_intrinsics)
            views.append((target.clamp(0, 1).permute(2, 0, 1).contiguous(), qv, scene.t_pointcloud_camera.clone(),
                          CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, 0, dist)))
        trainers = {}
        for v, rate in (("train", 0.0), ("train_joint_calibration", 1e-4)):
            cfg = GaussianPointCloudTrainer.TrainConfig(num_iterations=1, initial_downsample_factor=1,
                                                        camera_refinement_through_lens=True,
                                                        pose_learning_rate=rate, intrinsics_learning_rate=rate,
                                                        distortion_learning_rate=rate)
            sc = Scene(scene.point_cloud.detach().clone().requires_grad_(True),
                       scene.point_cloud_features.detach().clone().requires_grad_(True), scene.point_invalid_mask.clone(),
                       scene.point_object_id.clone())
            trainers[v] = GaussianPointCloudTrainer(cfg, sc, views)

        def wall(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        train_times = _alternate({v: tr.train for v, tr in trainers.items()}, args.regions, args.steps, args.warmup, wall)
        for v, tm in train_times.items():
            out[v + "_iteration"] = _stats(tm, args.regions, args.steps)
        res[lens] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
