"""Cost of the rolling shutter (``CameraInfo.rolling_shutter``, ``gsb200_forward_rolling_shutter`` /
``gsb200_backward_rolling_shutter``) at a bench configuration (default C3), without a lens and with the ``opencv`` lens of
``bench_lens.py``.

1. Forward + backward: per camera (global shutter, rolling shutter) the forward and the backward of an image loss are timed
   repeatedly in variants that alternate within the process (CUDA events; the order reverses every region):
     gs:       the global-shutter calls (gsb200_forward / _lens, gsb200_backward / _lens);
     rs:       the rolling-shutter calls without the motion gradient (preprocess_rs_kernel, backward_points_rs_kernel);
     rs_mgrad: the same with dL/dm (differentiable_rolling_shutter: the MGRAD per-point kernel, the finishing kernel and the
               24-byte read-back of the gradient).
   A torch.profiler pass then reports the device time per step of the per-point forward and backward kernels.
2. Training: the autograd loop (``GaussianPointCloudTrainer.train``) on one view, global shutter, rolling shutter, and rolling
   shutter with ``rolling_shutter_learning_rate``; wall time per iteration.
Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_rolling_shutter.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
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
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, RollingShutter  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene  # noqa: E402

MOTION = RollingShutter((0.03, -0.05, 0.02), (0.01, 0.02, -0.01))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rolling_shutter.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=torch.Generator().manual_seed(1)).cuda()
    q_normalised = scene.point_cloud_features.detach().clone()

    def render(op, camera, **kw):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3), **kw)[0]

    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps}
    for lens_name in ("pinhole", "opencv"):
        lens = LENSES[lens_name] if lens_name != "pinhole" else None
        gs_cam = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, lens)
        rs_cam = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, lens, MOTION)
        op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_rolling_shutter=True)
        m = torch.tensor(MOTION.motion, dtype=torch.float32, requires_grad=True)

        def step(camera, **kw):
            def run():
                with torch.no_grad():  # the forward normalises q in place: every step starts from the same rows
                    scene.point_cloud_features.copy_(q_normalised)
                image = render(op, camera, **kw)
                torch.autograd.grad([image], inputs + ([kw["rolling_shutter_motion"]] if kw else []), [g_img])
            return run

        variants = {"gs": step(gs_cam), "rs": step(rs_cam), "rs_mgrad": step(rs_cam, rolling_shutter_motion=m)}
        times = _alternate(variants, args.regions, args.steps, args.warmup, _event_time)
        out = {"M": op.last_frame.num_points_in_camera, "K": op.last_frame.num_keys}
        for v, t in times.items():
            out[v + "_forward_backward"] = _stats(t, args.regions, args.steps)
        kernels = {}
        for v, fn in variants.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = getattr(e, "cuda_time_total", 0.0)
                if t and ("preprocess" in e.key or "backward_points" in e.key or "_finish" in e.key):
                    per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per step
            kernels[v] = per
        out["kernels_ms_per_step"] = kernels

        # the autograd training loop on one view: global shutter, rolling shutter, rolling shutter with motion refinement
        with torch.no_grad():
            target = render(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), rs_cam).clamp(0, 1).permute(2, 0, 1)
        trainers = {}
        for v, camera, rate in (("train_gs", gs_cam, 0.0), ("train_rs", rs_cam, 0.0), ("train_rs_refine", rs_cam, 1e-3)):
            cfg = GaussianPointCloudTrainer.TrainConfig(num_iterations=1, initial_downsample_factor=1,
                                                        rolling_shutter_learning_rate=rate)
            sc = Scene(scene.point_cloud.detach().clone().requires_grad_(True),
                       scene.point_cloud_features.detach().clone().requires_grad_(True), scene.point_invalid_mask.clone(),
                       scene.point_object_id.clone())
            trainers[v] = GaussianPointCloudTrainer(
                cfg, sc, [(target.contiguous(), scene.q_pointcloud_camera, scene.t_pointcloud_camera, camera)])

        def wall(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        train_times = _alternate({v: tr.train for v, tr in trainers.items()}, args.regions, args.steps, args.warmup, wall)
        for v, t in train_times.items():
            out[v + "_iteration"] = _stats(t, args.regions, args.steps)
        res[lens_name] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
