"""Cost of the lens-coefficient gradient (``differentiable_distortion=True``, ``gsb200_backward_lens_grad``) at a bench
configuration (default C3), for the ``opencv`` and ``fisheye`` lenses of ``bench_lens.py``.

1. Backward: one forward of the scene per lens, then the backward of an image loss is timed repeatedly
   (``torch.autograd.grad`` with ``retain_graph``) in two variants that alternate within the process:
     lens:      dL/dxyz and dL/dfeatures -> gsb200_backward_lens, the LENS per-point kernel;
     lens_grad: the same plus dL/dlens_coefficients -> gsb200_backward_lens_grad, the LGRAD per-point kernel, the finishing
                kernel and the 20-byte read-back of the gradient to the host tensor.
   Each of --regions regions runs --steps timed steps of every variant (CUDA events; the order reverses every region) after
   --warmup untimed ones.  A torch.profiler pass then reports the device time per kernel.
2. Training: the autograd loop (``GaussianPointCloudTrainer.train``) on one view rendered through the lens, with and without
   ``distortion_learning_rate``, --steps iterations per region after --warmup, alternating; wall time per iteration.
Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_lens_grad.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_intrinsics_grad import card  # noqa: E402
from bench_lens import LENSES  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402
from taichi_3d_gaussian_splatting_b200.trainer import GaussianPointCloudTrainer, Scene  # noqa: E402


def _stats(v, regions, steps):
    a = np.asarray(v)
    return {"median_ms": round(float(np.median(a)), 4), "p90_ms": round(float(np.percentile(a, 90)), 4),
            "region_medians_ms": [round(float(np.median(a[i * steps:(i + 1) * steps])), 4) for i in range(regions)]}


def _alternate(variants, regions, steps, warmup, timer):
    times = {k: [] for k in variants}
    for region in range(regions):
        order = list(variants) if region % 2 == 0 else list(variants)[::-1]
        for k in order:
            for _ in range(warmup):
                variants[k]()
            for _ in range(steps):
                times[k].append(timer(variants[k]))
    return times


def _event_time(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lens_grad.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=torch.Generator().manual_seed(1)).cuda()

    def render(op, camera, **kw):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3), **kw)[0]

    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps}
    for lens in ("opencv", "fisheye"):
        dist = LENSES[lens]
        camera = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, dist)
        op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_distortion=True)
        k = torch.tensor(dist.coefficients, dtype=torch.float32, requires_grad=True)
        image = render(op, camera)
        image_k = render(op, camera, lens_coefficients=k)
        variants = {
            "lens": lambda: torch.autograd.grad([image], inputs, [g_img], retain_graph=True),
            "lens_grad": lambda: torch.autograd.grad([image_k], inputs + [k], [g_img], retain_graph=True),
        }
        times = _alternate(variants, args.regions, args.steps, args.warmup, _event_time)
        out = {"M": op.last_frame.num_points_in_camera, "K": op.last_frame.num_keys}
        for v, t in times.items():
            out[v] = _stats(t, args.regions, args.steps)
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
                if t and ("backward_points" in e.key or "_finish" in e.key):
                    per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per step
            kernels[v] = per
        out["kernels_ms_per_step"] = kernels

        # the autograd training loop on one view through the lens, with and without lens refinement
        with torch.no_grad():
            target = render(GPCR(GPCR.GaussianPointCloudRasterisationConfig()), camera).clamp(0, 1).permute(2, 0, 1)
        view = [(target.contiguous(), scene.q_pointcloud_camera, scene.t_pointcloud_camera, camera)]
        trainers = {}
        for v, rate in (("train", 0.0), ("train_distortion", 1e-3)):
            cfg = GaussianPointCloudTrainer.TrainConfig(num_iterations=1, initial_downsample_factor=1,
                                                        distortion_learning_rate=rate)
            sc = Scene(scene.point_cloud.detach().clone().requires_grad_(True),
                       scene.point_cloud_features.detach().clone().requires_grad_(True), scene.point_invalid_mask.clone(),
                       scene.point_object_id.clone())
            trainers[v] = GaussianPointCloudTrainer(cfg, sc, view)

        def wall(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        train_times = _alternate({v: tr.train for v, tr in trainers.items()}, args.regions, args.steps, args.warmup, wall)
        for v, t in train_times.items():
            out[v + "_iteration"] = _stats(t, args.regions, args.steps)
        res[lens] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
