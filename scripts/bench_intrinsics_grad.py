"""Cost of the camera-intrinsics gradient (``differentiable_intrinsics=True``, ``gsb200_backward_calib``) at a bench
configuration (default C3).

One forward of the scene per operator, then the backward of an image loss is timed repeatedly (``torch.autograd.grad`` with
``retain_graph``: no gradient accumulation kernels) in three variants that alternate within the process:
  image:           dL/dxyz and dL/dfeatures -> gsb200_backward, the default kernels;
  intrinsics:      the same plus dL/dK -> gsb200_backward_calib, the INTR per-point kernel and the finishing kernel;
  pose_intrinsics: the same plus dL/dq_pointcloud_camera and dL/dt_pointcloud_camera -> gsb200_backward_calib with a pose:
                   the combined per-point kernel (one pass) and both finishing kernels.
Each of --regions regions runs --steps timed steps of every variant (CUDA events around each backward call; the order of
the variants reverses every region), after --warmup untimed ones.  A torch.profiler pass then reports the device time per
kernel.  Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_intrinsics_grad.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:  # no nvidia-smi: the name from the runtime, the power limit unknown
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    cfg = CONFIGS[args.config]
    scene = make_scene(**cfg).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    q_pc = scene.q_pointcloud_camera.clone().requires_grad_(True)
    t_pc = scene.t_pointcloud_camera.clone().requires_grad_(True)
    ci = scene.camera_info
    K = ci.camera_intrinsics.clone().requires_grad_(True)
    camera_k = CameraInfo(K, ci.camera_height, ci.camera_width, ci.camera_id)
    Config = GPCR.GaussianPointCloudRasterisationConfig

    def render(op, q_in, t_in, camera):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask,
            camera_info=camera, q_pointcloud_camera=q_in, t_pointcloud_camera=t_in, color_max_sh_band=3))[0]

    op = GPCR(Config())
    op_intr = GPCR(Config(), differentiable_intrinsics=True)
    op_both = GPCR(Config(), differentiable_intrinsics=True, differentiable_pose=True)
    image = render(op, scene.q_pointcloud_camera, scene.t_pointcloud_camera, ci)
    image_intr = render(op_intr, scene.q_pointcloud_camera, scene.t_pointcloud_camera, camera_k)
    image_both = render(op_both, q_pc, t_pc, camera_k)
    gen = torch.Generator().manual_seed(1)
    g_img = torch.randn(image.shape, generator=gen).cuda()
    inputs = [scene.point_cloud, scene.point_cloud_features]
    variants = {
        "image": lambda: torch.autograd.grad([image], inputs, [g_img], retain_graph=True),
        "intrinsics": lambda: torch.autograd.grad([image_intr], inputs + [K], [g_img], retain_graph=True),
        "pose_intrinsics": lambda: torch.autograd.grad([image_both], inputs + [q_pc, t_pc, K], [g_img], retain_graph=True),
    }
    times = {k: [] for k in variants}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for region in range(args.regions):
        order = list(variants) if region % 2 == 0 else list(variants)[::-1]
        for k in order:
            for _ in range(args.warmup):
                variants[k]()
            for _ in range(args.steps):
                start.record()
                variants[k]()
                stop.record()
                stop.synchronize()
                times[k].append(start.elapsed_time(stop))
    kernels = {}
    for k, fn in variants.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t and ("blend_backward" in e.key or "backward_points" in e.key or "_finish" in e.key):
                per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per step
        kernels[k] = per
    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions,
           "steps": args.steps, "M": op.last_frame.num_points_in_camera, "K": op.last_frame.num_keys}
    for k, v in times.items():
        a = np.asarray(v)
        res[k] = {"median_ms": round(float(np.median(a)), 4), "p90_ms": round(float(np.percentile(a, 90)), 4),
                  "region_medians_ms": [round(float(np.median(a[i * args.steps:(i + 1) * args.steps])), 4)
                                        for i in range(args.regions)]}
    for k in list(variants)[1:]:
        res[f"{k}_over_image"] = round(res[k]["median_ms"] / res["image"]["median_ms"], 4)
    res["kernels_ms_per_step"] = kernels
    print(json.dumps(res))


if __name__ == "__main__":
    main()
