"""Cost of lens distortion (``CameraInfo.distortion``, ``gsb200_forward_lens`` / ``gsb200_backward_lens``) at a bench
configuration (default C3).

Three cameras on the same scene and K: pinhole (``distortion=None``: the default kernels), ``opencv`` (k1 k2 p1 p2 k3) and
``fisheye`` (k1..k4).  The forward+backward step of an image loss (forward, then ``torch.autograd.grad`` of the image) is
timed with CUDA events; each of --regions regions runs --steps timed steps of every camera after --warmup untimed ones, and
the order of the cameras reverses every region.  A torch.profiler pass per camera then reports the device time of the
per-point forward (``preprocess*kernel``) and the per-point backward (``backward_points*kernel``) per step.  Prints the
card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_lens.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_intrinsics_grad import card  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, LensDistortion  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402

LENSES = {
    "pinhole": None,
    "opencv": LensDistortion("opencv", (-0.12, 0.03, 1e-3, -2e-3, -0.004)),
    "fisheye": LensDistortion("fisheye", (0.06, -0.012, 0.003, -0.0005)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lens.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    ops = {k: GPCR(GPCR.GaussianPointCloudRasterisationConfig()) for k in LENSES}
    gen = torch.Generator().manual_seed(1)
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=gen).cuda()
    frames = {}

    def step(k):
        camera = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id, LENSES[k])
        image = ops[k](GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3))[0]
        torch.autograd.grad([image], inputs, [g_img])

    times = {k: [] for k in LENSES}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for region in range(args.regions):
        order = list(LENSES) if region % 2 == 0 else list(LENSES)[::-1]
        for k in order:
            for _ in range(args.warmup):
                step(k)
            for _ in range(args.steps):
                start.record()
                step(k)
                stop.record()
                stop.synchronize()
                times[k].append(start.elapsed_time(stop))
            frames[k] = (ops[k].last_frame.num_points_in_camera, ops[k].last_frame.num_keys)
    kernels = {}
    for k in LENSES:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step(k)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t and ("preprocess" in e.key or "backward_points" in e.key):
                per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per step
        kernels[k] = per
    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps,
           "lenses": {k: (None if v is None else [v.model, list(v.coefficients)]) for k, v in LENSES.items()}}
    for k, v in times.items():
        a = np.asarray(v)
        res[k] = {"M": frames[k][0], "K": frames[k][1], "step_median_ms": round(float(np.median(a)), 4),
                  "step_p90_ms": round(float(np.percentile(a, 90)), 4),
                  "region_medians_ms": [round(float(np.median(a[i * args.steps:(i + 1) * args.steps])), 4)
                                        for i in range(args.regions)],
                  "per_point_kernels_ms_per_step": kernels[k]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
