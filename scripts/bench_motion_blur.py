"""Cost of the motion blur (``CameraInfo.motion_blur``, ``gsb200_forward_motion_blur`` / ``gsb200_backward_motion_blur``) at a
bench configuration (default C3), pinhole camera, image loss.

Per median streak length L in {0, 4, 16} pixels (L = 0: the camera without blur; a sideways pan with a little rotation sized so
that the median splat streak |d| is L px), the forward and the backward are timed repeatedly in variants that alternate
within the process (CUDA events; the order reverses every region):
  sharp:        the calls without blur (gsb200_forward, gsb200_backward);
  blur_L:       the blurred calls without the motion gradient (preprocess_blur_kernel, backward_points_blur_kernel);
  blur_L_grad:  the same with dL/dm_b (the BGRAD per-point kernel, the finishing kernel and the 24-byte read-back).
It reports the number of (tile, splat) keys and of blended (pixel, splat) pairs of each: a blurred splat covers more tiles and
pixels, so the sort and both blend kernels do more work as the streak grows.  That cost is part of the model.  A
torch.profiler pass then reports the device time per step of the per-point forward and backward kernels.  Prints the card name
and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_motion_blur.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_intrinsics_grad import card  # noqa: E402
from bench_lens_grad import _alternate, _event_time, _stats  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, MotionBlur  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_motion_blur.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=torch.Generator().manual_seed(1)).cuda()
    q_normalised = scene.point_cloud_features.detach().clone()
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_motion_blur=True)

    def render(camera, **kw):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3), **kw)

    sharp_cam = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id)
    with torch.no_grad():
        render(sharp_cam)
        z = float(op.last_frame.point_in_camera[:, 2].median())
        scene.point_cloud_features.copy_(q_normalised)
    fx = float(ci.camera_intrinsics[0, 0])

    def camera(length):
        if length == 0:
            return sharp_cam
        v = length * z / fx  # a sideways pan: |d| ~ fx |v| / z
        return CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id,
                          motion_blur=MotionBlur((0.8 * v, 0.5 * v, 0.1 * v), (0.2 * v / z, -0.3 * v / z, 0.0)))

    def step(cam, grad):
        m = torch.tensor(cam.motion_blur.motion, requires_grad=True) if grad else None

        def run():
            with torch.no_grad():  # the forward normalises q in place: every step starts from the same rows
                scene.point_cloud_features.copy_(q_normalised)
            kw = {"exposure_motion": m} if grad else {}
            outs = render(cam, **kw)
            torch.autograd.grad([outs[0]], inputs + ([m] if grad else []), [g_img])
            return outs
        return run

    variants = {"sharp": step(sharp_cam, False)}
    for length in (4, 16):
        variants[f"blur_{length}"] = step(camera(length), False)
        variants[f"blur_{length}_grad"] = step(camera(length), True)
    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps,
           "median_depth": round(z, 4)}
    counts = {}
    for v, fn in variants.items():
        outs = fn()
        counts[v] = {"M": op.last_frame.num_points_in_camera, "keys": op.last_frame.num_keys,
                     "pixel_splat_pairs": int(outs[2].sum())}
    res["counts"] = counts
    times = _alternate(variants, args.regions, args.steps, args.warmup, _event_time)
    res["forward_backward"] = {v: _stats(t, args.regions, args.steps) for v, t in times.items()}
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
            if t and ("preprocess" in e.key or "backward_points" in e.key or "_finish" in e.key or "blend" in e.key
                      or "sort" in e.key):
                per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per step
        kernels[v] = per
    res["kernels_ms_per_step"] = kernels
    print(json.dumps(res))


if __name__ == "__main__":
    main()
