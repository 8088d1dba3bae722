"""Cost of the depth of field (``CameraInfo.defocus``, ``gsb200_forward_defocus`` / ``gsb200_backward_defocus``) at a bench
configuration (default C3), pinhole camera, image loss.

The focus is at the near quartile of the rendered depths, and per median blur diameter c in {0, 2, 8, 16} pixels the aperture
is a = c / (f_px |1/z_q1 - 1/z_median|) (c = 0: the pinhole camera).  The forward and the backward are timed repeatedly in
variants that alternate within the process (CUDA events; the order reverses every region):
  pinhole:       the calls without defocus (gsb200_forward, gsb200_backward);
  defocus_c:     the defocused calls without the (a, rho) gradient (preprocess_blur_kernel and backward_points_blur_kernel with
                 DEFOCUS);
  defocus_c_grad: the same with dL/d(a, rho) (the DGRAD per-point kernel, the finishing kernel and the 8-byte copy).
It reports the number of (tile, splat) keys and of blended (pixel, splat) pairs of each: a defocused splat covers more tiles
and pixels, so the sort and both blend kernels do more work as the blur grows.  That cost is part of the model.  A
torch.profiler pass then reports the device time per step of the per-point forward and backward kernels and of the blend
kernels.  Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_defocus.py [C3] [--regions 5] [--steps 20] [--warmup 3]
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
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo, Defocus  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_defocus.py measures on a CUDA device"
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    ci = scene.camera_info
    inputs = [scene.point_cloud, scene.point_cloud_features]
    g_img = torch.randn((ci.camera_height, ci.camera_width, 3), generator=torch.Generator().manual_seed(1)).cuda()
    q_normalised = scene.point_cloud_features.detach().clone()
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_defocus=True)

    def render(camera, **kw):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3), **kw)

    pinhole = CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id)
    with torch.no_grad():
        render(pinhole)
        depths = op.last_frame.point_in_camera[:, 2].double()
        zq, zm = float(depths.quantile(0.25)), float(depths.median())
        scene.point_cloud_features.copy_(q_normalised)
    fx = float(ci.camera_intrinsics[0, 0])

    def camera(diameter):
        return CameraInfo(ci.camera_intrinsics, ci.camera_height, ci.camera_width, ci.camera_id,
                          defocus=Defocus(diameter / (fx * abs(1 / zq - 1 / zm)), zq))

    def step(cam, grad):
        p = torch.tensor(cam.defocus.parameters, dtype=torch.float32, requires_grad=True) if grad else None

        def run():
            with torch.no_grad():  # the forward normalises q in place: every step starts from the same rows
                scene.point_cloud_features.copy_(q_normalised)
            kw = {"defocus_parameters": p} if grad else {}
            outs = render(cam, **kw)
            torch.autograd.grad([outs[0]], inputs + ([p] if grad else []), [g_img])
            return outs
        return run

    variants = {"pinhole": step(pinhole, False)}
    for diameter in (2, 8, 16):
        variants[f"defocus_{diameter}"] = step(camera(diameter), False)
        variants[f"defocus_{diameter}_grad"] = step(camera(diameter), True)
    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps,
           "near_quartile_depth": round(zq, 4), "median_depth": round(zm, 4),
           "apertures": {d: round(camera(d).defocus.aperture, 6) for d in (2, 8, 16)}}
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
