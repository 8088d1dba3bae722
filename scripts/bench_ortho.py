"""Cost of an orthographic view (``LensDistortion("orthographic", ())``, ``gsb200_forward_ortho`` / ``gsb200_backward_ortho``)
against a pinhole view of the same scene and footprint.

The scene is ``synthetic.make_aerial_scene`` (1e6 flat Gaussians on a textured ground with raised blocks, 1920 x 1072 at
0.01 scene units per pixel by default: the C3 scale of BASELINE.md).  Two views are timed, alternating within the process
(CUDA events; the order reverses every region): the nadir orthographic view of the scene, and a pinhole camera at the same
centre and orientation whose focal length (altitude / pixel size) gives the ground the same pixel size.  Forward alone (no
grad) and forward + backward of an image loss are timed.  It reports the in-view points and (tile, splat) keys of each view,
and a torch.profiler pass reports the device time per call of each stage's kernels (per-point stage, sort, tile ranges, blend
forward, loop A, per-point backward).  Prints the card name and power limit read in the same run, medians and p90 in ms, as
one JSON object.

    python scripts/bench_ortho.py [--size 1920x1072] [--points 1000000] [--regions 5] [--steps 10] [--warmup 3]
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
from taichi_3d_gaussian_splatting_b200.Camera import CameraInfo  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import make_aerial_scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="1920x1072")
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--pixel-size", type=float, default=0.01)
    ap.add_argument("--altitude", type=float, default=5.0)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ortho.py measures on a CUDA device"
    name, power = card()
    W, H = (int(v) for v in args.size.split("x"))
    res = {"card": name, "power_limit": power, "points": args.points, "size": args.size, "regions": args.regions,
           "steps": args.steps}
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    scene = make_aerial_scene(args.points, H, W, 2, pixel_size=args.pixel_size, altitude=args.altitude).to("cuda")
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    inputs = [scene.point_cloud, scene.point_cloud_features]
    q_normalised = scene.point_cloud_features.detach().clone()
    g_img = torch.randn((H, W, 3), generator=torch.Generator().manual_seed(1)).cuda()
    ortho = scene.camera_info
    f = args.altitude / args.pixel_size
    pinhole = CameraInfo(torch.tensor([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]], device="cuda"), H, W, 1)

    def render(camera):
        return op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
            point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask, camera_info=camera,
            q_pointcloud_camera=scene.q_pointcloud_camera, t_pointcloud_camera=scene.t_pointcloud_camera,
            color_max_sh_band=3))

    def step(camera, backward):
        def run():
            with torch.no_grad():  # the forward normalises q in place: every step starts from the same rows
                scene.point_cloud_features.copy_(q_normalised)
            if not backward:
                with torch.no_grad():
                    return render(camera)
            outs = render(camera)
            torch.autograd.grad([outs[0]], inputs, [g_img])
            return outs
        return run

    variants = {"ortho_forward": step(ortho, False), "pinhole_forward": step(pinhole, False),
                "ortho_forward_backward": step(ortho, True), "pinhole_forward_backward": step(pinhole, True)}
    res["counts"] = {}
    for v in ("ortho_forward", "pinhole_forward"):
        variants[v]()
        res["counts"][v.split("_")[0]] = {"M": op.last_frame.num_points_in_camera, "keys": op.last_frame.num_keys}
    times = _alternate(variants, args.regions, args.steps, args.warmup, _event_time)
    res["ms"] = {v: _stats(t, args.regions, args.steps) for v, t in times.items()}
    kernels = {}
    for v in ("ortho_forward_backward", "pinhole_forward_backward"):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                variants[v]()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t and any(k in e.key for k in ("preprocess", "pose_kernel", "sort", "tile", "blend", "backward_points")):
                per[e.key.split("(")[0][:120]] = round(t / 1e3 / args.steps, 4)  # ms per call
        kernels[v] = per
    res["kernels_ms_per_call"] = kernels
    print(json.dumps(res))


if __name__ == "__main__":
    main()
