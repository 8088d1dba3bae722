"""Cost of the per-Gaussian feature channels (``point_extra_features``) at a bench configuration (default C3).

Variants C = 0 (no features: gsb200_forward / gsb200_backward, the default kernels) and C = 3, 8, 16 (gsb200_forward_ext /
gsb200_backward_ext, the CF instantiations), alternated within the process: each of --regions regions runs --steps timed
steps of every variant (the order reverses every region) after --warmup untimed ones.  A step is one forward call and one
backward call (loss = <image, g> + <feature map, g_F>), each timed with CUDA events.  A torch.profiler pass then reports the
device time per step of the blend kernels.  The line the feature replaces: a user without it renders ceil(C / 3) more
frames through the colour channels, each a whole forward + backward -- that cost is ceil(C / 3) x the C = 0 step.
Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_extra_features.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_depth_grad import card  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="C3")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    scene = make_scene(**CONFIGS[args.config]).to("cuda")
    N = scene.point_cloud.shape[0]
    scene.point_cloud.requires_grad_(True)
    scene.point_cloud_features.requires_grad_(True)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    inp = GPCR.GaussianPointCloudRasterisationInput(
        point_cloud=scene.point_cloud, point_cloud_features=scene.point_cloud_features,
        point_object_id=scene.point_object_id, point_invalid_mask=scene.point_invalid_mask,
        camera_info=scene.camera_info, q_pointcloud_camera=scene.q_pointcloud_camera,
        t_pointcloud_camera=scene.t_pointcloud_camera, color_max_sh_band=3)
    H, W = scene.camera_info.camera_height, scene.camera_info.camera_width
    gen = torch.Generator().manual_seed(1)
    g_img = torch.randn((H, W, 3), generator=gen).cuda()
    widths = (0, 3, 8, 16)
    feats = {C: torch.randn((N, C), generator=gen).cuda().requires_grad_(True) for C in widths if C}
    g_map = {C: torch.randn((H, W, C), generator=gen).cuda() for C in widths if C}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def step(C, timed):
        ev[0].record()
        outs = op(inp) if C == 0 else op(inp, point_extra_features=feats[C])
        ev[1].record()
        if C == 0:
            torch.autograd.backward([outs[0]], [g_img])
        else:
            torch.autograd.backward([outs[0], outs[-1]], [g_img, g_map[C]])
        ev[2].record()
        ev[2].synchronize()
        if timed:
            return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
        return None

    fwd = {C: [] for C in widths}
    bwd = {C: [] for C in widths}
    for region in range(args.regions):
        order = widths if region % 2 == 0 else widths[::-1]
        for C in order:
            for _ in range(args.warmup):
                step(C, False)
            for _ in range(args.steps):
                f, b = step(C, True)
                fwd[C].append(f)
                bwd[C].append(b)
    kernels = {}
    for C in widths:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step(C, False)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0.0)
            if t and "blend_" in e.key:
                name = "blend_forward" if "blend_forward" in e.key else "blend_backward"
                per[name] = round(per.get(name, 0.0) + t / 1e3 / args.steps, 4)  # ms per step
        kernels[C] = per
    name, power = card()
    res = {"config": args.config, "card": name, "power_limit": power, "regions": args.regions, "steps": args.steps,
           "N": N, "M": op.last_frame.num_points_in_camera, "K": op.last_frame.num_keys}
    stat = lambda a: {"median_ms": round(float(np.median(a)), 4), "p90_ms": round(float(np.percentile(a, 90)), 4)}  # noqa: E731
    base = float(np.median(np.asarray(fwd[0]) + np.asarray(bwd[0])))
    for C in widths:
        tot = np.asarray(fwd[C]) + np.asarray(bwd[C])
        r = {"forward": stat(fwd[C]), "backward": stat(bwd[C]), "step": stat(tot), "kernels_ms_per_step": kernels[C]}
        if C:
            r["added_ms"] = round(float(np.median(tot)) - base, 4)
            r["extra_colour_passes"] = math.ceil(C / 3)
            r["extra_colour_passes_ms"] = round(math.ceil(C / 3) * base, 4)
        res[f"C{C}"] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
