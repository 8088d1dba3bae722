"""Cost of the supervision terms in the fused train step (``FusedTrainStep`` with ``depth_weight`` / ``mask_weight`` /
``background``: ``gsb200_train_step_aux``) at a bench configuration (default C3: 1e6 Gaussians, 1920 x 1072).

Four variants on one scene alternate within the process, on synthetic targets rendered from the scene itself (its depth
map with 60 % of the pixels set to NaN or 0, like a LiDAR target, and its accumulated alpha as the mask):
  image:        the image loss alone -> gsb200_train_step;
  depth:        + the depth term;
  mask_random:  + the mask term and a random background colour per step;
  all:          depth + mask + random background.
Each variant has its own scene copy and step object (so their Adam states do not mix).  Each of --regions regions runs
--steps timed steps of every variant (CUDA events around each call; the order reverses every region) after --warmup
untimed ones.  Prints the card name and power limit read in the same run, per-step medians and p90 in ms, as one JSON
object.

    python scripts/bench_supervised_step.py [C3] [--regions 5] [--steps 20] [--warmup 3]
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
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep, SupervisionTargets  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402

VARIANTS = {"image": (0.0, 0.0, False), "depth": (0.5, 0.0, False), "mask_random": (0.0, 0.5, True),
            "all": (0.5, 0.5, True)}


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
    base = make_scene(**cfg).to("cuda")
    ci = base.camera_info
    H, W = ci.camera_height, ci.camera_width
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig(), differentiable_alpha=True)
    with torch.no_grad():
        image, depth, _, alpha = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=base.point_cloud, point_cloud_features=base.point_cloud_features.clone(),
            point_object_id=base.point_object_id, point_invalid_mask=base.point_invalid_mask, camera_info=ci,
            q_pointcloud_camera=base.q_pointcloud_camera, t_pointcloud_camera=base.t_pointcloud_camera, color_max_sh_band=3))
    g = torch.Generator(device="cuda").manual_seed(0)
    gt = (image.clamp(0, 1) * 0.9 + 0.05).permute(2, 0, 1).contiguous()
    d = (depth * (1 + 0.05 * torch.randn(depth.shape, generator=g, device="cuda"))).contiguous()
    holes = torch.rand(depth.shape, generator=g, device="cuda")
    d[holes < 0.3] = float("nan")
    d[(holes >= 0.3) & (holes < 0.6)] = 0.0
    targets = SupervisionTargets(depth=d, mask=alpha.clone().contiguous())
    bg = torch.empty(3, device="cuda")
    steps = {}
    for name, (w_d, w_m, _) in VARIANTS.items():
        sc = make_scene(**cfg).to("cuda")
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2, depth_weight=w_d,
                                          mask_weight=w_m))

    def run(name):
        sc, step = steps[name]
        _, _, random_bg = VARIANTS[name]
        if random_bg:
            torch.rand(3, generator=g, out=bg)
        supervised = name != "image"
        step.run(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5,
                 targets=targets if supervised else None, background=bg if random_bg else None)

    for name in VARIANTS:
        for _ in range(args.warmup):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in VARIANTS}
    order = list(VARIANTS)
    for region in range(args.regions):
        for name in (order if region % 2 == 0 else order[::-1]):
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(name)
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1))
    skipped = {name: steps[name][1].num_skipped_steps for name in VARIANTS}
    name, power = card()
    out = dict(config=args.config, H=H, W=W, card=name, power_limit=power, regions=args.regions, steps=args.steps,
               skipped_steps=skipped)
    for v, ts in times.items():
        out[v] = dict(median_ms=round(float(np.median(ts)), 4), p90_ms=round(float(np.percentile(ts, 90)), 4))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
