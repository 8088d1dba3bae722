"""Cost of the feature term in the fused train step (``FusedTrainStep`` with ``extra_features`` / ``feature_loss``:
``gsb200_train_step_ext``) at a bench configuration (default C3: 1e6 Gaussians, 1920 x 1072).

Four variants on one scene alternate within the process:
  image:        the image loss alone -> gsb200_train_step;
  ce8:          + a cross-entropy feature term on C = 8 channels (random labels, 10 % of the pixels unlabelled);
  l2_16:        + an l2 feature term on C = 16 channels (a random target map);
  ce8_all:      ce8 + the depth and mask terms and a random background colour per step.
Each variant has its own scene copy and step object (so their Adam states do not mix).  Each of --regions regions runs
--steps timed steps of every variant (CUDA events around each call; the order reverses every region) after --warmup
untimed ones.  Prints the card name and power limit read in the same run, per-step medians and p90 in ms, as one JSON
object.

    python scripts/bench_feature_step.py [C3] [--regions 6] [--steps 20] [--warmup 3]
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

VARIANTS = {"image": (None, 0, False), "ce8": ("cross_entropy", 8, False), "l2_16": ("l2", 16, False),
            "ce8_all": ("cross_entropy", 8, True)}


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
    ap.add_argument("--regions", type=int, default=6)
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
    labels = torch.randint(-1, 9, (H, W), generator=g, device="cuda", dtype=torch.int32)  # -1 and 8: unlabelled
    feature_map = torch.randn((H, W, 16), generator=g, device="cuda")
    d = depth.clone().contiguous()
    targets = SupervisionTargets(depth=d, mask=alpha.clone().contiguous(), labels=labels, features=feature_map)
    bg = torch.empty(3, device="cuda")
    steps = {}
    for name, (kind, C, all_terms) in VARIANTS.items():
        sc = make_scene(**cfg).to("cuda")
        kw = {}
        if kind is not None:
            F = 0.1 * torch.randn((sc.point_cloud.shape[0], C), generator=g, device="cuda")
            kw = dict(extra_features=F, feature_loss=kind, feature_weight=0.5)
        if all_terms:
            kw.update(depth_weight=0.5, mask_weight=0.5)
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2, **kw))

    def run(name):
        sc, step = steps[name]
        kind, _, all_terms = VARIANTS[name]
        if all_terms:
            torch.rand(3, generator=g, out=bg)
        step.run(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5,
                 targets=targets if kind is not None else None, background=bg if all_terms else None)

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
