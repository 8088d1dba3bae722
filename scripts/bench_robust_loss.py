"""Cost of the per-pixel loss weights in the fused train step (``FusedTrainStep(robust=...)``: ``gsb200_train_step_robust``)
at a bench configuration (default C3: 1e6 Gaussians, 1920 x 1072).

Four variants on one scene alternate within the process: ``plain`` (gsb200_train_step), ``robust`` (the inlier mask of each
iteration's residual), ``robust_static`` (the mask and a static weight), all against a target with residuals spread over
many bins, and ``robust_converged`` (the mask against the scene's own render: nearly every residual falls into the lowest
bins, the case where same-address shared atomics would serialise).  Each has its own scene copy and step object.  Each of
--regions regions runs --steps timed steps of every variant (CUDA events around each call; the order reverses every region)
after --warmup untimed ones.  Then one profiled run each of ``robust_static`` and ``robust_converged`` (``torch.profiler``,
CUDA activity) gives the new kernels' device times, with the bytes each must move per step, counted from the shapes:
  histogram: x 12 B + gt 12 B + s 4 B per pixel;  mask: the same over the 18 x 18 halo of every tile (324 / 256 of it) plus
  x and gt once more for the composite, 4 B of w and 12 B of x' written;  post: w 4 B + x 12 B + dL/dx' 12 B read, 12 B
  written.
Prints the card name and power limit read in the same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_robust_loss.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_appearance import _stats, _timed, card  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR  # noqa: E402
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep  # noqa: E402
from taichi_3d_gaussian_splatting_b200.loss import RobustLossConfig, SupervisionTargets  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402

KERNELS = ("robust_hist_kernel", "robust_mask_kernel", "robust_post_kernel")


def kernel_bytes(H, W):
    n = H * W
    halo = 324 / 256
    return {"robust_hist_kernel": 28 * n, "robust_mask_kernel": int(28 * halo * n + 24 * n + 16 * n),
            "robust_post_kernel": 40 * n}


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
    H, W = int(ci.camera_height), int(ci.camera_width)
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        image, _, _ = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=base.point_cloud, point_cloud_features=base.point_cloud_features.clone(),
            point_object_id=base.point_object_id, point_invalid_mask=base.point_invalid_mask, camera_info=ci,
            q_pointcloud_camera=base.q_pointcloud_camera, t_pointcloud_camera=base.t_pointcloud_camera, color_max_sh_band=3))
    gt = (image.clamp(0, 1) * 0.9 + 0.05).permute(2, 0, 1).contiguous()
    gt[:, H // 4:H // 2, W // 3:W // 2] = torch.tensor([0.9, 0.1, 0.5], device="cuda")[:, None, None]  # a distractor
    static = torch.ones((H, W), device="cuda")
    static[:H // 8] = 0.0
    robust = RobustLossConfig(inlier_quantile=0.5)  # RobustNeRF's median: the most pixels to drop
    converged = image.clamp(0, 1).permute(2, 0, 1).contiguous()
    variants = {"plain": (None, None, gt), "robust": (robust, None, gt), "robust_static": (robust, static, gt),
                "robust_converged": (robust, None, converged)}
    steps = {}
    for name, (robust, _, _) in variants.items():
        sc = make_scene(**cfg).to("cuda")
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2, robust=robust))

    def run(name):
        sc, step = steps[name]
        _, s, target = variants[name]
        kw = {"targets": SupervisionTargets(loss_weight=s)} if s is not None else {}
        step.run(target, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5, **kw)

    for name in variants:
        for _ in range(args.warmup):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in variants}
    order = list(variants)
    for region in range(args.regions):
        for name in (order if region % 2 == 0 else order[::-1]):
            times[name] += _timed(lambda: run(name), args.steps)
    card_name, power = card()
    out = dict(config=args.config, H=H, W=W, card=card_name, power_limit=power, regions=args.regions, steps=args.steps,
               skipped_steps={n: steps[n][1].num_skipped_steps for n in variants},
               inlier_fraction=float(steps["robust"][1].robust_stats[0]),
               threshold_converged=float(steps["robust_converged"][1].robust_stats[1]))
    for v, ts in times.items():
        out["step_" + v] = _stats(ts)
    for v in ("robust", "robust_static", "robust_converged"):
        out[f"step_{v}_minus_plain_ms"] = round(out["step_" + v]["median_ms"] - out["step_plain"]["median_ms"], 4)

    # the new kernels' device times: one profiled run per variant, of its own (the profiler slows the host)
    from torch.profiler import ProfilerActivity, profile
    nbytes = kernel_bytes(H, W)
    for v in ("robust_static", "robust_converged"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                run(v)
            torch.cuda.synchronize()
        per = {k: [] for k in KERNELS}
        for ev in prof.events():
            for k in KERNELS:
                if k in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                    per[k].append(ev.device_time_total / 1e3)
        total_ms = 0.0
        kernels = {}
        for k, ts in per.items():
            if not ts:
                kernels[k] = "not found in the trace"
                continue
            st = _stats(ts)
            total_ms += st["median_ms"]
            kernels[k] = dict(**st, calls=len(ts), bytes=nbytes[k], gb_per_s=round(nbytes[k] / (st["median_ms"] * 1e-3) / 1e9, 1))
        out["kernels_" + v] = dict(kernels, total_median_ms=round(total_ms, 4))
    out["kernels_total_bytes"] = sum(nbytes.values())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
