"""Cost of the appearance grids in the fused train step (``FusedTrainStep(appearance_grids=...)``:
``gsb200_train_step_appearance``) at a bench configuration (default C3: 1e6 Gaussians, 1920 x 1072).

Three variants on one scene alternate within the process: ``none`` (gsb200_train_step), ``grid_1x1x1`` and
``grid_16x16x8``.  Each has its own scene copy and step object.  Each of --regions regions runs --steps timed steps of every
variant (CUDA events around each call; the order reverses every region) after --warmup untimed ones.  Then the slice kernels
alone (``gsb200_bilateral_grid_forward`` / ``_backward`` on the rendered image, the backward including its finishing
kernel), with the bytes each must move (forward: read the image, write the output; backward: read the image and dL/dout,
write dL/dimage) and the achieved bandwidth.  Prints the card name and power limit read in the same run, medians and p90 in
ms, as one JSON object.

    python scripts/bench_appearance.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR, _lib  # noqa: E402
from taichi_3d_gaussian_splatting_b200.appearance import identity_grids  # noqa: E402
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402

VARIANTS = {"none": None, "grid_1x1x1": (1, 1, 1), "grid_16x16x8": (16, 16, 8)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:  # no nvidia-smi: the name from the runtime, the power limit unknown
        return torch.cuda.get_device_name(0), "unknown"


def _timed(fn, n):
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def _stats(ts):
    return dict(median_ms=round(float(np.median(ts)), 4), p90_ms=round(float(np.percentile(ts, 90)), 4))


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
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        image, _, _ = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=base.point_cloud, point_cloud_features=base.point_cloud_features.clone(),
            point_object_id=base.point_object_id, point_invalid_mask=base.point_invalid_mask, camera_info=ci,
            q_pointcloud_camera=base.q_pointcloud_camera, t_pointcloud_camera=base.t_pointcloud_camera, color_max_sh_band=3))
    gt = (image.clamp(0, 1) * 0.9 + 0.05).permute(2, 0, 1).contiguous()
    steps = {}
    for name, shape in VARIANTS.items():
        sc = make_scene(**cfg).to("cuda")
        grids = identity_grids(1, shape, device="cuda") if shape else None
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2, appearance_grids=grids))

    def run(name):
        sc, step = steps[name]
        kw = {"appearance_view": 0} if VARIANTS[name] else {}
        step.run(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5, **kw)

    for name in VARIANTS:
        for _ in range(args.warmup):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in VARIANTS}
    order = list(VARIANTS)
    for region in range(args.regions):
        for name in (order if region % 2 == 0 else order[::-1]):
            times[name] += _timed(lambda: run(name), args.steps)
    name, power = card()
    out = dict(config=args.config, H=H, W=W, card=name, power_limit=power, regions=args.regions, steps=args.steps,
               skipped_steps={n: steps[n][1].num_skipped_steps for n in VARIANTS})
    for v, ts in times.items():
        out["step_" + v] = _stats(ts)

    # the slice kernels alone
    lib = _lib.load()
    img = image.contiguous()
    sliced, grad_out, grad_in = torch.empty_like(img), torch.randn_like(img) * 1e-7, torch.empty_like(img)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    image_bytes = img.numel() * 4
    for shape in ((1, 1, 1), (16, 16, 8)):
        gx, gy, gz = shape
        grid = (identity_grids(1, shape, device="cuda")[0] + 0.01 * torch.randn((12, gz, gy, gx), device="cuda")).contiguous()
        grad_grid = torch.empty_like(grid)
        tb = int(lib.gsb200_bilateral_grid_temp_bytes(H, W, gx, gy, gz))
        temp = torch.empty(tb, dtype=torch.uint8, device="cuda")
        fwd = lambda: _lib.check(lib.gsb200_bilateral_grid_forward(p(img), p(grid), H, W, gx, gy, gz, p(sliced), stream),  # noqa: E731
                                 "forward")
        bwd = lambda: _lib.check(lib.gsb200_bilateral_grid_backward(p(img), p(grid), H, W, gx, gy, gz, p(grad_out),  # noqa: E731
                                                                    p(grad_in), p(grad_grid), p(temp), tb, stream), "backward")
        for _ in range(args.warmup):
            fwd()
            bwd()
        tf, tbw = [], []
        for _ in range(args.regions):
            tf += _timed(fwd, args.steps)
            tbw += _timed(bwd, args.steps)
        key = f"kernels_{gx}x{gy}x{gz}"
        out[key] = dict(forward=_stats(tf), backward=_stats(tbw), forward_bytes=2 * image_bytes,
                        backward_bytes=3 * image_bytes,
                        forward_gb_per_s=round(2 * image_bytes / (np.median(tf) * 1e-3) / 1e9, 1),
                        backward_gb_per_s=round(3 * image_bytes / (np.median(tbw) * 1e-3) / 1e9, 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
