"""Cost of MCMC densification in the fused train step (``FusedTrainStep(mcmc=...)``: ``gsb200_train_step_mcmc``) at a bench
configuration (default C3: 1e6 Gaussians, 1920 x 1072).

Two variants on one scene alternate within the process: ``none`` (gsb200_train_step) and ``mcmc`` (the regulariser and the
position noise in the same call).  Each has its own scene copy and step object.  Each of --regions regions runs --steps timed
steps of both (CUDA events around each call; the order reverses every region) after --warmup untimed ones.  Then the two
per-iteration kernels alone (``gsb200_mcmc_regulariser``, ``gsb200_mcmc_noise``; many launches between one pair of events)
with the bytes each must move -- regulariser: 1 mask byte + 16 B of the row + 16 B of the gradient read, 16 B written;
noise: 1 mask byte + 32 B of the row + 12 B of xyz read, 12 B written, per valid row -- and the achieved bandwidth, and one
relocation of 5 % of the rows (``gsb200_mcmc_relocate``, both kernels).  Prints the card name and power limit read in the
same run, medians and p90 in ms, as one JSON object.

    python scripts/bench_mcmc.py [C3] [--regions 5] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_appearance import _stats, _timed, card  # noqa: E402
from taichi_3d_gaussian_splatting_b200 import GaussianPointCloudRasterisation as GPCR, _lib  # noqa: E402
from taichi_3d_gaussian_splatting_b200.fused_step import FusedTrainStep  # noqa: E402
from taichi_3d_gaussian_splatting_b200.mcmc import GaussianPointMCMCController, MCMCConfig, MCMCMoments  # noqa: E402
from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene  # noqa: E402

LAUNCHES = 50  # kernel launches between one pair of events


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
    N = base.point_cloud.shape[0]
    n_valid = int((base.point_invalid_mask == 0).sum())
    op = GPCR(GPCR.GaussianPointCloudRasterisationConfig())
    with torch.no_grad():
        image, _, _ = op(GPCR.GaussianPointCloudRasterisationInput(
            point_cloud=base.point_cloud, point_cloud_features=base.point_cloud_features.clone(),
            point_object_id=base.point_object_id, point_invalid_mask=base.point_invalid_mask, camera_info=ci,
            q_pointcloud_camera=base.q_pointcloud_camera, t_pointcloud_camera=base.t_pointcloud_camera, color_max_sh_band=3))
    gt = (image.clamp(0, 1) * 0.9 + 0.05).permute(2, 0, 1).contiguous()
    variants = {"none": None, "mcmc": MCMCConfig(cap_max=N)}
    steps = {}
    for name, mc in variants.items():
        sc = make_scene(**cfg).to("cuda")
        steps[name] = (sc, FusedTrainStep(sc, GPCR.GaussianPointCloudRasterisationConfig(), 0.2, mcmc=mc))

    def run(name):
        sc, step = steps[name]
        kw = {"mcmc_num_valid": n_valid} if variants[name] else {}
        step.run(gt, sc.q_pointcloud_camera, sc.t_pointcloud_camera, ci, 3, 1e-3, 1e-5, **kw)

    for name in variants:
        for _ in range(args.warmup):
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in variants}
    order = list(variants)
    for region in range(args.regions):
        for name in (order if region % 2 == 0 else order[::-1]):
            times[name] += _timed(lambda: run(name), args.steps)
    name, power = card()
    out = dict(config=args.config, N=N, num_valid=n_valid, card=name, power_limit=power, regions=args.regions, steps=args.steps,
               skipped_steps={n: steps[n][1].num_skipped_steps for n in variants})
    for v, ts in times.items():
        out["step_" + v] = _stats(ts)
    out["step_mcmc_minus_none_ms"] = round(out["step_mcmc"]["median_ms"] - out["step_none"]["median_ms"], 4)

    # the two per-iteration kernels alone
    lib = _lib.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sc = make_scene(**cfg).to("cuda")
    xyz, feat, mask = sc.point_cloud.contiguous(), sc.point_cloud_features.contiguous(), sc.point_invalid_mask
    grad = torch.zeros_like(feat)
    terms = torch.zeros(2, device="cuda")
    temp = torch.zeros(int(lib.gsb200_mcmc_temp_bytes()), dtype=torch.uint8, device="cuda")

    def regulariser():
        for _ in range(LAUNCHES):
            _lib.check(lib.gsb200_mcmc_regulariser(p(feat), p(mask), p(grad), N, n_valid, 0.01, 0.01, p(terms), p(temp), stream),
                       "regulariser")

    def noise():
        for k in range(LAUNCHES):  # a noise scale that leaves the scene where it is
            _lib.check(lib.gsb200_mcmc_noise(p(xyz), p(feat), p(mask), N, 1e-12, 100.0, 0.005, 1, k, stream), "noise")

    for fn, key, nbytes in ((regulariser, "regulariser", n_valid * 48 + N), (noise, "noise", n_valid * 56 + N)):
        fn()
        ts = [t / LAUNCHES for t in _timed(fn, args.regions * 4)]
        out["kernel_" + key] = dict(**_stats(ts), bytes=nbytes, gb_per_s=round(nbytes / (np.median(ts) * 1e-3) / 1e9, 1))

    # one relocation of 5 % of the rows: the dead rows are the last 5 %, their sources drawn by opacity from the others
    dead = N // 20
    with torch.no_grad():
        feat[N - dead:, 7] = -9.0
    moments = MCMCMoments((torch.zeros_like(feat), torch.zeros_like(feat)), (torch.zeros_like(xyz), torch.zeros_like(xyz)))
    mp = GaussianPointMCMCController.MaintainedParameters(xyz, feat, mask, sc.point_object_id)
    ctl = GaussianPointMCMCController(MCMCConfig(cap_max=N), mp, generator=torch.Generator(device="cuda").manual_seed(0))
    sources, counts, dest_sources = ctl._draw(dead)
    destinations = torch.arange(N - dead, N, device="cuda")
    relocate = lambda: ctl._apply_cuda(sources, counts, destinations, dest_sources, xyz, feat, None, moments)  # noqa: E731
    relocate()
    out["relocate_5_percent"] = dict(**_stats(_timed(relocate, args.regions * 4)), sources=int(sources.numel()),
                                     destinations=dead)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ctl.iteration_counter = ctl.config.refine_start - 1
    ctl.refinement(moments)
    e1.record()
    e1.synchronize()
    out["refinement_with_host_ms"] = round(e0.elapsed_time(e1), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
