"""-m gpu parity at the FULL sizes bench.py times: BASELINE config 2 (C2), the headline config C3 and the stress
variant C3s (sigma = 0.02), CUDA operator vs the CPU oracle on identical inputs, on BOTH arithmetic paths
(default ex2/rcp.approx path = what bench.py times; ``exact_exp`` = the reference's op order with expf).

Criteria (BASELINE.json north_star: RGB 1e-4 abs, gradients 1e-3 rel, floor 1e-6 max|g| as SURVEY 8(d)):
integer stages and per-point floats are bit-exact; image / gradient entries may leave the tolerance only where a
(pixel, splat) pair sits within rounding of the alpha >= 1/255 or T >= 1e-4 cut-offs and flips (the oracle's libm
expf and the GPU's exp differ in the last ulp; so do Taichi's LLVM expf and libm).  Every such pixel must show up
as a pixel-count or last-effective difference OR be within the cut-off's alpha step (4e-3); the number of flipped
pixels and of out-of-tolerance gradient entries is bounded and RECORDED (in the JSON file named by
$GSB200_PARITY_COUNTS, default parity_counts.json in the temporary directory) so that the allowance can be judged.
"""
import json
import os
import tempfile
import time

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200.synthetic import CONFIGS, make_scene

from helpers import grad_close, oracle_backward, oracle_forward
from gpu_helpers import count_above, cuda_scene, make_op, n, run_forward
from test_gpu_parity import _check_stages

pytestmark = pytest.mark.gpu

COUNTS_FILE = os.environ.get("GSB200_PARITY_COUNTS", os.path.join(tempfile.gettempdir(), "gsb200_parity_counts.json"))

_oracle_cache = {}


def _oracle(name):
    """Oracle forward + backward once per configuration (seconds on the box's host cores); both arithmetic paths
    of the CUDA operator are compared against the same result."""
    if name not in _oracle_cache:
        _oracle_cache.clear()  # one configuration resident at a time (C3: ~1 GB of numpy arrays)
        scene = make_scene(**CONFIGS[name])
        t0 = time.time()
        o, fwd, feats_n = oracle_forward(scene)
        g = torch.Generator().manual_seed(5)
        grad_image = torch.randn((scene.camera_info.camera_height, scene.camera_info.camera_width, 3), generator=g,
                                 dtype=torch.float32)
        bwd = oracle_backward(o, fwd, scene, feats_n, grad_image.numpy(), 3)
        _oracle_cache[name] = (scene, fwd, bwd, grad_image, time.time() - t0)
    return _oracle_cache[name]


def _record(key, entry):
    os.makedirs(os.path.dirname(os.path.abspath(COUNTS_FILE)), exist_ok=True)
    data = {}
    if os.path.exists(COUNTS_FILE):
        with open(COUNTS_FILE) as f:
            data = json.load(f)
    data[key] = entry
    with open(COUNTS_FILE, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


GROUPS = (("xyz", None), ("q", slice(0, 4)), ("s", slice(4, 7)), ("logit", slice(7, 8)), ("sh", slice(8, 56)))


@pytest.mark.parametrize("exact_exp", [False, True], ids=["default_fast_path", "exact_exp"])
@pytest.mark.parametrize("name", ["C2", "C3", "C3s"])
def test_full_size_forward_backward_vs_oracle(name, exact_exp):
    scene, fwd, bwd, grad_image, oracle_seconds = _oracle(name)
    sc = cuda_scene(scene, requires_grad=True)
    op = make_op(exact_exp=exact_exp)
    image, depth, count = run_forward(op, sc, band=3)
    frame = op.last_frame
    _check_stages(frame, fwd, max_tiles=100)  # ids, tile counts, per-point floats bit-exact; key lists: subsequence + dead pairs
    keys, vals = frame.sorted_keys, frame.point_offset_with_sort_key
    assert bool((keys[1:] >= keys[:-1]).all())
    same = keys[1:] == keys[:-1]
    assert bool((vals[1:][same] > vals[:-1][same]).all())  # stable: ties keep ascending in-camera offset
    assert bool(torch.isfinite(image).all()) and float(image.min()) >= 0.0

    H, W = fwd.image.shape[:2]
    d = np.abs(n(image) - fwd.image).max(axis=-1)
    cnt_diff = n(count) != fwd.pixel_valid_point_count
    bad = d > 1e-4
    entry = {
        "config": name, "path": "exact_exp" if exact_exp else "default", "pixels": int(H * W),
        "num_points_in_camera": int(frame.num_points_in_camera), "num_keys_emitted": int(frame.num_keys),
        "num_keys_reference": int(fwd.point_offset_with_sort_key.shape[0]),
        "image_max_abs_err": float(d.max()), "image_pixels_over_1e-4": int(bad.sum()),
        "image_pixels_over_1e-4_without_count_flip": int((bad & ~cnt_diff).sum()),
        "pixel_count_mismatches": int(cnt_diff.sum()), "oracle_seconds_fwd_bwd": round(oracle_seconds, 1),
    }
    image.backward(grad_image.cuda())
    gx, gf = n(sc.point_cloud.grad), n(sc.point_cloud_features.grad)
    worst_global = 0.0
    for gname, sl in GROUPS:
        got = gx if sl is None else gf[:, sl]
        exp = bwd.grad_pointcloud if sl is None else bwd.grad_pointcloud_features[:, sl]
        _, worst6, nviol6 = grad_close(got, exp, floor_frac=1e-6)
        _, worst5, nviol5 = grad_close(got, exp, floor_frac=1e-5)
        glob = float(np.abs(got - exp).max() / np.abs(exp).max())
        worst_global = max(worst_global, glob)
        entry["grad_" + gname] = {"entries": int(exp.size), "violations_floor_1e-6": nviol6, "violations_floor_1e-5": nviol5,
                                  "worst_excess_floor_1e-6": round(worst6, 2), "max_abs_err_over_max_abs_grad": glob}
    _record(f"{name}/{entry['path']}", entry)

    # ---- the assertions (allowances per 1e6 pixels / entries; the observed numbers are in the recorded file)
    px = H * W
    # The float atomics of loop A land in another order every run, so two GPU runs differ from each other as well (bench.py
    # exchange_check reports that noise at N > 1); the bound on the largest deviation is therefore north_star's 1e-3.
    assert d.max() <= 5e-3, entry                           # a flip moves a pixel by <= alpha_cut * T * |colour| ~ 4e-3
    assert bad.sum() <= max(4, 1e-5 * px), entry            # <= 10 flipped pixels per Mpix
    assert (bad & ~cnt_diff).sum() == 0, entry              # every pixel outside 1e-4 IS a cut-off flip (its count differs)
    assert cnt_diff.sum() <= max(8, 3e-5 * px), entry
    for gname, _ in GROUPS:
        e = entry["grad_" + gname]
        assert e["violations_floor_1e-6"] <= max(20, 1e-4 * e["entries"]), entry
        assert e["max_abs_err_over_max_abs_grad"] <= 1e-3, entry
