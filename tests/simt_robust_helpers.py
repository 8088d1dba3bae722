"""The per-pixel loss weights of the fused train step (``csrc/robust_loss.cu`` around ``csrc/image_loss.cu``) executed on
the CPU from the unmodified kernel sources (``tests/simt/emu_robust.cpp``, a library of its own).  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c


def build_robust_emulator():
    out = os.path.join(SIMT, "libsimt_emu_robust.so")
    tu = os.path.join(SIMT, "emu_robust.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_robust_step.restype = ctypes.c_longlong
    L.emu_robust_temp_bytes.restype = ctypes.c_longlong
    L.emu_robust_image_loss_temp_bytes.restype = ctypes.c_longlong
    return L


def new_temps(emu, H, W):
    """The two temp buffers of one resolution, zeroed (they must be zero before the first call)."""
    return (np.zeros(int(emu.emu_robust_temp_bytes()) + 16, np.uint8),
            np.zeros(int(emu.emu_robust_image_loss_temp_bytes(H, W)) + 16, np.uint8))


def emulated_robust_step(emu, image, gt, static_weight=None, config=None, lambda_value=0.2, temps=None):
    """One call of the pre-passes -> image loss -> post-pass chain.  ``config`` a ``loss.RobustLossConfig`` or None (static
    weight alone).  Returns the weight, the composite, the image loss triple, dL/dx and the stats."""
    H, W = image.shape[:2]
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    image, gt, static_weight = f32(image), f32(gt), f32(static_weight)
    temp, il_temp = temps if temps is not None else new_temps(emu, H, W)
    weight = np.full((H, W), np.nan, np.float32)
    composite = np.full((H, W, 3), np.nan, np.float32)
    il3, stats = np.zeros(3, np.float32), np.zeros(2, np.float32)
    grad = np.full((H, W, 3), np.nan, np.float32)
    f = ctypes.c_float
    q, bt, pt = (config.inlier_quantile, config.box_threshold, config.patch_threshold) if config else (1.0, 0.0, 0.0)
    ran = emu.emu_robust_step(c(image), c(gt), None if static_weight is None else c(static_weight), H, W, f(lambda_value),
                              int(config is not None), f(q), f(bt), f(pt), c(weight), c(composite), c(il3), c(grad),
                              c(stats), c(temp), c(il_temp))
    assert ran > 0
    return SimpleNamespace(weight=weight, composite=composite, image_loss=il3, grad=grad, stats=stats)
