"""The supervision terms of the fused train step (``csrc/supervision_loss.cu`` around ``csrc/image_loss.cu``) executed on
the CPU from the unmodified kernel sources (``tests/simt/emu_supervision_loss.cpp``, a library of its own).  Test
infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c


def build_supervision_emulator():
    out = os.path.join(SIMT, "libsimt_emu_supervision.so")
    tu = os.path.join(SIMT, "emu_supervision_loss.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_supervision_step.restype = ctypes.c_longlong
    L.emu_supervision_temp_bytes.restype = ctypes.c_longlong
    L.emu_supervision_image_loss_temp_bytes.restype = ctypes.c_longlong
    return L


def new_temps(emu, H, W):
    """The two temp buffers of one resolution, zeroed (their tickets must be zero before the first call)."""
    return (np.zeros(int(emu.emu_supervision_temp_bytes(H, W)) + 16, np.uint8),
            np.zeros(int(emu.emu_supervision_image_loss_temp_bytes(H, W)) + 16, np.uint8))


def emulated_supervision_step(emu, image, gt, alpha, depth, depth_target=None, mask_target=None, background=None,
                              lambda_value=0.2, depth_weight=0.0, mask_weight=0.0, temps=None):
    """One call of the pre-pass -> image loss -> post-pass chain.  Returns the image loss triple, the loss triple
    {total, mask term, depth term} and dL/dI, dL/dS, dL/dD (NaN-filled where a gradient is not written)."""
    H, W = image.shape[:2]
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    image, gt, alpha, depth = f32(image), f32(gt), f32(alpha), f32(depth)
    depth_target, mask_target, background = f32(depth_target), f32(mask_target), f32(background)
    temp, il_temp = temps if temps is not None else new_temps(emu, H, W)
    il3, loss3 = np.zeros(3, np.float32), np.zeros(3, np.float32)
    g_image = np.full((H, W, 3), np.nan, np.float32)
    g_alpha, g_depth = np.full((H, W), np.nan, np.float32), np.full((H, W), np.nan, np.float32)
    opt = lambda a: None if a is None else c(a)  # noqa: E731
    f = ctypes.c_float
    ran = emu.emu_supervision_step(c(image), c(gt), c(alpha), c(depth), opt(depth_target), opt(mask_target), opt(background),
                                   H, W, f(lambda_value), f(depth_weight), f(mask_weight), c(il3), c(g_image), c(g_alpha),
                                   c(g_depth), c(loss3), c(temp), c(il_temp))
    assert ran > 0
    return SimpleNamespace(image_loss=il3, loss=loss3, grad_image=g_image, grad_alpha=g_alpha, grad_depth=g_depth)
