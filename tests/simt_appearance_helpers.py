"""The bilateral-grid kernels (``csrc/appearance.cu``) executed on the CPU from the unmodified kernel sources
(``tests/simt/emu_appearance.cpp``, a library of its own).  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c


def build_appearance_emulator():
    out = os.path.join(SIMT, "libsimt_emu_appearance.so")
    tu = os.path.join(SIMT, "emu_appearance.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_bilateral_grid_temp_bytes.restype = ctypes.c_longlong
    L.emu_bilateral_grid_forward.restype = ctypes.c_longlong
    L.emu_bilateral_grid_backward.restype = ctypes.c_longlong
    return L


def emulated_slice(emu, image, grid):
    """image (H, W, 3), grid (12, Gz, Gy, Gx) -> the sliced (H, W, 3) image, float32."""
    image = np.ascontiguousarray(image, np.float32)
    grid = np.ascontiguousarray(grid, np.float32)
    H, W = image.shape[:2]
    gz, gy, gx = grid.shape[1:]
    out = np.full((H, W, 3), np.nan, np.float32)
    assert emu.emu_bilateral_grid_forward(c(image), c(grid), H, W, gx, gy, gz, c(out)) > 0
    return out


def emulated_slice_backward(emu, image, grid, grad_out, tv_weight=None):
    """dL/dimage and dL/dG of the slice (the first computed in place over a copy of grad_out, as the train step does); with
    ``tv_weight`` also the TV term, added into dL/dG, and its value ``tv`` (= tv_weight * tv(G))."""
    image = np.ascontiguousarray(image, np.float32)
    grid = np.ascontiguousarray(grid, np.float32)
    grad = np.array(grad_out, np.float32, order="C", copy=True)
    H, W = image.shape[:2]
    gz, gy, gx = grid.shape[1:]
    temp = np.full(int(emu.emu_bilateral_grid_temp_bytes(H, W, gx, gy, gz)) // 4, np.nan, np.float32)
    grad_grid = np.full(grid.shape, np.nan, np.float32)
    tv = np.full(1, np.nan, np.float32)
    ran = emu.emu_bilateral_grid_backward(c(image), c(grid), H, W, gx, gy, gz, c(grad), c(grad), c(grad_grid), c(temp),
                                          ctypes.c_float(tv_weight or 0.0), c(tv) if tv_weight is not None else None)
    assert ran > 0
    return SimpleNamespace(grad_image=grad, grad_grid=grad_grid, tv=float(tv[0]) if tv_weight is not None else None)
