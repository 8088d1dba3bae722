"""The accumulated-alpha-gradient backward (``gsb200_backward_aux`` with an alpha gradient) executed on the CPU from the
unmodified kernel sources: the ALPHA instantiations of the transposed loop A, alone and with DEPTH
(``tests/simt/emu_blend_alpha.cpp``, a library of its own), after the emulated forward of :mod:`simt_helpers` and followed
by the per-point kernel of :mod:`simt_depth_helpers` (the default one, or DEPTH with a depth term).  Test infrastructure."""
import ctypes
import os
import subprocess

import numpy as np

from simt_depth_helpers import emulated_points
from simt_helpers import CSRC, SIMT, c


def build_alpha_emulator():
    out = os.path.join(SIMT, "libsimt_emu_alpha.so")
    tu = os.path.join(SIMT, "emu_blend_alpha.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_blend_backward_alpha.restype = ctypes.c_longlong
    return L


def emulated_backward_alpha(emu, demu, aemu, st, grad_image, grad_alpha, grad_depth=None, band=3, stats=True):
    """Backward of the transposed path with an alpha gradient ((H,W)) for a state of :func:`simt_helpers.emulated_forward`:
    the ALPHA instantiation of loop A (ALPHA + DEPTH with ``grad_depth``), then the per-point kernel (DEPTH with
    ``grad_depth``).  Returns the dense gradients, loop A's accumulator rows (M,12) and the per-pixel magnitude image."""
    pre, M = st.pre, st.M
    H, W = pre.H, pre.W
    g = np.ascontiguousarray(grad_image, dtype=np.float32)
    ga = np.ascontiguousarray(grad_alpha, dtype=np.float32)
    gd = None if grad_depth is None else np.ascontiguousarray(grad_depth, dtype=np.float32)
    accum, mag = np.zeros((max(M, 1), 12), np.float32), np.zeros((H, W, 2), np.float32)
    if st.K:
        aemu.emu_blend_backward_alpha(int(st.exact), int(stats), H, W, c(st.start), c(st.end), c(st.sorted_vals),
                                      c(pre.records), c(g), c(st.acc_alpha), c(st.last_effective),
                                      None if gd is None else c(gd), None if gd is None else c(st.depth), c(ga), c(accum),
                                      c(mag))
    gx, gf = emulated_points(emu, demu, st, accum, band, depth=grad_depth is not None)
    return gx, gf, accum[:M].copy(), mag
