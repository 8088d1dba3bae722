"""The per-Gaussian feature channels (``gsb200_forward_ext`` / ``gsb200_backward_ext``) executed on the CPU from the
unmodified kernel sources: the CF instantiations of the forward blend and of the transposed loop A, alone and with the depth
and alpha terms (``tests/simt/emu_blend_features.cpp``, a library of its own), on the state of the emulated forward of
:mod:`simt_helpers` and followed by the per-point kernel of :mod:`simt_depth_helpers`.  Test infrastructure."""
import ctypes
import os
import subprocess

import numpy as np

from simt_depth_helpers import emulated_points
from simt_helpers import CSRC, SIMT, c


def build_feature_emulator():
    out = os.path.join(SIMT, "libsimt_emu_features.so")
    tu = os.path.join(SIMT, "emu_blend_features.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_blend_forward_features.restype = ctypes.c_longlong
    L.emu_blend_backward_features.restype = ctypes.c_longlong
    return L


def emulated_forward_features(femu, st, features):
    """The feature instantiation of the forward blend on a state of :func:`simt_helpers.emulated_forward` (same frame, same
    sorted list) with the (N,C) ``features``; returns (image, depth, acc_alpha, last_effective, count, feature_map)."""
    pre = st.pre
    H, W = pre.H, pre.W
    f = np.ascontiguousarray(features, dtype=np.float32)
    C = f.shape[1]
    image, depth, acc = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32)
    last, cnt = np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    fmap = np.zeros((H, W, C), np.float32)
    if st.K:
        femu.emu_blend_forward_features(int(st.exact), H, W, c(st.start), c(st.end), c(st.sorted_vals), c(pre.records),
                                        c(pre.point_id), C, c(f), c(image), c(depth), c(acc), c(last), c(cnt), c(fmap))
    return image, depth, acc, last, cnt, fmap


def emulated_backward_features(emu, demu, femu, st, features, grad_feature_map, grad_image, grad_depth=None,
                               grad_alpha=None, band=3, stats=True):
    """Backward of the transposed path with the feature channels for a state of :func:`simt_helpers.emulated_forward`: the CF
    instantiation of loop A (with DEPTH / ALPHA for ``grad_depth`` / ``grad_alpha``), then the per-point kernel (DEPTH with
    ``grad_depth``).  Returns the dense gradients, dL/dfeatures (N,C), loop A's accumulator rows (M,12) and the per-pixel
    magnitude image."""
    pre, M = st.pre, st.M
    H, W = pre.H, pre.W
    f = np.ascontiguousarray(features, dtype=np.float32)
    N, C = f.shape
    g = np.ascontiguousarray(grad_image, dtype=np.float32)
    gF = np.ascontiguousarray(grad_feature_map, dtype=np.float32)
    gd = None if grad_depth is None else np.ascontiguousarray(grad_depth, dtype=np.float32)
    ga = None if grad_alpha is None else np.ascontiguousarray(grad_alpha, dtype=np.float32)
    accum, mag = np.zeros((max(M, 1), 12), np.float32), np.zeros((H, W, 2), np.float32)
    gfeat = np.zeros((N, C), np.float32)  # zeroed, as gsb200_backward_ext does
    if st.K:
        femu.emu_blend_backward_features(int(st.exact), int(stats), H, W, c(st.start), c(st.end), c(st.sorted_vals),
                                         c(pre.records), c(g), c(st.acc_alpha), c(st.last_effective),
                                         None if gd is None else c(gd), None if gd is None else c(st.depth),
                                         None if ga is None else c(ga), c(pre.point_id), C, c(f), c(gF), c(gfeat), c(accum),
                                         c(mag))
    gx, gf = emulated_points(emu, demu, st, accum, band, depth=grad_depth is not None)
    return gx, gf, gfeat, accum[:M].copy(), mag
