"""The depth-gradient backward (``gsb200_backward_with_depth``) executed on the CPU from the unmodified kernel sources: the
DEPTH instantiations of the transposed loop A and of the per-point kernel (``tests/simt/emu_blend_depth.cpp``, a library
of its own) after the emulated forward of :mod:`simt_helpers`.  Test infrastructure."""
import ctypes
import os
import subprocess

import numpy as np

from simt_helpers import CSRC, SIMT, c


def build_depth_emulator():
    out = os.path.join(SIMT, "libsimt_emu_depth.so")
    tu = os.path.join(SIMT, "emu_blend_depth.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_blend_backward_depth.restype = ctypes.c_longlong
    L.emu_backward_points_depth.restype = ctypes.c_longlong
    return L


def emulated_points(emu, demu, st, accum, band=3, factors=(1.0, 0.5, 20.0, 5.0, 1.0), depth=False):
    """The dense per-point kernel (default, or DEPTH: word 11 of the rows is dL/dz) on the accumulator rows ``accum`` of a
    state of :func:`simt_helpers.emulated_forward`; returns the dense (N,3) and (N,56) gradients."""
    pre, scene = st.pre, st.scene
    N = pre.point_offset.shape[0]
    acc = np.zeros((max(st.M, 1), 12), np.float32)
    acc[:st.M] = accum[:st.M]
    q = scene.q_pointcloud_camera.numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.numpy().astype(np.float32).copy()
    poses = np.zeros((q.shape[0], 20), np.float32)
    emu.emu_pose(q.shape[0], c(q), c(t), c(poses))
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    K = scene.camera_info.camera_intrinsics.numpy().astype(np.float32).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    f = ctypes.c_float
    fn = demu.emu_backward_points_depth if depth else emu.emu_backward_points
    fn(ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
       c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), None, None, *([None] * 6))
    return gx, gf


def emulated_backward_depth(emu, demu, st, grad_image, grad_depth=None, band=3, stats=True):
    """Backward of the transposed path for a state of :func:`simt_helpers.emulated_forward`: with ``grad_depth`` ((H,W)) the
    DEPTH instantiations of loop A and of the per-point kernel, without it the default ones.  Returns the dense gradients,
    loop A's accumulator rows (M,12) and the per-pixel magnitude image."""
    pre, M = st.pre, st.M
    H, W = pre.H, pre.W
    g = np.ascontiguousarray(grad_image, dtype=np.float32)
    accum, mag = np.zeros((max(M, 1), 12), np.float32), np.zeros((H, W, 2), np.float32)
    args = (H, W, c(st.start), c(st.end), c(st.sorted_vals), c(pre.records), c(g), c(st.acc_alpha), c(st.last_effective))
    if st.K:
        if grad_depth is None:
            emu.emu_blend_backward(1, int(st.exact), int(stats), *args, c(accum), c(mag))
        else:
            gd = np.ascontiguousarray(grad_depth, dtype=np.float32)
            demu.emu_blend_backward_depth(int(st.exact), int(stats), *args, c(gd), c(st.depth), c(accum), c(mag))
    gx, gf = emulated_points(emu, demu, st, accum, band, depth=grad_depth is not None)
    return gx, gf, accum[:M].copy(), mag
