"""The camera-intrinsics gradient (``gsb200_backward_calib``) executed on the CPU from the unmodified kernel sources: the INTR
instantiations of the per-point kernel (intrinsics alone, or with the pose sums in the same pass) and the finishing kernels
(``tests/simt/emu_intrinsics.cpp``, a library of its own), on the accumulator rows that the emulated loop A left for a state
of :func:`simt_helpers.emulated_forward`.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c

INTRINSICS_PARTIAL_BLOCKS = 2048  # GSB_INTRINSICS_PARTIAL_BLOCKS of include/gsb200.h
POSE_PARTIAL_BLOCKS = 2048  # GSB_POSE_PARTIAL_BLOCKS


def build_intrinsics_emulator():
    out = os.path.join(SIMT, "libsimt_emu_intrinsics.so")
    tu = os.path.join(SIMT, "emu_intrinsics.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_backward_points_calib.restype = ctypes.c_int
    return L


def emulated_points_calib(emu, iemu, st, accum, band=3, depth=False, pose=False, K=None,
                          factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """The INTR per-point kernel (with ``pose`` the combined one; DEPTH: word 11 of the rows is dL/dz) and the finishing
    kernels on the accumulator rows ``accum`` of a state of :func:`simt_helpers.emulated_forward`.  ``K``: the (3,3)
    intrinsics the kernel reads (default: the scene's).  Returns the dense (N,3) / (N,56) gradients, dL/dK (3,3), with
    ``pose`` dL/dq_pc (K,4) and dL/dt_pc (K,3), the per-CTA intrinsics rows (grid, 6) and the grid size."""
    pre, scene = st.pre, st.scene
    N = pre.point_offset.shape[0]
    acc = np.zeros((max(st.M, 1), 12), np.float32)
    acc[:st.M] = accum[:st.M]
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    n_obj = q.shape[0]
    poses = np.zeros((n_obj, 20), np.float32)
    emu.emu_pose(n_obj, c(q), c(t), c(poses))
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    if K is None:
        K = scene.camera_info.camera_intrinsics.detach().numpy()
    K = np.ascontiguousarray(K, dtype=np.float32)
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    gq, gt = np.full((n_obj, 4), 7.0, np.float32), np.full((n_obj, 3), 7.0, np.float32)
    gK = np.full((3, 3), 7.0, np.float32)
    pose_partials = np.full((POSE_PARTIAL_BLOCKS, n_obj, 12), 7.0, np.float32)
    intr_partials = np.full((INTRINSICS_PARTIAL_BLOCKS, 6), 7.0, np.float32)
    f = ctypes.c_float
    blocks = iemu.emu_backward_points_calib(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), int(depth), int(pose),
        n_obj, c(q), c(pose_partials), c(gq), c(gt), c(intr_partials), c(gK))
    return SimpleNamespace(gx=gx, gf=gf, gK=gK, gq=gq if pose else None, gt=gt if pose else None,
                           partials=intr_partials[:blocks].copy(), blocks=blocks)
