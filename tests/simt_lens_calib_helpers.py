"""Pose and intrinsics gradients through a lens (``gsb200_backward_lens_calib``) executed on the CPU from the unmodified kernel
sources: the LENS instantiations of the per-point kernel with pose, intrinsics and coefficient sums and their finishing kernels
(``tests/simt/emu_lens_calib.cpp``, a library of its own), on the accumulator rows that the emulated loop A left for a state
of :func:`simt_lens_helpers.emulated_forward_lens`.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c
from simt_lens_helpers import MODELS, _coeffs

POSE_PARTIAL_BLOCKS = 2048  # GSB_POSE_PARTIAL_BLOCKS = GSB_INTRINSICS_PARTIAL_BLOCKS = GSB_LENS_GRAD_PARTIAL_BLOCKS


def build_lens_calib_emulator():
    out = os.path.join(SIMT, "libsimt_emu_lens_calib.so")
    tu = os.path.join(SIMT, "emu_lens_calib.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_backward_points_lens_calib.restype = ctypes.c_int
    return L


def emulated_points_lens_calib(emu, cemu, st, accum, band=3, depth=False, pose=True, intr=False, lgrad=False,
                               factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """The lens-calibration per-point kernel (``pose`` / ``intr`` / ``lgrad`` select the sums; one of the first two must be
    on) and the finishing kernels on the accumulator rows of a state of :func:`simt_lens_helpers.emulated_forward_lens`.
    Returns the dense (N,3) / (N,56) gradients, dL/dq_pc (K,4) and dL/dt_pc (K,3) with ``pose``, dL/dK (3,3) with ``intr``,
    dL/dk (5,) with ``lgrad`` (else None), the per-CTA rows of each sum and the grid size."""
    assert pose or intr
    pre, scene = st.pre, st.scene
    model, k = st.lens
    N = pre.point_offset.shape[0]
    acc = np.zeros((max(st.M, 1), 12), np.float32)
    acc[:st.M] = accum[:st.M]
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    n_obj = q.shape[0]
    poses = np.zeros((n_obj, 20), np.float32)
    emu.emu_pose(n_obj, c(q), c(t), c(poses))
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    K = scene.camera_info.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    gq, gt = np.full((n_obj, 4), 7.0, np.float32), np.full((n_obj, 3), 7.0, np.float32)
    gK, gk = np.full((3, 3), 7.0, np.float32), np.full(5, 7.0, np.float32)
    pose_partials = np.full((POSE_PARTIAL_BLOCKS, n_obj, 12), 7.0, np.float32)
    intr_partials = np.full((POSE_PARTIAL_BLOCKS, 6), 7.0, np.float32)
    lens_partials = np.full((POSE_PARTIAL_BLOCKS, 5), 7.0, np.float32)
    f = ctypes.c_float
    blocks = cemu.emu_backward_points_lens_calib(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), int(depth), MODELS[model],
        c(_coeffs(k)), int(pose), int(intr), int(lgrad), n_obj, c(q), c(pose_partials), c(gq), c(gt), c(intr_partials), c(gK),
        c(lens_partials), c(gk))
    return SimpleNamespace(gx=gx, gf=gf, gq=gq if pose else None, gt=gt if pose else None, gK=gK if intr else None,
                           gk=gk if lgrad else None, pose_partials=pose_partials[:blocks].copy() if pose else None,
                           intr_partials=intr_partials[:blocks].copy() if intr else None,
                           lens_partials=lens_partials[:blocks].copy() if lgrad else None, blocks=blocks)
