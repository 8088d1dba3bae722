"""The lens-coefficient gradient (``gsb200_backward_lens_grad``) executed on the CPU from the unmodified kernel sources: the
LGRAD instantiations of the per-point kernel, the finishing kernel and the coefficient helper (``tests/simt/emu_lens_grad.cpp``,
a library of its own), on the accumulator rows that the emulated loop A left for a state of
:func:`simt_lens_helpers.emulated_forward_lens`.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c
from simt_lens_helpers import MODELS, _coeffs

LENS_GRAD_PARTIAL_BLOCKS = 2048  # GSB_LENS_GRAD_PARTIAL_BLOCKS of include/gsb200.h


def build_lens_grad_emulator():
    out = os.path.join(SIMT, "libsimt_emu_lens_grad.so")
    tu = os.path.join(SIMT, "emu_lens_grad.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_backward_points_lens_grad.restype = ctypes.c_int
    return L


def coefficient_grad(gemu, model, xn, yn, gx, gy, w00, w01, w11):
    """The device helper lens_coefficient_grad in float32 on n points: (n, 5)."""
    arrs = [np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.float32), np.shape(xn))) for a in
            (xn, yn, gx, gy, w00, w01, w11)]
    n = arrs[0].shape[0]
    out = np.zeros((n, 5), np.float32)
    gemu.emu_lens_coefficient_grad(MODELS[model], ctypes.c_longlong(n), *(c(a) for a in arrs), c(out))
    return out


def coefficient_jacobian(gemu, model, xn, yn):
    """d(xd, yd)/dk of the helper in float32 (unit position weights, zero D weights): (n, 2, 5)."""
    z = np.zeros_like(np.asarray(xn, np.float32))
    cx = coefficient_grad(gemu, model, xn, yn, z + 1, z, z, z, z)
    cy = coefficient_grad(gemu, model, xn, yn, z, z + 1, z, z, z)
    return np.stack([cx, cy], 1)


def emulated_points_lens_grad(emu, gemu, st, accum, band=3, depth=False, factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """The LGRAD per-point kernel and the finishing kernel on the accumulator rows of a state of
    :func:`simt_lens_helpers.emulated_forward_lens`.  Returns the dense (N,3) / (N,56) gradients, dL/dk (5,), the per-CTA
    rows (grid, 5) and the grid size."""
    pre, scene = st.pre, st.scene
    model, k = st.lens
    N = pre.point_offset.shape[0]
    acc = np.zeros((max(st.M, 1), 12), np.float32)
    acc[:st.M] = accum[:st.M]
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    poses = np.zeros((q.shape[0], 20), np.float32)
    emu.emu_pose(q.shape[0], c(q), c(t), c(poses))
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    K = scene.camera_info.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    gk = np.full(5, 7.0, np.float32)
    partials = np.full((LENS_GRAD_PARTIAL_BLOCKS, 5), 7.0, np.float32)
    f = ctypes.c_float
    co = _coeffs(k)
    blocks = gemu.emu_backward_points_lens_grad(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), int(depth), MODELS[model],
        c(co), c(partials), c(gk))
    return SimpleNamespace(gx=gx, gf=gf, gk=gk, partials=partials[:blocks].copy(), blocks=blocks)
