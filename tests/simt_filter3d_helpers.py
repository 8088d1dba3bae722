"""The 3D smoothing filter executed on the CPU from the unmodified kernel sources: the views kernels of ``csrc/filter3d.cu``,
the FILTER instantiations of the per-point backward and of the per-point forward (``tests/simt/emu_filter3d.cpp``, a library of its own).  Test
infrastructure."""
import ctypes
import os
import subprocess

import numpy as np
import torch

from simt_helpers import CSRC, SIMT, c
from taichi_3d_gaussian_splatting_b200._lib import GsbFilter3dViewsArgs


def build_filter3d_emulator():
    out = os.path.join(SIMT, "libsimt_emu_filter3d.so")
    tu = os.path.join(SIMT, "emu_filter3d.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_filter3d_temp_bytes.restype = ctypes.c_longlong
    L.emu_filter3d_from_views.restype = ctypes.c_longlong
    L.emu_filter3d_from_views.argtypes = [ctypes.POINTER(GsbFilter3dViewsArgs)]
    L.emu_preprocess_filter.restype = ctypes.c_longlong
    vp, f = ctypes.c_void_p, ctypes.c_float
    L.emu_backward_points_filter.restype = None
    L.emu_backward_points_filter.argtypes = [ctypes.c_longlong] + [vp] * 10 + [ctypes.c_int] + [f] * 5 + [vp, vp, ctypes.c_int] + \
        [vp] * 3
    return L


def emulated_filter(emu, xyz, invalid, obj, views, near_plane, variance):
    """gsb200_filter3d_from_views under the emulator; views as ``mip_filter.compute_filter_3d`` takes them (CPU tensors)."""
    V, n_obj = len(views), views[0][0].shape[0]
    xyz = np.ascontiguousarray(xyz, np.float32)
    invalid = np.ascontiguousarray(invalid, np.int8)
    obj = np.ascontiguousarray(obj, np.int32)
    q = np.ascontiguousarray(torch.cat([v[0] for v in views]).numpy(), np.float32)
    t = np.ascontiguousarray(torch.cat([v[1] for v in views]).numpy(), np.float32)
    K = np.ascontiguousarray(np.stack([v[2].camera_intrinsics.numpy() for v in views]), np.float32)
    sizes = np.ascontiguousarray([[v[2].camera_width, v[2].camera_height] for v in views], np.int32)
    out = np.full(xyz.shape[0], np.nan, np.float32)
    temp = np.zeros(int(emu.emu_filter3d_temp_bytes(V, n_obj)) + 16, np.uint8)
    args = GsbFilter3dViewsArgs(num_points=xyz.shape[0], pointcloud=c(xyz), point_invalid_mask=c(invalid),
                                point_object_id=c(obj), num_objects=n_obj, num_views=V, q_pointcloud_camera=c(q),
                                t_pointcloud_camera=c(t), camera_intrinsics=c(K), camera_size=c(sizes), near_plane=near_plane,
                                variance=variance, filter3d=c(out), temp=(temp.ctypes.data + 15) // 16 * 16,
                                temp_bytes=temp.shape[0] - 16, stream=None)
    assert emu.emu_filter3d_from_views(ctypes.byref(args)) > 0
    return out


def emulated_backward(emu, st, features, records, accum, filter3d=None, depth=False, rolling=False):
    """The per-point backward on the frame state ``st`` (``records`` and ``accum`` given separately: they depend on the rows);
    factors 1.  Returns (dL/dxyz (N, 3), dL/dfeatures (N, 56))."""
    N = st.xyz.shape[0]
    gx, gf = np.full((N, 3), np.nan, np.float32), np.full((N, 56), np.nan, np.float32)
    feats = np.ascontiguousarray(features, np.float32)
    f3 = None if filter3d is None else np.ascontiguousarray(filter3d, np.float32)
    rt = np.array(st.row_time, np.float32) if rolling else None
    emu.emu_backward_points_filter(N, c(st.point_offset), c(np.ascontiguousarray(records, np.float32)), c(st.pic),
                                   c(np.ascontiguousarray(accum, np.float32)), c(st.poses), c(st.xyz), c(feats), c(st.obj),
                                   c(st.t_pc), c(st.K), 3, 1.0, 1.0, 1.0, 1.0, 1.0, c(gx), c(gf), int(depth),
                                   c(f3) if f3 is not None else None, c(st.motion) if rolling else None,
                                   c(rt) if rolling else None)
    return gx, gf
