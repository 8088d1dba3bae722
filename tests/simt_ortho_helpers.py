"""The orthographic view (``gsb200_forward_ortho`` / ``gsb200_backward_ortho``) executed on the CPU from the unmodified kernel
sources: the per-point forward (with or without the 3D filter), the default forward blend and transposed loop A, and the
per-point backward with its pose and intrinsics finishing kernels (``tests/simt/emu_ortho.cpp``, a library of its own), chained
with the emulated sort and tile ranges of :mod:`simt_helpers` exactly as ``csrc/api.cu`` chains them.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, _bit_width, c, emu_sort_frame

NEAR, FAR, SCALE = 0.8, 1000.0, 100.0
PARTIAL_BLOCKS = 2048  # GSB_POSE_PARTIAL_BLOCKS = GSB_INTRINSICS_PARTIAL_BLOCKS of include/gsb200.h


def build_ortho_emulator():
    out = os.path.join(SIMT, "libsimt_emu_ortho.so")
    tu = os.path.join(SIMT, "emu_ortho.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_preprocess_ortho.restype = ctypes.c_longlong
    L.emu_blend_forward_ortho.restype = ctypes.c_longlong
    L.emu_blend_backward_ortho.restype = ctypes.c_longlong
    L.emu_backward_points_ortho.restype = ctypes.c_int
    return L


def _np(t, dtype):
    return np.ascontiguousarray(t.detach().cpu().numpy(), dtype=dtype)


def emulated_forward_ortho(emu, oemu, scene, exact=True, features=None, filter3d=None, filter_tiles=True):
    """Forward of the orthographic path under the emulator: the state for the backward with the outputs (``fmap`` with
    ``features`` (N,C); ``filter3d`` (N,) selects the FILTER per-point kernel)."""
    xyz, feats = _np(scene.point_cloud, np.float32), _np(scene.point_cloud_features, np.float32)
    N = xyz.shape[0]
    ci = scene.camera_info
    H, W = ci.camera_height, ci.camera_width
    T = (H // 16) * (W // 16)
    tile_bits = _bit_width(max(T - 1, 0))
    depth_bits = max(_bit_width(int(np.float32(FAR) * np.float32(SCALE))), 1)
    key_bytes = 4
    if tile_bits + depth_bits > 32:
        key_bytes, depth_bits = 8, 32
    cap = T * N + 4096
    counters = np.zeros(8, np.int64)
    point_id, point_offset, num_tiles = (np.full(N, -9, np.int32) for _ in range(3))
    records, pic = np.zeros((N, 12), np.float32), np.zeros((N, 3), np.float32)
    keys = np.zeros(cap, np.uint32 if key_bytes == 4 else np.uint64)
    vals = np.zeros(cap, np.int32)
    q, t = _np(scene.q_pointcloud_camera, np.float32), _np(scene.t_pointcloud_camera, np.float32)
    K = _np(ci.camera_intrinsics, np.float32)
    inv, obj = _np(scene.point_invalid_mask, np.int8), _np(scene.point_object_id, np.int32)
    f3 = None if filter3d is None else np.ascontiguousarray(filter3d, dtype=np.float32)
    sw = oemu.emu_preprocess_ortho(
        ctypes.c_longlong(N), c(xyz), c(feats), c(inv), c(obj), q.shape[0], c(q), c(t), c(K), W, H, ctypes.c_float(NEAR),
        ctypes.c_float(FAR), ctypes.c_float(SCALE), depth_bits, key_bytes, int(filter_tiles), ctypes.c_longlong(cap),
        None if f3 is None else c(f3), c(counters), c(point_id), c(point_offset), c(num_tiles), c(records), c(pic), c(keys),
        c(vals))
    assert sw > 0 or N == 0
    pre = SimpleNamespace(feats=feats, counters=counters, point_id=point_id, point_offset=point_offset, num_tiles=num_tiles,
                          records=records, pic=pic, keys=keys, vals=vals, depth_bits=depth_bits, tile_bits=tile_bits, H=H, W=W,
                          T=T)
    M, Kk = int(counters[0]), int(counters[1])
    sk, sv = emu_sort_frame(emu, pre, Kk)
    start, end = np.zeros(T, np.int32), np.zeros(T, np.int32)
    emu.emu_tile_ranges(c(sk), ctypes.c_longlong(Kk), sk.dtype.itemsize, depth_bits, T, c(start), c(end))
    image, depth, acc = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32)
    last, cnt = np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    f = None if features is None else np.ascontiguousarray(features, dtype=np.float32)
    C = 0 if f is None else f.shape[1]
    fmap = np.zeros((H, W, max(C, 1)), np.float32)
    if Kk:
        oemu.emu_blend_forward_ortho(int(exact), H, W, c(start), c(end), c(sv), c(records), c(point_id), C,
                                     None if f is None else c(f), c(image), c(depth), c(acc), c(last), c(cnt), c(fmap))
    return SimpleNamespace(pre=pre, M=M, K=Kk, start=start, end=end, sorted_keys=sk, sorted_vals=sv, image=image, depth=depth,
                           acc_alpha=acc, last_effective=last, count=cnt, exact=exact, scene=scene, features=f,
                           fmap=fmap[..., :C] if C else None, filter3d=f3)


def emulated_backward_ortho(emu, oemu, st, grad_image, grad_depth=None, grad_alpha=None, grad_feature_map=None, pose=False,
                            intr=False, band=3, factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """Backward of a state of :func:`emulated_forward_ortho` (exact arithmetic): loop A (DEPTH / ALPHA / CF by the given
    gradients), then the per-point kernel (DEPTH with ``grad_depth``, FILTER with the state's filter, POSE / INTR as asked) and
    the finishing kernels.  Returns a namespace: gx (N,3), gf (N,56), gext (N,C) or None, gq (K,4) / gt (K,3) with ``pose``,
    gK (3,3) with ``intr``, accum (M,12), blocks."""
    pre, M, scene = st.pre, st.M, st.scene
    H, W = pre.H, pre.W
    N = pre.point_offset.shape[0]
    g = np.ascontiguousarray(grad_image, dtype=np.float32)
    gd = None if grad_depth is None else np.ascontiguousarray(grad_depth, dtype=np.float32)
    ga = None if grad_alpha is None else np.ascontiguousarray(grad_alpha, dtype=np.float32)
    f = st.features
    C = 0 if (f is None or grad_feature_map is None) else f.shape[1]
    gF = None if C == 0 else np.ascontiguousarray(grad_feature_map, dtype=np.float32)
    gfeat = np.zeros((N, max(C, 1)), np.float32)
    accum, mag = np.zeros((max(M, 1), 12), np.float32), np.zeros((H, W, 2), np.float32)
    if st.K:
        oemu.emu_blend_backward_ortho(H, W, c(st.start), c(st.end), c(st.sorted_vals), c(pre.records), c(g), c(st.acc_alpha),
                                      c(st.last_effective), None if gd is None else c(gd), None if gd is None else c(st.depth),
                                      None if ga is None else c(ga), c(pre.point_id), C, None if C == 0 else c(f),
                                      None if C == 0 else c(gF), c(gfeat), c(accum), c(mag))
    q, t = _np(scene.q_pointcloud_camera, np.float32), _np(scene.t_pointcloud_camera, np.float32)
    n_obj = q.shape[0]
    poses = np.zeros((n_obj, 20), np.float32)
    emu.emu_pose(n_obj, c(q), c(t), c(poses))
    xyz = _np(scene.point_cloud, np.float32)
    K = _np(scene.camera_info.camera_intrinsics, np.float32)
    obj = _np(scene.point_object_id, np.int32)
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    gq, gt = np.full((n_obj, 4), 7.0, np.float32), np.full((n_obj, 3), 7.0, np.float32)
    gK = np.full((3, 3), 7.0, np.float32)
    pose_partials = np.full((PARTIAL_BLOCKS, n_obj, 12), 7.0, np.float32)
    intr_partials = np.full((PARTIAL_BLOCKS, 6), 7.0, np.float32)
    fl = ctypes.c_float
    blocks = oemu.emu_backward_points_ortho(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(accum), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(fl(v) for v in factors), c(gx), c(gf), int(gd is not None),
        None if st.filter3d is None else c(st.filter3d), int(pose), int(intr), n_obj, c(q), c(pose_partials), c(gq), c(gt),
        c(intr_partials), c(gK))
    return SimpleNamespace(gx=gx, gf=gf, gext=gfeat[:, :C] if C else None, gq=gq if pose else None, gt=gt if pose else None,
                           gK=gK if intr else None, accum=accum[:M].copy(), blocks=blocks)
