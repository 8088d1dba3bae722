"""The equirectangular panorama (``gsb200_forward_equirect`` / ``gsb200_backward_equirect``) executed on the CPU from the
unmodified kernel sources: the per-point forward, the WRAP forward blend and loop A and the per-point backward
(``tests/simt/emu_equirect.cpp``, a library of its own), chained with the emulated sort and tile ranges of
:mod:`simt_helpers` exactly as ``csrc/api.cu`` chains them.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, _bit_width, c, emu_sort_frame

NEAR, FAR, SCALE = 0.8, 1000.0, 100.0


def build_equirect_emulator():
    out = os.path.join(SIMT, "libsimt_emu_equirect.so")
    tu = os.path.join(SIMT, "emu_equirect.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_preprocess_equirect.restype = ctypes.c_longlong
    L.emu_blend_forward_equirect.restype = ctypes.c_longlong
    L.emu_blend_backward_equirect.restype = ctypes.c_longlong
    L.emu_backward_points_equirect.restype = None
    return L


def run_preprocess_equirect(qemu, scene, filter_tiles=True):
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    feats = scene.point_cloud_features.detach().numpy().astype(np.float32).copy()
    N = xyz.shape[0]
    ci = scene.camera_info
    H, W = ci.camera_height, ci.camera_width
    T = (H // 16) * (W // 16)
    tile_bits = _bit_width(max(T - 1, 0))
    depth_bits = max(_bit_width(int(np.float32(FAR) * np.float32(SCALE))), 1)
    key_bytes = 4
    if tile_bits + depth_bits > 32:
        key_bytes, depth_bits = 8, 32
    cap = T * N + 4096  # a near-pole splat may key every tile
    counters = np.zeros(8, np.int64)
    point_id, point_offset, num_tiles = (np.full(N, -9, np.int32) for _ in range(3))
    records, pic = np.zeros((N, 12), np.float32), np.zeros((N, 3), np.float32)
    keys = np.zeros(cap, np.uint32 if key_bytes == 4 else np.uint64)
    vals = np.zeros(cap, np.int32)
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    K = ci.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    inv = scene.point_invalid_mask.numpy().astype(np.int8).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    sw = qemu.emu_preprocess_equirect(
        ctypes.c_longlong(N), c(xyz), c(feats), c(inv), c(obj), q.shape[0], c(q), c(t), c(K), W, H, ctypes.c_float(NEAR),
        ctypes.c_float(FAR), ctypes.c_float(SCALE), depth_bits, key_bytes, int(filter_tiles), ctypes.c_longlong(cap),
        c(counters), c(point_id), c(point_offset), c(num_tiles), c(records), c(pic), c(keys), c(vals))
    assert sw > 0 or N == 0
    return SimpleNamespace(feats=feats, counters=counters, point_id=point_id, point_offset=point_offset, num_tiles=num_tiles,
                           records=records, pic=pic, keys=keys, vals=vals, depth_bits=depth_bits, tile_bits=tile_bits, H=H, W=W,
                           T=T)


def emulated_forward_equirect(emu, qemu, scene, exact=True, features=None, filter_tiles=True):
    """Forward of the panorama path under the emulator: the state for the backward with the outputs (``fmap`` with
    ``features`` (N,C))."""
    pre = run_preprocess_equirect(qemu, scene, filter_tiles)
    M, Kk = int(pre.counters[0]), int(pre.counters[1])
    sk, sv = emu_sort_frame(emu, pre, Kk)
    start, end = np.zeros(pre.T, np.int32), np.zeros(pre.T, np.int32)
    emu.emu_tile_ranges(c(sk), ctypes.c_longlong(Kk), sk.dtype.itemsize, pre.depth_bits, pre.T, c(start), c(end))
    H, W = pre.H, pre.W
    image, depth, acc = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32)
    last, cnt = np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    f = None if features is None else np.ascontiguousarray(features, dtype=np.float32)
    C = 0 if f is None else f.shape[1]
    fmap = np.zeros((H, W, max(C, 1)), np.float32)
    if Kk:
        qemu.emu_blend_forward_equirect(int(exact), H, W, c(start), c(end), c(sv), c(pre.records), c(pre.point_id), C,
                                        None if f is None else c(f), c(image), c(depth), c(acc), c(last), c(cnt), c(fmap))
    return SimpleNamespace(pre=pre, M=M, K=Kk, start=start, end=end, sorted_keys=sk, sorted_vals=sv, image=image, depth=depth,
                           acc_alpha=acc, last_effective=last, count=cnt, exact=exact, scene=scene, features=f,
                           fmap=fmap[..., :C] if C else None)


def emulated_backward_equirect(emu, qemu, st, grad_image, grad_depth=None, grad_alpha=None, grad_feature_map=None, band=3,
                               stats=False, factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """Backward of a state of :func:`emulated_forward_equirect`: loop A (WRAP; DEPTH / ALPHA / CF by the given gradients),
    then the per-point kernel (DEPTH with ``grad_depth``).  Returns (dL/dxyz (N,3), dL/dfeatures (N,56), dL/dextra (N,C) or
    None, accumulator rows (M,12))."""
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
        qemu.emu_blend_backward_equirect(int(st.exact), int(stats), H, W, c(st.start), c(st.end), c(st.sorted_vals),
                                         c(pre.records), c(g), c(st.acc_alpha), c(st.last_effective),
                                         None if gd is None else c(gd), None if gd is None else c(st.depth),
                                         None if ga is None else c(ga), c(pre.point_id), C, None if C == 0 else c(f),
                                         None if C == 0 else c(gF), c(gfeat), c(accum), c(mag))
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    poses = np.zeros((q.shape[0], 20), np.float32)
    emu.emu_pose(q.shape[0], c(q), c(t), c(poses))
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    K = scene.camera_info.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)  # every row must be overwritten
    fl = ctypes.c_float
    qemu.emu_backward_points_equirect(ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(accum), c(poses),
                                      c(xyz), c(pre.feats), c(obj), c(t), c(K), int(band) if band in (0, 1, 2) else 3,
                                      *(fl(v) for v in factors), c(gx), c(gf), int(gd is not None))
    return gx, gf, (gfeat[:, :C] if C else None), accum[:M].copy()
