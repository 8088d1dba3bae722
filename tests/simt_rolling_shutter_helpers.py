"""The rolling shutter (``gsb200_forward_rolling_shutter`` / ``gsb200_backward_rolling_shutter``) executed on the CPU from the
unmodified kernel sources: the rolling-shutter instantiations of the per-point forward and backward, the finishing kernel and the
helpers of ``common.cuh`` (``tests/simt/emu_rolling_shutter.cpp``, a library of its own), chained with the emulated sort, tile
ranges, forward blend and loop A of the other emulator libraries exactly as ``csrc/api.cu`` chains them.  Test
infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, _bit_width, c, emu_sort_frame
from simt_lens_helpers import _coeffs

MODELS = {"pinhole": 0, "opencv": 1, "fisheye": 2}
RS_GRAD_PARTIAL_BLOCKS = 2048  # GSB_RS_GRAD_PARTIAL_BLOCKS of include/gsb200.h


def build_rolling_shutter_emulator():
    out = os.path.join(SIMT, "libsimt_emu_rolling_shutter.so")
    tu = os.path.join(SIMT, "emu_rolling_shutter.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_preprocess_rs.restype = ctypes.c_longlong
    L.emu_backward_points_rs.restype = ctypes.c_int
    return L


def rotation(remu, tau, w):
    """The device helper rolling_shutter_rotation in float32: (n, 3, 3)."""
    tau = np.ascontiguousarray(np.atleast_1d(tau), np.float32)
    w = np.ascontiguousarray(w, np.float32)
    R = np.zeros((tau.shape[0], 3, 3), np.float32)
    remu.emu_rolling_shutter_rotation(ctypes.c_longlong(tau.shape[0]), c(tau), c(w), c(R))
    return R


def run_preprocess_rs(remu, scene, model, k, motion, cfg=None, filter_tiles=True):
    """simt_lens_helpers.run_preprocess_lens with the rolling-shutter kernel (model "pinhole": no lens); also returns the
    row times (N,)."""
    cfg = cfg or {}
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    feats = scene.point_cloud_features.detach().numpy().astype(np.float32).copy()
    N = xyz.shape[0]
    ci = scene.camera_info
    H, W = ci.camera_height, ci.camera_width
    far, scale, near = cfg.get("far_plane", 1000.0), cfg.get("depth_to_sort_key_scale", 100.0), cfg.get("near_plane", 0.8)
    T = (H // 16) * (W // 16)
    tile_bits = _bit_width(max(T - 1, 0))
    depth_bits = max(_bit_width(int(np.float32(far) * np.float32(scale))), 1)
    key_bytes = 4
    if tile_bits + depth_bits > 32:
        key_bytes, depth_bits = 8, 32
    cap = 64 * N + 4096
    counters = np.zeros(8, np.int64)
    point_id, point_offset, num_tiles = (np.full(N, -9, np.int32) for _ in range(3))
    records, pic = np.zeros((N, 12), np.float32), np.zeros((N, 3), np.float32)
    keys = np.zeros(cap, np.uint32 if key_bytes == 4 else np.uint64)
    vals = np.zeros(cap, np.int32)
    row_time = np.full(N, 7.0, np.float32)  # every row must be overwritten
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    K = ci.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    inv = scene.point_invalid_mask.numpy().astype(np.int8).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    co = _coeffs(k)
    m = np.ascontiguousarray(motion, np.float32)
    sw = remu.emu_preprocess_rs(
        ctypes.c_longlong(N), c(xyz), c(feats), c(inv), c(obj), q.shape[0], c(q), c(t), c(K), W, H, ctypes.c_float(near),
        ctypes.c_float(far), ctypes.c_float(scale), depth_bits, key_bytes, int(filter_tiles), 0, ctypes.c_longlong(cap),
        c(counters), c(point_id), c(point_offset), c(num_tiles), c(records), c(pic), c(keys), c(vals), MODELS[model], c(co),
        c(m), c(row_time))
    assert sw > 0
    return SimpleNamespace(feats=feats, counters=counters, point_id=point_id, point_offset=point_offset, num_tiles=num_tiles,
                           records=records, pic=pic, keys=keys, vals=vals, depth_bits=depth_bits, tile_bits=tile_bits, H=H, W=W, T=T,
                           row_time=row_time)


def emulated_forward_rs(emu, remu, scene, model, k, motion, exact=True):
    """simt_lens_helpers.emulated_forward_lens through the rolling shutter: the rolling-shutter per-point kernel, then the
    unchanged sort, tile ranges and forward blend.  Returns the same state (``st.rs`` = (model, k, motion))."""
    pre = run_preprocess_rs(remu, scene, model, k, motion)
    M, Kk = int(pre.counters[0]), int(pre.counters[1])
    sk, sv = emu_sort_frame(emu, pre, Kk)
    start, end = np.zeros(pre.T, np.int32), np.zeros(pre.T, np.int32)
    emu.emu_tile_ranges(c(sk), ctypes.c_longlong(Kk), sk.dtype.itemsize, pre.depth_bits, pre.T, c(start), c(end))
    H, W = pre.H, pre.W
    image, depth, acc = np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.float32), np.zeros((H, W), np.float32)
    last, cnt = np.zeros((H, W), np.int32), np.zeros((H, W), np.int32)
    if Kk:
        emu.emu_blend_forward(0, int(exact), H, W, c(start), c(end), c(sv), c(pre.records), c(image), c(depth), c(acc), c(last),
                              c(cnt))
    return SimpleNamespace(pre=pre, M=M, K=Kk, start=start, end=end, sorted_vals=sv, image=image, depth=depth, acc_alpha=acc,
                           last_effective=last, count=cnt, exact=exact, scene=scene, rs=(model, k, tuple(motion)))


def emulated_points_rs(emu, remu, st, accum, band=3, depth=False, mgrad=True, factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """The RS per-point kernel (MGRAD with ``mgrad``; DEPTH: word 11 of the rows is dL/dz) on the accumulator rows of a state
    of :func:`emulated_forward_rs`.  Returns the dense (N,3) / (N,56) gradients, dL/dm (6,) (None without mgrad), the per-CTA
    rows and the grid size."""
    pre, scene = st.pre, st.scene
    model, k, motion = st.rs
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
    gm = np.full(6, 7.0, np.float32)
    partials = np.full((RS_GRAD_PARTIAL_BLOCKS, 6), 7.0, np.float32)
    f = ctypes.c_float
    co = _coeffs(k)
    m = np.ascontiguousarray(motion, np.float32)
    row_time = pre.row_time.copy()
    blocks = remu.emu_backward_points_rs(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), int(depth), MODELS[model],
        c(co), c(m), c(row_time), int(mgrad), c(partials), c(gm))
    return SimpleNamespace(gx=gx, gf=gf, gm=gm if mgrad else None, partials=partials[:blocks].copy() if mgrad else None,
                           blocks=blocks)
