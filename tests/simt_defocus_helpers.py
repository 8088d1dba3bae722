"""The depth of field (``gsb200_forward_defocus`` / ``gsb200_backward_defocus``) executed on the CPU from the unmodified kernel
sources: the DEFOCUS instantiations of the per-point forward and backward and the finishing kernel
(``tests/simt/emu_defocus.cpp``, a library of its own), chained with the emulated sort, tile ranges, forward blend and loop A
of the other emulator libraries exactly as ``csrc/api.cu`` chains them.  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, _bit_width, c, emu_sort_frame
from simt_lens_helpers import _coeffs
from simt_rolling_shutter_helpers import MODELS, RS_GRAD_PARTIAL_BLOCKS


def build_defocus_emulator():
    out = os.path.join(SIMT, "libsimt_emu_defocus.so")
    tu = os.path.join(SIMT, "emu_defocus.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_preprocess_defocus.restype = ctypes.c_longlong
    L.emu_backward_points_defocus.restype = ctypes.c_int
    return L


def run_preprocess_defocus(demu, scene, model, k, motion, blur, defocus, rolling, filter_tiles=True):
    """simt_motion_blur_helpers.run_preprocess_blur with the DEFOCUS kernel and the thin lens ``defocus`` = (a, rho)."""
    xyz = scene.point_cloud.detach().numpy().astype(np.float32).copy()
    feats = scene.point_cloud_features.detach().numpy().astype(np.float32).copy()
    N = xyz.shape[0]
    ci = scene.camera_info
    H, W = ci.camera_height, ci.camera_width
    far, scale, near = 1000.0, 100.0, 0.8
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
    row_time = np.full(N, 7.0, np.float32)
    q = scene.q_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    t = scene.t_pointcloud_camera.detach().numpy().astype(np.float32).copy()
    K = ci.camera_intrinsics.detach().numpy().astype(np.float32).copy()
    inv = scene.point_invalid_mask.numpy().astype(np.int8).copy()
    obj = scene.point_object_id.numpy().astype(np.int32).copy()
    co = _coeffs(k)
    m = np.ascontiguousarray(motion, np.float32)
    mb = np.ascontiguousarray(blur, np.float32)
    df = np.ascontiguousarray(defocus, np.float32)
    sw = demu.emu_preprocess_defocus(
        ctypes.c_longlong(N), c(xyz), c(feats), c(inv), c(obj), q.shape[0], c(q), c(t), c(K), W, H, ctypes.c_float(near),
        ctypes.c_float(far), ctypes.c_float(scale), depth_bits, key_bytes, int(filter_tiles), 0, ctypes.c_longlong(cap),
        c(counters), c(point_id), c(point_offset), c(num_tiles), c(records), c(pic), c(keys), c(vals), MODELS[model], c(co),
        c(m), c(row_time), int(rolling), c(mb), c(df))
    assert sw > 0
    return SimpleNamespace(feats=feats, counters=counters, point_id=point_id, point_offset=point_offset, num_tiles=num_tiles,
                           records=records, pic=pic, keys=keys, vals=vals, depth_bits=depth_bits, tile_bits=tile_bits, H=H, W=W, T=T,
                           row_time=row_time)


def emulated_forward_defocus(emu, demu, scene, model, k, motion, blur, defocus, rolling, exact=True):
    """simt_motion_blur_helpers.emulated_forward_blur with the DEFOCUS per-point kernel, then the unchanged sort, tile ranges and
    forward blend.  ``st.blur`` = (model, k, motion, blur, rolling), ``st.defocus`` = (a, rho)."""
    pre = run_preprocess_defocus(demu, scene, model, k, motion, blur, defocus, rolling)
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
                           last_effective=last, count=cnt, exact=exact, scene=scene,
                           blur=(model, k, tuple(motion), tuple(blur), rolling), rs=(model, k, tuple(motion)),
                           defocus=tuple(defocus))


def emulated_points_defocus(emu, demu, st, accum, band=3, depth=False, dgrad=True, factors=(1.0, 0.5, 20.0, 5.0, 1.0)):
    """The DEFOCUS per-point kernel (DGRAD with ``dgrad``) on the accumulator rows of a state of
    :func:`emulated_forward_defocus`.  Returns the dense (N,3) / (N,56) gradients, dL/d(a, rho) (2,) (None without dgrad),
    the per-CTA rows and the grid size."""
    pre, scene = st.pre, st.scene
    model, k, motion, blur, rolling = st.blur
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
    gx, gf = np.full((N, 3), 7.0, np.float32), np.full((N, 56), 7.0, np.float32)
    gd = np.full(2, 7.0, np.float32)
    partials = np.full((RS_GRAD_PARTIAL_BLOCKS + 1, 6), 7.0, np.float32)
    f = ctypes.c_float
    co = _coeffs(k)
    m = np.ascontiguousarray(motion, np.float32)
    mb = np.ascontiguousarray(blur, np.float32)
    df = np.ascontiguousarray(st.defocus, np.float32)
    row_time = pre.row_time.copy()
    blocks = demu.emu_backward_points_defocus(
        ctypes.c_longlong(N), c(pre.point_offset), c(pre.records), c(pre.pic), c(acc), c(poses), c(xyz), c(pre.feats), c(obj),
        c(t), c(K), int(band) if band in (0, 1, 2) else 3, *(f(v) for v in factors), c(gx), c(gf), int(depth), MODELS[model],
        c(co), c(m), c(row_time), int(rolling), c(mb), c(df), int(dgrad), c(partials), c(gd))
    return SimpleNamespace(gx=gx, gf=gf, gd=gd if dgrad else None, partials=partials[:blocks].copy() if dgrad else None,
                           blocks=blocks)
