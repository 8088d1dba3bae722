"""The MCMC densification kernels (``csrc/mcmc.cu``) executed on the CPU from the unmodified kernel sources
(``tests/simt/emu_mcmc.cpp``, a library of its own).  Test infrastructure."""
import ctypes
import os
import subprocess

import numpy as np

from simt_helpers import CSRC, SIMT, c
from taichi_3d_gaussian_splatting_b200._lib import GsbMcmcRelocateArgs


def build_mcmc_emulator():
    out = os.path.join(SIMT, "libsimt_emu_mcmc.so")
    tu = os.path.join(SIMT, "emu_mcmc.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
        [os.path.join(os.path.dirname(CSRC), "..", "include", "gsb200.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_mcmc_temp_bytes.restype = ctypes.c_longlong
    L.emu_mcmc_regulariser.restype = ctypes.c_longlong
    L.emu_mcmc_regulariser.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_longlong] * 2 + [ctypes.c_float] * 2 + \
        [ctypes.c_void_p] * 2
    L.emu_mcmc_noise.restype = None
    L.emu_mcmc_noise.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_longlong] + [ctypes.c_float] * 3 + \
        [ctypes.c_ulonglong, ctypes.c_longlong, ctypes.c_longlong]
    L.emu_mcmc_relocate.restype = None
    L.emu_mcmc_relocate.argtypes = [ctypes.POINTER(GsbMcmcRelocateArgs)]
    return L


def emulated_regulariser(emu, features, invalid_mask, grad, num_valid, lambda_opacity, lambda_scale):
    """Adds into a copy of ``grad`` (N, 56); returns (grad, terms (2,))."""
    features = np.ascontiguousarray(features, np.float32)
    invalid_mask = np.ascontiguousarray(invalid_mask, np.int8)
    grad = np.array(grad, np.float32, order="C", copy=True)
    terms = np.full(2, np.nan, np.float32)
    temp = np.zeros(int(emu.emu_mcmc_temp_bytes()), np.uint8)
    ran = emu.emu_mcmc_regulariser(c(features), c(invalid_mask), c(grad), features.shape[0], num_valid, lambda_opacity,
                                   lambda_scale, c(terms), c(temp))
    assert ran > 0 and not temp[:16].any()  # the ticket is left ready for the next call
    return grad, terms


def emulated_noise(emu, xyz, features, invalid_mask, noise_scale, seed, step, gate_k=100.0, min_opacity=0.005, skip=-1):
    """The noise on a copy of ``xyz`` (N, 3)."""
    xyz = np.array(xyz, np.float32, order="C", copy=True)
    features = np.ascontiguousarray(features, np.float32)
    invalid_mask = np.ascontiguousarray(invalid_mask, np.int8)
    emu.emu_mcmc_noise(c(xyz), c(features), c(invalid_mask), xyz.shape[0], noise_scale, gate_k, min_opacity, seed, step, skip)
    return xyz


def emulated_relocate(emu, xyz, features, invalid_mask, object_id, sources, counts, destinations, destination_sources,
                      extra=None, moments=(), min_opacity=0.005):
    """In place on the given float32 / int8 / int32 arrays; ``moments``: up to three (exp_avg, exp_avg_sq) pairs (features,
    positions, extra features), None for a missing pair."""
    i32 = lambda x: np.ascontiguousarray(x, np.int32)  # noqa: E731
    sources, counts, destinations, destination_sources = map(i32, (sources, counts, destinations, destination_sources))
    pairs = list(moments) + [None] * (3 - len(moments))
    pp = [c(a) if a is not None else None for pair in pairs for a in (pair or (None, None))]
    args = GsbMcmcRelocateArgs(
        num_points=xyz.shape[0], num_sources=len(sources), source_ids=c(sources), source_counts=c(counts),
        num_destinations=len(destinations), destination_ids=c(destinations), destination_sources=c(destination_sources),
        pointcloud=c(xyz), pointcloud_features=c(features), point_invalid_mask=c(invalid_mask), point_object_id=c(object_id),
        extra_features=c(extra) if extra is not None else None, channels=extra.shape[1] if extra is not None else 0,
        min_opacity=min_opacity, feature_exp_avg=pp[0], feature_exp_avg_sq=pp[1], position_exp_avg=pp[2],
        position_exp_avg_sq=pp[3], extra_exp_avg=pp[4], extra_exp_avg_sq=pp[5], stream=None)
    emu.emu_mcmc_relocate(ctypes.byref(args))
