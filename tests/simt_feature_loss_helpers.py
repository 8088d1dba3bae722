"""The feature term of the fused train step (``csrc/feature_loss.cu``: sum pass -> gradient pass) executed on the CPU from
the unmodified kernel source (``tests/simt/emu_feature_loss.cpp``, a library of its own).  Test infrastructure."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np

from simt_helpers import CSRC, SIMT, c


def build_feature_loss_emulator():
    out = os.path.join(SIMT, "libsimt_emu_feature_loss.so")
    tu = os.path.join(SIMT, "emu_feature_loss.cpp")
    deps = [tu, os.path.join(SIMT, "simt_emu.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I", cuda_inc, "-o", out, tu],
                       check=True)
    L = ctypes.CDLL(out)
    L.emu_feature_loss.restype = ctypes.c_longlong
    L.emu_feature_loss_temp_bytes.restype = ctypes.c_longlong
    return L


def new_temp(emu):
    """The temp buffer, zeroed (its ticket must be zero before the first call)."""
    return np.zeros(int(emu.emu_feature_loss_temp_bytes()) + 16, np.uint8)


def emulated_feature_loss(emu, fmap, labels=None, target=None, weight=1.0, temp=None):
    """One call of the two passes on the (H, W, C) feature map, with ``labels`` (H, W) int32 (cross entropy) or ``target``
    (H, W, C) float32 (l2).  Returns {feature term, n_supervised} and dL/dF (NaN-filled where not written)."""
    fmap = np.ascontiguousarray(fmap, dtype=np.float32)
    H, W, C = fmap.shape
    lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.int32)
    tgt = None if target is None else np.ascontiguousarray(target, dtype=np.float32)
    temp = temp if temp is not None else new_temp(emu)
    loss2 = np.zeros(2, np.float32)
    grad = np.full((H, W, C), np.nan, np.float32)
    ran = emu.emu_feature_loss(c(fmap), None if lab is None else c(lab), None if tgt is None else c(tgt), H, W, C,
                               ctypes.c_float(weight), c(grad), c(loss2), c(temp))
    assert ran > 0
    return SimpleNamespace(loss=loss2, grad=grad)
