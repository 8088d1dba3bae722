"""Build ``libgsb200.so`` in-tree with nvcc for sm_90a (H100; no JIT cache: the .so is built in the tree).

    python -m taichi_3d_gaussian_splatting_b200.build [--force] [--verbose]

``preprocess.cu`` and ``filter3d.cu`` are compiled with ``-fmad=false`` so that every per-point discrete decision is
bit-reproducible against the CPU oracle; the blend kernels use default FMA contraction.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, os.environ.get("GSB200_LIB_NAME", "libgsb200.so"))
EXTRA_DEFINES = os.environ.get("GSB200_DEFINES", "").split()  # e.g. "-DGSB_SORT_ITEMS=8" (tuning experiments)
OBJ_DIR = os.path.join(HERE, "build" + ("_" + os.environ["GSB200_LIB_NAME"] if "GSB200_LIB_NAME" in os.environ else ""))
STAMP = os.path.join(OBJ_DIR, "sources.sha1")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
          "--expt-relaxed-constexpr"]
SOURCES = {
    "api.cu": [],
    "preprocess.cu": ["-fmad=false"],
    "sort.cu": [],
    "blend_fwd.cu": [],
    "blend_bwd.cu": [],
    "blend_bwd_transposed.cu": [],
    "loss.cu": [],
    "image_loss.cu": [],
    "supervision_loss.cu": [],
    "feature_loss.cu": [],
    "appearance.cu": [],
    "adam.cu": [],
    "mcmc.cu": [],
    "filter3d.cu": ["-fmad=false"],
    "controller.cu": [],
    "exchange.cu": [],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _source_hash() -> str:
    h = hashlib.sha1()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    files.append(os.path.join(os.path.dirname(HERE), "include", "gsb200.h"))
    files.append(os.path.abspath(__file__))
    h.update(" ".join(EXTRA_DEFINES).encode())
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    digest = _source_hash()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == digest:
                return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
    objs = []
    procs = []
    for src, extra in SOURCES.items():
        obj = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        cmd = [nvcc, *ARCH_FLAGS, *COMMON, *ccbin, *extra, *EXTRA_DEFINES, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {src}\n{out}\n")
        elif verbose or "warning" in out:
            sys.stderr.write(f"--- {src}\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    # export only the extern "C" ABI (visibility=hidden elsewhere, default on the gsb200_* symbols)
    link = [nvcc, *ARCH_FLAGS, *ccbin, "-shared", "-o", LIB, *objs, "-cudart", "static"]
    subprocess.run(link, check=True)
    with open(STAMP, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
