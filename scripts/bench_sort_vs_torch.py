"""Sort stage against the reference's own primitive on the same box: torch.sort on int64 keys + gather (GPCR:947-950, CUB
under the hood) and torch.sort on the 30-bit keys as int32, next to gsb200_sort_pairs.  Output: one JSON line per K."""
import ctypes, json, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taichi_3d_gaussian_splatting_b200 import _lib
lib = _lib.load()
lib.gsb200_sort_temp_bytes.restype = ctypes.c_int64
lib.gsb200_sort_temp_bytes.argtypes = [ctypes.c_int64, ctypes.c_int32]
lib.gsb200_sort_pairs.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int64, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]


def timed(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # microseconds


for n in (2_741_293, 4_044_076, 10_000_000):
    torch.manual_seed(0)
    tile = torch.randint(0, 8040, (n,), dtype=torch.int64)
    depth = torch.randint(200, 1000, (n,), dtype=torch.int64)
    keys32 = ((tile << 17) | depth).to(torch.int32).cuda()
    keys64 = ((tile << 32) | depth).cuda()  # the reference's packing
    vals = torch.arange(n, dtype=torch.int32, device="cuda")
    tb = lib.gsb200_sort_temp_bytes(n, 4)
    temp = torch.empty(tb, dtype=torch.uint8, device="cuda")
    ko, vo = torch.empty_like(keys32), torch.empty_like(vals)
    st = torch.cuda.current_stream().cuda_stream

    def ours():
        assert lib.gsb200_sort_pairs(keys32.data_ptr(), vals.data_ptr(), ko.data_ptr(), vo.data_ptr(), n, 4, 30, temp.data_ptr(), tb, st) == 0

    def ref64():  # GPCR:947-950: sort the int64 keys, gather the offsets by the permutation
        k, perm = torch.sort(keys64)
        return k, vals[perm]

    def ref64_stable():
        k, perm = torch.sort(keys64, stable=True)
        return k, vals[perm]

    def torch32():
        k, perm = torch.sort(keys32, stable=True)
        return k, vals[perm]

    row = {"K": n, "gsb200_sort_pairs_us": round(timed(ours), 1), "torch_sort_i64_plus_gather_us": round(timed(ref64), 1),
           "torch_sort_i64_stable_plus_gather_us": round(timed(ref64_stable), 1), "torch_sort_i32_stable_plus_gather_us": round(timed(torch32), 1)}
    ek, perm = torch.sort(keys32.to(torch.int64) & 0xFFFFFFFF, stable=True)
    ours(); torch.cuda.synchronize()
    row["correct"] = bool(torch.equal(ko.to(torch.int64) & 0xFFFFFFFF, ek) and torch.equal(vo.to(torch.int64), perm))
    print(json.dumps(row), flush=True)
