"""Exact references for the device sort and the tile ranges, the frame layout table they are checked on, and that table
run through the kernel sources of csrc/sort.cu under the CPU emulator of tests/simt.

The references are plain numpy: a stable argsort for the sort and searchsorted for the tile ranges; every comparison is
bit for bit (keys, payloads, tile starts and ends).  ``test_gpu_sort_pipeline.py`` runs the same table on the GPU at scale
and imports the helpers from here.  The checker self-tests show that each assertion fails on the kind of error a broken
sort or range kernel would make (a swapped pair of tied payloads, a key out of order, a range off by one, a stale range
left in an empty tile), without running a broken kernel anywhere."""
import ctypes

import numpy as np
import pytest

from simt_helpers import build_emulator, c

SORT_TILE = 3072  # keys per CTA tile of the radix passes (csrc/common.cuh SORT_TILE)
GSB_FLAG_FORCE_KEY64 = 2
GSB_FLAG_KEEP_ALL_TILE_PAIRS = 8
CNT_K, CNT_MAX_DEPTH_KEY = 1, 4  # workspace counter slots (csrc/common.cuh)
TICKET_SORT0 = 1                 # first of the radix passes' ticket words; +8 is the histogram kernel's done count


# ------------------------------------------------------------------ exact references and checkers
def _first_diff(a, b):
    bad = np.flatnonzero(a != b)
    return f"{bad.size} mismatches, first at {bad[0]}: got {a[bad[0]]!r}, want {b[bad[0]]!r}" if bad.size else ""


def check_sorted_pairs(keys_in, vals_in, keys_out, vals_out):
    """keys_out / vals_out must be exactly the stable sort of (keys_in, vals_in): ties keep their input order."""
    keys_in, keys_out = np.asarray(keys_in), np.asarray(keys_out)
    vals_in, vals_out = np.asarray(vals_in), np.asarray(vals_out)
    assert keys_out.shape == keys_in.shape and vals_out.shape == vals_in.shape
    order = np.argsort(keys_in, kind="stable")
    want_k, want_v = keys_in[order], vals_in[order]
    assert np.array_equal(keys_out, want_k), "keys: " + _first_diff(keys_out, want_k)
    assert np.array_equal(vals_out, want_v), "payloads: " + _first_diff(vals_out, want_v)


def expected_tile_ranges(sorted_keys, depth_bits, num_tiles):
    """[start, end) of every tile in a sorted list of keys  tile << depth_bits | depth;  0, 0 for an empty tile."""
    tile = (np.asarray(sorted_keys).astype(np.uint64) >> np.uint64(depth_bits)).astype(np.int64)
    t = np.arange(num_tiles)
    start = np.searchsorted(tile, t, side="left").astype(np.int32)
    end = np.searchsorted(tile, t, side="right").astype(np.int32)
    empty = start == end
    start[empty] = 0
    end[empty] = 0
    return start, end


def check_tile_ranges(sorted_keys, depth_bits, tile_start, tile_end):
    want_s, want_e = expected_tile_ranges(sorted_keys, depth_bits, len(tile_start))
    tile_start, tile_end = np.asarray(tile_start), np.asarray(tile_end)
    assert np.array_equal(tile_start, want_s), "tile_start: " + _first_diff(tile_start, want_s)
    assert np.array_equal(tile_end, want_e), "tile_end: " + _first_diff(tile_end, want_e)


# ------------------------------------------------------------------ the frame layout table
# Every layout is reached the way a frame reaches it: through (H, W, far, scale, flags).  The tile-id width comes from the
# camera size, the depth width d from int32(far * scale) = 2^(d-1) (exact in float32).  Layouts whose tile + depth bits
# exceed 32 switch to the reference's 64-bit packing (depth field of 32 bits); GSB_FLAG_FORCE_KEY64 forces it.
TILE_SHAPES = {0: (16, 16), 1: (16, 32), 12: (1024, 1024), 13: (1072, 1920)}  # tile_bits -> (H, W)


def mirror_layout(tile_bits, depth_bits, flags):
    """(key_bytes, depth field width) that csrc/api.cu compute_layout picks."""
    if (flags & GSB_FLAG_FORCE_KEY64) or tile_bits + depth_bits > 32:
        return 8, 32
    return 4, depth_bits


def layout_table():
    """(tile_bits, d, flags): every 32-bit layout of each tile width, the first natural 64-bit one, and a forced one."""
    rows = []
    for tb in TILE_SHAPES:
        for d in range(1, 32):
            if tb + d > 32:
                rows.append((tb, d, 0))  # the first natural 64-bit layout; larger d give the same layout
                break
            rows.append((tb, d, 0))
        rows.append((tb, 17, GSB_FLAG_FORCE_KEY64))
    return rows


def layout_args(tb, d, flags):
    H, W = TILE_SHAPES[tb]
    return H, W, 1.0, float(2 ** (d - 1)), flags


def layout_id(row):
    tb, d, flags = row
    return f"t{tb}-d{d}" + ("-key64" if flags & GSB_FLAG_FORCE_KEY64 else "")


def max_depth_keys(tile_bits, depth_field):
    """The frame's largest depth key m for one layout: 0 and 1; for every live width b that puts the compacted key
    (tile_bits + b bits) exactly on a multiple of 8, 2^b - 1 (that width) and 2^b (one bit past it: one more pass); and
    the whole depth field.  Depth keys are non-negative int32, so at most 31 live bits."""
    top = min(depth_field, 31)
    ms = {0, 1, (1 << top) - 1}
    for b in range(0, top + 1):
        if (tile_bits + b) % 8 == 0:
            ms.add((1 << b) - 1)
            if b + 1 <= top:
                ms.add(1 << b)
    return sorted(ms)


def active_passes(tile_bits, m):
    """8-bit radix passes the compacted key  tile << bit_width(m) | depth  needs (at least one)."""
    return max((tile_bits + int(m).bit_length() + 7) // 8, 1)


def frame_keys(rng, n, tile_bits, depth_field, key_bytes, m, num_tiles, kind="mixed"):
    """Synthetic frame keys  tile << depth_field | depth  with depth <= m (m itself present when n > 0) and random int32
    payloads, negatives included.  kind: "mixed" (half the keys from a few tiles and depths: long runs of equal keys; the
    first and the last tile occupied), "one_tile" (every key in one tile), "first_last" (only the first and last tile)."""
    dtype = np.uint32 if key_bytes == 4 else np.uint64
    vals = rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64).astype(np.int32)
    if n == 0:
        return np.zeros(0, dtype), vals
    if kind == "one_tile":
        tile = np.full(n, int(rng.integers(0, num_tiles)), np.uint64)
    elif kind == "first_last":
        tile = np.where(rng.random(n) < 0.5, 0, num_tiles - 1).astype(np.uint64)
    else:
        pool = np.unique(np.concatenate([[0, num_tiles - 1], rng.integers(0, num_tiles, 6)])).astype(np.uint64)
        tile = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, num_tiles, n).astype(np.uint64))
        if n >= 2:
            tile[rng.integers(0, n)] = 0
            tile[rng.integers(0, n)] = num_tiles - 1
    dpool = np.unique(np.array([0, m, m // 2, m // 3, int(rng.integers(0, m + 1))], np.uint64))
    depth = np.where(rng.random(n) < 0.5, rng.choice(dpool, n), rng.integers(0, m + 1, n, dtype=np.uint64))
    depth[rng.integers(0, n)] = m
    keys = (tile << np.uint64(depth_field)) | depth
    return keys.astype(dtype), vals


def stage_cases(tile_bits, depth_field, small_n):
    """(m, n, kind) of one layout: every m of max_depth_keys() on mixed keys of a partial last tile, and, at the full depth
    field, no key, one key, all keys in one tile, and keys only in the first and the last tile."""
    ms = max_depth_keys(tile_bits, depth_field)
    cases = [(m, small_n, "mixed") for m in ms]
    top = ms[-1]
    cases += [(top, 0, "mixed"), (top, 1, "mixed"), (top, small_n, "one_tile"), (top, small_n, "first_last")]
    return cases


# ------------------------------------------------------------------ checker self-tests
def _sorted_example():
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 6, 400).astype(np.uint32)  # many ties
    vals = rng.integers(-(1 << 31), 1 << 31, 400, dtype=np.int64).astype(np.int32)
    order = np.argsort(keys, kind="stable")
    return keys, vals, keys[order].copy(), vals[order].copy()


def test_checker_accepts_the_stable_sort():
    keys, vals, ko, vo = _sorted_example()
    check_sorted_pairs(keys, vals, ko, vo)
    check_tile_ranges(ko, 0, *expected_tile_ranges(ko, 0, 8))


def test_checker_rejects_two_swapped_tied_payloads():
    keys, vals, ko, vo = _sorted_example()
    i = int(np.flatnonzero(ko[1:] == ko[:-1])[5])  # ko[i] == ko[i + 1]: the key list stays sorted
    vo[[i, i + 1]] = vo[[i + 1, i]]
    with pytest.raises(AssertionError, match="payloads"):
        check_sorted_pairs(keys, vals, ko, vo)


def test_checker_rejects_one_key_out_of_order():
    keys, vals, ko, vo = _sorted_example()
    i = int(np.flatnonzero(ko[1:] != ko[:-1])[2])  # ko[i] < ko[i + 1]
    ko[[i, i + 1]] = ko[[i + 1, i]]
    vo[[i, i + 1]] = vo[[i + 1, i]]
    with pytest.raises(AssertionError, match="keys"):
        check_sorted_pairs(keys, vals, ko, vo)


@pytest.mark.parametrize("which,delta", [("start", 1), ("start", -1), ("end", 1), ("end", -1)])
def test_checker_rejects_a_tile_range_off_by_one(which, delta):
    _, _, ko, _ = _sorted_example()
    start, end = expected_tile_ranges(ko, 0, 8)
    t = 3
    assert end[t] > start[t] > 0
    (start if which == "start" else end)[t] += delta
    with pytest.raises(AssertionError, match=f"tile_{which}"):
        check_tile_ranges(ko, 0, start, end)


def test_checker_rejects_a_stale_range_in_an_empty_tile():
    _, _, ko, _ = _sorted_example()
    start, end = expected_tile_ranges(ko, 0, 8)
    assert start[7] == end[7] == 0  # no key has tile 7
    start[7], end[7] = 120, 160      # what a previous, larger frame could have left there
    with pytest.raises(AssertionError, match="tile_start"):
        check_tile_ranges(ko, 0, start, end)


def test_tile_range_reference_known_answer():
    """The reference's own example (tile << 32 | depth, tiles 0 0 0 2 2 5 5 5 5 7 of 9)."""
    tiles = np.array([0, 0, 0, 2, 2, 5, 5, 5, 5, 7], np.uint64)
    keys = (tiles << np.uint64(32)) | np.arange(10, dtype=np.uint64)
    start, end = expected_tile_ranges(keys, 32, 9)
    assert start.tolist() == [0, 0, 3, 0, 0, 5, 0, 9, 0] and end.tolist() == [3, 0, 5, 0, 0, 9, 0, 10, 0]


def test_layout_table_matches_the_library_layout():
    """The mirror of compute_layout that the table relies on agrees with gsb200_workspace_layout for every row, and the
    table really reaches tile widths 0, 1, 12, 13, every depth width 1..31, and both ways to 64-bit keys."""
    from taichi_3d_gaussian_splatting_b200 import _lib
    seen_d, natural64, forced64 = set(), 0, 0
    for tb, d, flags in layout_table():
        H, W, far, scale, fl = layout_args(tb, d, flags)
        L = _lib.workspace_layout(0, 1, 5000, H, W, far, scale, fl)
        kb, depth_field = mirror_layout(tb, d, flags)
        assert (L.tile_bits, L.key_bytes, L.depth_bits) == (tb, kb, depth_field), (tb, d, flags)
        seen_d.add(d)
        natural64 += kb == 8 and not flags
        forced64 += bool(flags)
    assert seen_d == set(range(1, 32)) and natural64 == 2 and forced64 == 4
    assert active_passes(13, 1023) == 3 and active_passes(0, 0) == 1 and active_passes(8, 255) == 2


def test_binding_declares_the_signature_of_every_export():
    """Called through the binding without declared argtypes, ctypes passes each Python int as a 32-bit C int: the device
    pointers given to gsb200_find_tile_start_and_end were cut to their low 32 bits and the kernel wrote to a wild address.
    Every export must carry its signature from _lib.load() on, not only after some wrapper has set it."""
    from taichi_3d_gaussian_splatting_b200 import _lib
    lib = _lib.load()
    for name in _lib.EXPORTS:
        assert getattr(lib, name).argtypes is not None, f"{name} has no declared argtypes"
    fn = lib.gsb200_find_tile_start_and_end
    assert list(fn.argtypes) == [_lib.c_vp, _lib.c_i64, _lib.c_vp, _lib.c_vp, _lib.c_i32, _lib.c_vp]
    assert fn.restype is ctypes.c_int


# ------------------------------------------------------------------ the layout table under the emulator
@pytest.fixture(scope="module")
def emu():
    return build_emulator()


def emulate_stage(emu, keys, vals, key_bytes, tile_bits, depth_field, m, num_tiles):
    """launch_sort + launch_tile_ranges of one frame (csrc/sort.cu) under the emulator: the compacted sort from the frame's
    largest depth key m, then the tile ranges into zeroed arrays (the pose kernel zeroes them on the device)."""
    n = keys.shape[0]
    ko, vo = np.empty_like(keys), np.empty_like(vals)
    mk = np.array([m], np.int32)
    sw = emu.emu_sort_pairs_compacted(c(keys), c(vals), c(ko), c(vo), ctypes.c_longlong(n), key_bytes, depth_field,
                                      tile_bits + depth_field, c(mk))
    assert sw > 0 if n else sw == 0  # -1: the input buffer was written
    start, end = np.zeros(num_tiles, np.int32), np.zeros(num_tiles, np.int32)
    emu.emu_tile_ranges(c(ko), ctypes.c_longlong(n), key_bytes, depth_field, num_tiles, c(start), c(end))
    return ko, vo, start, end


@pytest.mark.parametrize("row", layout_table(), ids=layout_id)
def test_emulated_frame_sort_over_the_layout_table(emu, row):
    """Every layout of the table, every m that changes the pass count, the edge-case key sets: csrc/sort.cu's compacted
    sort (digits cut across the depth / tile boundary, device-side pass count, b / c buffer rotation) and its tile ranges
    against the exact references.  700 keys: one partial tile with a TMA tail."""
    tb, d, flags = row
    kb, depth_field = mirror_layout(tb, d, flags)
    H, W = TILE_SHAPES[tb]
    T = (H // 16) * (W // 16)
    rng = np.random.default_rng(1000 * tb + d + flags)
    for m, n, kind in stage_cases(tb, depth_field, 701):
        keys, vals = frame_keys(rng, n, tb, depth_field, kb, m, T, kind)
        ko, vo, start, end = emulate_stage(emu, keys, vals, kb, tb, depth_field, m, T)
        check_sorted_pairs(keys, vals, ko, vo)
        check_tile_ranges(ko, depth_field, start, end)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 3000])
@pytest.mark.parametrize("kind", ["mixed", "one_tile", "first_last"])
def test_emulated_raw_tile_ranges(emu, n, kind):
    """tile_ranges_kernel on the reference's packing (tile << 32 | depth, sorted int64), as gsb200_find_tile_start_and_end
    launches it: sizes around one 256-thread CTA, empty tiles, the first and the last tile occupied, one tile only."""
    rng = np.random.default_rng(n * 3 + len(kind))
    T = 40
    keys, _ = frame_keys(rng, n, 6, 32, 8, 1000, T, kind)
    keys = np.sort(keys)
    start, end = np.zeros(T, np.int32), np.zeros(T, np.int32)
    emu.emu_tile_ranges(c(keys), ctypes.c_longlong(n), 8, 32, T, c(start), c(end))
    check_tile_ranges(keys, 32, start, end)
