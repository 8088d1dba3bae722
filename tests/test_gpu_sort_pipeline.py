"""-m gpu: the device radix sort and the tile ranges at the sizes and in the states where the persistent passes can go
wrong, against exact numpy references (stable argsort, searchsorted), bit for bit.

- gsb200_sort_pairs at >= 13 M keys: a pass launches at most the CTAs the GPU holds at once (<= 8 x 132 on an H100), so
  at 4 x 1056 x 3072 keys some CTA sorts at least four tiles, flipping its mbarrier parity and fencing the async proxy
  between them.  The ticket words left in the temp buffer show how many CTAs each pass ran.
- The frame sort through the stage entry points on a workspace the test owns: synthetic keys and a largest depth key m
  written where the per-point kernel leaves them, over the layout table of test_sort_pipeline_cpu (tile widths 0, 1, 12,
  13; depth widths 1..31; 64-bit keys), with every m that changes the compacted pass count -- all on ONE workspace per
  layout, so every run follows a run with a different pass count, key count and buffer rotation.
- gsb200_find_tile_start_and_end beyond its grid-stride threshold (8 x 132 x 256 keys).
- Whole frames (gsb200_forward) on one reused workspace -- large, small, large, empty, a different pass count, a frame
  that overflows the key capacity, normal -- against the same frames rendered into fresh workspaces."""
import ctypes
import math

import numpy as np
import pytest
import torch

from taichi_3d_gaussian_splatting_b200 import _lib
from taichi_3d_gaussian_splatting_b200.GaussianPointCloudRasterisation import Frame
from taichi_3d_gaussian_splatting_b200.synthetic import make_scene
from test_sort_pipeline_cpu import (CNT_K, CNT_MAX_DEPTH_KEY, GSB_FLAG_KEEP_ALL_TILE_PAIRS, SORT_TILE, TICKET_SORT0,
                                    TILE_SHAPES, active_passes, check_sorted_pairs, check_tile_ranges, frame_keys,
                                    layout_args, layout_id, layout_table, mirror_layout, stage_cases)

pytestmark = pytest.mark.gpu

MAX_RESIDENT = 8 * 132                   # CTAs of 256 threads an H100 can hold at once
BIG = 4 * MAX_RESIDENT * SORT_TILE       # 12 976 128: at least four tiles for some CTA of every pass
LARGE = 13_000_000                       # its last tile holds 2368 keys


def _np_to_dev(a):
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view)).cuda()


def _dev_to_np(t, dtype):
    return t.cpu().numpy().view(dtype)


def _record(msg):
    print(f"\n[sort pipeline] {msg}")


def _check_pass_ctas(tickets, passes, tiles, what):
    """Ticket words after a sort: every CTA of an active pass takes tickets until one lies past the keys, so word p ends at
    tiles + (CTAs of pass p); passes that did not run leave theirs at 0.  Returns the CTAs of the passes."""
    ctas = [int(tickets[p]) - tiles for p in range(passes)]
    assert all(1 <= x <= MAX_RESIDENT for x in ctas), (what, ctas, tiles)
    assert len(set(ctas)) == 1, (what, ctas)
    assert all(int(tickets[p]) == 0 for p in range(passes, 8)), (what, tickets)
    return ctas[0]


# ------------------------------------------------------------------ 1. gsb200_sort_pairs
class _Sorter:
    """gsb200_sort_pairs on one temp buffer for every call of the module, sized for the largest (n, key width) used."""

    def __init__(self, max_n, key_bytes):
        self.lib = _lib.load()
        self.temp = torch.empty(int(self.lib.gsb200_sort_temp_bytes(max_n, key_bytes)), dtype=torch.uint8, device="cuda")

    def sort(self, keys, vals, end_bit, keys_out=None):
        n = keys.shape[0]
        ko = torch.empty_like(keys) if keys_out is None else keys_out
        vo = torch.empty_like(vals)
        _lib.check(self.lib.gsb200_sort_pairs(keys.data_ptr(), vals.data_ptr(), ko.data_ptr(), vo.data_ptr(), n,
                                              keys.element_size(), end_bit, self.temp.data_ptr(), self.temp.shape[0],
                                              torch.cuda.current_stream().cuda_stream), "gsb200_sort_pairs")
        torch.cuda.synchronize()
        return ko, vo

    def tickets(self):
        return self.temp[256:256 + 4 * 9].view(torch.int32).cpu().numpy()


@pytest.fixture(scope="module")
def sorter():
    return _Sorter(2 ** 24 + 5, 8)


def _sort_and_check(sorter, keys, vals, end_bit):
    """Sort on the device, check inputs unchanged and the result against the stable sort; returns the pass CTAs."""
    kd, vd = _np_to_dev(keys), _np_to_dev(vals)
    k0, v0 = kd.clone(), vd.clone()
    ko, vo = sorter.sort(kd, vd, end_bit)
    assert torch.equal(kd, k0) and torch.equal(vd, v0), "the input buffers were written"
    check_sorted_pairs(keys, vals, _dev_to_np(ko, keys.dtype), _dev_to_np(vo, np.int32))
    n = keys.shape[0]
    return _check_pass_ctas(sorter.tickets(), (end_bit + 7) // 8, (n + SORT_TILE - 1) // SORT_TILE, f"n={n}")


def _payloads(rng, n):
    return rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64).astype(np.int32)


def _frame_like(rng, n):
    """2^13 tiles x 10 live depth bits, heavy ties: 23-bit keys as a C3 frame makes them."""
    tile = rng.integers(0, 1 << 13, n, dtype=np.uint32)
    depth = np.where(rng.random(n) < 0.5, rng.integers(0, 1 << 10, n, dtype=np.uint32), np.uint32(517))
    return (tile << np.uint32(10)) | depth


@pytest.mark.parametrize("extra", [0, 1, 2, 3, 704])
def test_sort_pairs_many_tiles_per_cta(sorter, extra):
    """>= 4 x 1056 x 3072 keys: the last tile holds 2368 + extra keys -- TMA tails of 0, 1, 2, 3 keys, and (704) a full
    last tile.  Every pass must run at most as many CTAs as the GPU holds, so some CTA sorts at least four tiles."""
    n = LARGE + extra
    assert n >= BIG
    rng = np.random.default_rng(extra)
    ctas = _sort_and_check(sorter, _frame_like(rng, n), _payloads(rng, n), 23)
    tiles = (n + SORT_TILE - 1) // SORT_TILE
    assert math.ceil(tiles / ctas) >= 4
    _record(f"gsb200_sort_pairs n={n}: {tiles} tiles, {ctas} resident CTAs per pass -> up to {math.ceil(tiles / ctas)} "
            f"tiles per CTA")


def test_sort_pairs_4byte_keys_beyond_2_pow_24(sorter):
    n = 2 ** 24 + 5
    rng = np.random.default_rng(24)
    pool = rng.integers(0, 1 << 32, 1 << 20, dtype=np.uint64).astype(np.uint32)
    keys = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32))
    _sort_and_check(sorter, keys, _payloads(rng, n), 32)


def test_sort_pairs_8byte_keys_one_key_tail(sorter):
    """~13 M 64-bit keys, odd count: the last tile's bulk copy leaves one 8-byte key to the plain loads."""
    n = LARGE + 1
    rng = np.random.default_rng(64)
    pool = rng.integers(0, 1 << 63, 1 << 20, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    keys = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, 1 << 63, n, dtype=np.uint64) << np.uint64(1))
    _sort_and_check(sorter, keys, _payloads(rng, n), 64)


def _distribution(name, rng, n):
    if name == "all_equal":  # one digit receives every key in every pass: look-back sums reach n
        return np.full(n, 0x5A5A5A5A, np.uint32), 32
    if name == "sorted":
        return np.sort(rng.integers(0, 1 << 20, n, dtype=np.uint32)), 20
    if name == "reverse":
        return np.sort(rng.integers(0, 1 << 20, n, dtype=np.uint32))[::-1].copy(), 20
    if name == "top_digit":  # only the last pass sees more than one digit
        return rng.integers(0, 256, n, dtype=np.uint32) << np.uint32(24), 32
    if name == "low_digit":  # every later pass sees one digit
        return rng.integers(0, 256, n, dtype=np.uint32), 32
    if name == "one_live_bit":  # end_bit 25: the last pass sorts one bit
        return rng.integers(0, 1 << 25, n, dtype=np.uint32), 25
    if name == "frame_like":
        return _frame_like(rng, n), 23
    raise ValueError(name)


@pytest.mark.parametrize("name", ["all_equal", "sorted", "reverse", "top_digit", "low_digit", "one_live_bit", "frame_like"])
def test_sort_pairs_key_distributions(sorter, name):
    n = LARGE + 3
    rng = np.random.default_rng(len(name))
    keys, end_bit = _distribution(name, rng, n)
    _sort_and_check(sorter, keys, _payloads(rng, n), end_bit)


def test_sort_pairs_reuses_one_temp_buffer_across_sizes(sorter):
    """large -> small -> large -> 1 -> large on one temp buffer: each call clears only the look-back state of its own
    tiles, so what a larger call left behind must not leak into a smaller one, nor the reverse."""
    rng = np.random.default_rng(9)
    big_a = (_frame_like(rng, LARGE + 2), _payloads(rng, LARGE + 2))
    big_b = (rng.integers(0, 1 << 32, LARGE, dtype=np.uint64).astype(np.uint32), _payloads(rng, LARGE))
    small = (rng.integers(0, 1 << 32, 5000, dtype=np.uint64).astype(np.uint32), _payloads(rng, 5000))
    one = (np.array([0xDEADBEEF], np.uint32), np.array([-7], np.int32))
    for keys, vals in (big_a, small, big_b, one, big_a):
        _sort_and_check(sorter, keys, vals, 32)


@pytest.mark.parametrize("key_bytes", [4, 8])
def test_sort_pairs_offset_input_view(sorter, key_bytes):
    """keys_in 16 bytes into a larger tensor (the histogram kernel reads it with 16-byte vector loads, pass 0 with bulk
    copies): the sort must read exactly the viewed keys."""
    n = 1_000_003
    rng = np.random.default_rng(key_bytes)
    dt = np.uint32 if key_bytes == 4 else np.uint64
    pad = 16 // key_bytes
    base = rng.integers(0, 1 << 30, n + 2 * pad, dtype=np.uint64).astype(dt)
    vals = _payloads(rng, n)
    dev = _np_to_dev(base)
    kd = dev[pad:pad + n]
    assert kd.data_ptr() - dev.data_ptr() == 16
    vd = _np_to_dev(vals)
    ko, vo = sorter.sort(kd, vd, 30)
    assert torch.equal(dev, _np_to_dev(base))
    check_sorted_pairs(base[pad:pad + n], vals, _dev_to_np(ko, dt), _dev_to_np(vo, np.int32))


# ------------------------------------------------------------------ 2. the frame sort through the stage entry points
class _StageWorkspace:
    """A workspace the test owns, driven stage by stage: gsb200_stage_preprocess with no points (only the pose kernel's
    clears run), then keys / payloads / K / largest depth key written where the per-point kernel leaves them, then
    gsb200_stage_sort and gsb200_stage_tile_ranges."""

    def __init__(self, H, W, far, scale, flags, key_capacity):
        self.lib = _lib.load()
        self.L = _lib.workspace_layout(0, 1, key_capacity, H, W, far, scale, flags)
        self.T = (H // 16) * (W // 16)
        self.ws = torch.empty(self.L.total_bytes, dtype=torch.uint8, device="cuda")
        self.dummy = torch.zeros(64, device="cuda")  # camera_intrinsics / rasterized_image must be set; no stage reads them
        self.args = _lib.GsbForwardArgs(
            num_points=0, num_objects=0, camera_intrinsics=self.dummy.data_ptr(), camera_height=H, camera_width=W,
            near_plane=0.0, far_plane=far, depth_to_sort_key_scale=scale, rgb_only=1, flags=flags,
            workspace=self.ws.data_ptr(), workspace_bytes=self.L.total_bytes, key_capacity=key_capacity,
            rasterized_image=self.dummy.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
        self.key_dtype = torch.int32 if self.L.key_bytes == 4 else torch.int64

    def _view(self, off, count, dtype):
        size = torch.empty((), dtype=dtype).element_size()
        return self.ws[off:off + count * size].view(dtype)

    def run(self, keys, vals, m):
        n = keys.shape[0]
        _lib.check(self.lib.gsb200_stage_preprocess(ctypes.byref(self.args)), "gsb200_stage_preprocess")
        if n:
            self._view(self.L.keys_a, n, self.key_dtype).copy_(_np_to_dev(keys))
            self._view(self.L.vals_a, n, torch.int32).copy_(_np_to_dev(vals))
        counters = self._view(self.L.counters, 8, torch.int64)
        counters[CNT_K] = n
        counters[CNT_MAX_DEPTH_KEY] = m
        _lib.check(self.lib.gsb200_stage_sort(ctypes.byref(self.args)), "gsb200_stage_sort")
        _lib.check(self.lib.gsb200_stage_tile_ranges(ctypes.byref(self.args)), "gsb200_stage_tile_ranges")
        torch.cuda.synchronize()
        kt = np.uint32 if self.L.key_bytes == 4 else np.uint64
        ko = _dev_to_np(self._view(self.L.keys_b, n, self.key_dtype), kt)
        vo = _dev_to_np(self._view(self.L.vals_b, n, torch.int32), np.int32)
        start = self._view(self.L.tile_start, self.T, torch.int32).cpu().numpy()
        end = self._view(self.L.tile_end, self.T, torch.int32).cpu().numpy()
        tickets = self._view(self.L.tickets, 16, torch.int32).cpu().numpy()[TICKET_SORT0:TICKET_SORT0 + 8]
        return ko, vo, start, end, tickets


def _check_stage(sw, keys, vals, m, what):
    ko, vo, start, end, tickets = sw.run(keys, vals, m)
    check_sorted_pairs(keys, vals, ko, vo)
    check_tile_ranges(ko, sw.L.depth_bits, start, end)
    n = keys.shape[0]
    return _check_pass_ctas(tickets, active_passes(sw.L.tile_bits, m), (n + SORT_TILE - 1) // SORT_TILE, what)


@pytest.mark.parametrize("row", layout_table(), ids=layout_id)
def test_stage_sort_and_tile_ranges_over_the_layout_table(row):
    """Every m of the layout (0, 1, each width on and one past a multiple of 8, the whole depth field) and the edge-case key
    sets, on one workspace: the pass count decided on the device (read back from the ticket words: a pass beyond the
    compacted key exits before it takes a ticket), the digits cut across the depth / tile boundary, the b / c rotation,
    and tile ranges that the pose kernel must have cleared after the previous run."""
    tb, d, flags = row
    H, W, far, scale, fl = layout_args(tb, d, flags)
    sw = _StageWorkspace(H, W, far, scale, fl, 30_000)
    kb, depth_field = mirror_layout(tb, d, flags)
    assert (sw.L.tile_bits, sw.L.key_bytes, sw.L.depth_bits) == (tb, kb, depth_field)
    rng = np.random.default_rng(7000 + 100 * tb + d + flags)
    cases = stage_cases(tb, depth_field, 20_011)
    for m, n, kind in cases + cases[::-1]:  # and back: every pass count follows a larger and a smaller one
        keys, vals = frame_keys(rng, n, tb, depth_field, kb, m, sw.T, kind)
        _check_stage(sw, keys, vals, m, f"{layout_id(row)} m={m} n={n} {kind}")


def test_stage_sort_at_many_tiles_per_cta():
    """A C3-sized layout (1072 x 1920, far 1000, scale 100: 13 tile + 17 depth bits) with 13 M keys of 10 live depth bits
    (3 passes), then a small frame and a 2-pass frame on the same workspace, then the large one again."""
    n = LARGE + 3
    sw = _StageWorkspace(1072, 1920, 1000.0, 100.0, 0, n)
    assert (sw.L.key_bytes, sw.L.tile_bits, sw.L.depth_bits) == (4, 13, 17)
    rng = np.random.default_rng(13)
    big = frame_keys(rng, n, 13, 17, 4, 1023, sw.T)
    ctas = _check_stage(sw, *big, 1023, "C3 layout, 13 M keys")
    tiles = (n + SORT_TILE - 1) // SORT_TILE
    assert math.ceil(tiles / ctas) >= 4
    _record(f"frame sort n={n}: {tiles} tiles, {ctas} resident CTAs per pass -> up to {math.ceil(tiles / ctas)} tiles per CTA")
    _check_stage(sw, *frame_keys(rng, 7001, 13, 17, 4, 1023, sw.T), 1023, "small after large")
    _check_stage(sw, *frame_keys(rng, 50_000, 13, 17, 4, 7, sw.T), 7, "2 passes")
    _check_stage(sw, *big, 1023, "large again")


# ------------------------------------------------------------------ 3. gsb200_find_tile_start_and_end
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1_000_003])
@pytest.mark.parametrize("kind", ["mixed", "one_tile", "first_last"])
def test_find_tile_start_and_end(n, kind):
    T = 2000
    rng = np.random.default_rng(n + len(kind))
    keys, _ = frame_keys(rng, n, 11, 32, 8, 100_000, T, kind)
    keys = np.sort(keys)
    kd = _np_to_dev(keys)
    start = torch.zeros(T, dtype=torch.int32, device="cuda")
    end = torch.zeros(T, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    _lib.check(lib.gsb200_find_tile_start_and_end(kd.data_ptr(), n, start.data_ptr(), end.data_ptr(), T,
                                                  torch.cuda.current_stream().cuda_stream), "gsb200_find_tile_start_and_end")
    torch.cuda.synchronize()
    check_tile_ranges(keys, 32, start.cpu().numpy(), end.cpu().numpy())


# ------------------------------------------------------------------ 4. whole frames on one reused workspace
NEAR, FAR, SCALE = 0.8, 1000.0, 100.0
H4, W4 = 64, 96


def _base_scene():
    sc = make_scene(20_000, H4, W4, 0.06, 17, sh_degree=3, yaw_degrees=5.0)  # ~2e4 keys: several sort tiles
    sc.point_cloud[:, 2] *= 0.6               # depth keys <= 600: 10 live bits, 5 tile bits -> 2 passes
    sc.point_cloud_features[:, 7] += 1.0
    sc.point_cloud_features[:, :4] *= 1.7    # un-normalised q: every run gets its own copy to normalise
    sc.point_invalid_mask[::11] = 1
    return sc


def _variant(sc, name):
    """(xyz, features, invalid mask, extra flags) of one frame of the sequence; the point count never changes."""
    xyz, feats, mask = sc.point_cloud.clone(), sc.point_cloud_features.clone(), sc.point_invalid_mask.clone()
    flags = 0
    if name == "small":
        mask[:] = 1
        mask[::13] = 0
        flags = GSB_FLAG_KEEP_ALL_TILE_PAIRS
    elif name == "empty":
        mask[:] = 1
    elif name == "deeper":  # the same picture 4x further away: 12 live depth bits -> 3 passes
        xyz *= 4.0
        feats[:, 4:7] += math.log(4.0)
    elif name == "overflow":  # 5x larger splats: many more (tile, splat) pairs than the key capacity
        feats[:, 4:7] += math.log(5.0)
    return xyz, feats, mask, flags


class _FrameRunner:
    def __init__(self, sc, key_capacity):
        self.lib = _lib.load()
        self.sc = sc.to("cuda")
        self.cap = key_capacity
        self.L = _lib.workspace_layout(sc.point_cloud.shape[0], 1, key_capacity, H4, W4, FAR, SCALE, 0)

    def run(self, name, ws=None):
        """Render one frame into `ws` (a fresh zeroed workspace if None); returns the outputs and the sort's results."""
        xyz, feats, mask, flags = (t.cuda() if torch.is_tensor(t) else t for t in _variant(self.sc, name))
        if ws is None:
            ws = torch.zeros(self.L.total_bytes, dtype=torch.uint8, device="cuda")
        out = [torch.empty((H4, W4, 3), device="cuda"), torch.empty((H4, W4), device="cuda"),
               torch.empty((H4, W4), device="cuda"), torch.empty((H4, W4), dtype=torch.int32, device="cuda"),
               torch.empty((H4, W4), dtype=torch.int32, device="cuda")]
        sc = self.sc
        args = _lib.GsbForwardArgs(
            num_points=xyz.shape[0], pointcloud=xyz.data_ptr(), pointcloud_features=feats.data_ptr(),
            point_invalid_mask=mask.data_ptr(), point_object_id=sc.point_object_id.data_ptr(), num_objects=1,
            q_pointcloud_camera=sc.q_pointcloud_camera.data_ptr(), t_pointcloud_camera=sc.t_pointcloud_camera.data_ptr(),
            camera_intrinsics=sc.camera_info.camera_intrinsics.data_ptr(), camera_height=H4, camera_width=W4,
            near_plane=NEAR, far_plane=FAR, depth_to_sort_key_scale=SCALE, rgb_only=0, flags=flags, workspace=ws.data_ptr(),
            workspace_bytes=self.L.total_bytes, key_capacity=self.cap, rasterized_image=out[0].data_ptr(),
            rasterized_depth=out[1].data_ptr(), pixel_accumulated_alpha=out[2].data_ptr(),
            pixel_offset_of_last_effective_point=out[3].data_ptr(), pixel_valid_point_count=out[4].data_ptr(),
            stream=torch.cuda.current_stream().cuda_stream)
        _lib.check(self.lib.gsb200_forward(ctypes.byref(args)), "gsb200_forward")
        torch.cuda.synchronize()
        frame = Frame(ws, self.L, xyz.shape[0], self.cap, H4, W4, flags)
        counters = frame.counters.cpu().numpy()
        frame.num_points_in_camera, frame.num_keys = int(counters[0]), int(counters[1])
        tickets = ws[self.L.tickets:self.L.tickets + 64].view(torch.int32).cpu().numpy()[TICKET_SORT0:TICKET_SORT0 + 8]
        res = dict(image=out[0], depth=out[1], acc_alpha=out[2], last_effective=out[3], count=out[4],
                   sorted_keys=frame.sorted_keys, vals=frame.point_offset_with_sort_key,
                   tile_start=frame.tile_points_start, tile_end=frame.tile_points_end)
        res = {k: v.cpu().clone() for k, v in res.items()}
        res.update(M=int(counters[0]), K=int(counters[1]), overflow=int(counters[2]), passes=int((tickets > 0).sum()))
        return res, frame


def test_frames_on_one_reused_workspace():
    from helpers import oracle_forward
    from test_gpu_parity import _check_stages

    sc = _base_scene()
    probe = _FrameRunner(sc, 1 << 20)
    K = {name: probe.run(name)[0]["K"] for name in ("large", "small", "deeper", "overflow")}
    cap = max(K["large"], K["small"], K["deeper"]) + 100
    assert K["overflow"] > cap, K
    runner = _FrameRunner(sc, cap)
    ws = torch.empty(runner.L.total_bytes, dtype=torch.uint8, device="cuda")
    seq = ["large", "small", "large", "empty", "deeper", "overflow", "large", "small"]
    passes = []
    for name in seq:
        got, frame = runner.run(name, ws)
        if name == "overflow":
            assert got["overflow"] == 1 and got["K"] > cap  # only the next frame on this workspace is checked
            continue
        want, _ = runner.run(name)
        assert got["overflow"] == 0
        assert (got["M"], got["K"], got["passes"]) == (want["M"], want["K"], want["passes"]), name
        for k in ("image", "depth", "acc_alpha", "last_effective", "count", "sorted_keys", "vals", "tile_start", "tile_end"):
            assert torch.equal(got[k], want[k]), (name, k)
        check_tile_ranges(got["sorted_keys"].numpy(), runner.L.depth_bits, got["tile_start"].numpy(), got["tile_end"].numpy())
        if name == "empty":
            assert got["K"] == 0 and float(got["image"].abs().max()) == 0.0
        if name == "small":  # keep-all key list: exactly the reference's list
            scene = _base_scene()
            _, _, scene.point_invalid_mask, _ = _variant(scene, "small")
            _, fwd, _ = oracle_forward(scene, near_plane=NEAR, far_plane=FAR, depth_to_sort_key_scale=SCALE)
            _check_stages(frame, fwd)
        passes.append((name, got["passes"]))
    # the sequence really changed the compacted pass count between frames
    assert dict(passes)["deeper"] == dict(passes)["large"] + 1, passes
    _record(f"frames on one workspace (capacity {cap}): K = {K}, passes = {passes}")
