"""View-parallel multi-GPU plumbing (one process per GPU, ``torch.distributed``).

The reference is single-GPU and renders one view per step (GaussianPointTrainer.py:120-166).  The path
shards naturally by VIEW (SURVEY.md §8(e)): every rank holds a full replica of the scene, view ``i`` is
rendered by rank ``i mod R``, inference needs no communication, and training needs exactly one exchange
step per optimiser step: the sum over ranks of the per-Gaussian gradients (N,3)+(N,56).

Two ways to do that exchange:
* :func:`exchange_gradients` -- one all-reduce of the dense 59 floats per Gaussian (236 MB at 1e6 Gaussians);
* :class:`ViewParallelExchange` (what ``bench.py --gpus N`` uses), plugged INTO the operator's backward
  (``GaussianPointCloudRasterisation(..., gradient_exchange=...)``): 48 of the 56 feature gradients of a view are the
  outer product of 3 colour-argument gradients with the view's 16 SH basis values, and the basis depends only on the
  Gaussian's position and the view's camera centre, which every rank knows.  So the per-point kernel writes COMPACT rows
  (``GSB_FLAG_COMPACT_GRADS``), the ranks all-reduce the 11 columns that simply add up (xyz, q, s, logit) and all-gather
  the 3 colour-argument gradients plus the camera centres, and ``gsb200_expand_view_gradients`` rebuilds the dense sum on
  every rank: 14 instead of 59 floats per Gaussian cross NVLink (north_star: "NCCL all-gather only for the per-Gaussian
  gradient reduction"), and the per-point kernel writes 60 instead of 236 bytes per row.  Exact (same products, summed in
  rank order), not an approximation.
"""
from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist


def shard_views(num_views: int, rank: int, world_size: int) -> List[int]:
    """Indices of the views rank ``rank`` renders: i with i mod world_size == rank."""
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} outside world of size {world_size}")
    return list(range(rank, num_views, world_size))


def _aliases(buffer: torch.Tensor, grads) -> bool:
    """True if every gradient tensor is a view into ``buffer``'s allocation (then one collective covers all)."""
    lo = buffer.data_ptr()
    hi = lo + buffer.numel() * buffer.element_size()
    return all(g is None or (g.is_contiguous() and lo <= g.data_ptr() and
                             g.data_ptr() + g.numel() * g.element_size() <= hi) for g in grads)


def exchange_gradients(grads: Iterable[Optional[torch.Tensor]], group=None, average: bool = False,
                       async_op: bool = False, fused_buffer: Optional[torch.Tensor] = None):
    """Sum (or average) the dense gradient tensors over all ranks, in place.

    ``fused_buffer``: the operator's ``last_gradient_buffer``; when the gradients are views into it (autograd
    hands the operator's outputs to ``.grad`` without copying) the exchange is ONE all-reduce instead of one
    per tensor.

    Returns the list of work handles when ``async_op`` (so the exchange can overlap the next view's
    forward on another stream), else ``None``.  A no-op when torch.distributed is not initialised or
    the world has a single rank."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return [] if async_op else None
    handles = []
    world = dist.get_world_size(group)
    grads = list(grads)
    if fused_buffer is not None and _aliases(fused_buffer, grads):
        grads = [fused_buffer]
    for g in grads:
        if g is None:
            continue
        h = dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        if async_op:
            handles.append(h)
        if average:
            if async_op:
                h.wait()
            g.div_(world)
    return handles if async_op else None


class ViewParallelExchange:
    """The collectives of the compact exchange.  ``gradient_exchange=ViewParallelExchange(group)`` on the operator of every
    rank makes ``backward`` return -- and ``.grad`` receive -- the gradients summed over the ranks' views.

    ``run(grad_sum, blocks)``: ``grad_sum`` (N,12) f32 is summed over ranks in place; ``blocks`` (R, stride) f32 holds this
    rank's ``[3N colour-argument gradients | 3 n_obj camera centres]`` in row ``rank`` and receives the other ranks' rows
    (in-place all-gather: the send buffer is the rank's slot of the receive buffer)."""

    def __init__(self, group=None, gather_group=None, overlap_expansion: bool = False):
        """``gather_group``: optionally a SECOND process group over the same ranks (``dist.new_group()``): the all-gather
        then runs on its communicator concurrently with the all-reduce (two NCCL kernels in flight hide each other's
        latency) instead of behind it.  ``overlap_expansion``: gather first and expand the SH columns (they need only the
        gathered blocks) on a second stream while the all-reduce of the summed columns is on the wire (opt-in, off by
        default)."""
        if not dist.is_available() or not dist.is_initialized():
            raise RuntimeError("ViewParallelExchange needs an initialised torch.distributed process group")
        self.group = group
        self.gather_group = gather_group
        self._overlap = bool(overlap_expansion)
        self._side_stream = None
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if gather_group is not None and dist.get_world_size(gather_group) != self.world:
            raise ValueError("gather_group must span the same ranks as group")

    def allocate(self, num_points: int, num_objects: int, device):
        """The two exchange buffers of one backward: ``grad_sum`` (N,12) and ``blocks`` (R, stride), stride = 3N + 3 n_obj
        rounded up to 16 bytes.  Plain device tensors here; the multicast variant hands out views of a symmetric allocation."""
        stride = (3 * num_points + 3 * num_objects + 3) // 4 * 4
        return (torch.empty((num_points, 12), dtype=torch.float32, device=device),
                torch.empty((self.world, stride), dtype=torch.float32, device=device))

    def rows_written(self, grad_sum: torch.Tensor, blocks: torch.Tensor) -> None:
        """Called by the operator right after this rank's compact rows have been enqueued (before ``run``); the multicast
        variant starts pushing its block here."""

    def run(self, grad_sum: torch.Tensor, blocks: torch.Tensor) -> None:
        if blocks.shape[0] != self.world or not blocks.is_contiguous() or not grad_sum.is_contiguous():
            raise ValueError("blocks must be a contiguous (world, stride) tensor and grad_sum contiguous")
        mine = blocks[self.rank]
        if not mine.is_cuda:  # gloo (CPU tests): no in-place all-gather
            mine = mine.clone()
        if self.gather_group is None:
            dist.all_reduce(grad_sum, op=dist.ReduceOp.SUM, group=self.group)
            dist.all_gather_into_tensor(blocks.view(-1), mine, group=self.group)
        else:
            w1 = dist.all_reduce(grad_sum, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
            w2 = dist.all_gather_into_tensor(blocks.view(-1), mine, group=self.gather_group, async_op=True)
            w1.wait()
            w2.wait()


    def _side(self, device) -> "torch.cuda.Stream":
        if self._side_stream is None or self._side_stream.device != device:
            self._side_stream = torch.cuda.Stream(device=device)
        return self._side_stream

    def run_and_expand(self, grad_sum: torch.Tensor, blocks: torch.Tensor, expand) -> None:
        """The collectives followed by the expansion to dense gradients.  ``expand(part)`` enqueues
        ``gsb200_expand_view_gradients`` on the current stream (0 = everything, 1 = SH columns, 2 = summed columns).

        Default: the collectives, then one expansion pass.  With ``overlap_expansion=True`` (CUDA tensors, one communicator) the
        blocks are gathered FIRST and the 48 SH columns -- 4/5 of the expansion's traffic, HBM-bound -- are expanded on a second
        stream while the all-reduce of the summed columns is on the wire; only the small part 2 (xyz, q, s, logit) waits for the
        sums.  The two parts write disjoint pieces of the dense gradients.  (Opt-in.)"""
        if not (self._overlap and grad_sum.is_cuda) or self.gather_group is not None:
            self.run(grad_sum, blocks)
            return expand(0)
        if blocks.shape[0] != self.world or not blocks.is_contiguous() or not grad_sum.is_contiguous():
            raise ValueError("blocks must be a contiguous (world, stride) tensor and grad_sum contiguous")
        dev = grad_sum.device
        main, side = torch.cuda.current_stream(dev), self._side(dev)
        dist.all_gather_into_tensor(blocks.view(-1), blocks[self.rank], group=self.group)
        side.wait_stream(main)                      # the gathered blocks are in place
        dist.all_reduce(grad_sum, op=dist.ReduceOp.SUM, group=self.group)  # NCCL's stream; main waits for it
        with torch.cuda.stream(side):
            expand(1)                               # runs beside the all-reduce
        expand(2)
        main.wait_stream(side)


class MulticastViewParallelExchange(ViewParallelExchange):
    """The same exchange with BOTH collectives done by one hand-written kernel over NVSwitch multicast memory
    (``gsb200_exchange_multimem``, csrc/exchange.cu: ``multimem.ld_reduce`` / ``multimem.st``) instead of ncclAllReduce +
    ncclAllGather.  The buffers of a scene size live in one symmetric allocation (``torch.distributed._symmetric_memory``:
    same offset on every rank, mapped to a multicast address), created once and reused every step; the per-point backward
    kernel writes its compact rows straight into it.  ``run`` = cross-rank barrier (every rank's rows are written), the
    kernel, cross-rank barrier (every multicast store has landed).  Needs NVLS multicast support (one NVSwitch domain)."""

    def __init__(self, group=None, barrier_timeout_ms: int = 20000, num_blocks: int = 0, overlap_expansion: bool = False):
        """``num_blocks``: CTAs of the exchange kernel (0 = two per SM).  ``overlap_expansion``: expand the SH columns (they
        need only the gathered blocks) on a second stream while the all-reduce of the summed columns is on the wire.  Off by
        default: the expansion's 128-register CTAs and its HBM traffic compete with the wire-bound exchange kernel."""
        super().__init__(group, overlap_expansion=overlap_expansion)
        self._num_blocks = int(num_blocks)
        self._overlap = bool(overlap_expansion)
        import torch.distributed._symmetric_memory as symm_mem
        self._symm_mem = symm_mem
        self._group = group if group is not None else dist.group.WORLD
        self._cache = {}
        self._timeout = int(barrier_timeout_ms)

    def allocate(self, num_points: int, num_objects: int, device):
        key = (num_points, num_objects, torch.device(device).index)
        entry = self._cache.get(key)
        if entry is None:
            stride = (3 * num_points + 3 * num_objects + 3) // 4 * 4
            sum_floats = 12 * num_points
            # [grad_sum | blocks of even steps | blocks of odd steps]: a rank pushes its block BEFORE the step's barrier, so
            # the buffer it writes must not be the one a slow peer may still be expanding from (the previous step's)
            flat = self._symm_mem.empty(sum_floats + 2 * self.world * stride, dtype=torch.float32, device=device)
            hdl = self._symm_mem.rendezvous(flat, self._group)
            if not hdl.multicast_ptr:
                raise RuntimeError("MulticastViewParallelExchange: no NVLS multicast support for this group "
                                   "(use ViewParallelExchange, the NCCL path)")
            # multicast address of `flat`: the handle's pointers are those of the symmetric block, the tensor may sit at an offset
            mc_flat = int(hdl.multicast_ptr) + (flat.data_ptr() - int(hdl.buffer_ptrs[hdl.rank]))
            blocks = [flat[sum_floats + b * self.world * stride:sum_floats + (b + 1) * self.world * stride].view(self.world, stride)
                      for b in range(2)]
            entry = dict(flat=flat, hdl=hdl, grad_sum=flat[:sum_floats].view(num_points, 12), blocks=blocks, mc_sum=mc_flat,
                         mc_blocks=[mc_flat + 4 * (sum_floats + b * self.world * stride) for b in range(2)], stride=stride,
                         num_points=num_points, num_objects=num_objects, parity=1)
            self._cache[key] = entry
        entry["parity"] ^= 1  # one allocate() per backward on every rank: the parities stay in step
        self._current = entry
        return entry["grad_sum"], entry["blocks"][entry["parity"]]

    def _launch(self, phases: int, blocks: torch.Tensor) -> None:
        import ctypes
        from . import _lib
        e = self._current
        with torch.cuda.device(blocks.device):
            args = _lib.GsbMultimemExchangeArgs(
                num_points=e["num_points"], num_objects=e["num_objects"], rank=self.rank, world_size=self.world,
                num_blocks=self._num_blocks, phases=phases, multicast_grad_sum=e["mc_sum"],
                multicast_blocks=e["mc_blocks"][e["parity"]], local_block=blocks[self.rank].data_ptr(), block_stride=e["stride"],
                stream=torch.cuda.current_stream(blocks.device).cuda_stream)
            _lib.check(_lib.load().gsb200_exchange_multimem(ctypes.byref(args)), "gsb200_exchange_multimem")

    def _check(self, grad_sum, blocks):
        e = self._current
        if grad_sum.data_ptr() != e["grad_sum"].data_ptr() or blocks.data_ptr() != e["blocks"][e["parity"]].data_ptr():
            raise ValueError("MulticastViewParallelExchange needs the buffers handed out by the latest allocate()")
        return e

    def rows_written(self, grad_sum: torch.Tensor, blocks: torch.Tensor) -> None:
        """This rank's rows are enqueued: push its block to every rank now, without waiting for the others -- early ranks'
        pushes run under the slowest rank's compute.  Safe without a barrier: the destination is the buffer of this step's
        parity, and a peer can only still be reading the OTHER one (to get here this rank has passed both barriers of the
        previous step, which every peer enqueues behind its expansion of the step before that)."""
        self._check(grad_sum, blocks)
        self._launch(1, blocks)

    def run(self, grad_sum: torch.Tensor, blocks: torch.Tensor) -> None:
        e = self._check(grad_sum, blocks)
        hdl = e["hdl"]
        with torch.cuda.device(grad_sum.device):
            hdl.barrier(channel=0, timeout_ms=self._timeout)  # every rank's compact rows are in its buffer
            self._launch(2, blocks)                            # two-shot all-reduce of the summable columns
            hdl.barrier(channel=1, timeout_ms=self._timeout)  # every rank's multicast stores (sums and blocks) have landed


    def run_and_expand(self, grad_sum: torch.Tensor, blocks: torch.Tensor, expand) -> None:
        """Default: ``run`` (barrier, all-reduce kernel, barrier), then one expansion pass.  With ``overlap_expansion=True``:
        every rank's block is in place after the FIRST barrier (the pushes were launched before it), so the 48 SH columns
        -- 4/5 of the expansion's traffic, HBM-bound -- are expanded on a second stream while the all-reduce of the summed
        columns is still bound by the NVLink wire; only the small part 2 (xyz, q, s, logit) follows the second barrier.
        (Opt-in, see ``__init__``.)"""
        if not self._overlap:
            return super().run_and_expand(grad_sum, blocks, expand)
        e = self._check(grad_sum, blocks)
        hdl = e["hdl"]
        dev = grad_sum.device
        with torch.cuda.device(dev):
            main, side = torch.cuda.current_stream(dev), self._side(dev)
            hdl.barrier(channel=0, timeout_ms=self._timeout)  # rows written and blocks pushed on every rank
            side.wait_stream(main)
            self._launch(2, blocks)                            # two-shot all-reduce of the summed columns: launched FIRST, so
            with torch.cuda.stream(side):                      #   that the wire-bound kernel gets its CTAs before the expansion
                expand(1)                                      #   (SH columns from the gathered blocks) fills the rest of the SMs
            hdl.barrier(channel=1, timeout_ms=self._timeout)  # the sums have landed everywhere
            expand(2)                                          # xyz / q / s / logit columns
            main.wait_stream(side)


def render_views(op, make_input, view_ids: Sequence[int], streams: Optional[Sequence["torch.cuda.Stream"]] = None):
    """Inference helper: render this rank's shard of views (no communication). ``make_input(i)`` builds the
    ``GaussianPointCloudRasterisationInput`` of view i.

    ``streams``: two (or more) CUDA streams -> consecutive frames go to alternating streams, so that the latency-bound
    stages of frame i+1 (per-point stage, radix sort: a few hundred resident warps) run under the issue-bound blend of frame i
    instead of behind it.  Every frame owns its workspace and outputs, the operator's only host wait per frame ends after that
    frame's first kernel, so nothing else changes; the caller must synchronise the streams (or wait on the outputs' stream)
    before reading the images.  ``ValueError`` for an equirectangular or orthographic view (not implemented here; render it
    with ``op`` directly), raised before the view is rendered."""
    out = {}
    with torch.no_grad():
        for n, i in enumerate(view_ids):
            inp = make_input(i)
            distortion = getattr(inp.camera_info, "distortion", None)
            if distortion is not None and distortion.model in ("equirectangular", "orthographic"):
                raise ValueError(f"parallel.render_views does not render {distortion.model} views")
            if streams:
                with torch.cuda.stream(streams[n % len(streams)]):
                    image, depth, count = op(inp)
            else:
                image, depth, count = op(inp)
            out[i] = (image, depth, count)
    return out
