"""Data-parallel training of the temporal models: one process per GPU, batches sharded by rank,
one gradient all-reduce per step over NCCL (NVLink 5 / NVSwitch) — SURVEY.md §8e.

The reference is single-GPU (no torch.distributed anywhere), so this module has no reference
counterpart.  By default it adds exactly one collective and BatchNorm statistics stay per-GPU
(north_star: "allreduce on gradients only"); `broadcast_buffers` aligns the running statistics
before a checkpoint / evaluation, as DistributedDataParallel does.

`GradientReducer(sync_bn=True)` is synchronized BatchNorm (what nn.SyncBatchNorm gives a PyTorch
model): every training BatchNorm takes its batch statistics, and its backward sums, over the rows of
all ranks, so W ranks with B/W rows each train the model one process trains on B rows.  The kernels
write each rank's per-channel moments (forward) or sums (backward) into its slot of a zeroed
[W][k][C] buffer and call back into Python (vp3d_set_bn_sync); the exchange is an fp32 SUM
all-reduce of that buffer, i.e. an exact all-gather, after which every rank merges the slots in rank
order and computes identical statistics.

Overlap: the C backward (`vp3d_backward_ex` with a stage callback) reports, stage by stage, when the
kernels producing a group of gradients have been enqueued (shrink first, expand last).  All
gradients of a step live in one flat fp32 buffer laid out in that completion order, so each stage is
a contiguous slice whose all-reduce is launched on a side stream behind an event while the remaining
backward GEMMs run.
"""
import torch
import torch.distributed as dist


class _DeviceFloats:
    """A zero-copy view of `n` fp32 device floats at `ptr` (CUDA array interface)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False),
                                         "strides": None, "version": 2}


def stage_order(module):
    """Parameter names grouped by backward completion stage (the stage callback of
    vp3d_backward_ex)."""
    nb = len(module.layers_conv) // 2
    stages = [["shrink.weight", "shrink.bias"]]
    for i in range(nb, 0, -1):
        c1, c2 = 2 * (i - 1), 2 * (i - 1) + 1
        stages.append([f"layers_conv.{c2}.weight", f"layers_bn.{c2}.weight", f"layers_bn.{c2}.bias",
                       f"layers_conv.{c1}.weight", f"layers_bn.{c1}.weight", f"layers_bn.{c1}.bias"])
    stages.append(["expand_conv.weight", "expand_bn.weight", "expand_bn.bias"])
    return stages


class GradientReducer:
    """Averages gradients across the ranks of `process_group`.

    attach(module) makes the module's training backward write its gradients into a flat buffer and
    all-reduce it stage by stage (overlapped on CUDA); `reduce_flat` is the device-agnostic core and
    is what the CPU (gloo) tests exercise."""

    def __init__(self, process_group=None, overlap=True, compress=None, reserve_sms=0,
                 sync_bn=False):
        """compress: None (fp32 all-reduce) or "bf16" (each slice is rounded to bf16 for the wire
        and widened back: half the NVLink bytes; the rounding error, 2^-9 relative per rank
        contribution, is below the bf16 training noise floor).
        reserve_sms: with overlap, cap the persistent GEMM grids at (SM count - reserve_sms) so
        that the NCCL kernels of the side stream always find free SMs (pair it with
        NCCL_MAX_CTAS <= reserve_sms in the environment).
        sync_bn: synchronized BatchNorm -- batch statistics and BatchNorm-backward sums over the
        rows of every rank (1 + 2B exchanges in the forward and as many in the backward, on a
        process group of their own, always fp32: `compress` applies to gradients only)."""
        if compress not in (None, "bf16"):
            raise ValueError("compress must be None or 'bf16'")
        self.reserve_sms = int(reserve_sms)
        self.group = process_group
        self.overlap = overlap
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.comm_stream = None
        self.launched = 0
        self.step_scale = 1.0
        self.compress = compress
        self.sync_bn = bool(sync_bn)
        self.bn_group = None    # the exchanges' own process group (attach, world > 1)
        self.exchanges = 0      # BatchNorm exchanges made (forward and backward)
        self.errors = []        # raised by the exchange callback, re-raised after the C call

    # ---------------------------------------------------------------- layout
    def plan_layout(self, module):
        """-> (names in flat order, {name: (offset, numel)}, [(lo, hi)] per stage); offsets are
        padded to 4 elements so that every slice stays 16-byte aligned."""
        params = dict(module.named_parameters())
        names, spans, stage_spans = [], {}, []
        off = 0
        for group in stage_order(module):
            lo = off
            for n in group:
                numel = params[n].numel()
                spans[n] = (off, numel)
                names.append(n)
                off += (numel + 3) // 4 * 4
            stage_spans.append((lo, off))
        return names, spans, stage_spans, off

    def attach(self, module):
        """Route `module`'s training backward through this reducer; returns the reducer.

        With more than one rank on CUDA devices the kernels' programmatic dependent launch is
        switched off for the process: kernels that hand every SM over without a gap leave the NCCL
        kernels nowhere to run (with it on, a step is fast only in one of two regimes -- launch
        queue full or a host sync every step, as run.py's `loss.item()` does -- and slow in the
        other; since
        the small kernels between the GEMMs also chain programmatically this holds without
        overlap too)."""
        object.__setattr__(module, "_grad_reducer", self)
        if self.sync_bn and self.world > 1 and self.bn_group is None:
            # a group of their own: a BatchNorm exchange in the backward must not queue behind the
            # gradient slices the stage callback has just handed to the shared NCCL stream
            group = self.group if self.group is not None else dist.group.WORLD
            self.bn_group = dist.new_group(ranks=dist.get_process_group_ranks(group),
                                           backend=dist.get_backend(group))
        if self.world > 1 and torch.cuda.is_available():
            from . import _capi
            _capi.check(_capi.load().vp3d_set_pdl(0), "vp3d_set_pdl")
            if self.overlap and self.reserve_sms > 0:
                sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
                limit = sms - self.reserve_sms
                if limit >= 2:
                    _capi.check(_capi.load().vp3d_set_sm_limit(limit), "vp3d_set_sm_limit")
        return self

    def set_step_rows(self, local_rows, global_rows):
        """Weight this rank's gradient by its share of the step's batch rows.  With equal shards
        (the usual case) the weight is 1 and the all-reduce is a plain mean; with a ragged last
        batch the mean of per-rank means would over-weight the short shards, so each rank's
        gradient is scaled by n_local * world / n_global before the average."""
        if global_rows <= 0:
            raise ValueError("global_rows must be positive")
        self.step_scale = float(local_rows) * self.world / float(global_rows)
        # (with sync_bn the backward applies the weight to dy instead, see reduce_flat)

    # ---------------------------------------------------------------- collective
    def reduce_flat(self, flat):
        """In-place (weighted) average of a flat gradient slice over the group."""
        if self.world == 1:
            return flat
        # sync_bn: the BatchNorm backward mixes the ranks' dY, so the weight was applied to dY
        # before the backward (on every rank) and must not be applied a second time
        if self.step_scale != 1.0 and not self.sync_bn:
            flat.mul_(self.step_scale)
        wire = flat.to(torch.bfloat16) if self.compress == "bf16" else flat
        backend = dist.get_backend(self.group)
        if backend == "nccl":
            dist.all_reduce(wire, op=dist.ReduceOp.AVG, group=self.group)
        else:  # gloo (CPU tests): no AVG
            dist.all_reduce(wire, op=dist.ReduceOp.SUM, group=self.group)
            wire.div_(self.world)
        if wire is not flat:
            flat.copy_(wire)
        self.launched += 1
        return flat

    # ---------------------------------------------------------------- synchronized BatchNorm
    def exchange(self, slots):
        """Fill every rank's slot of `slots`, this rank's zero-padded fp32 slot buffer (its own
        slot written, all others zero), in place: a SUM all-reduce, exact because every element
        has one non-zero contribution.  On CUDA it is enqueued on the current stream, which the
        next kernel reads the slots from; gloo stages the buffer through host memory."""
        self.exchanges += 1
        if self.world == 1:
            return slots
        group = self.bn_group if self.bn_group is not None else self.group
        if slots.is_cuda and dist.get_backend(group) != "nccl":
            host = slots.cpu()
            dist.all_reduce(host, op=dist.ReduceOp.SUM, group=group)
            slots.copy_(host)
        else:
            dist.all_reduce(slots, op=dist.ReduceOp.SUM, group=group)
        return slots

    def bn_exchange_fn(self):
        """The vp3d_bn_exchange_fn of this reducer (a ctypes object: keep it alive as long as a
        plan may call it).  Exceptions are collected in `errors`, never raised through C."""
        from . import _capi

        def _exchange(_layer, _phase, slots, floats_per_rank, _user):
            try:
                buf = torch.as_tensor(_DeviceFloats(slots, floats_per_rank * self.world))
                self.exchange(buf)
            except Exception as e:  # never raise through the C frame
                self.errors.append(e)

        return _capi.BN_EXCHANGE_FN(_exchange)

    def raise_errors(self):
        """Re-raise the first exception an exchange collected during the last C call."""
        if self.errors:
            err = self.errors[0]
            self.errors = []
            raise err

    def stage_ready(self, flat, lo, hi):
        """Called (from the C backward's stage callback) once the kernels writing flat[lo:hi] are
        enqueued on the current stream."""
        if hi <= lo:
            return
        piece = flat[lo:hi]
        if not flat.is_cuda or not self.overlap:
            self.reduce_flat(piece)
            return
        cur = torch.cuda.current_stream(flat.device)
        if self.comm_stream is None:
            # (high priority: the collective's kernels must not queue behind the compute grids)
            self.comm_stream = torch.cuda.Stream(device=flat.device, priority=-1)
        ev = torch.cuda.Event()
        ev.record(cur)
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            self.reduce_flat(piece)
        flat.record_stream(self.comm_stream)

    def finish(self, flat):
        """Make the current stream wait for every outstanding all-reduce."""
        if flat.is_cuda and self.comm_stream is not None:
            torch.cuda.current_stream(flat.device).wait_stream(self.comm_stream)


def broadcast_buffers(module, src=0, process_group=None):
    """Copy rank `src`'s BatchNorm running statistics to every rank (checkpoint / eval alignment)."""
    if not dist.is_initialized() or dist.get_world_size(process_group) == 1:
        return
    for b in module.buffers():
        dist.broadcast(b, src=src, group=process_group)
    if hasattr(module, "_stats_epoch"):
        module._stats_epoch += 1


def shard_batch(batch_index, rank, world):
    """Weak scaling as SURVEY.md §8e prefers: rank r takes batches b with b % world == r, each of
    the full per-GPU batch size (keeps the BatchNorm population per GPU equal to the reference's)."""
    return batch_index % world == rank
