"""Offline inference on a known list of clips of any lengths, as few large GEMM chains.

``model.predict(sequences)`` is the offline counterpart of ``StreamingSession.predict``: same
input and output contract, but every clip is known up front, so the clips are edge-padded as
UnchunkedGenerator pads them (run.py:186-193, common/generators.py:216-238), concatenated, and run
through the eval forward's dilated GEMM chain as one long sample (``include/vp3d_b200.h``,
vp3d_forward_clips).  Output row t of that chain depends on input rows [t, t + RF - 1] only, so each
clip's rows are exactly its own forward, bit for bit; the RF - 1 rows between two clips straddle
them and are discarded.

    with torch.no_grad():
        ys = model.predict([x0, x1, ...])                  # x_i: CUDA fp32 (T_i, J_in, F)
        ys = model.predict(xs, augment=True, kps_left=kl, kps_right=kr,
                           joints_left=jl, joints_right=jr)  # run.py's flip average

Clips are grouped greedily, in input order, into chains of at most ``max_rows`` packed rows
(``clip_chains``); a clip and its mirrored copy share a chain, and a clip longer than ``max_rows``
runs alone.  The grouping follows from the lengths alone, so one host-to-device copy carries every
chain's clip table and nothing is read back.
"""
import numpy as np
import torch

from . import _capi
from .streaming import _check_sequence, augment_maps

# Packed rows per chain by default: 2^18 rows (0.26 M frames) fill every SM for many waves, and one
# chain's workspace stays about 2 GB at channels = 1024 (DESIGN.md, "Offline clips").
DEFAULT_MAX_ROWS = 1 << 18


def clip_rows(length, rf, augment):
    """Packed rows one clip of `length` frames takes in a chain: its padded copy (and the
    mirrored one with augment), T + RF - 1 rows each."""
    return (2 if augment else 1) * (int(length) + int(rf) - 1)


def clip_chains(lengths, rf, augment, max_rows=DEFAULT_MAX_ROWS):
    """Group clips of `lengths` frames, in input order, into chains of at most `max_rows` packed
    rows; a clip that alone exceeds `max_rows` gets a chain of its own.  Returns a list of
    (first clip, end clip) index ranges covering 0..len(lengths)."""
    max_rows = int(max_rows)
    if max_rows < 1:
        raise ValueError("max_rows must be >= 1")
    chains, start, rows = [], 0, 0
    for i, n in enumerate(lengths):
        r = clip_rows(n, rf, augment)
        if i > start and rows + r > max_rows:
            chains.append((start, i))
            start, rows = i, 0
        rows += r
    if len(lengths) > start:
        chains.append((start, len(lengths)))
    return chains


def clip_tables(lengths, rf, augment, max_rows=DEFAULT_MAX_ROWS):
    """The host side of every chain: (chains, first, rows) with first[i] the row of clip i in both
    the concatenated input and the concatenated output (the clips' lengths summed before it) and
    rows[c] the packed rows of chain c."""
    chains = clip_chains(lengths, rf, augment, max_rows)
    first = np.zeros(len(lengths), np.int64)
    if len(lengths) > 1:
        first[1:] = np.cumsum(np.asarray(lengths, np.int64))[:-1]
    rows = [sum(clip_rows(n, rf, augment) for n in lengths[a:b]) for a, b in chains]
    return chains, first, rows


def predict(model, sequences, augment=False, kps_left=None, kps_right=None, joints_left=None,
            joints_right=None, max_rows=None):
    """TemporalModel.predict (see there and the module docstring)."""
    from .temporal_model import TemporalModel
    if type(model)._variant != TemporalModel._variant:
        raise NotImplementedError(
            "predict needs a TemporalModel; a TemporalModelOptimized1f state_dict loads into "
            "TemporalModel(..., same arguments) unchanged -- predict with that model instead")
    if model.precision == "mixed":
        raise NotImplementedError(
            "precision 'mixed' cannot predict clip chains: its per-layer split choice depends on "
            "the geometry; use 'fp16', 'bf16', 'bf16x3' or 'int8'")
    if model.training:
        raise RuntimeError("predict is an eval-mode computation: call model.eval() first")
    kps, joints = augment_maps(model, augment, kps_left, kps_right, joints_left, joints_right)
    seqs = list(sequences)
    if not seqs:
        raise ValueError("predict needs at least one sequence")
    if torch.is_grad_enabled() and (any(torch.is_tensor(x) and x.requires_grad for x in seqs)
                                    or any(p.requires_grad for p in model.parameters())):
        raise RuntimeError("predict is inference-only (no autograd graph): call it under "
                           "torch.no_grad() or with inputs and parameters that do not require grad")
    device = model.expand_conv.weight.device
    J, F = model.num_joints_in, model.in_features
    for x in seqs:
        _check_sequence(x, J, F, device)
    lengths = [int(x.shape[0]) for x in seqs]
    rf = model.receptive_field()
    chains, first, rows = clip_tables(lengths, rf, augment,
                                      DEFAULT_MAX_ROWS if max_rows is None else max_rows)
    flags = _capi.VP3D_CLIPS_AUGMENT if augment else 0
    lib = _capi.load()
    n = len(seqs)
    # the clip table of every chain in one buffer: first (int64) | y_first (int64) | len (int32);
    # chain c reads entries [a, b) of each part
    host = np.zeros(20 * n, np.uint8)
    host[:8 * n] = first.view(np.uint8)
    host[8 * n:16 * n] = first.view(np.uint8)
    host[16 * n:] = np.asarray(lengths, np.int32).view(np.uint8)
    host_ptr = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    with torch.cuda.device(device):
        plan = model._use_plan(device, model.precision)
        stream = torch.cuda.current_stream(device).cuda_stream
        model._sync_weights(plan, stream)
        nbytes = max(lib.vp3d_clips_workspace_bytes(plan, r, flags) for r in rows)
        if nbytes == 0:
            raise ValueError(f"a chain of {max(rows)} rows is too large")
        ws = model._get_workspace(nbytes, device)
        table = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
        xs = torch.cat(seqs)
        y = torch.empty((sum(lengths), model.num_joints_out, 3), dtype=torch.float32, device=device)
        base = table.data_ptr()
        launches = 0
        for (a, b), r in zip(chains, rows):
            _capi.check(lib.vp3d_forward_clips(
                plan, xs.data_ptr(), base + 8 * a, base + 16 * n + 4 * a, b - a, r, flags,
                host_ptr(kps), host_ptr(joints), y.data_ptr(), base + 8 * (n + a), ws.data_ptr(),
                ws.numel(), stream), "vp3d_forward_clips")
            launches += lib.vp3d_last_launch_count(plan)
    model.last_predict_launches = launches
    return [y[int(f):int(f) + T] for f, T in zip(first, lengths)]
