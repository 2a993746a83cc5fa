"""Streaming (frame-by-frame) inference of a TemporalModel: one 3-D pose per new 2-D frame.

The reference's causal models exist for real-time use (DOCUMENTATION.md: causal convolutions are
"suitable for real-time applications"), but ``model(x)`` recomputes a whole receptive field per
output frame.  A session keeps every conv layer's past activations in device rings and computes only
the new frames' share (``include/vp3d_b200.h``, vp3d_stream_*):

    sess = model.streaming(streams=S, max_frames=K)   # TemporalModel in eval()
    y, frame = sess.push(x, start=None, end=None, count=None)   # x: (S, k, J_in, F) CUDA fp32,
                                                               # 1 <= k <= K
    y, frame = sess.finish()              # the look-ahead tail of every slot; slots become idle
    sess.reset()                          # drop all history
    ys = sess.predict([x0, x1, ...])      # whole (T_i, J_in, F) sequences, scheduled over the slots

Per slot, the outputs of frames 0..T-1 of a sequence are exactly ``model(xp)`` with ``xp`` the
sequence padded as run.py's UnchunkedGenerator pads it (run.py:186-193, common/generators.py:
216-238): ``np.pad(x, (pad + shift, pad - shift), 'edge')``, pad = (RF - 1) // 2, shift = pad
for a causal model and 0 otherwise.  Output frame t comes back in the push that delivers input frame
t + lookahead (lookahead = pad - shift, 0 for a causal model); ``frame`` numbers every returned row
within its slot's sequence and is -1 for rows that are no frame yet.

``end[s] = n`` (0 <= n <= k) ends slot s's sequence after frame n - 1 of the push: from then on the
slot is fed its last frame repeated (the generator's end padding), its last `lookahead` frames come
out over the following pushes while the other slots go on, and the slot is idle once the last one is
out.  ``predict`` uses this to run a list of sequences of any lengths through the slots, longest
first, each slot taking the next sequence once the previous one has drained.

``count[s] = n`` (0 <= n <= k) gives slot s only the n real frames x[s, :n] in this push, so
cameras that drop frames, deliver late or run at different rates share one session: each slot's
outputs stay those of the offline forward on its own padded sequence, and rows f >= n get frame -1.

Test-time flip augmentation, run.py's default (common/arguments.py:43):

    sess = model.streaming(streams=S, max_frames=K, augment=True,
                           kps_left=kl, kps_right=kr, joints_left=jl, joints_right=jr)

runs every slot twice in the same launches, plain and mirrored as UnchunkedGenerator(augment=True)
mirrors it (common/generators.py:223-237), and returns the flip average of run.py:674-680: per slot
bit-identical to ``metrics.flip_average(model(b), jl, jr)[0]`` with ``b`` the generator's (2, T +
2 pad, J, F) batch.  The trajectory model (num_joints_out = 1) takes no joints lists (negate x only,
run.py:678).

Provisional poses for the frames still inside the look-ahead (non-causal models):

    sess = model.streaming(streams=S, max_frames=K, provisional=True)
    y, frame, y_prov, frame_prov = sess.push(x, start, end, count, provisional=True)

``y_prov`` (S, lookahead, J_out, 3) / ``frame_prov`` (S, lookahead) are what ``finish()`` would
return if it were called right after this push, bit for bit and with the same frame numbers, but
nothing ends: the push's own ``y, frame`` and every later push are what they would be without the
request.  Per slot they cover the frames [c - lookahead, c) of its sequence (c = frames pushed so
far) that are not final yet, -1 below frame 0, past an ended sequence and for idle slots; each is
the offline forward on the sequence as pushed so far, edge-padded.  Frame t thus gets a provisional
pose as soon as its input arrives and its final one `lookahead` frames later, from one session.  The
look-ahead tail rides in the push's own launches (its GEMMs run over k + lookahead frame rows), and
the flag makes every ring hold `lookahead` positions more (``ring_bytes_per_stream(...,
provisional=True)``).  A published checkpoint (arc 3,3,3,3,3, not causal) has a look-ahead of 121
frames, 2.4 s at 50 fps, which this removes from the latency of a first estimate.

int8 sessions, for a model calibrated for ``set_precision('int8')``:

    sess = model.streaming(streams=S, max_frames=K, int8=True)   # with augment / provisional too

Every output is bit for bit the offline int8 forward ``model(xp)`` on the padded sequence: the
blocks of ``model.int8_blocks`` run u8 x s8, the rest fp16, in the push's own launches (one quantise
launch more per fp16 -> int8 block transition).  The rings of the residual blocks keep a u8 copy of
their history (``ring_bytes_per_stream(..., int8=True)``, about 1.5x the 16-bit bytes).  The history
holds one calibration's quantisation: ``calibrate_int8``, ``load_int8_calibration`` or
``set_int8_blocks`` under a session with history make its next push raise until ``reset()``, as a
parameter change does.  An int8 model without ``int8=True`` cannot stream.

Sessions fed by a 2-D detector (``detections=True``, ``push_detections``) take pixel keypoints and a
host "person detected" flag per frame; frames after a slot's last detection are pending until the
next detection, the video's end, finish() or max_gap.  With ``max_gap=G`` they can also return
provisional poses, for the look-ahead and for the pending frames:

    sess = model.streaming(streams=S, max_frames=K, detections=True, provisional=True, max_gap=G)
    y, frame, y_prov, frame_prov = sess.push_detections(kps_px, detected, start, end, resolution,
                                                        provisional=True)

``y_prov`` (S, lookahead + G, J_out, 3) / ``frame_prov`` (S, lookahead + G) are what finish() would
return right after the call, bit for bit: the pending frames held (the last detection repeated),
then the look-ahead tail.  Causal models are accepted with G >= 1 (their provisional rows are the
pending frames alone).  A push computes at most receptive_field - 1 tail rows however long the gap
(past that every row is a copy), and the rings hold that many positions more
(``ring_bytes_per_stream(..., held=True)``).

A slot's state can move to another session, of any streams / max_frames / provisional sizing, on
any device, as long as the model, precision, weights, int8 calibration, augmentation and detector
settings are the same:

    state = old.export_slots(range(S))        # StreamSlots; .to(device), torch.save / torch.load
    new = model.streaming(streams=2 * S, max_frames=K2)
    new.import_slots(state, range(S))          # each camera goes on as if it had never moved

Every imported slot continues bit for bit as the uninterrupted stream.  To move a camera rather than
copy it, free the old slot at its next push with start=True, end=0.
"""
import hashlib
import weakref

import numpy as np
import torch

from . import _capi
from .generators import mirror_source


def lookahead(model):
    """Input frames a session needs past output frame t before it can return t: pad - shift with
    shift = pad for a causal model (run.py:186-193)."""
    return 0 if model._causal else (model.receptive_field() - 1) // 2


def ring_history(filter_widths, dense=False):
    """Frames of history each ring keeps next to the new ones: ring 0 holds the network input (the
    expand conv's w0 - 1 frames), ring i the input of residual block i (its first conv spans
    (w_i - 1) * dilation_i = 2 * pad_i frames; the same for the dense ablation).  They add up to
    receptive_field - 1."""
    hist = [filter_widths[0] - 1]
    d = filter_widths[0]
    for w in filter_widths[1:]:
        hist.append((w - 1) * d)
        d *= w
    return hist


def ring_bytes_per_stream(model, max_frames, planes=1, augment=False, provisional=False,
                          int8=False, held=False):
    """Device bytes of history one stream slot occupies (both mirror halves, every plane; twice that
    with augment: the slot's mirrored copy has rings of its own).  provisional: every ring also
    holds the `lookahead` positions of the tail a provisional push appends (not for causal
    models, whose look-ahead is 0).  held: every ring holds receptive_field - 1 tail positions
    instead, the most a provisional push of a detector-fed session computes (causal models too;
    not together with provisional).  int8: the rings of the residual blocks also hold a u8 plane
    with the same positions (one byte per channel, every block whatever the int8 block set)."""
    fw = model.filter_widths
    c_in = -(-model.num_joints_in * model.in_features // 64) * 64
    c = -(-model._channels // 64) * 64
    tail = 0
    if provisional:
        tail = lookahead(model)
        if tail == 0:
            raise ValueError("provisional outputs need a non-causal model (a causal one has no "
                             "look-ahead: every output is final)")
    if held:
        if provisional:
            raise ValueError("held and provisional exclude each other: held rings already hold "
                             "the provisional tail")
        tail = model.receptive_field() - 1
    total = 0
    for i, h in enumerate(ring_history(fw)):
        positions = 2 * (h + max_frames + tail + 1)
        total += positions * (c_in if i == 0 else c) * 2 * planes
        if int8 and i > 0:
            total += positions * c
    return 2 * total if augment else total


def _check_pair(left, right, n, what):
    if (left is None) != (right is None):
        raise ValueError(f"{what}_left and {what}_right go together: give both or neither")
    if left is None:
        return
    for j in list(left) + list(right):
        if not 0 <= int(j) < n:
            raise ValueError(f"{what} index {j} is out of range for {n} joints")


def augment_maps(model, augment, kps_left=None, kps_right=None, joints_left=None,
                 joints_right=None):
    """The (kps_src, joints_src) int32 mirror maps of a session (generators.mirror_source), or
    (None, None) without augmentation; joints_src is None for the trajectory model.  Raises
    ValueError for lists that are missing, unpaired, out of range, or given with augment=False."""
    lists = (kps_left, kps_right, joints_left, joints_right)
    if not augment:
        if any(v is not None for v in lists):
            raise ValueError("kps_left / kps_right / joints_left / joints_right are only used with "
                             "augment=True")
        return None, None
    j_in, j_out = model.num_joints_in, model.num_joints_out
    _check_pair(kps_left, kps_right, j_in, "kps")
    _check_pair(joints_left, joints_right, j_out, "joints")
    if kps_left is None:
        raise ValueError("augment=True needs kps_left/kps_right (and joints_left/joints_right "
                         "unless num_joints_out == 1)")
    if joints_left is None and j_out > 1:
        raise ValueError("augment=True needs joints_left/joints_right for a model with "
                         f"num_joints_out = {j_out}: only the trajectory model (num_joints_out == 1) "
                         "skips the joint swap (run.py:678)")
    kps = mirror_source(j_in, kps_left, kps_right)
    joints = None if joints_left is None else mirror_source(j_out, joints_left, joints_right)
    return kps, joints


class FrameBook:
    """Host model of the frame bookkeeping the session's input kernel does on the device (used by
    the tests and by predict's scheduler): per slot a frame counter, an active flag and the length of
    an ended sequence (-1 while it is open)."""

    def __init__(self, streams, lookahead):
        self.count = np.zeros(streams, np.int64)
        self.active = np.zeros(streams, bool)
        self.length = np.full(streams, -1, np.int64)
        self.lookahead = lookahead

    def push(self, k, start=None, end=None, count=None, provisional=False, held=None, rows=None):
        """The (S, k) frame numbers of a push; provisional=True also returns the (S, rows) numbers
        of its provisional rows (rows = lookahead by default), those finish() would give right after
        it.  held: per slot the pending frames finish() would first push held (a detector-fed
        slot's frames after its last detection, read for open sequences only): row j is a frame
        for j < lookahead + held[s] (vp3d_stream_push_held)."""
        S = len(self.count)
        start = np.zeros(S, bool) if start is None else np.asarray(start, bool)
        self.count[start] = 0
        self.active[start] = True
        self.length[start] = -1
        end = np.full(S, -1, np.int64) if end is None else np.asarray(end, np.int64)
        end = np.where((end < -1) | (end > k), -1, end)   # as the device reads it
        is_open = self.active & (self.length < 0)
        ends = is_open & (end >= 0)
        self.length[ends] = self.count[ends] + end[ends]
        # frames each slot advances by: count[s] for an open sequence that does not end here, read
        # as the device reads it (outside [0, k], or 0 on a starting slot: k), k for every other slot
        n = np.full(S, k, np.int64)
        if count is not None:
            c = np.asarray(count, np.int64)
            c = np.where((c < 0) | (c > k) | (start & (c == 0)), k, c)
            counted = is_open & (end < 0)
            n[counted] = c[counted]
        f = np.arange(k)[None, :]
        idx = self.count[:, None] + f - self.lookahead
        length = self.length[:, None]
        frame = np.where(self.active[:, None] & (f < n[:, None]) & (idx >= 0)
                         & ((length < 0) | (idx < length)), idx, -1)
        self.count += n
        # idle once frame length - 1 is out (at once for a sequence without frames)
        done = self.active & (self.length >= 0) & ((self.count - self.lookahead >= self.length)
                                                   | (self.length == 0))
        self.active[done] = False
        if not provisional:
            return frame
        j = np.arange(self.lookahead if rows is None else rows)[None, :]
        h = np.zeros(S, np.int64) if held is None else np.maximum(np.asarray(held, np.int64), 0)
        h = np.where(self.active & (self.length < 0), h, 0)
        idx = self.count[:, None] + j - self.lookahead
        length = self.length[:, None]
        prov = np.where(self.active[:, None] & (j < self.lookahead + h[:, None]) & (idx >= 0)
                        & ((length < 0) | (idx < length)), idx, -1)
        return frame, prov

    def finish(self):
        frame = self.push(self.lookahead) if self.lookahead else \
            np.zeros((len(self.count), 0), np.int64)
        self.active[:] = False
        return frame

    def export_slots(self, slots):
        """The bookkeeping rows of `slots` (what vp3d_stream_export copies of them on the device)."""
        i = np.asarray(slots, np.int64)
        return dict(lookahead=self.lookahead, count=torch.from_numpy(self.count[i].copy()),
                    active=torch.from_numpy(self.active[i].copy()),
                    length=torch.from_numpy(self.length[i].copy()))

    def import_slots(self, rows, slots):
        """Replace the rows of `slots` with those export_slots returned (the same look-ahead)."""
        if rows["lookahead"] != self.lookahead:
            raise ValueError(f"the slots come from a book with lookahead {rows['lookahead']}, this "
                             f"one has {self.lookahead}")
        i = np.asarray(slots, np.int64)
        self.count[i] = rows["count"].numpy()
        self.active[i] = rows["active"].numpy()
        self.length[i] = rows["length"].numpy()


class DetectionCall:
    """What one push_detections (or finish) call sends to the device, as DetectionBook plans it.

    pushes: the internal pushes, each a dict of k (<= max_frames) and the per-slot arrays start
    (bool), end (int32, -1 = none) and count (int32, frames released into this push), plus
    `counted`: whether the push needs its count array (some open slot releases fewer than k).
    records: (rows, 5) int32, one per input row of the pushes in order (push, slot, row) -- slot,
    left, right, num, den as vp3d_stream_pack_detections reads them.  slots: (S, 3) int32 --
    w, h and the row of this call's newest detection (-1 = keep the stored one).  frames: per slot
    the video frame indices released, in order.  realigned: (slot, push) pairs that take the
    realign path (an open slot with fewer frames than the push).  out: (S, n) int64, the frame
    numbers of the rows the call returns (for finish() including the device finish's look-ahead
    rows).  held: (S,) int32, per slot the pending frames after the call (DetectionBook.push).
    prov_frames: for a provisional request, (S, lookahead + max_gap) int64, the frame numbers of
    its rows, those finish() would return right after the call; else None."""

    def __init__(self, pushes, records, slots, frames, realigned, out, held, prov_frames=None):
        self.pushes, self.records, self.slots = pushes, records, slots
        self.frames, self.realigned = frames, realigned
        self.out, self.held, self.prov_frames = out, held, prov_frames

    @property
    def rows(self):
        return len(self.records)

    def table(self):
        """The bytes copied to the device once per call, and the offsets (from its start) of each
        push's end / count (int32, S each) and start (uint8, S) arrays: slots and records (int32,
        vp3d_stream_pack_detections' table) | per push end, count | per push start, and for a
        provisional request the held counts (int32, S) in the last 4 S bytes."""
        S, n = len(self.slots), len(self.pushes)
        tab = np.concatenate([self.slots.reshape(-1), self.records.reshape(-1)]).astype(np.int32)
        head = -(-tab.nbytes // 8) * 8
        tail = 4 * S if self.prov_frames is not None else 0
        host = np.zeros(head + 8 * S * n + -(-S * n // 8) * 8 + tail, np.uint8)
        if tail:
            host[-tail:] = self.held.view(np.uint8)
        host[:tab.nbytes] = tab.view(np.uint8)
        offsets = []
        for i, p in enumerate(self.pushes):
            e, c, st = head + 8 * S * i, head + 8 * S * i + 4 * S, head + 8 * S * n + S * i
            host[e:e + 4 * S] = p["end"].view(np.uint8)
            host[c:c + 4 * S] = p["count"].view(np.uint8)
            host[st:st + S] = p["start"]
            offsets.append((e, c, st))
        return host, offsets


class DetectionBook:
    """Host bookkeeping of a session fed by a 2-D detector (StreamingSession.push_detections):
    which video frames each call releases to the network, and what each is made from, under the
    rules of the reference's decode (data/prepare_data_2d_custom.py:39-49, np.interp over the
    frames without a detection).  Per slot: the open video's frames seen so far, its newest
    detection, the frames released so far (the run between them is pending), the video's
    resolution, and whether the device slot holds the video yet (from its first released frame,
    which is always video frame 0, so the device's frame numbers are the video's).

    Release rules: a detection releases the pending frames before it (interpolated from the
    previous detection, or equal to it before the first one: np.interp's left value) and itself;
    frames after the last detection are released held (np.interp's right value) by the video's end
    or finish(); with max_gap = G, a (G + 1)-th pending frame after a detection releases the oldest
    one held.  A video without detections releases nothing.  Pure host code: the CPU tests drive
    it, and the session turns each DetectionCall into one table copy, one pack launch and its
    pushes.

    Every call reports each slot's pending held count P = seen - released of an open video with a
    detection (0 otherwise: finish() releases nothing before a first detection), at most G.  A
    provisional call (max_gap given) also numbers the la + G rows finish() would return right
    after it: the released frames' look-ahead, then the P pending ones."""

    def __init__(self, streams, max_frames, max_gap=None, lookahead=0):
        self.streams, self.max_frames = int(streams), int(max_frames)
        if max_gap is not None and (isinstance(max_gap, bool) or int(max_gap) != max_gap
                                    or int(max_gap) < 0):
            raise ValueError(f"max_gap must be None or an int >= 0 (got {max_gap!r})")
        self.max_gap = None if max_gap is None else int(max_gap)
        S = self.streams
        self.open = np.zeros(S, bool)               # a video is open: started, not ended
        self.seen = np.zeros(S, np.int64)           # its frames seen so far
        self.last = np.full(S, -1, np.int64)        # its newest detection, -1 before the first
        self.released = np.zeros(S, np.int64)       # its frames released so far
        self.on_device = np.zeros(S, bool)          # the device slot holds it as an open sequence
        self.resolution = np.zeros((S, 2), np.int64)
        self.device = FrameBook(S, lookahead)       # the device's bookkeeping under the pushes

    def check(self, detected, start=None, end=None, resolution=None):
        """The validated (detected (S, k) bool, start (S,) bool, end (S,) int64, resolution (S, 2))
        of a call; raises ValueError / TypeError before anything changes."""
        S = self.streams
        if isinstance(detected, torch.Tensor) and detected.is_cuda:
            raise TypeError("detected must be a host array: how many frames a slot releases depends "
                            "on it, and reading it back from the device would synchronise")
        detected = np.asarray(detected)
        if detected.dtype != np.bool_:
            raise TypeError(f"detected must be a bool array, got {detected.dtype}")
        if detected.ndim != 2 or detected.shape[0] != S or not 1 <= detected.shape[1] <= \
                self.max_frames:
            raise ValueError(f"detected must have shape ({S}, k) with 1 <= k <= max_frames = "
                             f"{self.max_frames}, got {detected.shape}")
        k = detected.shape[1]
        if isinstance(start, torch.Tensor) or isinstance(end, torch.Tensor):
            raise TypeError("push_detections takes start and end as host lists (the host plans "
                            "the releases from them)")
        start = np.zeros(S, bool) if start is None else np.array([bool(v) for v in start])
        if start.shape != (S,):
            raise ValueError(f"start must list {S} slots")
        end = np.full(S, -1, np.int64) if end is None else np.array([int(v) for v in end],
                                                                    np.int64).reshape(-1)
        if end.shape != (S,):
            raise ValueError(f"end must list {S} slots")
        for s in range(S):
            if not -1 <= end[s] <= k:
                raise ValueError(f"end[{s}] = {end[s]} is outside [-1, k = {k}]")
            if end[s] == 0 and start[s]:
                raise ValueError(f"slot {s} starts and ends with end = 0: a video without frames")
        res = self.resolution.copy()
        if resolution is not None:
            resolution = list(resolution)
            if len(resolution) != S:
                raise ValueError(f"resolution must list {S} slots (a (w, h) pair or None each)")
        for s in np.nonzero(start)[0]:
            r = None if resolution is None else resolution[s]
            if r is None:
                raise ValueError(f"slot {s} starts without a resolution: give resolution[{s}] = "
                                 "(w, h), the camera's frame size in pixels")
            w, h = (int(v) for v in r)
            if w <= 0 or h <= 0:
                raise ValueError(f"resolution[{s}] = ({w}, {h}): width and height must be > 0")
            res[s] = (w, h)
        return detected, start, end, res

    def push(self, detected, start=None, end=None, resolution=None, provisional=False):
        """Plan one push_detections call (k = detected.shape[1] video frames per slot);
        provisional=True also plans the provisional rows of its last push (needs max_gap)."""
        if provisional and self.max_gap is None:
            raise ValueError("provisional rows need max_gap: with max_gap=None the frames after a "
                             "slot's last detection may wait without bound")
        detected, start, end, res = self.check(detected, start, end, resolution)
        S, k = detected.shape
        rel = [[] for _ in range(S)]       # per slot: (t, left, right, num, den)
        keep = np.full(S, -1, np.int64)
        drop = np.zeros(S, bool)           # started: without a frame yet, start + end 0 on an active
                                           # device slot
        ending = np.zeros(S, bool)         # the device ends the slot's sequence in this call
        for s in range(S):
            if start[s]:
                # (a start that releases nothing yet still ends what the device slot held, a
                # draining tail included, as a start does in push)
                drop[s] = True
                self.open[s], self.on_device[s] = True, False
                self.seen[s], self.last[s], self.released[s] = 0, -1, 0
                self.resolution[s] = res[s]
            if not self.open[s]:
                continue
            last_row = -1                  # row of the newest detection in this call, -1 = stored
            for f in range(k if end[s] < 0 else int(end[s])):
                t = int(self.seen[s])
                self.seen[s] += 1
                if detected[s, f]:
                    a = int(self.last[s])
                    for u in range(int(self.released[s]), t):
                        rel[s].append((u, f, -1, 0, 0) if a < 0 else (u, last_row, f, u - a, t - a))
                    rel[s].append((t, f, -1, 0, 0))
                    self.last[s], self.released[s] = t, t + 1
                    last_row = keep[s] = f
                elif self.last[s] >= 0 and self.max_gap is not None and \
                        self.seen[s] - self.released[s] > self.max_gap:
                    rel[s].append((int(self.released[s]), last_row, -1, 0, 0))
                    self.released[s] += 1
            if end[s] >= 0:
                if self.last[s] >= 0:
                    for u in range(int(self.released[s]), int(self.seen[s])):
                        rel[s].append((u, last_row, -1, 0, 0))
                    self.released[s] = self.seen[s]
                self.open[s] = False
                ending[s] = True
        pending = np.where(self.open & (self.last >= 0), self.seen - self.released, 0)
        return self._plan(k, rel, keep, drop, ending, pending.astype(np.int32), provisional)

    def finish(self):
        """Plan the pushes finish() makes before the device finish: every open video's pending
        frames released held; every slot then idle."""
        S = self.streams
        rel = [[] for _ in range(S)]
        for s in np.nonzero(self.open & (self.last >= 0))[0]:
            rel[s] = [(u, -1, -1, 0, 0) for u in range(int(self.released[s]), int(self.seen[s]))]
            self.released[s] = self.seen[s]
        none = np.zeros(S, bool)
        call = self._plan(0, rel, np.full(S, -1, np.int64), none, none, np.zeros(S, np.int32))
        self.open[:] = False
        self.on_device[:] = False
        call.out = np.concatenate([call.out, self.device.finish()], 1)
        return call

    _SLOT_FIELDS = ("open", "seen", "last", "released", "on_device", "resolution")

    def export_slots(self, slots):
        """Everything the book keeps of `slots`, its FrameBook rows included, for import_slots of
        another book with the same max_gap and look-ahead (max_frames and streams may differ)."""
        i = np.asarray(slots, np.int64)
        rows = {f: torch.from_numpy(getattr(self, f)[i].copy()) for f in self._SLOT_FIELDS}
        rows.update(max_gap=self.max_gap, device=self.device.export_slots(i))
        return rows

    def import_slots(self, rows, slots):
        """Replace what `slots` hold with the rows export_slots returned: each video goes on as in
        the book it left (its frames, releases and pending ones)."""
        if rows["max_gap"] != self.max_gap:
            raise ValueError(f"the slots come from a book with max_gap {rows['max_gap']}, this one "
                             f"has {self.max_gap}")
        i = np.asarray(slots, np.int64)
        self.device.import_slots(rows["device"], i)
        for f in self._SLOT_FIELDS:
            getattr(self, f)[i] = rows[f].numpy()

    def _plan(self, k, rel, keep, drop, ending, pending, provisional=False):
        """Split the released frames into pushes of at most max_frames, k rows in all at least;
        with provisional, the last push also numbers the provisional rows (pending: P per slot)."""
        S, K = self.streams, self.max_frames
        n = np.array([len(r) for r in rel], np.int64)
        total = max(k, int(n.max()))
        ks = [min(K, total - o) for o in range(0, total, K)]
        offs = np.concatenate([[0], np.cumsum(ks)]).astype(np.int64)
        pushes = [dict(k=kk, start=np.zeros(S, bool), end=np.full(S, -1, np.int32),
                       count=np.zeros(S, np.int32)) for kk in ks]
        for i, p in enumerate(pushes):
            p["count"][:] = np.clip(n - offs[i], 0, ks[i])
        # the push in which the device's sequence of each slot ends (len(pushes) = it goes on)
        end_push = np.full(S, len(pushes), np.int64)
        open_dev = np.zeros(S, bool)   # the device slot holds an open sequence from push 0 on
        for s in range(S):
            first = n[s] > 0 and not self.on_device[s]
            if first:
                assert rel[s][0][0] == 0, "a video's first released frame is its frame 0"
                pushes[0]["start"][s] = True
                self.on_device[s] = True
            elif drop[s] and self.device.active[s]:
                pushes[0]["start"][s] = True
                pushes[0]["end"][s] = 0
                end_push[s] = 0
            open_dev[s] = self.on_device[s]
            if ending[s] and self.on_device[s]:
                i = int(np.searchsorted(offs, n[s] - 1, side="right")) - 1 if n[s] > 0 else 0
                pushes[i]["end"][s] = pushes[i]["count"][s]
                end_push[s] = i
                self.on_device[s] = False
        realigned, out, prov = [], [np.zeros((S, 0), np.int64)], None
        for i, p in enumerate(pushes):
            # count is read for a slot whose open sequence does not end in this push
            held = [s for s in range(S) if open_dev[s] and i < end_push[s]
                    and p["count"][s] < p["k"]]
            p["counted"] = bool(held)
            realigned += [(s, i) for s in held]
            fr = self.device.push(p["k"], p["start"], p["end"], p["count"] if held else None,
                                  provisional and i == len(pushes) - 1, pending,
                                  self.device.lookahead + (self.max_gap or 0))
            if provisional and i == len(pushes) - 1:
                fr, prov = fr
            out.append(fr)
        records = np.zeros((int(offs[-1]) * S, 5), np.int32)
        r = 0
        for i, kk in enumerate(ks):
            for s in range(S):
                chunk = rel[s][offs[i]:offs[i] + kk]
                for f in range(kk):
                    if f < len(chunk):
                        records[r] = (s,) + chunk[f][1:]
                    else:
                        records[r] = (s, -2, -1, 0, 0)
                    r += 1
        slots = np.zeros((S, 3), np.int32)
        slots[:, :2] = self.resolution
        slots[:, 2] = keep
        frames = [[u[0] for u in r] for r in rel]
        return DetectionCall(pushes, records, slots, frames, realigned, np.concatenate(out, 1),
                             pending, prov)


def predict_schedule(lengths, streams, max_frames, lookahead):
    """The pushes StreamingSession.predict makes for sequences of `lengths` frames: a list of dicts
    with k and the per-slot arrays start (bool), end (int32), x_rows and y_rows (int64), rows
    counted in the concatenation of the sequences (input and output alike).

    Sequences go longest first (ties: input order) to the slots that are free; a slot is free in
    the push after the one that returned its previous sequence's last frame.  Pushes carry
    max_frames frames, fewer only once no sequence waits and the remaining drains are shorter."""
    lengths = [int(n) for n in lengths]
    if any(n < 1 for n in lengths):
        raise ValueError("every sequence needs at least one frame")
    S, K = int(streams), int(max_frames)
    order = sorted(range(len(lengths)), key=lambda i: (-lengths[i], i))
    offset = np.concatenate([[0], np.cumsum(lengths, dtype=np.int64)])
    book = FrameBook(S, lookahead)
    seq = np.full(S, -1, np.int64)     # sequence each slot holds
    fed = np.zeros(S, np.int64)        # its frames pushed so far
    pushes, q = [], 0
    while True:
        start = np.zeros(S, bool)
        for s in range(S):
            if not book.active[s] and q < len(order):
                seq[s], fed[s], start[s] = order[q], 0, True
                q += 1
        busy = book.active | start
        if not busy.any():
            return pushes
        if q < len(order):
            k = K
        else:
            count = np.where(start, 0, book.count)
            need = max(lengths[seq[s]] + lookahead - int(count[s]) for s in np.nonzero(busy)[0])
            k = min(K, need)
        end = np.full(S, -1, np.int32)
        x_rows = np.zeros(S, np.int64)
        y_rows = np.zeros(S, np.int64)
        for s in np.nonzero(busy)[0]:
            i = seq[s]
            rest = lengths[i] - fed[s]
            if rest > 0:
                x_rows[s] = offset[i] + fed[s]
                if rest <= k:
                    end[s] = rest
                fed[s] += min(rest, k)
            y_rows[s] = offset[i]
        book.push(k, start, end)
        pushes.append(dict(k=k, start=start, end=end, x_rows=x_rows, y_rows=y_rows))


def _check_sequence(x, joints, features, device):
    if not isinstance(x, torch.Tensor):
        raise TypeError("predict expects a list of torch tensors")
    # (shape and dtype first: they are checked the same way whatever device the tensor is on)
    if x.dim() != 3 or x.shape[1] != joints or x.shape[2] != features or x.shape[0] < 1:
        raise ValueError(f"expected sequences of shape (T >= 1, {joints}, {features}), "
                         f"got {tuple(x.shape)}")
    if x.dtype != torch.float32:
        raise TypeError(f"expected float32 sequences, got {x.dtype}")
    if not x.is_cuda:
        raise RuntimeError("videopose3d_b200 runs on CUDA (sm_90a) tensors only; there is no CPU "
                           "fallback")
    if x.device != device:
        raise RuntimeError("input and parameters are on different devices")


def check_push_input(x, streams, max_frames, joints, features):
    """The validation push() applies to x (raises like the model's forward does)."""
    if not isinstance(x, torch.Tensor):
        raise TypeError("push expects a torch tensor")
    if not x.is_cuda:
        raise RuntimeError("videopose3d_b200 streaming runs on CUDA (sm_90a) tensors only; "
                           "there is no CPU fallback")
    if x.dtype != torch.float32:
        raise TypeError(f"expected a float32 input, got {x.dtype}")
    if x.dim() != 4 or x.shape[0] != streams or x.shape[2] != joints or x.shape[3] != features:
        raise ValueError(f"expected x of shape ({streams}, k, {joints}, {features}), "
                         f"got {tuple(x.shape)}")
    k = int(x.shape[1])
    if not 1 <= k <= max_frames:
        raise ValueError(f"push of {k} frames: k must be in [1, max_frames = {max_frames}]")
    return k


def weights_fingerprint(model):
    """A digest of the values of every tensor the eval forward reads (conv weights, BatchNorm
    parameters and running statistics, shrink bias), whatever device they are on.  Taken once per
    parameter version: the first call after a change reads the parameters back to the host."""
    eng = model._engine
    versions = model._versions()
    cached = getattr(eng, "fingerprint", None)
    if cached is not None and cached[0] == versions:
        return cached[1]
    conv, bn = model._param_tensors()
    h = hashlib.sha256()
    for t in conv + bn:
        a = t.detach().to("cpu", torch.float32).contiguous().numpy()
        h.update(repr(a.shape).encode())
        h.update(a.tobytes())
    eng.fingerprint = (versions, h.hexdigest())
    return eng.fingerprint[1]


def int8_fingerprint(model):
    """A digest of an int8 model's calibration (activation amax per block conv) and block set."""
    eng = model._engine
    key = (model._int8, tuple(model.int8_blocks))
    cached = getattr(eng, "int8_fingerprint", None)
    if cached is not None and cached[0][0] is key[0] and cached[0][1] == key[1]:
        return cached[1]
    h = hashlib.sha256()
    if model._int8 is not None:
        h.update(model._int8[0].detach().to("cpu", torch.float32).contiguous().numpy().tobytes())
    h.update(repr(key[1]).encode())
    eng.int8_fingerprint = (key, h.hexdigest())
    return eng.int8_fingerprint[1]


class StreamSlots:
    """Slots exported from a StreamingSession (export_slots), to be imported into slots of a
    compatible session (import_slots), on this device or another one.

    blob: the DEVICE (or CPU, after .to("cpu")) uint8 records of vp3d_stream_export, one per slot.
    header: the vp3d_stream_slots_header bytes import checks on the host.  compat: what import
    compares with the destination (architecture, precision, augmentation and its mirror maps, the
    detector settings, look-ahead, and fingerprints of the weights and the int8 calibration).  book /
    last: for a detector-fed session, the DetectionBook rows of the slots and their last detections
    (n, J_in, 2).  Survives torch.save / torch.load (also with weights_only=True)."""

    def __init__(self, blob, header, compat, book=None, last=None):
        self.blob, self.header, self.compat, self.book, self.last = blob, header, compat, book, last

    def __len__(self):
        return _capi.StreamSlotsHeader.from_buffer_copy(self.header.numpy().tobytes()).n

    @property
    def device(self):
        return self.blob.device

    def to(self, device):
        """The same slots with the device tensors on `device` (a CUDA device or the CPU)."""
        return StreamSlots(self.blob.to(device), self.header, self.compat, self.book,
                           None if self.last is None else self.last.to(device))


torch.serialization.add_safe_globals([StreamSlots])


class StreamingSession:
    """S stream slots running a TemporalModel frame by frame (see the module docstring).  Create it
    with ``model.streaming(streams, max_frames)``; ``augment=True`` with the left / right lists of
    UnchunkedGenerator returns the test-time flip average instead."""

    detections = False   # fed by push_detections (model.streaming(..., detections=True))

    def __init__(self, model, streams, max_frames, augment=False, kps_left=None, kps_right=None,
                 joints_left=None, joints_right=None, provisional=False, int8=False,
                 detections=False, max_gap=None):
        from .temporal_model import TemporalModel
        if type(model)._variant != TemporalModel._variant:
            raise NotImplementedError(
                "streaming needs a TemporalModel; a TemporalModelOptimized1f state_dict loads into "
                "TemporalModel(..., same arguments) unchanged -- stream that model instead")
        if model.precision == "mixed":
            raise NotImplementedError(
                "precision 'mixed' cannot stream: its per-layer split choice depends on the "
                "sequence length; use 'fp16', 'bf16' or 'bf16x3'")
        self.int8 = bool(int8)
        if self.int8 and model.precision != "int8":
            raise ValueError(f"int8=True streams a model in precision 'int8' (this one is "
                             f"{model.precision!r}: call set_precision('int8') first)")
        if model.precision == "int8" and not self.int8:
            raise NotImplementedError(
                "precision 'int8' streams only in an int8 session: model.streaming(..., "
                "int8=True), whose rings also keep the u8 history; or use 'fp16', 'bf16' or "
                "'bf16x3'")
        if model.training:
            raise RuntimeError("streaming is an eval-mode computation: call model.eval() first")
        streams, max_frames = int(streams), int(max_frames)
        if streams < 1 or max_frames < 1:
            raise ValueError("streams and max_frames must be >= 1")
        self.detections = bool(detections)
        if self.detections:
            if model.in_features != 2:
                raise ValueError(f"detections=True takes 2-D keypoints (in_features == 2); this "
                                 f"model has in_features = {model.in_features}")
            DetectionBook(streams, max_frames, max_gap)   # (checks max_gap)
            if provisional and max_gap is None:
                raise NotImplementedError(
                    "provisional=True with detections=True needs max_gap = G (an int >= 0): the "
                    "provisional rows cover the look-ahead and the at most G frames waiting after "
                    "a slot's last detection, which max_gap=None leaves unbounded")
            if provisional and lookahead(model) == 0 and max_gap == 0:
                raise ValueError("provisional=True on a causal model with max_gap = 0 has nothing "
                                 "provisional: every output is final and no frame waits (give "
                                 "max_gap >= 1)")
        elif max_gap is not None:
            raise ValueError("max_gap is only used with detections=True")
        self.max_gap = max_gap
        # host-side int32 maps; vp3d_stream_init_ex copies them into the session state
        self._kps_src, self._joints_src = augment_maps(model, augment, kps_left, kps_right,
                                                       joints_left, joints_right)
        self.augment = bool(augment)
        self.provisional = bool(provisional)
        if self.provisional and not self.detections and lookahead(model) == 0:
            raise ValueError("provisional=True needs a non-causal model: a causal model has no "
                             "look-ahead, every output of a push is already final")
        # a detections session's provisional rows also cover held frames: HELD rings
        prov_flag = _capi.VP3D_STREAM_HELD if self.detections else _capi.VP3D_STREAM_PROVISIONAL
        self._flags = (_capi.VP3D_STREAM_AUGMENT if self.augment else 0) | \
            (prov_flag if self.provisional else 0) | \
            (_capi.VP3D_STREAM_INT8 if self.int8 else 0)
        device = model.expand_conv.weight.device
        if device.type != "cuda":
            raise RuntimeError("streaming needs the model on a CUDA device; there is no CPU fallback")
        self.model = model
        self.streams = streams
        self.max_frames = max_frames
        self.precision = model.precision
        self.device = device
        self.lookahead = lookahead(model)
        self.last_predict_launches = 0   # kernels the last predict() launched
        lib = _capi.load()
        # the model's plan of this precision (same packed eval weights as model(x))
        self._plan = model._get_plan(device, self.precision)
        with torch.cuda.device(device):
            nbytes = lib.vp3d_stream_state_bytes_ex(self._plan, streams, max_frames, self._flags)
            if nbytes == 0:
                raise ValueError(f"{streams} streams x {max_frames} frames is too large a session")
            self._state = torch.empty(nbytes, dtype=torch.uint8, device=device)
            if self.detections:
                # the last detection of every slot, double-buffered (vp3d_stream_pack_detections)
                self._last = torch.zeros((2, streams, model.num_joints_in, 2), dtype=torch.float32,
                                         device=device)
        self._finalizer = weakref.finalize(self, _release, self._plan, self._state.data_ptr(),
                                           model._engine)
        self.reset()

    def reset(self):
        """Drop all history: every slot idle, weights re-read at the next push."""
        host_ptr = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _capi.check(_capi.load().vp3d_stream_init_ex(
                self._plan, self._state.data_ptr(), self._state.numel(), self.streams,
                self.max_frames, self._flags, host_ptr(self._kps_src), host_ptr(self._joints_src),
                stream), "vp3d_stream_init_ex")
        self._versions = self._quant = None
        if self.detections:
            self._book = DetectionBook(self.streams, self.max_frames, self.max_gap, self.lookahead)
            self._parity = 0
        self.last_call_pushes = 0        # internal pushes of the last push_detections / finish
        self.last_call_launches = 0      # kernels it launched
        self.last_call_realigned = 0     # (slot, push) pairs of it that took the realign path
        self.last_call_prov_rows = 0     # provisional tail rows it computed
        return self

    def _prepare(self):
        m = self.model
        if m.training:
            raise RuntimeError("the model is in train() mode: streaming is an eval-mode computation")
        current = m._versions()
        if self._versions is not None and current != self._versions:
            raise RuntimeError("the model's parameters changed since this session started; call "
                               "reset() before pushing again (old and new weights never mix)")
        # an int8 history is also made from the calibration (the `_int8` tuple itself: every
        # calibrate_int8 / load_int8_calibration makes a new one) and the int8 block set
        quant = (m._int8, m.int8_blocks) if self.int8 else None
        if self._versions is not None and self.int8 and (
                quant[0] is not self._quant[0] or quant[1] != self._quant[1]):
            raise RuntimeError("the model's int8 calibration or int8 blocks changed since this "
                               "session started; call reset() before pushing again (old and new "
                               "quantisations never mix)")
        stream = torch.cuda.current_stream(self.device).cuda_stream
        # (an int8 plan also takes the model's block set and calibration here: _sync_int8)
        m._sync_weights(self._plan, stream)
        self._versions = current
        self._quant = quant
        return stream

    def _slot_tensor(self, v, name):
        if v.shape != (self.streams,):
            raise ValueError(f"{name} must have shape ({self.streams},)")
        if v.device != self.device:
            raise RuntimeError(f"{name} must be on the session's device (or a list)")

    def _start_list(self, start):
        """None, a device tensor, or the validated host list of bools."""
        if start is None:
            return None
        if isinstance(start, torch.Tensor):
            self._slot_tensor(start, "start")
            return start
        start = [bool(v) for v in start]
        if len(start) != self.streams:
            raise ValueError(f"start must list {self.streams} slots")
        return start

    def _end_list(self, end, k, start):
        """None, a device tensor, or the validated host list of ints in [-1, k]."""
        if end is None:
            return None
        if isinstance(end, torch.Tensor):
            self._slot_tensor(end, "end")
            if end.dtype != torch.int32:
                raise TypeError(f"end must be an int32 tensor, got {end.dtype}")
            return end
        end = [int(v) for v in end]
        if len(end) != self.streams:
            raise ValueError(f"end must list {self.streams} slots")
        for s, e in enumerate(end):
            if not -1 <= e <= k:
                raise ValueError(f"end[{s}] = {e} is outside [-1, k = {k}]")
            if e == 0 and isinstance(start, list) and start[s]:
                raise ValueError(f"slot {s} starts and ends with end = 0: a sequence without frames")
        return end

    def _count_list(self, count, k, start):
        """None, a device tensor, or the validated host list of ints in [0, k]."""
        if count is None:
            return None
        if isinstance(count, torch.Tensor):
            self._slot_tensor(count, "count")
            if count.dtype != torch.int32:
                raise TypeError(f"count must be an int32 tensor, got {count.dtype}")
            return count
        count = [int(v) for v in count]
        if len(count) != self.streams:
            raise ValueError(f"count must list {self.streams} slots")
        for s, n in enumerate(count):
            if not 0 <= n <= k:
                raise ValueError(f"count[{s}] = {n} is outside [0, k = {k}]")
            if n == 0 and isinstance(start, list) and start[s]:
                raise ValueError(f"slot {s} starts with count = 0: a start needs its first frame")
        return count

    def _start_mask(self, start):
        start = self._start_list(start)
        if start is None:
            return None
        if isinstance(start, torch.Tensor):
            return start.to(torch.uint8).contiguous()
        if not any(start):
            return None
        return torch.tensor(start, dtype=torch.uint8).to(self.device)

    def push(self, x, start=None, end=None, count=None, provisional=False):
        """Push up to k new frames per slot; returns (y (S, k, J_out, 3), frame (S, k) int64).

        start: S bools (list or device tensor), slots that begin a new sequence with x[s, 0].
        end: S ints in [-1, k] (list or CUDA int32 tensor), end[s] = n >= 0 ends slot s's sequence
        after frame n - 1 of this push (x[s, n:] is not read), -1 = it continues.  Values of a
        device tensor outside [-1, k] count as -1.
        count: S ints in [0, k] (list or CUDA int32 tensor), the real frames x[s, :count[s]] slot s
        has in this push (x[s, count[s]:] is not read, its rows get frame -1), for streams that skip
        or drop frames; None = k for every slot.  Read for open sequences that do not end in this
        push; at least 1 on a starting slot.  Values of a device tensor outside [0, k] (and 0 on a
        starting slot) count as k.  Counts below k add two launches.
        provisional: also return y_prov (S, lookahead, J_out, 3) and frame_prov (S, lookahead)
        int64, what finish() would return right after this push (module docstring); needs a
        session made with provisional=True."""
        if self.detections:
            raise RuntimeError("a session made with detections=True is fed by push_detections")
        if provisional and not self.provisional:
            raise RuntimeError("push(provisional=True) needs a session made with "
                               "model.streaming(..., provisional=True)")
        k = check_push_input(x, self.streams, self.max_frames, self.model.num_joints_in,
                             self.model.in_features)
        if x.device != self.device:
            raise RuntimeError("input and parameters are on different devices")
        start = self._start_list(start)
        end = self._end_list(end, k, start)   # host lists are checked before any device work
        count = self._count_list(count, k, start)
        x = x.contiguous()
        mask = self._start_mask(start)
        if isinstance(end, list):
            end = torch.tensor(end, dtype=torch.int32).to(self.device) if max(end) >= 0 else None
        elif end is not None:
            end = end.contiguous()
        if isinstance(count, list):   # every slot full: the plain push's launches
            count = torch.tensor(count, dtype=torch.int32).to(self.device) if min(count) < k else None
        elif count is not None:
            count = count.contiguous()
        y = torch.empty((self.streams, k, self.model.num_joints_out, 3), dtype=torch.float32,
                        device=self.device)
        frame = torch.empty((self.streams, k), dtype=torch.int64, device=self.device)
        if provisional:
            la = self.lookahead
            y_prov = torch.empty((self.streams, la, self.model.num_joints_out, 3),
                                 dtype=torch.float32, device=self.device)
            frame_prov = torch.empty((self.streams, la), dtype=torch.int64, device=self.device)
            ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
            with torch.cuda.device(self.device):
                stream = self._prepare()
                _capi.check(_capi.load().vp3d_stream_push_provisional(
                    self._plan, self._state.data_ptr(), x.data_ptr(), k, ptr(mask), ptr(end),
                    ptr(count), y.data_ptr(), frame.data_ptr(), y_prov.data_ptr(),
                    frame_prov.data_ptr(), stream), "vp3d_stream_push_provisional")
            return y, frame, y_prov, frame_prov
        with torch.cuda.device(self.device):
            stream = self._prepare()
            _capi.check(_capi.load().vp3d_stream_push_counts(
                self._plan, self._state.data_ptr(), x.data_ptr(), k,
                None if mask is None else mask.data_ptr(), None if end is None else end.data_ptr(),
                None, None, y.data_ptr(), frame.data_ptr(),
                None if count is None else count.data_ptr(), stream), "vp3d_stream_push_counts")
        return y, frame

    def predict(self, sequences):
        """Run whole sequences through the slots: a list of CUDA fp32 (T_i, J_in, F) tensors, T_i >= 1,
        in; the list of their (T_i, J_out, 3) outputs (views into one buffer) out, in input order,
        each equal to the offline forward on the edge-padded sequence (the flip average with
        augment=True).  The session is reset first and left idle.

        The schedule (predict_schedule) follows from the lengths alone, so nothing is read back from
        the device: one host-to-device copy of the whole schedule, then one push per step, each
        reading its frames from and writing its outputs to rows of the two flat buffers."""
        if self.detections:
            raise RuntimeError("a session made with detections=True is fed by push_detections")
        seqs = list(sequences)
        J, F = self.model.num_joints_in, self.model.in_features
        for x in seqs:
            _check_sequence(x, J, F, self.device)
        lengths = [int(x.shape[0]) for x in seqs]
        pushes = predict_schedule(lengths, self.streams, self.max_frames, self.lookahead)
        self.reset()
        self.last_predict_launches = 0
        if not seqs:
            return []
        S, n = self.streams, len(pushes)
        # one row per push: x_rows | y_rows (int64) | end (int32) | start (uint8), 8-byte aligned
        row = -(-(20 * S + S) // 8) * 8
        host = np.zeros((n, row), np.uint8)
        for i, p in enumerate(pushes):
            host[i, :8 * S] = p["x_rows"].view(np.uint8)
            host[i, 8 * S:16 * S] = p["y_rows"].view(np.uint8)
            host[i, 16 * S:20 * S] = p["end"].view(np.uint8)
            host[i, 20 * S:21 * S] = p["start"]
        with torch.cuda.device(self.device):
            sched = torch.from_numpy(host).pin_memory().to(self.device, non_blocking=True)
            xs = torch.cat(seqs)
            y = torch.empty((sum(lengths), self.model.num_joints_out, 3), dtype=torch.float32,
                            device=self.device)
            frame = torch.empty((S, self.max_frames), dtype=torch.int64, device=self.device)
            lib = _capi.load()
            base = sched.data_ptr()
            for i, p in enumerate(pushes):
                stream = self._prepare()
                b = base + i * row
                _capi.check(lib.vp3d_stream_push_ex(
                    self._plan, self._state.data_ptr(), xs.data_ptr(), p["k"],
                    b + 20 * S if p["start"].any() else None,
                    b + 16 * S if (p["end"] >= 0).any() else None,
                    b, b + 8 * S, y.data_ptr(), frame.data_ptr(), stream), "vp3d_stream_push_ex")
                self.last_predict_launches += lib.vp3d_last_launch_count(self._plan)
        offset = np.concatenate([[0], np.cumsum(lengths)])
        return [y[int(offset[i]):int(offset[i + 1])] for i in range(len(seqs))]

    def push_detections(self, kps_px, detected, start=None, end=None, resolution=None,
                        provisional=False):
        """Push k video frames per slot straight from a 2-D detector (a session made with
        detections=True); returns (y (S, n, J_out, 3), frame (S, n) int64), n >= k.

        kps_px: (S, k, J_in, 2) CUDA fp32 pixel keypoints, 1 <= k <= max_frames.
        detected: HOST bool array (S, k), False = no person in that frame (its kps_px values are
        never read and may be NaN).  It is a host array on purpose: how many frames a slot releases
        depends on it, and the host sizes the pushes from it without reading anything back from
        the device.
        start / end: host lists as for push, counted in video frames (this call's k rows, detected
        or not).  resolution: per slot None or the camera's (w, h) in pixels, read for the slots
        that start in this call (required there, both > 0) and kept until the slot's next start.

        Per slot the network receives the video's frames in order, each once, as the reference's
        in-the-wild pipeline prepares them (decode's np.interp over the missed frames, then
        run.py's normalize_screen_coordinates): a detection releases itself and the missed frames
        before it; missed frames after the last detection are released held by `end` or finish();
        with max_gap = G at most G missed frames wait for the next detection (DetectionBook).
        A video without any detection releases nothing.  `frame` numbers the video's frames from
        its start, -1 for rows that are no frame.  A call that releases more than max_frames
        frames for a slot runs several pushes and returns their rows concatenated.

        provisional (a session made with provisional=True and max_gap = G): also return y_prov
        (S, lookahead + G, J_out, 3) and frame_prov (S, lookahead + G) int64, what finish() would
        return right after this call, bit for bit: row j of slot s is frame c - lookahead + j (c =
        its released frames) for j < lookahead + P (P = its pending frames after its last
        detection), under push's rules for ended, draining and idle slots; other rows have frame -1.
        Nothing of it persists.  The tail rides in the call's last push; last_call_prov_rows says
        how many rows it computed, min(lookahead + max P, receptive_field - 1)."""
        if not self.detections:
            raise RuntimeError("push_detections needs a session made with "
                               "model.streaming(..., detections=True)")
        if provisional and not self.provisional:
            raise RuntimeError("push_detections(provisional=True) needs a session made with "
                               "model.streaming(..., detections=True, provisional=True, "
                               "max_gap=G)")
        J = self.model.num_joints_in
        k = check_push_input(kps_px, self.streams, self.max_frames, J, 2)
        if kps_px.device != self.device:
            raise RuntimeError("input and parameters are on different devices")
        det = self._book.check(detected, start, end, resolution)[0]   # before anything changes
        if det.shape != (self.streams, k):
            raise ValueError(f"detected must have shape ({self.streams}, {k}) like kps_px's first "
                             f"two dimensions, got {det.shape}")
        call = self._book.push(det, start, end, resolution, provisional)
        return self._run_detections(call, kps_px.contiguous(), k)

    def _run_detections(self, call, kps, k):
        """One table copy, one pack launch and the pushes of a DetectionCall; the last one asks for
        the provisional rows of a provisional call."""
        S, J = self.streams, self.model.num_joints_in
        pushes = call.pushes
        self.last_call_pushes = len(pushes)
        self.last_call_realigned = len(call.realigned)
        self.last_call_launches = 0
        self.last_call_prov_rows = 0
        outs = []
        if not pushes:
            return None
        host, offsets = call.table()
        lib = _capi.load()
        with torch.cuda.device(self.device):
            stream = self._prepare()
            buf = torch.from_numpy(host).pin_memory().to(self.device, non_blocking=True)
            base = buf.data_ptr()
            xs = torch.empty((call.rows, J, 2), dtype=torch.float32, device=self.device)
            if kps is None:   # finish: every record reads the stored detection
                kps, k = self._last, 1
            _capi.check(lib.vp3d_stream_pack_detections(
                kps.data_ptr(), S, k, J, base, call.rows, self._last.data_ptr(), self._parity,
                xs.data_ptr(), stream), "vp3d_stream_pack_detections")
            self._parity ^= 1
            self.last_call_launches = 1
            row = 0
            for i, p in enumerate(pushes):
                kk = p["k"]
                y = torch.empty((S, kk, self.model.num_joints_out, 3), dtype=torch.float32,
                                device=self.device)
                frame = torch.empty((S, kk), dtype=torch.int64, device=self.device)
                e, c, st = (base + o for o in offsets[i])
                args = (self._plan, self._state.data_ptr(), xs[row:row + S * kk].data_ptr(), kk,
                        st if p["start"].any() else None, e if (p["end"] >= 0).any() else None)
                if call.prov_frames is not None and i == len(pushes) - 1:
                    max_held = int(call.held.max())
                    rows = call.prov_frames.shape[1]
                    prov = (torch.empty((S, rows, self.model.num_joints_out, 3),
                                        dtype=torch.float32, device=self.device),
                            torch.empty((S, rows), dtype=torch.int64, device=self.device))
                    _capi.check(lib.vp3d_stream_push_held(
                        *args, c if p["counted"] else None, base + host.nbytes - 4 * S, max_held,
                        rows, y.data_ptr(), frame.data_ptr(), prov[0].data_ptr(),
                        prov[1].data_ptr(), stream), "vp3d_stream_push_held")
                    self.last_call_prov_rows = min(self.lookahead + max_held,
                                                   self.model.receptive_field() - 1)
                else:
                    _capi.check(lib.vp3d_stream_push_counts(
                        *args, None, None, y.data_ptr(), frame.data_ptr(),
                        c if p["counted"] else None, stream), "vp3d_stream_push_counts")
                self.last_call_launches += lib.vp3d_last_launch_count(self._plan)
                outs.append((y, frame))
                row += S * kk
        if len(outs) == 1:
            y, frame = outs[0]
        else:
            y, frame = torch.cat([o[0] for o in outs], 1), torch.cat([o[1] for o in outs], 1)
        return (y, frame) if call.prov_frames is None else (y, frame) + prov

    def finish(self):
        """Emit the last `lookahead` frames of every slot (its last frame repeated, as the
        generator's end padding does), then mark every slot idle.  A slot whose sequence ended
        earlier returns what is left of its tail, -1 after that.  A detections session first
        releases every open video's missed frames after its last detection (held, np.interp's
        right value) in pushes of its own; their rows come first."""
        if self.detections:
            outs = self._run_detections(self._book.finish(), None, 0)
            launches = self.last_call_launches
            y, frame = self._finish()
            self.last_call_launches = launches + self.last_launch_count()
            if outs is None:
                return y, frame
            return torch.cat([outs[0], y], 1), torch.cat([outs[1], frame], 1)
        return self._finish()

    def _finish(self):
        la = self.lookahead
        y = torch.empty((self.streams, la, self.model.num_joints_out, 3), dtype=torch.float32,
                        device=self.device)
        frame = torch.empty((self.streams, la), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            stream = self._prepare()
            _capi.check(_capi.load().vp3d_stream_finish(self._plan, self._state.data_ptr(),
                                                        y.data_ptr(), frame.data_ptr(), stream),
                        "vp3d_stream_finish")
        return y, frame

    def last_launch_count(self):
        """Kernels the last push (or finish) launched."""
        return _capi.load().vp3d_last_launch_count(self._plan)

    def _slot_list(self, slots, distinct):
        """The validated host list of slot indices of export_slots / import_slots."""
        if isinstance(slots, torch.Tensor):
            if slots.is_cuda:
                raise TypeError("slots must be a host list (the indices are checked on the host)")
            slots = slots.tolist()
        out = []
        for s in slots:
            if isinstance(s, bool) or int(s) != s:
                raise TypeError(f"slot indices must be ints, got {s!r}")
            out.append(int(s))
        if not out:
            raise ValueError("no slots listed")
        for s in out:
            if not 0 <= s < self.streams:
                raise ValueError(f"slot {s} is out of range for {self.streams} slots")
        if distinct and len(set(out)) != len(out):
            dup = next(s for s in out if out.count(s) > 1)
            raise ValueError(f"slot {dup} is listed twice")
        return out

    def _compat(self):
        """What a slot's state depends on besides S, K, provisional sizing and device."""
        m = self.model
        tup = lambda a: None if a is None else tuple(int(v) for v in a)  # noqa: E731
        return dict(
            architecture=(m.num_joints_in, m.in_features, m.num_joints_out,
                          tuple(int(w) for w in m.filter_widths), int(m._channels),
                          bool(m._causal), bool(m._dense)),
            precision=self.precision, lookahead=self.lookahead, augment=self.augment,
            kps_src=tup(self._kps_src), joints_src=tup(self._joints_src),
            detections=self.detections, max_gap=self.max_gap,
            weights=weights_fingerprint(m), int8=int8_fingerprint(m) if self.int8 else None)

    def _unchanged_since_push(self):
        """Raise if the parameters or the int8 quantisation changed under the session's history (as
        the next push would)."""
        m = self.model
        if self._versions is not None and m._versions() != self._versions:
            raise RuntimeError("the model's parameters changed since this session started; call "
                               "reset() first (old and new weights never mix)")
        if self._versions is not None and self.int8 and (
                m._int8 is not self._quant[0] or m.int8_blocks != self._quant[1]):
            raise RuntimeError("the model's int8 calibration or int8 blocks changed since this "
                               "session started; call reset() first")

    def _device_index(self, slots):
        idx = torch.tensor(slots, dtype=torch.int64).pin_memory()
        return idx.to(self.device, non_blocking=True)

    def export_slots(self, slots):
        """Copy the listed slots (host ints in [0, S), any state: idle, open or draining) into a
        StreamSlots, for import_slots of a compatible session; the session is not changed.  One
        launch (vp3d_stream_export) on the current stream, no host synchronisation once the weights'
        fingerprint of this parameter version is known; a detector-fed session also copies the
        slots' last detections."""
        slots = self._slot_list(slots, distinct=False)
        self._unchanged_since_push()
        compat = self._compat()
        lib = _capi.load()
        nbytes = lib.vp3d_stream_slot_bytes(self._plan, self._flags)
        header = _capi.StreamSlotsHeader()
        idx = np.asarray(slots, np.int32)
        book = last = None
        with torch.cuda.device(self.device):
            blob = torch.empty(len(slots) * nbytes, dtype=torch.uint8, device=self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _capi.check(lib.vp3d_stream_export(self._plan, self._state.data_ptr(), idx.ctypes.data,
                                               len(slots), blob.data_ptr(), blob.numel(),
                                               _capi.ctypes.byref(header), stream),
                        "vp3d_stream_export")
            if self.detections:
                book = self._book.export_slots(slots)
                last = self._last[self._parity].index_select(0, self._device_index(slots))
        raw = torch.frombuffer(bytearray(bytes(header)), dtype=torch.uint8)
        return StreamSlots(blob, raw, compat, book, last)

    def import_slots(self, state, slots):
        """Replace what the listed slots (distinct host ints in [0, S), one per exported slot, in
        order) hold with the exported ones, as a start replaces a sequence; the other slots are not
        disturbed.  Each imported slot continues as if every push had gone to the session it came
        from: its frame numbers, end, draining tail, provisional rows and detection gaps, bit for
        bit.  The sessions must be compatible: the same architecture, precision, weights, int8
        calibration and blocks, augment and mirror maps, detections and max_gap (streams,
        max_frames, provisional and device may differ); anything else raises before any device
        work.  One launch (vp3d_stream_import), no host synchronisation once the weights'
        fingerprint of this parameter version is known."""
        if not isinstance(state, StreamSlots):
            raise TypeError(f"import_slots takes the StreamSlots of export_slots, got "
                            f"{type(state).__name__}")
        slots = self._slot_list(slots, distinct=True)
        if len(slots) != len(state):
            raise ValueError(f"{len(slots)} slots listed for {len(state)} exported ones")
        if state.device != self.device:
            raise RuntimeError(f"the exported slots are on {state.device}, the session on "
                               f"{self.device}: call .to({str(self.device)!r}) first")
        self._unchanged_since_push()
        mine = self._compat()
        for key, value in mine.items():
            if state.compat.get(key) != value:
                raise ValueError(f"the exported slots come from an incompatible session: {key} "
                                 f"differs ({state.compat.get(key)!r} there, {value!r} here)")
        header = _capi.StreamSlotsHeader.from_buffer_copy(state.header.numpy().tobytes())
        idx = np.asarray(slots, np.int32)
        lib = _capi.load()
        with torch.cuda.device(self.device):
            stream = self._prepare()
            _capi.check(lib.vp3d_stream_import(self._plan, self._state.data_ptr(), idx.ctypes.data,
                                               len(slots), state.blob.data_ptr(),
                                               state.blob.numel(), _capi.ctypes.byref(header),
                                               stream), "vp3d_stream_import")
            if self.detections:
                self._last[self._parity].index_copy_(0, self._device_index(slots), state.last)
                self._book.import_slots(state.book, slots)
        return self


def _release(plan, state_ptr, engine):
    # `engine` keeps the model's engine state (and with it the plan) alive until the session is gone
    try:
        _capi.load().vp3d_stream_release(plan, state_ptr)
    except Exception:  # pragma: no cover - interpreter shutdown
        pass
