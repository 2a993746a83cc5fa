"""GPU: moving slots between sessions (export_slots / import_slots).

A camera exported from one session and imported into a slot of another compatible one -- other
streams, max_frames, provisional sizing or device -- must go on bit for bit as the uninterrupted
stream: every frame of every sequence that passes through either session is the offline forward on
its padded sequence (``metrics.flip_average`` of it with augmentation, decode -> normalise ->
evaluate() for detector input), and comes out exactly once across both sessions when the source
slot is freed with start=True, end=0.  The source window has wrapped and the destination's last push
carried k > 1 frames, so mirror copies are pending on both sides when the slots move.
"""
import copy
import io

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200.streaming import ring_history

import detections_oracle as dorc
import test_gpu_streaming_counts as counts
import test_gpu_streaming_int8 as int8
from test_streaming_detections_cpu import _random_video

pytestmark = pytest.mark.gpu

SRC = (3, 2)   # (streams, max_frames) of the exporting session
DST = (5, 3)   # of the importing one
SLOT_MAP = [4, 1, 2]   # destination slot of source slots 0 (open), 1 (draining), 2 (idle)


def _rings_R(m, K, provisional):
    tail = vp.streaming.lookahead(m) if provisional else 0
    return [h + K + tail + 1 for h in ring_history(m.filter_widths)], ring_history(m.filter_widths)


def _wrapped(m, K, provisional, pushes):
    """Every ring saw a push whose window [w0, w0 + H + k) crossed its mirror boundary R."""
    Rs, Hs = _rings_R(m, K, provisional)
    return all(any((q - H) % R + H + k > R for q, k in pushes) for R, H in zip(Rs, Hs))


class Run:
    """Sequences by id, and the rows each session returned for them ({frame: y row})."""

    def __init__(self, m, augment):
        self.m, self.augment = m, augment
        self.dev = m.expand_conv.weight.device
        self.seqs, self.rows = {}, {}

    def seq(self, key, T, seed):
        self.seqs[key] = orc.make_input(1, T, 17, self.m.in_features, seed=seed)[0].to(self.dev)
        self.rows[key] = {}
        return self.seqs[key]

    def collect(self, y, frame, owner):
        fr = frame.cpu().numpy()
        for s, f in zip(*np.nonzero(fr >= 0)):
            key = owner[s]
            assert key is not None, ("a frame from a slot without a sequence", s)
            assert int(fr[s, f]) not in self.rows[key], ("frame returned twice", key)
            self.rows[key][int(fr[s, f])] = y[s, f]

    def check(self, keys, partial=()):
        for key in keys:
            x, rows = self.seqs[key], self.rows[key]
            want = counts._offline(self.m, x, self.augment)
            if key not in partial:
                assert sorted(rows) == list(range(len(x))), key
            if not rows:
                continue
            got = torch.stack([rows[t] for t in sorted(rows)])
            assert torch.equal(got, want[sorted(rows)]), (key, float((got - want[sorted(rows)])
                                                                     .abs().max()))


def _push(sess, run, owner, feed, k, start=None, end=None, count=None, provisional=False):
    """One push: feed[s] = (key, first frame) for slots that read x; NaN elsewhere."""
    S = sess.streams
    x = torch.full((S, k, 17, run.m.in_features), float("nan"), device=run.dev)
    for s, (key, f0) in feed.items():
        n = min(k, len(run.seqs[key]) - f0)
        x[s, :n] = run.seqs[key][f0:f0 + n]
    out = sess.push(x, start, end, count, provisional=provisional)
    run.collect(out[0], out[1], owner)
    return out


def _move_and_check(m, augment=False, src_prov=False, dst_prov=False, check_prov=True):
    """Source session A (S = 3, K = 2): slot 0 open (fed with host counts, then exported mid-
    sequence), slot 1 draining after its end, slot 2 idle after a short sequence.  Destination B
    (S = 5, K = 3): slots 0 and 3 run sequences of their own throughout, slot 4 is replaced while
    open, slot 2 while draining, slot 1 while idle; its last push before the import has k = 3.
    After the import A frees its slots (start, end = 0) and B goes on, its first push with a device
    count tensor (the realign path); provisional rows of B are checked against the offline forward
    of the sequence as pushed so far, i.e. what finish() of the uninterrupted session returns."""
    la = vp.streaming.lookahead(m)
    lists = counts._lists(m, augment)
    A = m.streaming(streams=SRC[0], max_frames=SRC[1], augment=augment, provisional=src_prov,
                    **lists)
    B = m.streaming(streams=DST[0], max_frames=DST[1], augment=augment, provisional=dst_prov,
                    **lists)
    run = Run(m, augment)
    R_max = max(_rings_R(m, SRC[1], src_prov)[0])
    n_before = R_max + 8                   # source frames before the export: the window wraps
    T0 = n_before + 40
    x0 = run.seq("x0", T0, 1)
    run.seq("x1", n_before - max(la // 2, 1), 2)   # ends la // 2 frames before the export
    run.seq("x2", 3, 3)
    rng = np.random.RandomState(7)

    # ---- A: counted pushes of k = 2; x1 drains at the export, x2 is idle again
    owner_a = ["x0", "x1", "x2"]
    fed = {"x0": 0, "x1": 0, "x2": 0}
    q, pushes_a, first = 0, [], True
    while q < n_before:
        k = 2
        start = [first] * 3
        end, count, feed = [-1] * 3, [k] * 3, {}
        for s, key in enumerate(owner_a):
            rest = len(run.seqs[key]) - fed[key]
            if rest <= 0:
                continue
            feed[s] = (key, fed[key])
            n = k if s > 0 else int(rng.randint(1 if first else 0, k + 1))
            if rest <= n:
                n = end[s] = rest
            else:
                count[s] = n
            fed[key] += n
        _push(A, run, owner_a, feed, k, start, end, count)
        pushes_a.append((q, k))
        q += k
        first = False
    assert _wrapped(m, SRC[1], src_prov, pushes_a)

    # ---- B: y0 / y3 run throughout; slot 4 open, slot 2 draining, slot 1 idle before the import
    for key, T, seed in (("y0", 70, 4), ("y3", 70, 5), ("y4", 40, 6), ("y2", 4, 7)):
        run.seq(key, T, seed)
    owner_b = ["y0", None, "y2", "y3", "y4"]
    fed_b = {"y0": 0, "y2": 0, "y3": 0, "y4": 0}
    for i in range(4):
        k = 3   # the last push before the import: k > 1 rows whose mirror copy is pending
        start = [i == 0 and owner_b[s] is not None for s in range(5)]
        end, feed = [-1] * 5, {}
        for s, key in enumerate(owner_b):
            if key is None or fed_b[key] >= len(run.seqs[key]):
                continue
            feed[s] = (key, fed_b[key])
            rest = len(run.seqs[key]) - fed_b[key]
            if rest <= k:
                end[s] = rest
            fed_b[key] += min(k, rest)
        _push(B, run, owner_b, feed, k, start, end)
    assert B._versions is not None and k > 1

    # ---- the move
    state = A.export_slots([0, 1, 2])
    B.import_slots(state, SLOT_MAP)
    for s, key in zip(SLOT_MAP, owner_a):
        owner_b[s] = key
    # the move idiom: the freed source slots start a sequence without frames (end = 0, a device
    # tensor: a host list refuses a start with end = 0)
    free = torch.zeros(3, dtype=torch.int32, device=run.dev)
    y_a, frame_a = _push(A, run, [None] * 3, {}, 1, start=[True] * 3, end=free)
    assert (frame_a < 0).all()

    # ---- B goes on: device counts first (realign path), then plain pushes, ends, finish
    i = 0
    while True:
        k = 3
        end, feed = [-1] * 5, {}
        count = [k] * 5
        for s, key in enumerate(owner_b):
            f = fed[key] if key in fed else fed_b.get(key)
            if f is None or f >= len(run.seqs[key]):   # idle or draining: x is not read
                continue
            rest = len(run.seqs[key]) - f
            n = 1 if (i == 0 and key == "x0") else k
            feed[s] = (key, f)
            if rest <= n:
                n = end[s] = rest
            else:
                count[s] = n
            if key in fed:
                fed[key] += n
            else:
                fed_b[key] += n
        if not feed and i > 0:
            break
        dev_count = torch.tensor(count, dtype=torch.int32, device=run.dev) if i == 0 else None
        prov = dst_prov and check_prov and i in (0, 3)
        out = _push(B, run, owner_b, feed, k, end=end, count=dev_count, provisional=prov)
        if prov:
            y_prov, f_prov = out[2], out[3].cpu().numpy()
            c = fed["x0"]   # x0's frames pushed so far: the rows are its forward on x0[:c]
            want = counts._offline(m, run.seqs["x0"][:c], augment)
            rows = f_prov[4][f_prov[4] >= 0]
            assert len(rows) > 0 and (rows < c).all()
            assert torch.equal(y_prov[4][f_prov[4] >= 0], want[rows])
        i += 1
    run.collect(*B.finish(), owner_b)
    run.check(["x0", "x1", "x2", "y0", "y3"])
    run.check(["y4", "y2"], partial=("y4", "y2"))   # replaced by the import: no frame after it
    return A, B


# name: (filter widths, channels, causal, num_joints_out)
ARCHS = {
    "333_c64": ([3, 3, 3], 64, False, 17),
    "333_c128_causal": ([3, 3, 3], 128, True, 17),
    "33333_c1024": ([3, 3, 3, 3, 3], 1024, False, 17),
}


@pytest.mark.parametrize("precision", ["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("arch", list(ARCHS))
def test_moved_slots_bit_identical(cuda_device, arch, precision):
    fw, C, causal, jout = ARCHS[arch]
    m = counts._model(cuda_device, fw, C, causal, precision, jout)
    _move_and_check(m)


@pytest.mark.parametrize("jout", [17, 1])
def test_moved_slots_with_augmentation(cuda_device, jout):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16", jout)
    _move_and_check(m, augment=True)


@pytest.mark.parametrize("src_prov, dst_prov", [(False, True), (True, False), (True, True)])
def test_moves_between_plain_and_provisional_sessions(cuda_device, src_prov, dst_prov):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "bf16x3")
    _move_and_check(m, src_prov=src_prov, dst_prov=dst_prov)


@pytest.mark.parametrize("blocks", [None, [2]])
def test_moved_int8_slots_with_augmentation(cuda_device, blocks):
    m = int8._model(cuda_device, [3, 3, 3], 64, blocks=blocks)
    _move_and_check(m, augment=True, dst_prov=True)


def test_resize_recipe_keeps_every_slot(cuda_device):
    """The README's recipe: a bigger session takes every slot of the old one, in place."""
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    old = m.streaming(streams=2, max_frames=2)
    run = Run(m, False)
    xs = [run.seq(f"x{s}", 50, 10 + s) for s in range(2)]
    for f in range(0, 20, 2):
        _push(old, run, ["x0", "x1"], {0: ("x0", f), 1: ("x1", f)}, 2, start=[f == 0] * 2)
    new = m.streaming(streams=5, max_frames=4)
    new.import_slots(old.export_slots(range(2)), range(2))
    for f in range(20, 50, 4):
        k = min(4, 50 - f)
        _push(new, run, ["x0", "x1", None, None, None], {0: ("x0", f), 1: ("x1", f)}, k,
              end=[k, k, -1, -1, -1] if f + k == 50 else None)
    run.collect(*new.finish(), ["x0", "x1", None, None, None])
    run.check(["x0", "x1"])
    assert len(xs) == 2


def test_round_trip_through_the_cpu_and_torch_save(cuda_device):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    A = m.streaming(streams=1, max_frames=2)
    run = Run(m, False)
    run.seq("x", 40, 3)
    for f in range(0, 20, 2):
        _push(A, run, ["x"], {0: ("x", f)}, 2, start=[f == 0])
    buf = io.BytesIO()
    torch.save(A.export_slots([0]).to("cpu"), buf)
    buf.seek(0)
    state = torch.load(buf).to(cuda_device)
    B = m.streaming(streams=2, max_frames=2)
    B.import_slots(state, [1])
    for f in range(20, 40, 2):
        _push(B, run, [None, "x"], {1: ("x", f)}, 2, end=[-1, 2] if f == 38 else None)
    run.collect(*B.finish(), [None, "x"])
    run.check(["x"])


def test_move_across_devices(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    m1 = copy.deepcopy(m).to("cuda:1")
    A = m.streaming(streams=1, max_frames=2)
    run = Run(m, False)
    x = run.seq("x", 40, 3)
    for f in range(0, 20, 2):
        _push(A, run, ["x"], {0: ("x", f)}, 2, start=[f == 0])
    B = m1.streaming(streams=2, max_frames=3)
    B.import_slots(A.export_slots([0]).to("cuda:1"), [1])
    for f in range(20, 40, 2):
        xb = torch.full((2, 2, 17, 2), float("nan"), device="cuda:1")
        xb[1] = x[f:f + 2].to("cuda:1")
        y, frame = B.push(xb, end=[-1, 2] if f == 38 else None)
        run.collect(y.to(cuda_device), frame, [None, "x"])
    y, frame = B.finish()
    run.collect(y.to(cuda_device), frame, [None, "x"])
    run.check(["x"])


def test_one_launch_each_without_host_synchronisation(cuda_device):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    A = m.streaming(streams=3, max_frames=2, augment=True, **counts.H36M)
    B = m.streaming(streams=4, max_frames=3, augment=True, **counts.H36M)
    x = torch.rand(3, 2, 17, 2, device=cuda_device)
    A.push(x, start=[True] * 3)
    B.push(torch.rand(4, 3, 17, 2, device=cuda_device), start=[True] * 4)
    B.import_slots(A.export_slots([0, 2]), [3, 0])   # (fingerprints taken once per version)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        state = A.export_slots([0, 2])
        assert A.last_launch_count() == 1
        B.import_slots(state, [3, 0])
        assert B.last_launch_count() == 1
    finally:
        torch.cuda.set_sync_debug_mode(0)
    lib = vp._capi.load()
    # bytes per slot, from shapes: bookkeeping, then per physical row H_l rows of ld_l 16-bit values
    hist = ring_history(m.filter_widths)
    row = sum(h * 64 * 2 for h in hist)   # (c_in_pad = C = 64 here)
    assert lib.vp3d_stream_slot_bytes(A._plan, A._flags) == 32 + 2 * row
    assert state.blob.numel() == 2 * (32 + 2 * row)


def test_incompatible_imports_leave_the_destination_untouched(cuda_device):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    perturbed = copy.deepcopy(m)
    with torch.no_grad():
        perturbed.layers_conv[2].weight[5, 7, 1] += 1e-3
    bf16 = counts._model(cuda_device, [3, 3, 3], 64, False, "bf16")
    q8 = int8._model(cuda_device, [3, 3, 3], 64)
    q8b = int8._model(cuda_device, [3, 3, 3], 64, blocks=[1])
    B = m.streaming(streams=3, max_frames=2)
    B.push(torch.rand(3, 2, 17, 2, device=cuda_device), start=[True] * 3)
    before = B._state.clone()
    good = m.streaming(streams=2, max_frames=2)
    good.push(torch.rand(2, 2, 17, 2, device=cuda_device), start=[True] * 2)
    state = good.export_slots([0, 1])
    bad = []
    for other, kw in ((perturbed, {}), (bf16, {}), (m, dict(augment=True, **counts.H36M)),
                      (m, dict(detections=True)), (q8, {})):
        s = other.streaming(streams=2, max_frames=2, **kw)
        if not kw.get("detections"):
            s.push(torch.rand(2, 2, 17, 2, device=cuda_device), start=[True] * 2)
        bad.append(s.export_slots([0, 1]))
    for st in bad:
        with pytest.raises(ValueError, match="incompatible"):
            B.import_slots(st, [0, 1])
    with pytest.raises(ValueError, match="out of range"):
        B.import_slots(state, [0, 3])
    with pytest.raises(ValueError, match="listed twice"):
        B.import_slots(state, [1, 1])
    with pytest.raises(ValueError, match="exported"):
        B.import_slots(state, [0])
    with pytest.raises(RuntimeError, match=r"\.to\("):
        B.import_slots(state.to("cpu"), [0, 1])
    torch.cuda.synchronize()
    assert torch.equal(B._state, before)
    # int8: another block set is another quantisation
    s8 = q8.streaming(streams=2, max_frames=2)
    s8.push(torch.rand(2, 2, 17, 2, device=cuda_device), start=[True] * 2)
    d8 = q8b.streaming(streams=2, max_frames=2)
    with pytest.raises(ValueError, match="incompatible"):
        d8.import_slots(s8.export_slots([0]), [1])
    # and the C header check, under the Python one: a blob of another configuration
    st = s8.export_slots([0])
    st.compat = d8._compat()
    with pytest.raises(RuntimeError, match="stream_import"):
        d8.import_slots(st, [1])
    # the compatible import works afterwards, and the outputs are those of the plain session
    B.import_slots(state, [2, 0])


def test_detector_session_moved_inside_an_open_gap(cuda_device):
    """A detector-fed camera with max_gap exported while a gap is holding frames, imported into a
    running detector session; every frame is decode -> normalise -> evaluate() of its video, and the
    provisional rows after the move are those of the uninterrupted session."""
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    G = 6
    rng = np.random.RandomState(3)
    T = 90
    kps, _, w, h = _random_video(rng, T, 1920, 1080, 0.0)
    mask = np.ones(T, bool)
    mask[[5, 6, 20, 21, 22, 23, 24, 25, 26, 27, 28]] = False
    mask[44:48] = False          # the gap open at the export (frame 48 is the export point)
    mask[60:62] = False
    A = m.streaming(streams=3, max_frames=2, detections=True, provisional=True, max_gap=G)
    U = m.streaming(streams=3, max_frames=2, detections=True, provisional=True, max_gap=G)
    B = m.streaming(streams=5, max_frames=3, detections=True, provisional=True, max_gap=G)
    dev = cuda_device
    got = {}

    def collect(y, frame, s):
        fr = frame[s].cpu().numpy()
        for f in np.nonzero(fr >= 0)[0]:
            assert int(fr[f]) not in got, "frame returned twice"
            got[int(fr[f])] = y[s, f]

    def call(sess, slot, t0, k, start=False, end=-1, prov=True):
        S = sess.streams
        x = torch.full((S, k, 17, 2), float("nan"), device=dev)
        x[slot] = torch.from_numpy(kps[t0:t0 + k]).to(dev)
        det = np.zeros((S, k), bool)
        det[slot] = mask[t0:t0 + k]
        st = [False] * S
        st[slot] = start
        en = [-1] * S
        en[slot] = end
        res = [None] * S
        res[slot] = (w, h)
        return sess.push_detections(x, det, st, en, res, provisional=prov)

    other = np.random.RandomState(9).rand(20, 3) < 0.7   # B's own camera on slot 0
    okps = torch.rand(20, 3, 17, 2, device=dev) * 1000
    for t in range(0, 48, 2):
        out = call(A, 1, t, 2, start=t == 0)
        call(U, 1, t, 2, start=t == 0)
        collect(out[0], out[1], 1)
    for i in range(3):
        x = torch.full((5, 3, 17, 2), float("nan"), device=dev)
        x[0] = okps[i]
        det = np.zeros((5, 3), bool)
        det[0] = other[i]
        B.push_detections(x, det, [i == 0] + [False] * 4, None, [(640, 480)] + [None] * 4)
    assert A._book.seen[1] - A._book.released[1] > 0   # the gap is holding frames
    B.import_slots(A.export_slots([1]), [3])
    for t in range(48, T, 2):
        end = 2 if t + 2 >= T else -1
        yb = call(B, 3, t, 2, end=end)
        yu = call(U, 1, t, 2, end=end)
        collect(yb[0], yb[1], 3)
        if end < 0:   # provisional rows: the uninterrupted session's
            assert torch.equal(yb[3][3], yu[3][1])
            sel = (yb[3][3] >= 0).cpu()
            assert torch.equal(yb[2][3][sel], yu[2][1][sel])
    y, frame = B.finish()
    collect(y, frame, 3)
    xn = dorc.reference_sequence(kps, mask, w, h, G)
    want = counts._offline(m, torch.from_numpy(xn).to(dev))
    assert sorted(got) == list(range(T))
    assert torch.equal(torch.stack([got[t] for t in range(T)]), want)
