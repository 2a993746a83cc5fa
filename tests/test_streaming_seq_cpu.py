"""CPU: the host side of per-slot sequence ends and of StreamingSession.predict -- the frame
bookkeeping model against a brute-force per-frame one, predict's schedule, argument validation
before any device work, the C-ABI error paths of vp3d_stream_push_ex, and the reference-produced
fixtures."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import FrameBook, StreamingSession, predict_schedule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "stream_seq")


def _maker():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_stream_seq_golden as mk
    finally:
        sys.path.pop(0)
    return mk


class BruteSlots:
    """Frame-by-frame model of the slots: each pushed frame advances every slot by one."""

    def __init__(self, S, la):
        self.S, self.la = S, la
        self.mode = ["idle"] * S     # idle / open / ended
        self.c = [0] * S             # frames of the current sequence pushed (padding included)
        self.L = [None] * S          # length once ended

    def push(self, k, start=None, end=None):
        frame = np.full((self.S, k), -1, np.int64)
        for s in range(self.S):
            if start is not None and start[s]:
                self.mode[s], self.c[s], self.L[s] = "open", 0, None
            e = -1 if end is None else int(end[s])
            if not -1 <= e <= k:
                e = -1
            if self.mode[s] != "open":
                e = -1
            for f in range(k):
                if f == e:
                    self.mode[s], self.L[s] = "ended", self.c[s]
                idx = self.c[s] - self.la
                if self.mode[s] != "idle" and idx >= 0 and (self.L[s] is None or idx < self.L[s]):
                    frame[s, f] = idx
                self.c[s] += 1
            if e == k:
                self.mode[s], self.L[s] = "ended", self.c[s]
            if self.mode[s] == "ended" and (self.c[s] - self.la >= self.L[s] or self.L[s] == 0):
                self.mode[s] = "idle"
        return frame

    def active(self):
        return np.array([m != "idle" for m in self.mode])


@pytest.mark.parametrize("la", [0, 1, 4, 121])
@pytest.mark.parametrize("seed", range(4))
def test_framebook_matches_brute_force(la, seed):
    """Random schedules: starts, ends mid-push, end = k, end = 0, out-of-range ends (read as -1),
    starts during a drain, ends of idle or already ended slots (ignored)."""
    rng = np.random.RandomState(seed * 10 + la)
    S, K = 5, 9
    book, brute = FrameBook(S, la), BruteSlots(S, la)
    for i in range(300):
        k = int(rng.randint(1, K + 1))
        start = rng.rand(S) < 0.08
        end = np.where(rng.rand(S) < 0.15, rng.randint(-3, k + 3, S), -1)
        if i % 7 == 0:
            end[rng.randint(S)] = 0
        if i % 11 == 0:
            end[rng.randint(S)] = k
        args = dict(start=start if start.any() or i % 2 else None,
                    end=end if (end >= 0).any() or i % 3 else None)
        got = book.push(k, **args)
        want = brute.push(k, **args)
        assert np.array_equal(got, want), i
        assert np.array_equal(book.active, brute.active()), i
    want = brute.push(la) if la else np.zeros((S, 0), np.int64)
    assert np.array_equal(book.finish(), want)
    assert not book.active.any()


@pytest.mark.parametrize("la", [0, 4, 121])
def test_an_ended_slot_drains_and_idles(la):
    """End in the middle of a push: the slot returns frames 0..n-1 exactly once, lookahead frames
    later, then stays idle; the other slot is undisturbed."""
    book = FrameBook(2, la)
    got = {0: [], 1: []}
    book_frames = [book.push(5, start=[True, True], end=[-1, 3])]
    for _ in range(40):
        book_frames.append(book.push(5))
    for fr in book_frames:
        for s in range(2):
            got[s] += [int(v) for v in fr[s] if v >= 0]
    assert got[1] == [0, 1, 2]
    assert got[0] == list(range(len(got[0]))) and len(got[0]) == 205 - la
    assert not book.active[1] and book.active[0]
    book.push(2, start=[False, True], end=[-1, 0])   # start with end = 0: idle at once
    assert not book.active[1]


def _replay(lengths, S, K, la):
    """Replay predict's schedule on the brute-force slots; returns the pushes and, per output row,
    how often it was delivered."""
    pushes = predict_schedule(lengths, S, K, la)
    brute = BruteSlots(S, la)
    offset = np.concatenate([[0], np.cumsum(lengths)])
    delivered = np.zeros(int(offset[-1]), np.int64)
    read = np.zeros(int(offset[-1]), np.int64)
    queued = len(lengths)
    for p in pushes:
        k = p["k"]
        assert 1 <= k <= K
        before = brute.active()
        for s in np.nonzero(p["start"])[0]:
            assert not before[s], "slot reused before its drain"
            queued -= 1
        if queued > 0:
            assert k == K
        for s in range(S):
            open_ = brute.mode[s] == "open" or p["start"][s]
            if open_:
                n = p["end"][s] if p["end"][s] >= 0 else k
                read[p["x_rows"][s]:p["x_rows"][s] + n] += 1
        frame = brute.push(k, p["start"], p["end"])
        for s, f in zip(*np.nonzero(frame >= 0)):
            row = p["y_rows"][s] + frame[s, f]
            seq = np.searchsorted(offset, p["y_rows"][s], side="right") - 1
            assert offset[seq] == p["y_rows"][s] and row < offset[seq + 1]
            delivered[row] += 1
    assert not brute.active().any() and queued == 0
    return pushes, delivered, read


@pytest.mark.parametrize("la", [0, 1, 13, 121])
@pytest.mark.parametrize("S,K", [(1, 1), (3, 4), (8, 16), (50, 7)])
def test_predict_schedule_delivers_every_frame_once(la, S, K):
    rng = np.random.RandomState(S * 100 + K + la)
    lengths = [1, 2] + [int(v) for v in rng.randint(1, 300, 38)]
    pushes, delivered, read = _replay(lengths, S, K, la)
    assert (delivered == 1).all()
    assert (read == 1).all()
    again = predict_schedule(lengths, S, K, la)
    assert len(again) == len(pushes)
    for a, b in zip(pushes, again):
        assert a["k"] == b["k"]
        for key in ("start", "end", "x_rows", "y_rows"):
            assert np.array_equal(a[key], b[key])
            assert a[key].dtype == b[key].dtype


def test_predict_schedule_takes_longest_first():
    pushes = predict_schedule([3, 10, 7, 10], 2, 4, 0)
    first = pushes[0]
    assert first["start"].all()
    # slot 0 holds sequence 1 (rows 3..12), slot 1 sequence 3 (rows 20..29)
    assert first["x_rows"].tolist() == [3, 20] and first["y_rows"].tolist() == [3, 20]
    assert first["end"].dtype == np.int32 and first["x_rows"].dtype == np.int64
    assert predict_schedule([], 4, 4, 3) == []
    with pytest.raises(ValueError, match="at least one frame"):
        predict_schedule([4, 0], 2, 2, 0)


def _bare_session(S=3, K=4):
    """The host-side attributes of a session, without the device state a real one allocates."""
    sess = StreamingSession.__new__(StreamingSession)
    sess.model = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    sess.streams, sess.max_frames, sess.lookahead = S, K, 4
    sess.device = torch.device("cuda", 0)
    return sess


def test_end_validation_before_device_work():
    sess = _bare_session()
    assert sess._end_list(None, 4, None) is None
    assert sess._end_list([-1, 0, 4], 4, None) == [-1, 0, 4]
    with pytest.raises(ValueError, match="outside"):
        sess._end_list([-1, 5, 0], 4, None)
    with pytest.raises(ValueError, match="outside"):
        sess._end_list([-2, 1, 0], 4, None)
    with pytest.raises(ValueError, match="list 3 slots"):
        sess._end_list([1, 1], 4, None)
    with pytest.raises(ValueError, match="without frames"):
        sess._end_list([-1, 0, 2], 4, [False, True, True])
    assert sess._end_list([-1, 0, 2], 4, [True, False, True]) == [-1, 0, 2]
    with pytest.raises(ValueError, match="list 3 slots"):
        sess._start_list([True])
    with pytest.raises(ValueError, match=r"shape \(3,\)"):
        sess._end_list(torch.zeros(4, dtype=torch.int32), 4, None)
    with pytest.raises(RuntimeError, match="device"):
        sess._end_list(torch.zeros(3, dtype=torch.int32), 4, None)


def test_cpu_tensors_are_refused():
    sess = _bare_session()
    with pytest.raises(RuntimeError, match="CUDA"):
        sess.push(torch.zeros(3, 2, 17, 2), end=[-1, 1, 2])
    with pytest.raises(RuntimeError, match="CUDA"):
        sess.predict([torch.zeros(5, 17, 2)])
    with pytest.raises(TypeError, match="torch tensors"):
        sess.predict([np.zeros((5, 17, 2), np.float32)])
    m = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.streaming(streams=2).predict([torch.zeros(5, 17, 2)])


def test_push_ex_reports_errors_without_gpu():
    """Argument checks of vp3d_stream_push_ex run before any device work: status codes, not
    crashes."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    push = lib.vp3d_stream_push_ex
    assert push(fake, None, fake, 1, None, None, None, None, fake, fake, None) == -1
    assert b"null state" in lib.vp3d_last_error()
    for k in (0, -1):
        assert push(fake, fake, fake, k, None, None, None, None, fake, fake, None) == -1
        assert b"k must be >= 1" in lib.vp3d_last_error()
    assert push(None, fake, fake, 1, None, None, None, None, fake, fake, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, fake, fake, fake, fake, None, None) == -1
    assert b"y_rows needs frame" in lib.vp3d_last_error()
    assert push(fake, fake, None, 1, None, fake, fake, None, fake, fake, None) == -1
    assert b"null x, y or frame" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, None, None, fake, None, fake, None) == -1
    assert b"null x, y or frame" in lib.vp3d_last_error()
    assert b"stream_push_ex" in lib.vp3d_last_error()
    # the plain entry reports under its own name
    assert lib.vp3d_stream_push(fake, None, fake, 1, None, fake, fake, None) == -1
    assert b"stream_push: null state" in lib.vp3d_last_error()


def test_fixture_set_covers_the_cases():
    mk = _maker()
    names = sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))
    assert names == sorted(mk.CASES)
    kinds = set()
    for n in names:
        assert os.path.getsize(os.path.join(GOLDEN, n + ".npz")) < 1 << 20
        z = np.load(os.path.join(GOLDEN, n + ".npz"))
        meta = json.loads(str(z["meta"]))
        lengths = meta["lengths"]
        rf = int(np.prod(meta["fw"]))
        assert 1 in lengths and min(lengths) < rf and len(set(lengths)) == len(lengths)
        assert z["lengths"].tolist() == lengths
        assert z["x"].shape == (sum(lengths), meta["J"], meta["F"])
        assert z["y"].shape == (sum(lengths), meta["Jout"], 3)
        kinds.add((meta["causal"], meta["augment"], meta["Jout"]))
    assert {(False, True, 17), (True, False, 17), (False, True, 1)} <= kinds


@pytest.mark.parametrize("name", ["seq_333_c64_tta", "seq_333_c64_causal", "seq_353_c128_traj_tta"])
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    fresh = _maker().make_case(name, ref)
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    for key in ("x", "y", "lengths"):
        assert np.array_equal(fresh[key], z[key]), key
    assert str(fresh["meta"]) == str(z["meta"])

