"""CPU: the host side of provisional outputs (push(..., provisional=True)) -- FrameBook's provisional
frame numbers against a per-slot restatement of what finish() would number right after each push,
the ring sizes of a provisional session, the validation push() and streaming() apply before any
device work, and the C-ABI error paths of vp3d_stream_push_provisional and the new init flag."""
import copy

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi, streaming
from videopose3d_b200.streaming import FrameBook, StreamingSession


class SlotTail:
    """Each slot on its own: the frames fed to its current sequence (True = real, False = end
    padding).  finish() right after a push would feed `la` padding frames more; its row j is then
    the frame fed `la` frames before it, fed index len(fed) - la + j, while that is a real frame of
    a slot that is still active."""

    def __init__(self, S, la):
        self.S, self.la = S, la
        self.fed = [[] for _ in range(S)]
        self.open = [False] * S
        self.active = [False] * S

    def push(self, k, start, end, count):
        for s in range(self.S):
            if start[s]:
                self.fed[s], self.open[s], self.active[s] = [], True, True
            e = int(end[s]) if -1 <= int(end[s]) <= k else -1
            n = int(count[s])
            if not 0 <= n <= k or (n == 0 and start[s]):
                n = k
            if not self.active[s]:
                continue
            if self.open[s] and e >= 0:
                self.fed[s] += [True] * e + [False] * (k - e)
                self.open[s] = False
            elif self.open[s]:
                self.fed[s] += [True] * n
            else:
                self.fed[s] += [False] * k
            if not self.open[s] and (len(self.fed[s]) - self.la >= sum(self.fed[s])
                                     or sum(self.fed[s]) == 0):
                self.active[s] = False

    def tail(self):
        out = np.full((self.S, self.la), -1, np.int64)
        for s in range(self.S):
            if not self.active[s]:
                continue
            for j in range(self.la):
                idx = len(self.fed[s]) - self.la + j
                if idx >= 0 and self.fed[s][idx]:
                    out[s, j] = idx
        return out


@pytest.mark.parametrize("la", [1, 4, 13, 121])
@pytest.mark.parametrize("seed", range(3))
def test_framebook_provisional_frames_are_finish_right_after_the_push(la, seed):
    """Random schedules with starts, restarts during a drain, ends (also end = 0 and out of range),
    counts of 0, partial, full and out of range, and sequences shorter than the look-ahead."""
    rng = np.random.RandomState(seed * 100 + la)
    S, K = 6, 5
    book, plain, sim = FrameBook(S, la), FrameBook(S, la), SlotTail(S, la)
    for i in range(300):
        k = int(rng.randint(1, K + 1))
        start = rng.rand(S) < 0.1
        end = np.where(rng.rand(S) < 0.15, rng.randint(-2, k + 2, S), -1)
        if i % 11 == 0:
            s = rng.randint(S)
            start[s], end[s] = True, 0
        count = rng.randint(0, k + 1, S)
        if i % 7 == 0:
            count[rng.randint(S)] = rng.choice([-1, k + 1])
        frame, prov = book.push(k, start, end, count, provisional=True)
        assert np.array_equal(frame, plain.push(k, start, end, count)), i
        for a in ("count", "active", "length"):
            assert np.array_equal(getattr(book, a), getattr(plain, a)), (i, a)
        sim.push(k, start, end, count)
        assert prov.shape == (S, la)
        assert np.array_equal(prov, sim.tail()), i
        assert np.array_equal(prov, copy.deepcopy(book).finish()), i


def test_provisional_frames_of_a_short_sequence_lead_with_minus_one():
    la = 6
    book = FrameBook(1, la)
    _, prov = book.push(2, start=[True], provisional=True)
    assert prov.tolist() == [[-1, -1, -1, -1, 0, 1]]
    _, prov = book.push(1, end=[1], provisional=True)    # a 3-frame sequence, ended
    assert prov.tolist() == [[-1, -1, -1, 0, 1, 2]]
    _, prov = book.push(2, provisional=True)              # draining: frames past the end are -1
    assert prov.tolist() == [[-1, 0, 1, 2, -1, -1]]
    frame, prov = book.push(3, provisional=True)
    assert frame.tolist() == [[-1, 0, 1]] and prov.tolist() == [[2, -1, -1, -1, -1, -1]]
    frame, prov = book.push(1, provisional=True)           # the last frame is out: idle
    assert frame.tolist() == [[2]] and (prov < 0).all() and not book.active[0]


@pytest.mark.parametrize("fw", [[3, 3, 3], [3, 3, 3, 3, 3], [3, 5, 3]])
@pytest.mark.parametrize("max_frames", [1, 4])
def test_provisional_rings_hold_the_lookahead_more(fw, max_frames):
    m = vp.TemporalModel(17, 2, 17, fw, channels=1024)
    la = streaming.lookahead(m)
    c_in = 64
    per_position = 2 * (c_in + (len(fw) - 1) * 1024) * 2   # both copies, every ring, 16-bit
    plain = streaming.ring_bytes_per_stream(m, max_frames)
    assert streaming.ring_bytes_per_stream(m, max_frames, provisional=True) == \
        plain + la * per_position
    assert streaming.ring_bytes_per_stream(m, max_frames, provisional=True) == \
        streaming.ring_bytes_per_stream(m, max_frames + la)
    assert streaming.ring_bytes_per_stream(m, max_frames, planes=2, augment=True,
                                           provisional=True) == \
        4 * streaming.ring_bytes_per_stream(m, max_frames, provisional=True)
    if fw == [3, 3, 3, 3, 3] and max_frames == 1:
        # rings of the published H36M architecture: about 3 MB per slot (1 MB without the tail)
        assert 2.9e6 < streaming.ring_bytes_per_stream(m, 1, provisional=True) < 3.1e6
    causal = vp.TemporalModel(17, 2, 17, fw, causal=True, channels=64)
    with pytest.raises(ValueError, match="non-causal"):
        streaming.ring_bytes_per_stream(causal, max_frames, provisional=True)


def _bare_session(provisional, S=3, K=4):
    """The host-side attributes of a session, without the device state a real one allocates."""
    sess = StreamingSession.__new__(StreamingSession)
    sess.model = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    sess.streams, sess.max_frames, sess.lookahead = S, K, 4
    sess.device = torch.device("cuda", 0)
    sess.provisional = provisional
    return sess


def test_provisional_validation_before_device_work():
    with pytest.raises(RuntimeError, match="provisional=True"):
        _bare_session(False).push(torch.zeros(3, 2, 17, 2), provisional=True)
    # a flagged session goes on to the input checks (x on the CPU is refused)
    with pytest.raises(RuntimeError, match="CUDA"):
        _bare_session(True).push(torch.zeros(3, 2, 17, 2), provisional=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        _bare_session(False).push(torch.zeros(3, 2, 17, 2))
    causal = vp.TemporalModel(17, 2, 17, [3, 3], causal=True, channels=64).eval()
    with pytest.raises(ValueError, match="non-causal"):
        causal.streaming(2, 1, provisional=True)
    # the flag itself is accepted on a non-causal model (then the CPU model is refused)
    with pytest.raises(RuntimeError, match="CUDA device"):
        vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval().streaming(2, 1, provisional=True)


def test_push_provisional_reports_errors_without_gpu():
    """Argument checks of vp3d_stream_push_provisional and of the flag run before any device work."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    push = lib.vp3d_stream_push_provisional
    assert push(fake, fake, fake, 1, None, None, None, fake, fake, None, fake, None) == -1
    assert b"stream_push_provisional: null y_prov or frame_prov" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, None, None, fake, fake, fake, None, None) == -1
    assert b"null y_prov or frame_prov" in lib.vp3d_last_error()
    assert push(fake, None, fake, 1, None, None, None, fake, fake, fake, fake, None) == -1
    assert b"stream_push_provisional: null state" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 0, None, None, None, fake, fake, fake, fake, None) == -1
    assert b"k must be >= 1" in lib.vp3d_last_error()
    assert push(None, fake, fake, 1, None, None, None, fake, fake, fake, fake, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert push(fake, fake, None, 1, None, None, None, fake, fake, fake, fake, None) == -1
    assert b"null x, y or frame" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, None, None, fake, None, fake, fake, None) == -1
    assert b"null x, y or frame" in lib.vp3d_last_error()
    prov = _capi.VP3D_STREAM_PROVISIONAL
    assert prov == 4
    aug = _capi.VP3D_STREAM_AUGMENT
    assert lib.vp3d_stream_state_bytes_ex(None, 4, 1, prov) == 0
    for flags in (2, 8, prov | 2, prov | aug | 8, -1):
        assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, flags, None, None, None) == -1
        assert b"unknown flags" in lib.vp3d_last_error()
    # the flag passes the flag check (the null plan is reported next)
    assert lib.vp3d_stream_init_ex(None, fake, 1 << 20, 4, 1, prov, None, None, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
