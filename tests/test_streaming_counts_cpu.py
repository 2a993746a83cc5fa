"""CPU: the host side of per-slot frame counts (push's `count`) -- FrameBook against a per-slot
simulation that keeps each slot's own list of real frames, the validation push() applies before any
device work, and the C-ABI error paths of vp3d_stream_push_counts."""
import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import FrameBook, StreamingSession


class SlotFrames:
    """Each slot on its own: the frames of its current sequence it has been fed, real ones and the
    end padding after them.  A push hands slot s the frames it has in that push -- count[s] real
    ones for an open sequence that does not end, end[s] real ones then padding for one that ends,
    padding while it drains, nothing that counts while idle -- and output row f is the frame fed
    `lookahead` frames before row f's input, while it is a real frame."""

    def __init__(self, S, la):
        self.S, self.la = S, la
        self.fed = [[] for _ in range(S)]    # per fed frame: True = real, False = end padding
        self.open = [False] * S
        self.active = [False] * S

    def push(self, k, start=None, end=None, count=None):
        frame = np.full((self.S, k), -1, np.int64)
        for s in range(self.S):
            if start is not None and start[s]:
                self.fed[s], self.open[s], self.active[s] = [], True, True
            e = -1 if end is None else int(end[s])
            e = e if -1 <= e <= k else -1
            n = k if count is None else int(count[s])
            if not 0 <= n <= k or (n == 0 and start is not None and start[s]):
                n = k
            if not self.active[s]:
                continue
            if self.open[s] and e >= 0:
                new = [True] * e + [False] * (k - e)
                self.open[s] = False
            elif self.open[s]:
                new = [True] * n
            else:
                new = [False] * k
            for f, real in enumerate(new):
                self.fed[s].append(real)
                idx = len(self.fed[s]) - 1 - self.la
                if idx >= 0 and self.fed[s][idx]:
                    frame[s, f] = idx
            length = sum(self.fed[s])
            if not self.open[s] and (len(self.fed[s]) - self.la >= length or length == 0):
                self.active[s] = False
        return frame


@pytest.mark.parametrize("la", [0, 1, 4, 121])
@pytest.mark.parametrize("seed", range(4))
def test_framebook_counts_match_per_slot_frames(la, seed):
    """Random schedules: counts in [0, k] and out of range (read as k), all-zero pushes, starts
    with count 0 (read as k), starts with end = 0, ends while counted, starts during a drain, ends
    of idle or ended slots."""
    rng = np.random.RandomState(seed * 10 + la)
    S, K = 6, 9
    book, sim = FrameBook(S, la), SlotFrames(S, la)
    for i in range(400):
        k = int(rng.randint(1, K + 1))
        start = rng.rand(S) < 0.08
        end = np.where(rng.rand(S) < 0.1, rng.randint(-2, k + 2, S), -1)
        if i % 13 == 0:
            s = rng.randint(S)
            start[s], end[s] = True, 0
        count = rng.randint(0, k + 1, S)
        if i % 5 == 0:
            count[rng.randint(S)] = rng.choice([-3, -1, k + 1, 1000])
        if i % 17 == 0:
            count[:] = 0
        if i % 19 == 0:
            count[rng.randint(S)] = 0
            start[:] = count == 0
        args = dict(start=start if start.any() or i % 2 else None,
                    end=end if (end >= 0).any() or i % 3 else None,
                    count=None if i % 11 == 0 else count)
        got = book.push(k, **args)
        want = sim.push(k, **args)
        assert np.array_equal(got, want), i
        assert np.array_equal(book.active, np.array(sim.active)), i
        for s in range(S):
            if sim.open[s]:
                assert book.length[s] == -1 and book.count[s] == len(sim.fed[s]), (i, s)
            elif sim.active[s]:
                assert book.length[s] == sum(sim.fed[s]), (i, s)
    assert book.finish().shape == (S, la)
    assert not book.active.any()


def test_count_none_and_all_k_are_the_plain_push():
    rng = np.random.RandomState(5)
    a, b, c = FrameBook(4, 3), FrameBook(4, 3), FrameBook(4, 3)
    for i in range(60):
        k = int(rng.randint(1, 6))
        start = rng.rand(4) < 0.1
        end = np.where(rng.rand(4) < 0.1, rng.randint(0, k + 1, 4), -1)
        fa = a.push(k, start, end)
        fb = b.push(k, start, end, count=None)
        fc = c.push(k, start, end, count=np.full(4, k))
        assert np.array_equal(fa, fb) and np.array_equal(fa, fc), i
        for x, y in ((a, b), (a, c)):
            assert np.array_equal(x.count, y.count) and np.array_equal(x.active, y.active)
            assert np.array_equal(x.length, y.length)


def test_a_slot_fed_in_bursts_numbers_its_frames_as_one_per_push():
    la = 4
    burst, single = FrameBook(1, la), FrameBook(1, la)
    counts = [3, 0, 0, 2, 5, 0, 1, 4, 0, 5]
    got, want = [], []
    for i, n in enumerate(counts):
        fr = burst.push(5, start=[i == 0], count=[n])
        got += [int(v) for v in fr[0] if v >= 0]
    for i in range(sum(counts)):
        fr = single.push(1, start=[i == 0])
        want += [int(v) for v in fr[0] if v >= 0]
    assert got == want == list(range(sum(counts) - la))
    assert burst.count[0] == single.count[0] == sum(counts)


def _bare_session(S=3, K=4):
    """The host-side attributes of a session, without the device state a real one allocates."""
    sess = StreamingSession.__new__(StreamingSession)
    sess.model = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    sess.streams, sess.max_frames, sess.lookahead = S, K, 4
    sess.device = torch.device("cuda", 0)
    return sess


def test_count_validation_before_device_work():
    sess = _bare_session()
    assert sess._count_list(None, 4, None) is None
    assert sess._count_list([0, 4, 2], 4, None) == [0, 4, 2]
    assert sess._count_list((1, 0, 2), 2, [True, False, False]) == [1, 0, 2]
    for bad in ([-1, 0, 0], [0, 5, 0]):
        with pytest.raises(ValueError, match="outside"):
            sess._count_list(bad, 4, None)
    with pytest.raises(ValueError, match="list 3 slots"):
        sess._count_list([1, 1], 4, None)
    with pytest.raises(ValueError, match="start needs its first frame"):
        sess._count_list([1, 0, 2], 4, [False, True, False])
    with pytest.raises(ValueError, match=r"shape \(3,\)"):
        sess._count_list(torch.zeros(4, dtype=torch.int32), 4, None)
    with pytest.raises(RuntimeError, match="device"):
        sess._count_list(torch.zeros(3, dtype=torch.int32), 4, None)
    cpu = _bare_session()
    cpu.device = torch.device("cpu")   # the dtype check, on a tensor of the session's device
    with pytest.raises(TypeError, match="int32"):
        cpu._count_list(torch.zeros(3, dtype=torch.int64), 4, None)
    assert cpu._count_list(torch.zeros(3, dtype=torch.int32), 4, None) is not None
    # push checks the list before it touches the device (x on the CPU is refused first)
    with pytest.raises(RuntimeError, match="CUDA"):
        sess.push(torch.zeros(3, 2, 17, 2), count=[0, 1, 2])


def test_push_counts_reports_errors_without_gpu():
    """Argument checks of vp3d_stream_push_counts run before any device work, under its own name."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    push = lib.vp3d_stream_push_counts
    assert push(fake, None, fake, 1, None, None, None, None, fake, fake, fake, None) == -1
    assert b"stream_push_counts: null state" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 0, None, None, None, None, fake, fake, fake, None) == -1
    assert b"k must be >= 1" in lib.vp3d_last_error()
    assert push(None, fake, fake, 1, None, None, None, None, fake, fake, fake, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, None, None, None, None, fake, fake, None) == -1
    assert b"null x, y or frame" in lib.vp3d_last_error()
    assert push(fake, fake, fake, 1, None, None, None, fake, fake, None, fake, None) == -1
    assert b"y_rows needs frame" in lib.vp3d_last_error()
