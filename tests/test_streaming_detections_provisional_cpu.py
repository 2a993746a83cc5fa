"""CPU: the host side of provisional outputs in detector-fed sessions (push_detections(...,
provisional=True)) -- DetectionBook's pending counts and provisional frame numbers against a copy of
the book that runs finish() right after each call, the held ring sizes, the validation the
constructor and push_detections apply before any device work, and the C-ABI error paths of
vp3d_stream_push_held and the VP3D_STREAM_HELD flag."""
import copy

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi, streaming
from videopose3d_b200.streaming import DetectionBook, StreamingSession


def _call_masks(rng, S, k, p_miss, gap):
    """(S, k) detected flags: misses at rate p_miss, and per slot now and then a run of `gap`
    missed frames (the run may go on over the next calls through `gap`'s state)."""
    det = rng.rand(S, k) >= p_miss
    for s in range(S):
        if gap[s] > 0:
            n = min(gap[s], k)
            det[s, :n] = False
            gap[s] -= n
        elif rng.rand() < 0.05:
            gap[s] = int(rng.randint(1, 60))
    return det


@pytest.mark.parametrize("la", [0, 4, 13])
@pytest.mark.parametrize("max_gap", [0, 3, 20])
@pytest.mark.parametrize("K", [1, 4])
def test_provisional_frames_are_finish_right_after_the_call(la, max_gap, K):
    """Random calls with misses, gaps shorter and longer than max_gap, starts (restarts too) and
    ends in the middle of a call, videos nobody is in, and bursts of several pushes per call: the
    provisional frame numbers are, slot by slot, the frames finish() returns on a copy of the book,
    row j being frame c - la + j; the call's own pushes are those of a call without the request."""
    rng = np.random.RandomState(la * 100 + max_gap * 10 + K)
    S = 5
    book, twin = DetectionBook(S, K, max_gap, la), DetectionBook(S, K, max_gap, la)
    gap = [0] * S
    res = [(640, 480)] * S
    n_pending = n_rows = 0
    for i in range(150):
        k = int(rng.randint(1, K + 1))
        det = _call_masks(rng, S, k, rng.choice([0.0, 0.3, 0.9]), gap)
        start = [bool(not book.open[s] and rng.rand() < 0.5 or rng.rand() < 0.02)
                 for s in range(S)]
        end = [int(rng.randint(0, k + 1)) if rng.rand() < 0.04 else -1 for s in range(S)]
        end = [-1 if e == 0 and start[s] else e for s, e in enumerate(end)]   # (no empty video)
        call = book.push(det, start, end, res, provisional=True)
        plain = twin.push(det, start, end, res)
        assert [p["k"] for p in call.pushes] == [p["k"] for p in plain.pushes], i
        for a, b in zip(call.pushes, plain.pushes):
            for key in ("start", "end", "count", "counted"):
                assert np.array_equal(a[key], b[key]), (i, key)
        assert np.array_equal(call.records, plain.records) and np.array_equal(call.out, plain.out)
        assert np.array_equal(call.held, plain.held), i
        prov = call.prov_frames
        assert prov.shape == (S, la + max_gap) and prov.dtype == np.int64
        assert ((call.held >= 0) & (call.held <= max_gap)).all()
        fin = copy.deepcopy(book).finish().out
        c = book.device.count
        for s in range(S):
            want = fin[s][fin[s] >= 0]
            got = prov[s][prov[s] >= 0]
            assert np.array_equal(got, want), (i, s, got, want)
            j = np.nonzero(prov[s] >= 0)[0]
            assert np.array_equal(prov[s, j], c[s] - la + j), (i, s)
            assert (j < la + call.held[s]).all()
            pend = book.seen[s] - book.released[s] if book.open[s] and book.last[s] >= 0 else 0
            assert call.held[s] == pend, (i, s)
        n_pending += int((call.held > 0).sum())
        n_rows += int((prov >= 0).sum())
        if i % 37 == 36:
            assert np.array_equal(book.finish().out, twin.finish().out)
    # (la = 0 with max_gap = 0 has no provisional row: the constructor refuses that session)
    assert (n_rows > 0 or la + max_gap == 0) and (n_pending > 0 or max_gap == 0)


def test_pending_frames_extend_the_provisional_rows():
    la, G = 2, 3
    book = DetectionBook(1, 4, G, la)
    c = book.push(np.array([[True, True, True]]), [True], None, [(10, 10)], provisional=True)
    # 3 frames released, none pending: the look-ahead rows [1, 3)
    assert c.held.tolist() == [0] and c.prov_frames.tolist() == [[1, 2, -1, -1, -1]]
    c = book.push(np.array([[False, False]]), provisional=True)
    assert c.held.tolist() == [2] and c.prov_frames.tolist() == [[1, 2, 3, 4, -1]]
    c = book.push(np.array([[False, False]]), provisional=True)
    # the 4th missed frame goes out held (max_gap = 3): 4 released, 3 pending
    assert c.frames[0] == [3] and c.held.tolist() == [3]
    assert c.prov_frames.tolist() == [[2, 3, 4, 5, 6]]
    assert c.table()[0][-4:].view(np.int32).tolist() == [3]
    c = book.push(np.array([[True]]), provisional=True)       # the gap closes: nothing pending
    assert c.frames[0] == [4, 5, 6, 7] and c.held.tolist() == [0]
    assert c.prov_frames.tolist() == [[6, 7, -1, -1, -1]]
    c = book.push(np.array([[False]]), None, [1], provisional=True)   # the end releases it held
    assert c.frames[0] == [8] and c.held.tolist() == [0]
    assert c.prov_frames.tolist() == [[7, 8, -1, -1, -1]]
    # before a video's first detection nothing is pending (finish() does not release it)
    book = DetectionBook(1, 4, G, la)
    c = book.push(np.array([[False, False]]), [True], None, [(10, 10)], provisional=True)
    assert c.held.tolist() == [0] and (c.prov_frames < 0).all()
    with pytest.raises(ValueError, match="max_gap"):
        DetectionBook(1, 4, None, la).push(np.array([[True]]), [True], None, [(10, 10)],
                                           provisional=True)


def _model(fw, causal=False, C=64):
    return vp.TemporalModel(17, 2, 17, fw, causal=causal, channels=C).eval()


@pytest.mark.parametrize("fw", [[3, 3, 3], [3, 3, 3, 3, 3], [3, 5, 3]])
@pytest.mark.parametrize("max_frames", [1, 4])
def test_held_rings_hold_the_receptive_field_more(fw, max_frames):
    for causal in (False, True):
        m = _model(fw, causal, 1024)
        rf = m.receptive_field()
        held = streaming.ring_bytes_per_stream(m, max_frames, held=True)
        assert held == streaming.ring_bytes_per_stream(m, max_frames + rf - 1)
        assert streaming.ring_bytes_per_stream(m, max_frames, planes=2, augment=True, held=True,
                                               int8=True) == \
            2 * streaming.ring_bytes_per_stream(m, max_frames + rf - 1, planes=2, int8=True)
        if not causal:
            assert held == streaming.ring_bytes_per_stream(
                m, max_frames + streaming.lookahead(m), provisional=True)
            with pytest.raises(ValueError, match="exclude"):
                streaming.ring_bytes_per_stream(m, max_frames, provisional=True, held=True)
    if fw == [3, 3, 3, 3, 3] and max_frames == 1:
        # the published architecture at C = 1024, fp16: about 5 MB per slot (3 MB provisional)
        assert 4.9e6 < streaming.ring_bytes_per_stream(_model(fw, C=1024), 1, held=True) < 5.1e6


def test_constructor_rules_before_device_work():
    m = _model([3, 3])
    with pytest.raises(NotImplementedError, match="provisional.*max_gap"):
        StreamingSession(m, 2, 4, detections=True, provisional=True)
    with pytest.raises(ValueError, match="max_gap"):
        StreamingSession(m, 2, 4, detections=True, provisional=True, max_gap=-1)
    causal = _model([3, 3], causal=True)
    with pytest.raises(ValueError, match="nothing provisional"):
        StreamingSession(causal, 2, 4, detections=True, provisional=True, max_gap=0)
    with pytest.raises(ValueError, match="non-causal"):
        StreamingSession(causal, 2, 4, provisional=True)
    # accepted: then the CPU model is refused
    for model, G in ((m, 0), (m, 5), (causal, 1)):
        with pytest.raises(RuntimeError, match="CUDA device"):
            StreamingSession(model, 2, 4, detections=True, provisional=True, max_gap=G)


def test_push_detections_provisional_needs_the_flag():
    sess = StreamingSession.__new__(StreamingSession)
    sess.model = _model([3, 3])
    sess.streams, sess.max_frames, sess.lookahead = 2, 4, 4
    sess.device = torch.device("cuda", 0)
    sess.detections, sess.provisional = True, False
    with pytest.raises(RuntimeError, match="provisional=True"):
        sess.push_detections(torch.zeros(2, 1, 17, 2), np.ones((2, 1), bool), provisional=True)
    sess.provisional = True   # a flagged session goes on to the input checks
    with pytest.raises(RuntimeError, match="CUDA"):
        sess.push_detections(torch.zeros(2, 1, 17, 2), np.ones((2, 1), bool), provisional=True)


def test_push_held_reports_errors_without_gpu():
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    push = lib.vp3d_stream_push_held

    def call(plan=fake, state=fake, x=fake, k=1, held=fake, max_held=0, rows=4, y=fake,
             frame=fake, y_prov=fake, frame_prov=fake):
        return push(plan, state, x, k, None, None, None, held, max_held, rows, y, frame, y_prov,
                    frame_prov, None)

    for kw in (dict(y_prov=None), dict(frame_prov=None), dict(held=None)):
        assert call(**kw) == -1
        assert b"stream_push_held: null y_prov, frame_prov or held" in lib.vp3d_last_error()
    assert call(max_held=-1) == -1 and b"max_held must be >= 0" in lib.vp3d_last_error()
    assert call(state=None) == -1 and b"stream_push_held: null state" in lib.vp3d_last_error()
    assert call(k=0) == -1 and b"k must be >= 1" in lib.vp3d_last_error()
    assert call(plan=None) == -1 and b"null plan" in lib.vp3d_last_error()
    assert call(x=None) == -1 and b"null x, y or frame" in lib.vp3d_last_error()
    held, prov = _capi.VP3D_STREAM_HELD, _capi.VP3D_STREAM_PROVISIONAL
    aug, i8 = _capi.VP3D_STREAM_AUGMENT, _capi.VP3D_STREAM_INT8
    assert held == 64
    assert lib.vp3d_stream_state_bytes_ex(None, 4, 1, held) == 0
    for flags in (held | 2, held | 8, held | 32, held | 1 << 30, -1):
        assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, flags, None, None, None) == -1
        assert b"unknown flags" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, held | prov, None, None, None) == -1
    assert b"exclude each other" in lib.vp3d_last_error()
    # the flag passes the flag checks alone and with AUGMENT / INT8 (the null plan is reported next)
    for flags in (held, held | i8):
        assert lib.vp3d_stream_init_ex(None, fake, 1 << 20, 4, 1, flags, None, None, None) == -1
        assert b"null plan" in lib.vp3d_last_error()
    kps = np.arange(17, dtype=np.int32)
    assert lib.vp3d_stream_init_ex(None, fake, 1 << 20, 4, 1, held | aug, kps.ctypes.data, None,
                                   None) == -1
    assert b"null plan" in lib.vp3d_last_error()
