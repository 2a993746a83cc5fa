"""CPU: the host side of detector-fed streaming (push_detections) -- the numpy restatement of the
pack arithmetic against the reference's golden keypoints, DetectionBook's release rules on random
videos, the validation before any device work, and the C-ABI error paths of the pack entry."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import DetectionBook, FrameBook, StreamingSession

import detections_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "detections")
CASES = ["gaps_1920x1080", "random_1000x1002", "single_640x480"]


def _golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return z["kps_px"], z["mask"], z["xn"], json.loads(str(z["meta"]))


def _drive(videos, S, K, max_gap, rng, use_finish=False):
    """Push every slot's list of videos (kps_px, mask, w, h) through a DetectionBook in calls of
    random k, starting each video after a random idle stretch and ending it with `end` (or, for
    the last video of every slot with use_finish, leaving it to finish()).  Each call's records go
    through pack_restated, and its pushes through a FrameBook (lookahead 0), whose frame numbers
    say which video frame every input row is.  Returns, per video, {frame: normalised row}, the
    list of internal pushes and the detected flags of the frames pushed (past the video's own
    frames for one left open to finish())."""
    J = videos[0][0][0].shape[1]
    book, frames = DetectionBook(S, K, max_gap), FrameBook(S, 0)
    last = np.zeros((S, J, 2), np.float32)
    got = [[{} for _ in v] for v in videos]
    pushed = [[[] for _ in v] for v in videos]   # per video the detected flags of its pushed frames
    cur, pos, pushes = [-1] * S, [0] * S, []

    def end_at(s, n):
        """n if this call ends slot s's video (its last frames are in it), else -1."""
        last_video = cur[s] + 1 == len(videos[s])
        if pos[s] + n < len(videos[s][cur[s]][1]) or (use_finish and last_video):
            return -1
        return n

    def run(call, kps):
        nonlocal last
        k = kps.shape[1]
        out, last = orc.pack_restated(kps, call.slots, call.records, last)
        row = 0
        for p in call.pushes:
            assert 1 <= p["k"] <= K
            pushes.append(p)
            fr = frames.push(p["k"], p["start"], p["end"], p["count"] if p["counted"] else None)
            for s in range(S):
                for f in range(p["k"]):
                    if fr[s, f] >= 0:
                        rows = got[s][cur[s]]
                        assert int(fr[s, f]) not in rows, "frame released twice"
                        assert int(fr[s, f]) == len(rows), "frames out of order"
                        rows[int(fr[s, f])] = out[row + s * p["k"] + f]
            row += S * p["k"]
        assert row == call.rows and row >= S * k

    def done(s):
        return cur[s] + 1 == len(videos[s]) and (
            not book.open[s] or pos[s] >= len(videos[s][cur[s]][1]))

    while not all(done(s) for s in range(S)):
        k = int(rng.randint(1, K + 1))
        kps = np.full((S, k, J, 2), np.nan, np.float32)
        det = np.zeros((S, k), bool)
        start, end, res = [False] * S, [-1] * S, [None] * S
        for s in range(S):
            if not book.open[s] and cur[s] + 1 < len(videos[s]) and rng.rand() < 0.6:
                cur[s] += 1
                pos[s] = 0
                start[s] = True
                res[s] = videos[s][cur[s]][2:]
            if not book.open[s] and not start[s]:
                continue
            x, m = videos[s][cur[s]][:2]
            n = max(0, min(k, len(m) - pos[s]))
            kps[s, :n] = x[pos[s]:pos[s] + n]
            det[s, :n] = m[pos[s]:pos[s] + n]
            end[s] = end_at(s, n)
            # an open video past its frames (left to finish()) takes k more missed frames
            pushed[s][cur[s]].append(det[s] if end[s] < 0 else det[s, :n])
            pos[s] += n
        run(book.push(det, start, end, res), kps)
    run(book.finish(), np.zeros((S, 0, J, 2), np.float32))
    masks = [[np.concatenate(d) if d else np.zeros(0, bool) for d in v] for v in pushed]
    return got, pushes, masks


def _random_video(rng, T, w, h, p_miss, J=17):
    m = rng.rand(T) >= p_miss
    if rng.rand() < 0.3:                      # a long gap
        a = int(rng.randint(0, T))
        m[a:a + int(rng.randint(5, 40))] = False
    if rng.rand() < 0.1:
        m[:] = False                          # nobody in the whole video
    x = rng.uniform(0, 1, (T, J, 2)) * [w, h]
    x = x.astype(np.float32)
    x[~m] = np.nan
    return x, m, w, h


def _expected(video, m, max_gap):
    x, _, w, h = video
    x = np.concatenate([x, np.full((len(m) - len(x),) + x.shape[1:], np.nan, np.float32)])
    if not m.any():
        return {}
    xn = orc.reference_sequence(x, m, w, h, max_gap)
    return {t: xn[t] for t in range(len(m))}


@pytest.mark.parametrize("name", CASES)
def test_golden_is_the_reference_pipeline(name):
    """The golden keypoints are np.interp + normalize_screen_coordinates of the detector's pixels,
    and the float64 restatement of the pack kernel's arithmetic gives the same bits."""
    kps, mask, xn, meta = _golden(name)
    assert kps.shape == xn.shape == (meta["T"], 17, 2) and mask.shape == (meta["T"],)
    assert np.isnan(kps[~mask]).all() and np.isfinite(kps[mask]).all()
    ref = orc.reference_sequence(kps, mask, meta["w"], meta["h"])
    assert np.array_equal(ref.view(np.uint32), xn.view(np.uint32))


@pytest.mark.parametrize("K", [1, 4, 16])
@pytest.mark.parametrize("name", CASES)
def test_book_and_pack_reproduce_the_golden_bits(name, K):
    kps, mask, xn, meta = _golden(name)
    video = (kps, mask, meta["w"], meta["h"])
    for use_finish in (False, True):
        got, _, masks = _drive([[video]], 1, K, None, np.random.RandomState(K), use_finish)
        # (a video left to finish() takes the rest of its last call as missed frames: held)
        T = len(masks[0][0])
        assert np.array_equal(masks[0][0][:meta["T"]], mask) and not masks[0][0][meta["T"]:].any()
        want = np.concatenate([xn, np.repeat(xn[-1:], T - meta["T"], 0)])
        rows = got[0][0]
        assert sorted(rows) == list(range(T))
        out = np.stack([rows[t] for t in range(T)])
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), use_finish


@pytest.mark.parametrize("max_gap", [None, 0, 1, 5])
@pytest.mark.parametrize("seed", range(4))
def test_book_releases_every_frame_once_in_order(seed, max_gap):
    """Random masks (misses of 0-60 %, long gaps, videos nobody is in), random k, starts, ends and
    finish(): every video frame is released once, in order, under its own index, with at most K
    frames per internal push, and its value is the reference's (or the G rule's) bit for bit."""
    rng = np.random.RandomState(seed * 7 + (max_gap or 0))
    S, K = 5, 4
    videos = [[_random_video(rng, int(rng.randint(1, 60)), int(rng.choice([640, 1000, 1920])),
                             int(rng.choice([480, 1002, 1080])), rng.uniform(0, 0.6))
               for _ in range(int(rng.randint(1, 4)))] for _ in range(S)]
    got, pushes, masks = _drive(videos, S, K, max_gap, rng, use_finish=seed % 2 == 1)
    for s in range(S):
        for i, v in enumerate(videos[s]):
            want = _expected(v, masks[s][i], max_gap)
            assert sorted(got[s][i]) == sorted(want), (s, i)
            for t, row in want.items():
                assert np.array_equal(got[s][i][t].view(np.uint32), row.view(np.uint32)), (s, i, t)
    assert all(1 <= p["k"] <= K for p in pushes)


def test_bursts_and_max_gap_push_counts():
    # a detection after 6 missed frames releases 7 frames: pushes of 2, 2, 2, 1 at K = 2
    book = DetectionBook(1, 2)
    c = book.push(np.array([[True, False]]), [True], None, [(10, 10)])
    assert [p["k"] for p in c.pushes] == [2] and list(c.pushes[0]["count"]) == [1]
    for _ in range(2):
        c = book.push(np.array([[False, False]]))
        assert [p["k"] for p in c.pushes] == [2] and list(c.pushes[0]["count"]) == [0]
    c = book.push(np.array([[False, True]]))
    assert [p["k"] for p in c.pushes] == [2, 2, 2, 1]
    assert [int(p["count"][0]) for p in c.pushes] == [2, 2, 2, 1]
    assert c.frames[0] == list(range(1, 8))
    assert len(c.realigned) == 0
    # max_gap = 0: every missed frame goes out at once, held
    book = DetectionBook(1, 1, max_gap=0)
    book.push(np.array([[True]]), [True], None, [(10, 10)])
    for t in range(1, 5):
        c = book.push(np.array([[False]]))
        assert len(c.pushes) == 1 and c.frames[0] == [t]
        assert tuple(c.records[0]) == (0, -1, -1, 0, 0)      # the stored detection
    # max_gap = 2: a gap of 5 is held for 3 frames, the last 2 wait and are interpolated
    book = DetectionBook(1, 8, max_gap=2)
    c = book.push(np.array([[True, False, False, False, False, False, True]]), [True], None,
                  [(10, 10)])
    assert len(c.pushes) == 1 and c.frames[0] == list(range(7))
    assert [tuple(r[1:]) for r in c.records[:7]] == [
        (0, -1, 0, 0), (0, -1, 0, 0), (0, -1, 0, 0), (0, -1, 0, 0),
        (0, 6, 4, 6), (0, 6, 5, 6), (6, -1, 0, 0)]
    # frames before the first detection wait whatever max_gap is
    book = DetectionBook(1, 4, max_gap=0)
    c = book.push(np.array([[False, False, False]]), [True], None, [(10, 10)])
    assert c.frames[0] == [] and not c.pushes[0]["start"][0]      # the device slot stays idle
    c = book.push(np.array([[True]]))
    assert c.frames[0] == [0, 1, 2, 3] and c.pushes[0]["start"][0]
    # a restart that releases nothing yet ends what the device slot held: start with end 0
    c = book.push(np.array([[False]]), [True], None, [(10, 10)])
    assert c.frames[0] == [] and c.pushes[0]["start"][0] and c.pushes[0]["end"][0] == 0
    assert not book.device.active[0]
    # a video nobody is in releases nothing, and its end leaves the device slot as it was
    book = DetectionBook(2, 3)
    c = book.push(np.array([[False, False], [True, True]]), [True, True], [2, -1],
                  [(10, 10), (10, 10)])
    assert c.frames == [[], [0, 1]] and not book.open[0]
    assert c.pushes[0]["counted"] is False


def test_validation_before_device_work():
    book = DetectionBook(2, 4)
    det = np.ones((2, 3), bool)
    with pytest.raises(ValueError, match="without a resolution"):
        book.push(det, [True, False])
    with pytest.raises(ValueError, match="without a resolution"):
        book.push(det, [True, False], None, [None, (640, 480)])
    for bad in ((0, 480), (640, -1)):
        with pytest.raises(ValueError, match="must be > 0"):
            book.push(det, [True, False], None, [bad, None])
    with pytest.raises(ValueError, match="list 2 slots"):
        book.push(det, [True, False], None, [(640, 480)])
    with pytest.raises(ValueError, match="shape"):
        book.push(np.ones((3, 3), bool))
    with pytest.raises(ValueError, match="shape"):
        book.push(np.ones((2, 5), bool))
    with pytest.raises(TypeError, match="bool"):
        book.push(np.ones((2, 3), np.int32))
    with pytest.raises(ValueError, match="outside"):
        book.push(det, None, [4, -1])
    with pytest.raises(ValueError, match="without frames"):
        book.push(det, [True, False], [0, -1], [(640, 480), None])
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="max_gap"):
            DetectionBook(2, 4, bad)
    assert not book.open.any() and (book.resolution == 0).all()   # nothing changed
    # the session's constructor: before any device allocation (these models are on the CPU)
    m = vp.TemporalModel(17, 3, 17, [3, 3], channels=64).eval()
    with pytest.raises(ValueError, match="in_features"):
        StreamingSession(m, 2, 4, detections=True)
    m = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    with pytest.raises(NotImplementedError, match="provisional"):
        StreamingSession(m, 2, 4, detections=True, provisional=True)
    with pytest.raises(ValueError, match="max_gap"):
        StreamingSession(m, 2, 4, detections=True, max_gap=-2)
    with pytest.raises(ValueError, match="only used with detections"):
        StreamingSession(m, 2, 4, max_gap=3)


def test_push_detections_checks_its_session_and_shapes():
    sess = StreamingSession.__new__(StreamingSession)
    sess.model = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    sess.streams, sess.max_frames, sess.lookahead = 2, 4, 4
    sess.device = torch.device("cuda", 0)
    sess.detections = False
    with pytest.raises(RuntimeError, match="detections=True"):
        sess.push_detections(torch.zeros(2, 1, 17, 2), np.ones((2, 1), bool))
    sess.detections = True
    with pytest.raises(RuntimeError, match="is fed by push_detections"):
        sess.push(torch.zeros(2, 1, 17, 2))
    with pytest.raises(RuntimeError, match="CUDA"):
        sess.push_detections(torch.zeros(2, 1, 17, 2), np.ones((2, 1), bool))


def test_pack_detections_reports_errors_without_gpu():
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    pack = lib.vp3d_stream_pack_detections
    assert pack(fake, 0, 1, 17, fake, 1, fake, 0, fake, None) == -1
    assert b"stream_pack_detections: S (0)" in lib.vp3d_last_error()
    assert pack(fake, 1, 1, 17, fake, -1, fake, 0, fake, None) == -1
    assert b"rows must be >= 0" in lib.vp3d_last_error()
    assert pack(fake, 1, 1, 17, fake, 1, fake, 2, fake, None) == -1
    assert b"parity must be 0 or 1" in lib.vp3d_last_error()
    assert pack(None, 1, 1, 17, fake, 1, fake, 0, fake, None) == -1
    assert b"null kps_px" in lib.vp3d_last_error()
    assert pack(fake + 4, 1, 1, 17, fake, 1, fake, 0, fake, None) == -1
    assert b"8-byte aligned" in lib.vp3d_last_error()


@pytest.mark.parametrize("name", CASES)
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None or not os.path.exists(os.path.join(ref, "data", "prepare_data_2d_custom.py")):
        pytest.skip("no reference checkout with data/prepare_data_2d_custom.py")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_detections_golden as mk
    finally:
        sys.path.pop(0)
    fresh = mk.make_case(name, ref)
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    for key in ("kps_px", "mask", "xn"):
        assert np.array_equal(fresh[key], z[key], equal_nan=key == "kps_px"), key
    assert str(fresh["meta"]) == str(z["meta"])
