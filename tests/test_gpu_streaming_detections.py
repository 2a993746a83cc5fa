"""GPU: sessions fed by a 2-D detector (push_detections).

A video goes in as the detector gives it -- pixel keypoints, a per-frame "person detected" flag and
the camera resolution -- and must come out bit for bit as the reference's in-the-wild pipeline
would give it: decode's np.interp over the missed frames, normalize_screen_coordinates, then
``model(np.pad(xn, (pad + shift, pad - shift), 'edge'))`` (the flip average with augment).  Missed
frames are NaN in kps_px, so a read of one would show in every later output of its slot.
"""
import numpy as np
import pytest
import torch

from videopose3d_b200 import _capi
from videopose3d_b200.streaming import DetectionBook

import detections_oracle as dorc
import test_gpu_streaming_counts as counts
import test_gpu_streaming_int8 as int8
from test_streaming_detections_cpu import CASES, _golden, _random_video

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", CASES)
def test_pack_kernel_matches_the_golden_keypoints(cuda_device, name):
    """vp3d_stream_pack_detections alone: every call's rows are the reference's normalised
    keypoints of the frames it releases, bit for bit, and the stored last detection carries over."""
    kps_px, mask, xn, meta = _golden(name)
    T, J = len(mask), 17
    rng = np.random.RandomState(3)
    book = DetectionBook(1, 8)
    lib = _capi.load()
    last = torch.zeros((2, 1, J, 2), dtype=torch.float32, device=cuda_device)
    parity, t, nxt = 0, 0, 0
    while t < T:
        k = int(min(rng.randint(1, 9), T - t))
        call = book.push(mask[None, t:t + k], [t == 0], [k] if t + k == T else None,
                         [(meta["w"], meta["h"])])
        host, _ = call.table()
        tab = torch.from_numpy(host).to(cuda_device)
        kps = torch.from_numpy(kps_px[None, t:t + k].copy()).to(cuda_device)
        out = torch.full((call.rows, J, 2), float("nan"), device=cuda_device)
        _capi.check(lib.vp3d_stream_pack_detections(
            kps.data_ptr(), 1, k, J, tab.data_ptr(), call.rows, last.data_ptr(), parity,
            out.data_ptr(), torch.cuda.current_stream().cuda_stream), "pack_detections")
        parity ^= 1
        got = out.cpu().numpy()
        frames = call.frames[0]
        assert frames == list(range(nxt, nxt + len(frames)))
        nxt += len(frames)
        rows = got[:len(frames)]
        assert np.array_equal(rows.view(np.uint32), xn[frames].view(np.uint32)), (t, frames)
        assert (got[len(frames):] == 0).all()
        t += k
    assert nxt == T


def _drive_session(sess, m, S, K, videos, rng, max_gap):
    """Push every slot's videos with random k, starts after a random idle stretch, ends (or the
    last video left to finish()), each video only once the previous one's outputs are all back.
    Returns per video ({frame: y row}, detected flags as pushed)."""
    dev = m.expand_conv.weight.device
    J = m.num_joints_in
    got = [[{} for _ in v] for v in videos]
    pushed = [[[] for _ in v] for v in videos]
    cur, pos, want_len = [-1] * S, [0] * S, [[None] * len(v) for v in videos]
    open_ = [False] * S

    def collect(y, frame):
        fr = frame.cpu().numpy()
        for s, f in zip(*np.nonzero(fr >= 0)):
            rows = got[s][cur[s]]
            assert int(fr[s, f]) not in rows, "frame returned twice"
            rows[int(fr[s, f])] = y[s, f]

    def drained(s):
        return cur[s] < 0 or (not open_[s] and len(got[s][cur[s]]) == want_len[s][cur[s]])

    while True:
        if all(cur[s] + 1 == len(videos[s]) and (drained(s) or open_[s] and
                                                 pos[s] >= len(videos[s][cur[s]][1]))
               for s in range(S)):
            break
        k = int(rng.randint(1, K + 1))
        kps = torch.full((S, k, J, 2), float("nan"))
        det = np.zeros((S, k), bool)
        start, end, res = [False] * S, [-1] * S, [None] * S
        for s in range(S):
            if drained(s) and cur[s] + 1 < len(videos[s]) and rng.rand() < 0.6:
                cur[s] += 1
                pos[s] = 0
                start[s] = open_[s] = True
                res[s] = videos[s][cur[s]][2:]
            if not open_[s]:
                continue
            x, msk = videos[s][cur[s]][:2]
            n = max(0, min(k, len(msk) - pos[s]))
            kps[s, :n] = torch.from_numpy(x[pos[s]:pos[s] + n])
            det[s, :n] = msk[pos[s]:pos[s] + n]
            last_video = cur[s] + 1 == len(videos[s])
            if pos[s] + n >= len(msk) and not last_video:
                end[s] = n
                open_[s] = False
            pushed[s][cur[s]].append(det[s] if end[s] < 0 else det[s, :n])
            pos[s] += n
            if not open_[s]:
                d = np.concatenate(pushed[s][cur[s]])
                want_len[s][cur[s]] = len(d) if d.any() else 0
        y, frame = sess.push_detections(kps.to(dev), det, start, end, res)
        assert y.shape[1] >= k and frame.shape[1] == y.shape[1]
        collect(y, frame)
    collect(*sess.finish())
    return got, [[np.concatenate(d) if d else np.zeros(0, bool) for d in v] for v in pushed]


def _check(m, videos, got, masks, max_gap, augment):
    dev = m.expand_conv.weight.device
    n_frames = 0
    for s in range(len(videos)):
        for i, v in enumerate(videos[s]):
            x, _, w, h = v
            msk = masks[s][i]
            rows = got[s][i]
            if not msk.any():
                assert rows == {}, (s, i)
                continue
            x = np.concatenate([x, np.full((len(msk) - len(x), 17, 2), np.nan, np.float32)])
            xn = dorc.reference_sequence(x, msk, w, h, max_gap)
            want = counts._offline(m, torch.from_numpy(xn).to(dev), augment)
            assert sorted(rows) == list(range(len(msk))), (s, i)
            out = torch.stack([rows[t] for t in range(len(msk))])
            assert torch.equal(out, want), (s, i, float((out - want).abs().max()))
            n_frames += len(msk)
    assert n_frames > 0


def _videos(rng, S, n_max=3, T_max=40):
    # (videos of 2 frames or more: a one-frame sequence in a non-causal bf16x3 session differs from
    # the offline forward in the last bits whether it is pushed plainly or from detections)
    return [[_random_video(rng, int(rng.randint(2, T_max)), int(rng.choice([640, 1000, 1920])),
                           int(rng.choice([480, 1002, 1080])), rng.uniform(0, 0.5))
             for _ in range(int(rng.randint(1, n_max + 1)))] for _ in range(S)]


MODES = {   # name: (precision, augment)
    "fp16": ("fp16", False),
    "bf16x3": ("bf16x3", False),
    "int8_augment": ("int8", True),
}


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("mode", list(MODES))
def test_detection_sessions_bit_identical(cuda_device, mode, causal, K):
    precision, augment = MODES[mode]
    if precision == "int8":
        m = int8._model(cuda_device, [3, 3, 3], 64, causal=causal)
    else:
        m = counts._model(cuda_device, [3, 3, 3], 64, causal, precision)
    rng = np.random.RandomState(K * 10 + causal)
    S = 8 if K == 1 else 5
    videos = _videos(rng, S)
    sess = m.streaming(streams=S, max_frames=K, augment=augment, detections=True,
                       **counts._lists(m, augment))
    got, masks = _drive_session(sess, m, S, K, videos, rng, None)
    _check(m, videos, got, masks, None, augment)


@pytest.mark.parametrize("max_gap", [0, 3])
def test_max_gap_sessions_follow_the_gap_rule(cuda_device, max_gap):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    rng = np.random.RandomState(50 + max_gap)
    S, K = 6, 4
    videos = _videos(rng, S, T_max=60)
    sess = m.streaming(streams=S, max_frames=K, detections=True, max_gap=max_gap)
    got, masks = _drive_session(sess, m, S, K, videos, rng, max_gap)
    _check(m, videos, got, masks, max_gap, False)


def test_golden_video_through_a_session(cuda_device):
    """The golden 1000 x 1002 video, pushed one frame per call into slot 1 of a session whose
    other slots run their own videos: its outputs are the offline forward of the reference's
    normalised keypoints."""
    kps_px, mask, xn, meta = _golden("random_1000x1002")
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    rng = np.random.RandomState(9)
    videos = _videos(rng, 3, n_max=1, T_max=30)
    videos[1] = [(kps_px, mask, meta["w"], meta["h"])]
    sess = m.streaming(streams=3, max_frames=1, detections=True)
    got, masks = _drive_session(sess, m, 3, 1, videos, rng, None)
    rows = got[1][0]
    want = counts._offline(m, torch.from_numpy(xn).to(cuda_device))
    out = torch.stack([rows[t] for t in range(len(mask))])
    assert torch.equal(out, want)


def test_launches_and_plain_push_compatibility(cuda_device):
    """Every slot detected in every frame: one pack launch plus the plain push's launches, and
    the outputs of a plain push of the normalised frames."""
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    S, K = 4, 2
    sess = m.streaming(streams=S, max_frames=K, detections=True)
    plain = m.streaming(streams=S, max_frames=K)
    rng = np.random.RandomState(1)
    res = [(1920, 1080)] * S
    for i in range(6):
        px = (rng.uniform(0, 1, (S, K, 17, 2)) * [1920, 1080]).astype(np.float32)
        xn = dorc.normalize(px, 1920, 1080)
        start = [i == 0] * S
        y, frame = sess.push_detections(torch.from_numpy(px).to(cuda_device),
                                        np.ones((S, K), bool), start, None, res if i == 0 else None)
        assert sess.last_call_pushes == 1 and sess.last_call_realigned == 0
        y2, frame2 = plain.push(torch.from_numpy(xn).to(cuda_device), start)
        assert sess.last_call_launches == 1 + plain.last_launch_count()
        assert torch.equal(y, y2) and torch.equal(frame, frame2)
    y, frame = sess.finish()
    y2, frame2 = plain.finish()
    assert torch.equal(y, y2) and torch.equal(frame, frame2)


def test_session_rules(cuda_device):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    sess = m.streaming(streams=2, max_frames=2, detections=True)
    x = torch.zeros(2, 2, 17, 2, device=cuda_device)
    with pytest.raises(RuntimeError, match="push_detections"):
        sess.push(x)
    with pytest.raises(RuntimeError, match="push_detections"):
        sess.predict([x[0]])
    with pytest.raises(ValueError, match="shape"):
        sess.push_detections(x, np.ones((2, 1), bool))
    with pytest.raises(TypeError, match="host"):
        sess.push_detections(x, torch.ones(2, 2, dtype=torch.bool, device=cuda_device))
    with pytest.raises(ValueError, match="resolution"):
        sess.push_detections(x, np.ones((2, 2), bool), [True, False])
    with pytest.raises(RuntimeError, match="detections=True"):
        m.streaming(streams=2, max_frames=2).push_detections(x, np.ones((2, 2), bool))
    # a video nobody is in: every row -1, the slot idle after its end
    y, frame = sess.push_detections(x + float("nan"), np.zeros((2, 2), bool), [True, True],
                                    [2, -1], [(640, 480), (640, 480)])
    assert (frame.cpu() == -1).all()
    y, frame = sess.finish()
    assert (frame.cpu() == -1).all()
