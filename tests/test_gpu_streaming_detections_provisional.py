"""GPU: provisional outputs of detector-fed sessions (push_detections(..., provisional=True),
vp3d_stream_push_held).

A provisional call also returns what finish() would return right after it: the look-ahead tail of
the frames released so far and, per slot, the frames still pending after its last detection, held.
Checked on every call of random videos (misses, gaps shorter and longer than max_gap, trailing gaps,
starts and ends in the middle of a call, bursts of several pushes per call):
  * every provisional row with a frame >= 0 is the offline forward on the video as seen so far,
    decoded as the reference decodes it (np.interp, the held frames after the last detection) and
    edge-padded, bit for bit (the flip average with augment);
  * every few calls both sessions finish() (then start new videos): the last call's provisional
    rows are finish()'s rows;
  * a twin session without the flag, fed the same calls, returns the same y / frame on every call
    and the same finish(), and the launches are its launches plus the output kernel where it shrinks
    straight into y; last_call_prov_rows = min(lookahead + max pending, receptive_field - 1).
A video seen for one frame only is left to the finish() comparison: the offline forward of a
one-frame sequence takes the dependency-cone schedule, which sums the taps in another order.
"""
import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import DetectionBook

import detections_oracle as dorc
import test_gpu_streaming_counts as counts
import test_gpu_streaming_int8 as int8
from test_gpu_streaming_detections import MODES, _videos
from test_streaming_detections_cpu import _random_video

pytestmark = pytest.mark.gpu


def _with_trailing_gaps(rng, videos, longest):
    """Every video followed by a run of 0..longest missed frames (NaN keypoints), so that the
    frames after its last detection wait as a live camera's would."""
    out = []
    for vs in videos:
        row = []
        for x, msk, w, h in vs:
            n = int(rng.randint(0, longest + 1))
            row.append((np.concatenate([x, np.full((n,) + x.shape[1:], np.nan, np.float32)]),
                        np.concatenate([msk, np.zeros(n, bool)]), w, h))
        out.append(row)
    return out


def _run(m, S, K, videos, rng, max_gap, augment, episode=None):
    dev = m.expand_conv.weight.device
    J = m.num_joints_in
    la = vp.streaming.lookahead(m)
    rf = m.receptive_field()
    # calls between finish() comparisons: long enough at K = 1 for a gap to pend past RF - 2
    episode = episode or (24 if K == 1 else 12)
    kw = dict(augment=augment, detections=True, max_gap=max_gap, **counts._lists(m, augment))
    sess = m.streaming(streams=S, max_frames=K, provisional=True, **kw)
    twin = m.streaming(streams=S, max_frames=K, **kw)
    book = DetectionBook(S, K, max_gap, la)
    cur, pos, open_ = [-1] * S, [0] * S, [False] * S
    offline = {}
    n_checked = n_finish = n_copied = 0
    calls = since = 0
    while any(open_[s] or cur[s] + 1 < len(videos[s]) for s in range(S)):
        k = int(rng.randint(1, K + 1))
        kps = torch.full((S, k, J, 2), float("nan"))
        det = np.zeros((S, k), bool)
        start, end, res = [False] * S, [-1] * S, [None] * S
        for s in range(S):
            if not open_[s] and cur[s] + 1 < len(videos[s]) and rng.rand() < 0.6:
                cur[s] += 1
                pos[s] = 0
                start[s] = open_[s] = True
                res[s] = videos[s][cur[s]][2:]
            if not open_[s]:
                continue
            x, msk = videos[s][cur[s]][:2]
            n = min(k, len(msk) - pos[s])
            kps[s, :n] = torch.from_numpy(x[pos[s]:pos[s] + n])
            det[s, :n] = msk[pos[s]:pos[s] + n]
            pos[s] += n
            if pos[s] == len(msk):
                end[s] = n
                open_[s] = False
        call = book.push(det, start, end, res, provisional=True)
        y, frame, yp, fp = sess.push_detections(kps.to(dev), det, start, end, res,
                                                provisional=True)
        y2, frame2 = twin.push_detections(kps.to(dev), det, start, end, res)
        calls += 1
        assert torch.equal(y, y2) and torch.equal(frame, frame2), calls
        direct = not augment and (call.pushes[-1]["k"] == 1 or S == 1)
        assert sess.last_call_launches == twin.last_call_launches + int(direct), calls
        assert sess.last_call_pushes == twin.last_call_pushes == len(call.pushes)
        assert sess.last_call_prov_rows == min(la + int(call.held.max()), rf - 1), calls
        assert tuple(yp.shape) == (S, la + max_gap, m.num_joints_out, 3)
        fp_h = fp.cpu().numpy()
        assert np.array_equal(fp_h, call.prov_frames), calls
        for s in range(S):
            rows = np.nonzero(fp_h[s] >= 0)[0]
            x, msk, w, h = videos[s][cur[s]] if cur[s] >= 0 else (None,) * 4
            seen = pos[s]
            if not len(rows) or seen < 2:
                continue
            key = (s, cur[s], seen)
            if key not in offline:
                xn = dorc.reference_sequence(x[:seen], msk[:seen], w, h, max_gap)
                offline[key] = counts._offline(m, torch.from_numpy(xn).to(dev), augment)
            want = offline[key][torch.from_numpy(fp_h[s, rows]).to(dev)]
            assert torch.equal(yp[s, torch.from_numpy(rows).to(dev)], want), (calls, s)
            n_checked += len(rows)
            n_copied += int((rows >= rf - 2).sum())
        since += 1
        # finish() once `episode` calls have passed and this call has provisional rows, and at the end
        if since >= episode and (fp_h >= 0).any() or not any(
                open_[s] or cur[s] + 1 < len(videos[s]) for s in range(S)):
            since = 0
            yf, ff = sess.finish()
            yf2, ff2 = twin.finish()
            assert torch.equal(yf, yf2) and torch.equal(ff, ff2), calls
            ff_h = ff.cpu().numpy()
            assert np.array_equal(ff_h, book.finish().out), calls
            for s in range(S):
                got = {int(t): i for i, t in enumerate(fp_h[s]) if t >= 0}
                fin = {int(t): i for i, t in enumerate(ff_h[s]) if t >= 0}
                assert sorted(got) == sorted(fin), (calls, s)
                for t in got:
                    assert torch.equal(yp[s, got[t]], yf[s, fin[t]]), (calls, s, t)
                    n_finish += 1
            open_ = [False] * S   # finish() ended every video
    assert n_checked > 0 and n_finish > 0
    return n_copied


@pytest.mark.parametrize("max_gap", [0, 3, 20])
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("mode", list(MODES))
def test_provisional_calls_are_finish_and_the_offline_forward(cuda_device, mode, causal, K,
                                                               max_gap):
    """Arc 3,3,3 (receptive field 27, look-ahead 13): max_gap = 20 pends up to 20 frames, so
    provisional rows j >= RF - 2 = 25 are copies of row 25."""
    if causal and max_gap == 0:
        pytest.skip("a causal model with max_gap = 0 has nothing provisional (refused)")
    precision, augment = MODES[mode]
    if precision == "int8":
        m = int8._model(cuda_device, [3, 3, 3], 64, causal=causal)
    else:
        m = counts._model(cuda_device, [3, 3, 3], 64, causal, precision)
    rng = np.random.RandomState(K * 100 + causal * 10 + max_gap)
    S = 6 if K == 1 else 4
    videos = _with_trailing_gaps(rng, _videos(rng, S, n_max=2, T_max=40), 30)
    n_copied = _run(m, S, K, videos, rng, max_gap, augment)
    if max_gap == 20 and not causal:
        assert n_copied > 0


def test_trajectory_model(cuda_device):
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16", jout=1)
    rng = np.random.RandomState(77)
    videos = _with_trailing_gaps(rng, _videos(rng, 4, n_max=2, T_max=40), 20)
    _run(m, 4, 3, videos, rng, 5, True)


def test_a_gap_longer_than_the_published_lookahead(cuda_device):
    """Arc 3,3,3,3,3 (look-ahead 121, RF - 1 = 242) at C = 128, K = 1: gaps of 150 frames in the
    middle and at the end of a video, with max_gap = 130, pend more than 121 frames, and no call
    computes more than 242 tail rows."""
    m = counts._model(cuda_device, [3, 3, 3, 3, 3], 128, False, "fp16", seed=5)
    rng = np.random.RandomState(5)
    videos = []
    for s in range(2):
        x, msk, w, h = _random_video(rng, 200, 1920, 1080, 0.2)
        msk[:3] = True
        msk[20:170] = False
        x[~msk] = np.nan
        videos.append([(x, msk, w, h)])
    videos = _with_trailing_gaps(rng, videos, 160)
    assert _run(m, 2, 1, videos, rng, 130, False, episode=10 ** 6) > 0


def test_state_size_and_entry_errors(cuda_device):
    lib = _capi.load()
    held, prov = _capi.VP3D_STREAM_HELD, _capi.VP3D_STREAM_PROVISIONAL
    m = counts._model(cuda_device, [3, 3, 3], 64, False, "fp16")
    rf, la = m.receptive_field(), vp.streaming.lookahead(m)
    sess = m.streaming(streams=3, max_frames=2, detections=True, provisional=True, max_gap=4)
    plan = sess._plan
    assert sess._state.numel() == lib.vp3d_stream_state_bytes_ex(plan, 3, 2, held)
    # the held rings and buffers are those of K + RF - 1 rows
    assert lib.vp3d_stream_state_bytes_ex(plan, 3, 2, held) == \
        lib.vp3d_stream_state_bytes_ex(plan, 3, 2 + rf - 1, 0)
    assert lib.vp3d_stream_state_bytes_ex(plan, 3, 2, held | prov) == 0
    x = torch.zeros(3, 2, 17, 2, device=cuda_device)
    y = torch.empty((3, 2, 17, 3), device=cuda_device)
    fr = torch.empty((3, 2), dtype=torch.int64, device=cuda_device)
    yp = torch.empty((3, la + 4, 17, 3), device=cuda_device)
    fp = torch.empty((3, la + 4), dtype=torch.int64, device=cuda_device)
    h = torch.zeros(3, dtype=torch.int32, device=cuda_device)
    stream = sess._prepare()
    st = lib.vp3d_stream_push_held(plan, sess._state.data_ptr(), x.data_ptr(), 2, None, None, None,
                                   h.data_ptr(), 5, la + 4, y.data_ptr(), fr.data_ptr(),
                                   yp.data_ptr(), fp.data_ptr(), stream)
    assert st == -1 and b"rows = 17 < lookahead 13 + max_held 5" in lib.vp3d_last_error()
    st = lib.vp3d_stream_push_held(plan, sess._state.data_ptr(), x.data_ptr(), 3, None, None, None,
                                   h.data_ptr(), 4, la + 4, y.data_ptr(), fr.data_ptr(),
                                   yp.data_ptr(), fp.data_ptr(), stream)
    assert st == -1 and b"exceeds max_frames" in lib.vp3d_last_error()
    # a provisional (not held) session refuses push_held, and a held one push_provisional
    other = m.streaming(streams=3, max_frames=2, provisional=True)
    st = lib.vp3d_stream_push_held(other._plan, other._state.data_ptr(), x.data_ptr(), 2, None, None,
                                   None, h.data_ptr(), 4, la + 4, y.data_ptr(), fr.data_ptr(),
                                   yp.data_ptr(), fp.data_ptr(), stream)
    assert st == -5 and b"VP3D_STREAM_HELD" in lib.vp3d_last_error()
    st = lib.vp3d_stream_push_provisional(plan, sess._state.data_ptr(), x.data_ptr(), 2, None,
                                          None, None, y.data_ptr(), fr.data_ptr(), yp.data_ptr(),
                                          fp.data_ptr(), stream)
    assert st == -5 and b"VP3D_STREAM_PROVISIONAL" in lib.vp3d_last_error()
    torch.cuda.synchronize()
    # a causal session with max_gap >= 1 is made, and its rings are sized as the non-causal ones
    causal = counts._model(cuda_device, [3, 3, 3], 64, True, "fp16")
    cs = causal.streaming(streams=2, max_frames=1, detections=True, provisional=True, max_gap=1)
    assert cs._state.numel() == lib.vp3d_stream_state_bytes_ex(cs._plan, 2, 1, held) > 0
