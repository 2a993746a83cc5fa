"""GPU: sequences that end on their own slot (push's `end`) and StreamingSession.predict.

Every sequence that goes through a slot must come out as the offline forward on the sequence
edge-padded as UnchunkedGenerator pads it, ``model(np.pad(x, (pad + shift, pad - shift), 'edge'))``,
or ``metrics.flip_average(model(b))[0]`` with test-time augmentation, bit for bit, whatever the
other slots do: after its end a slot is fed the end padding (its last frame, repacked from x or
copied from the ring, the same bits), and the GEMMs never mix rows.  A one-frame sequence is the
exception on the offline side only: model(x) then takes the dependency-cone schedule, which sums
the taps in another order (tests/test_gpu_streaming.py), so it is checked against a session of its
own and against the reference fixtures' tolerance.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi, metrics
from videopose3d_b200.generators import UnchunkedGenerator
from videopose3d_b200.streaming import FrameBook

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_seq")
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
H36M = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
TRAJ = dict(kps_left=LEFT, kps_right=RIGHT)


def _model(dev, fw, C, causal, precision, dense=False, jout=17, F=2, seed=0):
    m = vp.TemporalModel(17, F, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(17, F, jout, fw, C, dense=dense, seed=seed))
    return m.to(dev).eval().set_precision(precision)


def _lists(m, augment):
    if not augment:
        return {}
    return TRAJ if m.num_joints_out == 1 else H36M


def _offline(m, x, augment=False):
    """run.py's evaluate(return_predictions=True) for one (T, J, F) sequence."""
    pad = (m.receptive_field() - 1) // 2
    shift = pad if m._causal else 0          # run.py:186-193
    if not augment:
        xp = np.pad(x.cpu().numpy(), ((pad + shift, pad - shift), (0, 0), (0, 0)), "edge")
        with torch.no_grad():
            return m(torch.from_numpy(xp)[None].to(x.device))[0]
    lists = _lists(m, True)
    gen = UnchunkedGenerator(None, None, [x.cpu().numpy()], pad=pad, causal_shift=shift,
                             augment=True, kps_left=LEFT, kps_right=RIGHT, device=x.device)
    with torch.no_grad():
        for _, _, b in gen.next_epoch():
            return metrics.flip_average(m(b), lists.get("joints_left"), lists.get("joints_right"))[0]


def _live_session(m, S, K, seqs_per_slot, seed, augment=False, drain_starts=False,
                  finish_at=None):
    """Drive a session push by push: every slot runs its own list of sequences, started after a
    random idle gap, ended with `end` in the middle of a random push.  Frames past a sequence's end
    are NaN in x (they must never be read).  With drain_starts, some sequences start while the
    previous one still drains (its undelivered tail is dropped).  finish_at: stop feeding after that
    many pushes and call finish().  Returns {(slot, j): (x, {frame: y row}, dropped)}."""
    rng = np.random.RandomState(seed)
    la = vp.streaming.lookahead(m)
    dev = m.expand_conv.weight.device
    J, F = m.num_joints_in, m.in_features
    sess = m.streaming(streams=S, max_frames=K, augment=augment, **_lists(m, augment))
    book = FrameBook(S, la)
    queue = {s: [orc.make_input(1, int(T), J, F, seed=seed * 1000 + s * 10 + j)[0].to(dev)
                 for j, T in enumerate(seqs_per_slot[s])] for s in range(S)}
    cur = [-1] * S            # index of the sequence each slot holds
    fed = [0] * S
    out = {}
    n_push = 0
    while any(book.active) or any(cur[s] + 1 < len(queue[s]) for s in range(S)):
        if finish_at is not None and n_push == finish_at:
            break
        k = int(rng.randint(1, K + 1))
        start = [False] * S
        end = [-1] * S
        x = torch.rand(S, k, J, F, device=dev) * 2 - 1
        for s in range(S):
            nxt = cur[s] + 1 < len(queue[s])
            draining = book.active[s] and cur[s] >= 0 and fed[s] == len(queue[s][cur[s]])
            if nxt and (not book.active[s] and rng.rand() < 0.5 or
                        drain_starts and draining and rng.rand() < 0.3):
                if cur[s] >= 0 and book.active[s]:
                    out[(s, cur[s])] = out[(s, cur[s])][:2] + (True,)
                cur[s] += 1
                fed[s] = 0
                start[s] = True
                out[(s, cur[s])] = (queue[s][cur[s]], {}, False)
            if cur[s] < 0 or not (book.active[s] or start[s]):
                continue
            seq = queue[s][cur[s]]
            rest = len(seq) - fed[s]
            if rest <= 0:   # draining: x is not read
                x[s] = float("nan")
                continue
            n = min(rest, k)
            x[s, :n] = seq[fed[s]:fed[s] + n]
            if rest <= k:
                end[s] = rest
                x[s, rest:] = float("nan")
            fed[s] += n
        y, frame = sess.push(x, start=start, end=end)
        want = book.push(k, start, end)
        assert np.array_equal(frame.cpu().numpy(), want), n_push
        for s, f in zip(*np.nonzero(want >= 0)):
            rows = out[(s, cur[s])][1]
            assert int(want[s, f]) not in rows, "frame returned twice"
            rows[int(want[s, f])] = y[s, f]
        n_push += 1
    if finish_at is not None:
        for s in range(S):   # an open sequence ends where finish() finds it
            if cur[s] >= 0 and book.active[s]:
                x, rows, dropped = out[(s, cur[s])]
                out[(s, cur[s])] = (x[:fed[s]], rows, dropped)
        y, frame = sess.finish()
        want = book.finish()
        assert np.array_equal(frame.cpu().numpy(), want)
        for s, f in zip(*np.nonzero(want >= 0)):
            out[(s, cur[s])][1][int(want[s, f])] = y[s, f]
    return out


def _check_live(m, out, augment=False, complete=True):
    checked = 0
    for key, (x, rows, dropped) in out.items():
        T = len(x)
        got = sorted(rows)
        assert got == list(range(len(got))), key          # a prefix, each frame once
        if complete and not dropped:
            assert len(got) == T, key
        if not got or T < 2:   # one frame: the offline cone schedule (module docstring)
            continue
        ref = _offline(m, x, augment)
        assert torch.equal(torch.stack([rows[f] for f in got]), ref[:len(got)]), key
        checked += 1
    assert checked > 0


@pytest.mark.parametrize("precision", ["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("K", [1, 5, 13])
def test_end_on_a_live_session(cuda_device, precision, causal, K):
    m = _model(cuda_device, [3, 3, 3], 64, causal, precision, seed=K)
    rng = np.random.RandomState(K + 7 * causal)
    S = 6
    seqs = {s: [int(v) for v in rng.randint(2, 45, 3)] for s in range(S)}
    _check_live(m, _live_session(m, S, K, seqs, seed=K))


def test_end_on_a_live_session_arc_3_pow_5(cuda_device):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, False, "fp16", seed=81)
    seqs = {0: [150, 2], 1: [40, 130], 2: [300], 3: [7, 90, 20]}
    _check_live(m, _live_session(m, 4, 16, seqs, seed=82))


@pytest.mark.parametrize("causal", [False, True])
def test_start_during_a_drain_drops_the_tail(cuda_device, causal):
    """Restarts while the previous sequence still drains: the dropped tail never comes back, the
    delivered prefix and the next sequence are exact."""
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=83)
    seqs = {s: [20, 9, 31, 14, 25] for s in range(5)}
    out = _live_session(m, 5, 3, seqs, seed=84, drain_starts=True)
    if not causal:
        assert any(d for _, _, d in out.values())
    _check_live(m, out)


@pytest.mark.parametrize("causal", [False, True])
def test_end_with_augment_and_finish(cuda_device, causal):
    m = _model(cuda_device, [3, 3, 3], 64, causal, "bf16x3", seed=85)
    seqs = {s: [12, 30, 7] for s in range(5)}
    _check_live(m, _live_session(m, 5, 4, seqs, seed=86, augment=True), augment=True)
    # finish() while some slots have ended and drain, others are open, some idle
    out = _live_session(m, 5, 4, seqs, seed=87, augment=True, finish_at=14)
    _check_live(m, out, augment=True, complete=False)


def test_finish_returns_an_ended_slot_s_tail(cuda_device):
    """Slot 1 ends at frame 16 in the second push; finish() returns the rest of its tail and -1
    after it, and slot 0's tail as before."""
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=88)
    la = vp.streaming.lookahead(m)
    x = orc.make_input(2, 20, 17, 2, seed=89).to(cuda_device)
    sess = m.streaming(streams=2, max_frames=10)
    outs = [sess.push(x[:, :10], start=[True, True]), sess.push(x[:, 10:], end=[-1, 6])]
    y, frame = sess.finish()
    idx = np.arange(20 - la, 20)
    assert frame[0].tolist() == np.where(idx >= 0, idx, -1).tolist()
    assert frame[1].tolist() == np.where((idx >= 0) & (idx < 16), idx, -1).tolist()
    for s, T in ((0, 20), (1, 16)):
        rows = {}
        for yy, fr in outs + [(y, frame)]:
            for f, t in enumerate(fr[s].tolist()):
                if t >= 0:
                    assert t not in rows
                    rows[t] = yy[s, f]
        assert sorted(rows) == list(range(T))
        assert torch.equal(torch.stack([rows[t] for t in range(T)]), _offline(m, x[s, :T]))


def _seq_set(dev, n, J, F, seed, shortest=1):
    rng = np.random.RandomState(seed)
    lengths = [1, 2, 3] + [int(v) for v in rng.randint(shortest, 300, n - 3)]
    return [orc.make_input(1, T, J, F, seed=seed * 100 + i)[0].to(dev) for i, T in enumerate(lengths)]


def _check_predict(m, seqs, ys, augment):
    assert len(ys) == len(seqs)
    for x, y in zip(seqs, ys):
        assert tuple(y.shape) == (len(x), m.num_joints_out, 3)
        if len(x) >= 2:
            assert torch.equal(y, _offline(m, x, augment)), len(x)
        else:   # the offline cone schedule sums in another order: a session of its own
            alone = m.streaming(streams=1, max_frames=1, augment=augment, **_lists(m, augment))
            assert torch.equal(y, alone.predict([x])[0])
            assert float((y - _offline(m, x, augment)).abs().max()) <= 1e-3 * float(y.abs().max())


@pytest.mark.parametrize("causal", [False, True])
def test_predict_is_exact_and_schedule_independent(cuda_device, causal):
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=91)
    seqs = _seq_set(cuda_device, 40, 17, 2, seed=92)
    first = None
    for S, K in ((1, 1), (3, 4), (8, 16), (64, 8)):
        sess = m.streaming(streams=S, max_frames=K)
        ys = sess.predict(seqs)
        if first is None:
            first = ys
            _check_predict(m, seqs, ys, False)
        else:
            for a, b in zip(first, ys):
                assert torch.equal(a, b), (S, K)
        assert not sess.predict([])   # empty list, session idle and usable


@pytest.mark.parametrize("S,K", [(3, 4), (8, 16), (50, 3)])
def test_predict_with_augment(cuda_device, S, K):
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=93)
    seqs = _seq_set(cuda_device, 40, 17, 2, seed=94)
    sess = m.streaming(streams=S, max_frames=K, augment=True, **H36M)
    _check_predict(m, seqs, sess.predict(seqs), True)


@pytest.mark.parametrize("dense,jout,F,augment", [(True, 17, 2, False), (False, 1, 2, True),
                                                  (False, 1, 2, False), (False, 17, 3, False)])
def test_predict_dense_trajectory_and_3d_inputs(cuda_device, dense, jout, F, augment):
    fw = [3, 3] if dense else [3, 5, 3]
    m = _model(cuda_device, fw, 128, False, "bf16", dense=dense, jout=jout, F=F, seed=95)
    seqs = _seq_set(cuda_device, 20, 17, F, seed=96)
    sess = m.streaming(streams=3, max_frames=4, augment=augment, **_lists(m, augment))
    _check_predict(m, seqs, sess.predict(seqs), augment)


def test_predict_arc_3_pow_5(cuda_device):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, False, "fp16", seed=97)
    seqs = _seq_set(cuda_device, 12, 17, 2, seed=98)
    sess = m.streaming(streams=5, max_frames=16, augment=True, **H36M)
    _check_predict(m, seqs, sess.predict(seqs), True)


def _golden_names():
    return sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))


@pytest.mark.parametrize("precision,tol", [("fp16", 1e-3), ("bf16x3", 1e-3), ("bf16", 3e-2)])
@pytest.mark.parametrize("name", _golden_names())
def test_against_reference_goldens(cuda_device, name, precision, tol):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    m = _model(cuda_device, meta["fw"], meta["C"], meta["causal"], precision, dense=meta["dense"],
               jout=meta["Jout"], F=meta["F"], seed=meta["seed"])
    x = torch.from_numpy(z["x"]).to(cuda_device)
    seqs = list(torch.split(x, meta["lengths"]))
    sess = m.streaming(streams=2, max_frames=3, augment=meta["augment"],
                       **_lists(m, meta["augment"]))
    got = torch.cat(sess.predict(seqs)).cpu().numpy()
    y = z["y"].astype(np.float64)
    assert got.shape == y.shape
    off = np.concatenate([[0], np.cumsum(meta["lengths"])])
    for i in range(len(meta["lengths"])):
        a, b = off[i], off[i + 1]
        assert float(np.abs(got[a:b] - y[a:b]).max() / np.abs(y[a:b]).max()) <= tol, i


@pytest.mark.parametrize("S,k", [(1, 1), (3, 1), (1, 4), (3, 4)])
@pytest.mark.parametrize("augment", [False, True])
def test_nothing_changed_for_existing_callers(cuda_device, S, k, augment):
    """push(end=None) is vp3d_stream_push: same bits, same launches; `end` adds no launch; y_rows
    adds the output kernel only where a push would shrink straight into y."""
    lib = _capi.load()
    m = _model(cuda_device, [3, 3, 3, 3, 3], 64, False, "fp16", seed=99)
    kw = _lists(m, augment)
    a = m.streaming(streams=S, max_frames=k, augment=augment, **kw)
    b = m.streaming(streams=S, max_frames=k, augment=augment, **kw)
    c = m.streaming(streams=S, max_frames=k, augment=augment, **kw)
    direct = not augment and (k == 1 or S == 1)
    stream = torch.cuda.current_stream().cuda_stream
    rows = torch.arange(S, dtype=torch.int64, device=cuda_device) * 1000
    flat = torch.full((S * 1000, 17, 3), float("nan"), device=cuda_device)
    for i in range(4):
        x = orc.make_input(S, k, 17, 2, seed=100 + i).to(cuda_device)
        st = [True] * S if i == 0 else None
        ya, fa = a.push(x, start=st)
        n_a = a.last_launch_count()
        yb = torch.empty_like(ya)
        fb = torch.empty_like(fa)
        mask = torch.ones(S, dtype=torch.uint8, device=cuda_device) if i == 0 else None
        b._prepare()
        _capi.check(lib.vp3d_stream_push(b._plan, b._state.data_ptr(), x.data_ptr(), k,
                                         None if mask is None else mask.data_ptr(), yb.data_ptr(),
                                         fb.data_ptr(), stream), "vp3d_stream_push")
        assert lib.vp3d_last_launch_count(b._plan) == n_a
        assert torch.equal(ya, yb) and torch.equal(fa, fb)
        # the same push through row-addressed x and y, with an end past this test's pushes
        fc = torch.empty_like(fa)
        end = torch.full((S,), k if i == 3 else -1, dtype=torch.int32, device=cuda_device)
        c._prepare()
        _capi.check(lib.vp3d_stream_push_ex(
            c._plan, c._state.data_ptr(), x.reshape(S * k, 17, 2).data_ptr(), k,
            None if mask is None else mask.data_ptr(), end.data_ptr(), (rows // 1000 * k).data_ptr(),
            rows.data_ptr(), flat.data_ptr(), fc.data_ptr(), stream), "vp3d_stream_push_ex")
        assert lib.vp3d_last_launch_count(c._plan) == n_a + direct
        assert torch.equal(fc, fa)
        for s in range(S):
            for f in range(k):
                if fa[s, f] >= 0:
                    assert torch.equal(flat[1000 * s + int(fa[s, f])], ya[s, f])
        # `end` adds no launch
        a.push(x, end=[-1] * S)
        n_none = a.last_launch_count()
        a.push(x, end=torch.full((S,), -1, dtype=torch.int32, device=cuda_device))
        assert a.last_launch_count() == n_none
        b._prepare()
        _capi.check(lib.vp3d_stream_push(b._plan, b._state.data_ptr(), x.data_ptr(), k, None,
                                         yb.data_ptr(), fb.data_ptr(), stream), "vp3d_stream_push")
        b._prepare()
        _capi.check(lib.vp3d_stream_push(b._plan, b._state.data_ptr(), x.data_ptr(), k, None,
                                         yb.data_ptr(), fb.data_ptr(), stream), "vp3d_stream_push")
        assert lib.vp3d_last_launch_count(b._plan) == n_none
        c.push(x)
        c.push(x)


def test_push_ex_needs_a_known_session_and_k_in_range(cuda_device):
    lib = _capi.load()
    m = _model(cuda_device, [3, 3], 64, False, "fp16", seed=101)
    sess = m.streaming(streams=2, max_frames=2)
    x = torch.zeros(2, 3, 17, 2, device=cuda_device)
    y = torch.empty(2, 3, 17, 3, device=cuda_device)
    fr = torch.empty(2, 3, dtype=torch.int64, device=cuda_device)
    args = (x.data_ptr(), 3, None, None, None, None, y.data_ptr(), fr.data_ptr(), None)
    assert lib.vp3d_stream_push_ex(sess._plan, sess._state.data_ptr(), *args) == -1
    assert b"exceeds max_frames" in lib.vp3d_last_error()
    assert lib.vp3d_stream_push_ex(sess._plan, fr.data_ptr(), *args) == -5
    assert b"not initialised" in lib.vp3d_last_error()
    with pytest.raises(ValueError, match="outside"):
        sess.push(x[:, :2], end=[3, -1])
    with pytest.raises(TypeError, match="int32"):
        sess.push(x[:, :2], end=torch.zeros(2, dtype=torch.int64, device=cuda_device))


def test_predict_makes_no_synchronisation(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=103)
    seqs = _seq_set(cuda_device, 10, 17, 2, seed=104)
    sess = m.streaming(streams=3, max_frames=4, augment=True, **H36M)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ys = sess.predict(seqs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _check_predict(m, seqs, ys, True)


def test_weight_changes_between_predicts_are_picked_up(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, True, "fp16", seed=105)
    seqs = _seq_set(cuda_device, 8, 17, 2, seed=106, shortest=2)[3:]
    sess = m.streaming(streams=2, max_frames=4)
    before = sess.predict(seqs)
    with torch.no_grad():
        m.shrink.bias.add_(0.5)
    after = sess.predict(seqs)
    for x, a, b in zip(seqs, before, after):
        assert not torch.equal(a, b)
        assert torch.equal(b, _offline(m, x))
