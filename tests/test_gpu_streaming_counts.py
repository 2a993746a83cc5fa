"""GPU: per-slot frame counts (push's `count`): streams that skip or drop frames share one session.

Slot s takes the first count[s] frames of x[s] in a push, anywhere from 0 to k, in the same launches
as the other slots.  Every sequence that goes through a slot must still come out as the offline
forward on the sequence edge-padded as UnchunkedGenerator pads it,
``model(np.pad(x, (pad + shift, pad - shift), 'edge'))``, or ``metrics.flip_average(model(b))[0]``
with test-time augmentation, bit for bit, whatever the counts.  Frames past a slot's count are NaN
in x, so a read of one would show in every later output of that slot.
"""
import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi, metrics
from videopose3d_b200.generators import UnchunkedGenerator
from videopose3d_b200.streaming import FrameBook

pytestmark = pytest.mark.gpu

LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
H36M = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
TRAJ = dict(kps_left=LEFT, kps_right=RIGHT)


def _model(dev, fw, C, causal, precision, jout=17, F=2, seed=0):
    m = vp.TemporalModel(17, F, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C)
    m.load_state_dict(orc.make_state_dict(17, F, jout, fw, C, seed=seed))
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


def _collect(rows, want, y, key_of):
    """Store y[s, f] under frame want[s, f] of the sequence key_of(s); each frame once."""
    for s, f in zip(*np.nonzero(want >= 0)):
        got = rows[key_of(s)]
        assert int(want[s, f]) not in got, "frame returned twice"
        got[int(want[s, f])] = y[s, f]


def _counted_session(m, S, K, seqs_per_slot, seed, augment=False, row_addressed=False,
                     skip_runs=False):
    """Drive a session push by push with random per-slot counts: every slot runs its own list of
    sequences, started after a random idle gap, fed count[s] in [0, k] of its frames per push (k
    random in [1, K]), and ended with `end` once its remaining frames fit the push.  Counts go as a
    host list or as a device tensor (then some full slots carry an out-of-range value, read as k).
    skip_runs: slots also skip 3-12 pushes in a row (count 0).  row_addressed: frames are read from
    one flat store through x_rows and outputs written through y_rows.  Returns [(x, {frame: y})]."""
    rng = np.random.RandomState(seed)
    la = vp.streaming.lookahead(m)
    dev = m.expand_conv.weight.device
    J, F = m.num_joints_in, m.in_features
    sess = m.streaming(streams=S, max_frames=K, augment=augment, **_lists(m, augment))
    book = FrameBook(S, la)
    seqs = []
    queue = {}
    for s in range(S):
        queue[s] = []
        for j, T in enumerate(seqs_per_slot[s]):
            queue[s].append(len(seqs))
            seqs.append(orc.make_input(1, int(T), J, F, seed=seed * 1000 + s * 10 + j)[0].to(dev))
    offset = np.concatenate([[0], np.cumsum([len(x) for x in seqs])]).astype(np.int64)
    if row_addressed:
        store = torch.cat(seqs)
        flat = torch.full((int(offset[-1]), m.num_joints_out, 3), float("nan"), device=dev)
        lib = _capi.load()
    rows = {i: {} for i in range(len(seqs))}
    cur = [-1] * S            # position in queue[s] of the sequence slot s holds
    fed = [0] * S
    skip = [0] * S
    n_push = 0
    while any(book.active) or any(cur[s] + 1 < len(queue[s]) for s in range(S)):
        k = int(rng.randint(1, K + 1))
        start = [False] * S
        end = [-1] * S
        count = [int(v) for v in rng.randint(0, k + 1, S)]   # idle / draining slots ignore it
        x = torch.rand(S, k, J, F, device=dev) * 2 - 1
        x_rows = np.zeros(S, np.int64)
        y_rows = np.zeros(S, np.int64)
        for s in range(S):
            if cur[s] + 1 < len(queue[s]) and not book.active[s] and rng.rand() < 0.5:
                cur[s] += 1
                fed[s] = 0
                start[s] = True
                count[s] = max(count[s], 1)   # a host list may not start a slot with count 0
            if cur[s] < 0 or not (book.active[s] or start[s]):
                continue
            i = queue[s][cur[s]]
            seq = seqs[i]
            y_rows[s] = offset[i]
            rest = len(seq) - fed[s]
            if rest <= 0:   # draining: x is not read
                x[s] = float("nan")
                continue
            x_rows[s] = offset[i] + fed[s]
            if skip_runs and skip[s] == 0 and not start[s] and rng.rand() < 0.1:
                skip[s] = int(rng.randint(3, 13))
            if skip[s] > 0:
                skip[s] -= 1
                n = 0
            else:
                n = int(rng.randint(1 if start[s] else 0, k + 1))
            if rest <= n:
                n = end[s] = rest
            else:
                count[s] = n
            x[s, :n] = seq[fed[s]:fed[s] + n]
            x[s, n:] = float("nan")
            fed[s] += n
        if rng.rand() < 0.5:
            arg = count
        else:   # a device tensor: k may also be sent as an out-of-range value
            dev_count = [c if c < k or rng.rand() < 0.5 else int(rng.choice([-7, k + 1, 1 << 30]))
                         for c in count]
            arg = torch.tensor(dev_count, dtype=torch.int32, device=dev)
        want = book.push(k, start, end, count)
        if row_addressed:
            mask = torch.tensor(start, dtype=torch.uint8, device=dev)
            e = torch.tensor(end, dtype=torch.int32, device=dev)
            c = arg if isinstance(arg, torch.Tensor) else torch.tensor(arg, dtype=torch.int32,
                                                                       device=dev)
            xr = torch.from_numpy(x_rows).to(dev)
            yr = torch.from_numpy(y_rows).to(dev)
            frame = torch.empty((S, k), dtype=torch.int64, device=dev)
            stream = sess._prepare()
            _capi.check(lib.vp3d_stream_push_counts(
                sess._plan, sess._state.data_ptr(), store.data_ptr(), k, mask.data_ptr(),
                e.data_ptr(), xr.data_ptr(), yr.data_ptr(), flat.data_ptr(), frame.data_ptr(),
                c.data_ptr(), stream), "vp3d_stream_push_counts")
        else:
            y, frame = sess.push(x, start=start, end=end, count=arg)
            _collect(rows, want, y, lambda s: queue[s][cur[s]])
        assert np.array_equal(frame.cpu().numpy(), want), n_push
        if row_addressed:
            for s, f in zip(*np.nonzero(want >= 0)):
                rows[queue[s][cur[s]]][int(want[s, f])] = None
        n_push += 1
    out = []
    for i, x in enumerate(seqs):
        assert sorted(rows[i]) == list(range(len(x))), i   # every frame once
        if row_addressed:
            out.append((x, flat[int(offset[i]):int(offset[i + 1])]))
        else:
            out.append((x, torch.stack([rows[i][t] for t in range(len(x))])))
    return out


def _check(m, out, augment=False):
    for j, (x, y) in enumerate(out):
        assert torch.equal(y, _offline(m, x, augment)), (j, len(x))


def _lengths(rng, S, n, lo=2, hi=45):
    return {s: [int(v) for v in rng.randint(lo, hi, n)] for s in range(S)}


@pytest.mark.parametrize("precision", ["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("C,K", [(64, 5), (100, 13)])
def test_counts_on_a_live_session(cuda_device, precision, causal, C, K):
    m = _model(cuda_device, [3, 3, 3], C, causal, precision, seed=C + K)
    rng = np.random.RandomState(C + 7 * causal)
    S = 6
    _check(m, _counted_session(m, S, K, _lengths(rng, S, 3), seed=K + causal))


@pytest.mark.parametrize("precision,causal", [("fp16", False), ("bf16x3", True)])
def test_counts_arc_3_pow_5(cuda_device, precision, causal):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, causal, precision, seed=111)
    seqs = {0: [150, 2], 1: [40, 130], 2: [300], 3: [7, 90, 20]}
    _check(m, _counted_session(m, 4, 16, seqs, seed=112 + causal))


@pytest.mark.parametrize("jout,F", [(17, 2), (1, 2), (17, 3)])
def test_counts_with_augment(cuda_device, jout, F):
    m = _model(cuda_device, [3, 3, 3], 64, False, "bf16x3", jout=jout, F=F, seed=113 + jout + F)
    rng = np.random.RandomState(114)
    _check(m, _counted_session(m, 5, 6, _lengths(rng, 5, 3), seed=115 + F, augment=True),
           augment=True)


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("causal", [False, True])
def test_counts_row_addressed_with_skip_runs(cuda_device, augment, causal):
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=116)
    rng = np.random.RandomState(117 + augment)
    out = _counted_session(m, 5, 4, _lengths(rng, 5, 2, hi=60), seed=118 + 2 * augment + causal,
                           augment=augment, row_addressed=True, skip_runs=True)
    _check(m, out, augment)


def test_counts_over_more_rows_than_one_realign_tile(cuda_device):
    """700 augmented slots are 1400 physical rows, more than the 1024 the realign lists at a time:
    every slot runs one sequence under random counts (some whole pushes at 0), checked against the
    frame bookkeeping, and a spread of slots bit for bit against the offline flip average."""
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=125)
    S, K, T = 700, 3, 40
    la = vp.streaming.lookahead(m)
    rng = np.random.RandomState(126)
    seqs = orc.make_input(S, T, 17, 2, seed=127).to(cuda_device)
    sess = m.streaming(streams=S, max_frames=K, augment=True, **H36M)
    book = FrameBook(S, la)
    watch = [0, 1, 300, 323, 324, 511, 512, 699]
    rows = {s: {} for s in watch}
    fed = np.zeros(S, np.int64)
    slot = torch.arange(S, device=cuda_device)[:, None]
    i = 0
    while book.active.any() or i == 0:
        k = int(rng.randint(1, K + 1))
        n = rng.randint(1 if i == 0 else 0, k + 1, S)
        if i % 5 == 4:
            n[rng.rand(S) < 0.5] = 0
        n = np.minimum(n, T - fed)
        ends = (fed < T) & (fed + n >= T) & (n > 0)
        end = np.where(ends, n, -1).astype(np.int32)
        idx = torch.from_numpy(np.minimum(fed[:, None] + np.arange(k), T - 1)).to(cuda_device)
        x = seqs[slot, idx]
        x[torch.from_numpy(np.arange(k)[None, :] >= n[:, None]).to(cuda_device)] = float("nan")
        start = [True] * S if i == 0 else None
        y, frame = sess.push(x, start=start, end=end.tolist(),
                             count=torch.from_numpy(n.astype(np.int32)).to(cuda_device))
        want = book.push(k, start, end, n)
        assert np.array_equal(frame.cpu().numpy(), want), i
        _collect(rows, np.where(np.isin(np.arange(S), watch)[:, None], want, -1), y, lambda s: s)
        fed += n
        i += 1
    for s in watch:
        assert sorted(rows[s]) == list(range(T)), s
        assert torch.equal(torch.stack([rows[s][t] for t in range(T)]),
                           _offline(m, seqs[s], augment=True)), s


@pytest.mark.parametrize("causal", [False, True])
def test_a_push_where_every_slot_has_count_zero(cuda_device, causal):
    """No frame comes out of such a push, and the outputs after it are still exact."""
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=119)
    S, K, T = 3, 4, 30
    la = vp.streaming.lookahead(m)
    x = orc.make_input(S, T, 17, 2, seed=120).to(cuda_device)
    sess = m.streaming(streams=S, max_frames=K)
    book = FrameBook(S, la)
    rows = {s: {} for s in range(S)}
    # (k, count of every slot); the push that reaches frame T ends every sequence instead
    schedule = [(K, K), (2, 2), (K, 0), (1, 0), (K, 0)] + [(K, K)] * (T // K + 1)
    fed = 0
    for i, (k, n) in enumerate(schedule):
        n = min(n, T - fed)
        last = fed + n == T
        count, end = [n] * S, ([n] * S if last else None)
        start = [True] * S if i == 0 else None
        xk = torch.full((S, k, 17, 2), float("nan"), device=cuda_device)
        xk[:, :n] = x[:, fed:fed + n]
        y, frame = sess.push(xk, start=start, end=end, count=count)
        want = book.push(k, start, end, count)
        assert np.array_equal(frame.cpu().numpy(), want), i
        if n == 0:
            assert (want < 0).all()
        _collect(rows, want, y, lambda s: s)
        fed += n
        if last:
            break
    y, frame = sess.finish()
    want = book.finish()
    assert np.array_equal(frame.cpu().numpy(), want)
    _collect(rows, want, y, lambda s: s)
    for s in range(S):
        assert sorted(rows[s]) == list(range(T))
        assert torch.equal(torch.stack([rows[s][t] for t in range(T)]), _offline(m, x[s]))


def test_a_slot_fed_in_bursts_equals_one_frame_per_push(cuda_device):
    """Slot 0 gets its frames in bursts (3, 0, 0, 2, ...) next to slot 1, fed k every push; a
    second session gets slot 0's frames one per push.  Same bits, frame for frame, and slot 1 is
    untouched by its neighbour's bursts."""
    m = _model(cuda_device, [3, 3, 3], 100, False, "fp16", seed=121)
    la = vp.streaming.lookahead(m)
    K = 5
    bursts = [3, 0, 0, 2, 5, 0, 1, 4, 0, 0, 0, 5, 2, 0, 3, 1, 5, 5, 0, 4]
    T, T1 = sum(bursts), K * len(bursts)
    x = orc.make_input(2, T1, 17, 2, seed=122).to(cuda_device)
    a = m.streaming(streams=2, max_frames=K)
    b = m.streaming(streams=1, max_frames=1)
    got = {0: {}, 1: {}}
    ref = {0: {}}
    fed = 0
    for i, n in enumerate(bursts):
        xk = x[:, i * K:(i + 1) * K].clone()
        xk[0, :n] = x[0, fed:fed + n]
        xk[0, n:] = float("nan")
        y, frame = a.push(xk, start=[True, True] if i == 0 else None, count=[n, K])
        _collect(got, frame.cpu().numpy(), y, lambda s: s)
        fed += n
    for t in range(T):
        y, frame = b.push(x[:1, t:t + 1], start=[True] if t == 0 else None)
        _collect(ref, frame.cpu().numpy(), y, lambda s: s)
    assert sorted(got[0]) == sorted(ref[0]) == list(range(T - la))
    for t in range(T - la):
        assert torch.equal(got[0][t], ref[0][t]), t
    assert torch.equal(torch.stack([got[0][t] for t in range(T - la)]),
                       _offline(m, x[0, :T])[:T - la])
    assert sorted(got[1]) == list(range(T1 - la))
    assert torch.equal(torch.stack([got[1][t] for t in range(T1 - la)]),
                       _offline(m, x[1])[:T1 - la])


@pytest.mark.parametrize("S,k", [(1, 1), (3, 1), (1, 4), (3, 4)])
@pytest.mark.parametrize("augment", [False, True])
def test_count_none_and_all_k_are_the_plain_push(cuda_device, S, k, augment):
    """count=None and a host list of all k: push_ex's bits and launches; a device tensor of all k:
    the same bits, two realign launches more."""
    lib = _capi.load()
    m = _model(cuda_device, [3, 3, 3, 3, 3], 64, False, "fp16", seed=123)
    kw = _lists(m, augment)
    sessions = [m.streaming(streams=S, max_frames=k, augment=augment, **kw) for _ in range(4)]
    stream = torch.cuda.current_stream().cuda_stream
    for i in range(5):
        x = orc.make_input(S, k, 17, 2, seed=124 + i).to(cuda_device)
        st = [True] * S if i == 0 else None
        end = [k] * S if i == 4 else None
        base = sessions[0]
        yb = torch.empty((S, k, 17, 3), device=cuda_device)
        fb = torch.empty((S, k), dtype=torch.int64, device=cuda_device)
        mask = torch.ones(S, dtype=torch.uint8, device=cuda_device) if i == 0 else None
        e = None if end is None else torch.tensor(end, dtype=torch.int32, device=cuda_device)
        stream = base._prepare()
        _capi.check(lib.vp3d_stream_push_ex(
            base._plan, base._state.data_ptr(), x.data_ptr(), k,
            None if mask is None else mask.data_ptr(), None if e is None else e.data_ptr(),
            None, None, yb.data_ptr(), fb.data_ptr(), stream), "vp3d_stream_push_ex")
        n_ex = lib.vp3d_last_launch_count(base._plan)
        for j, count in enumerate([None, [k] * S,
                                   torch.full((S,), k, dtype=torch.int32, device=cuda_device)]):
            sess = sessions[j + 1]
            y, frame = sess.push(x, start=st, end=end, count=count)
            assert torch.equal(y, yb) and torch.equal(frame, fb), (i, j)
            assert sess.last_launch_count() == n_ex + (2 if j == 2 else 0), (i, j)
