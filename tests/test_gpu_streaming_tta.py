"""GPU: augmented streaming sessions (test-time flip augmentation) against run.py's evaluate().

Per slot, the concatenated session output must equal ``metrics.flip_average(model(b), jl, jr)[0]``
bit for bit, ``b`` the (2, T + 2 pad, J, F) batch of the device UnchunkedGenerator with
augment=True: every physical row of the session is the offline forward of its own padded sequence
(the offline dilated forward never mixes samples) and the output kernel averages with the same
expression as the metrics kernel.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi, metrics
from videopose3d_b200.generators import UnchunkedGenerator, mirror_source
from videopose3d_b200.streaming import FrameBook

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_tta")
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
H36M = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)


def _model(dev, fw, C, causal, precision, dense=False, jout=17, F=2, seed=0, jin=17):
    m = vp.TemporalModel(jin, F, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(jin, F, jout, fw, C, dense=dense, seed=seed))
    return m.to(dev).eval().set_precision(precision)


def _generator(m, x, lists):
    pad = (m.receptive_field() - 1) // 2
    shift = pad if m._causal else 0          # run.py:186-193
    return UnchunkedGenerator(None, None, [x.cpu().numpy()], pad=pad, causal_shift=shift,
                              augment=True, kps_left=lists["kps_left"],
                              kps_right=lists["kps_right"], device=x.device)


def _offline_tta(m, x, lists):
    """run.py's evaluate(return_predictions=True) with TTA for one (T, J, F) sequence."""
    with torch.no_grad():
        for _, _, b in _generator(m, x, lists).next_epoch():
            return metrics.flip_average(m(b), lists.get("joints_left"),
                                        lists.get("joints_right"))[0]


def _collect(outs, S):
    """{slot: {frame: y row}} from a list of (y, frame) pairs."""
    got = {s: {} for s in range(S)}
    for y, frame in outs:
        fr = frame.cpu().numpy()
        for s, f in zip(*np.nonzero(fr >= 0)):
            assert int(fr[s, f]) not in got[s], "frame returned twice"
            got[s][int(fr[s, f])] = y[s, f]
    return got


def _stream_all(m, xs, chunks, max_frames, lists):
    """Every slot starts at the first push; the sequences are pushed in `chunks`, then finished."""
    S, T = xs.shape[0], xs.shape[1]
    sess = m.streaming(streams=S, max_frames=max_frames, augment=True, **lists)
    assert sess.augment
    outs, t = [], 0
    for k in chunks:
        outs.append(sess.push(xs[:, t:t + k], start=[True] * S if t == 0 else None))
        t += k
    assert t == T
    outs.append(sess.finish())
    got = _collect(outs, S)
    return [torch.stack([got[s][f] for f in range(T)]) for s in range(S)]


def _chunkings(T, rf, seed):
    rng = np.random.RandomState(seed)
    mix, t = [], 0
    while t < T:
        k = int(min(T - t, rng.randint(1, 12)))
        mix.append(k)
        t += k
    big = min(T, rf + 5)
    return {"k1": ([1] * T, 1), "k7": ([7] * (T // 7) + ([T % 7] if T % 7 else []), 7),
            "rf+5": ([big] * (T // big) + ([T % big] if T % big else []), big),
            "random": (mix, 12)}


CASES = [([3, 3, 3], 64), ([3, 3, 3], 100), ([3, 3, 3, 3, 3], 1024)]


@pytest.mark.parametrize("precision", ["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("fw,C", CASES)
def test_session_equals_offline_tta_bitwise(cuda_device, precision, causal, fw, C):
    m = _model(cuda_device, fw, C, causal, precision, seed=C)
    T = 40 if len(fw) == 3 else 30
    xs = orc.make_input(2, T, 17, 2, seed=C + 1).to(cuda_device)
    ref = [_offline_tta(m, xs[s], H36M) for s in range(2)]
    names = ["k1", "k7", "rf+5", "random"] if len(fw) == 3 else ["k1", "random", "rf+5"]
    for name in names:
        chunks, K = _chunkings(T, m.receptive_field(), seed=C)[name]
        got = _stream_all(m, xs, chunks, K, H36M)
        for s in range(2):
            assert torch.equal(got[s], ref[s]), (name, s, float((got[s] - ref[s]).abs().max()))


def test_offline_reference_is_metrics_evaluate(cuda_device):
    """The offline result the tests compare against is metrics.evaluate(return_predictions=True)."""
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=5)
    x = orc.make_input(1, 40, 17, 2, seed=6)[0].to(cuda_device)
    want = metrics.evaluate(m, _generator(m, x, H36M), LEFT, RIGHT, return_predictions=True)
    assert torch.equal(_offline_tta(m, x, H36M), want)


@pytest.mark.parametrize("dense,jout,F", [(True, 17, 2), (False, 1, 2), (False, 17, 3)])
def test_dense_trajectory_and_3d_inputs(cuda_device, dense, jout, F):
    fw = [3, 3] if dense else [3, 5, 3]
    m = _model(cuda_device, fw, 128, jout == 1, "fp16", dense=dense, jout=jout, F=F, seed=7)
    lists = dict(kps_left=LEFT, kps_right=RIGHT) if jout == 1 else H36M   # trajectory: negate x only
    xs = orc.make_input(3, 33, 17, F, seed=8).to(cuda_device)
    for name in ("k1", "random"):
        chunks, K = _chunkings(33, m.receptive_field(), seed=9)[name]
        got = _stream_all(m, xs, chunks, K, lists)
        for s in range(3):
            assert torch.equal(got[s], _offline_tta(m, xs[s], lists)), (name, s)


@pytest.mark.parametrize("causal", [False, True])
def test_input_map_differs_from_output_map(cuda_device, causal):
    """15 input joints with their own lists, 17 output joints with H36M's: a mix-up of kps_src and
    joints_src cannot pass."""
    lists = dict(kps_left=[1, 2, 3, 9], kps_right=[4, 5, 6, 12], joints_left=LEFT,
                 joints_right=RIGHT)
    assert not np.array_equal(mirror_source(15, lists["kps_left"], lists["kps_right"]),
                              mirror_source(17, LEFT, RIGHT)[:15])
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", jin=15, seed=15)
    xs = orc.make_input(2, 30, 15, 2, seed=16).to(cuda_device)
    chunks, K = _chunkings(30, m.receptive_field(), seed=17)["random"]
    got = _stream_all(m, xs, chunks, K, lists)
    for s in range(2):
        assert torch.equal(got[s], _offline_tta(m, xs[s], lists)), s
    # the lists matter: swapping the input map for the plain one changes the answer
    plain = _offline_tta(m, xs[0], dict(lists, kps_left=[0], kps_right=[0]))
    assert not torch.equal(got[0], plain)


def _golden_names():
    return sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))


@pytest.mark.parametrize("precision,tol", [("fp16", 1e-3), ("bf16x3", 1e-3), ("bf16", 3e-2)])
@pytest.mark.parametrize("name", _golden_names())
def test_against_reference_goldens(cuda_device, name, precision, tol):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    m = _model(cuda_device, meta["fw"], meta["C"], meta["causal"], precision, dense=meta["dense"],
               jout=meta["Jout"], F=meta["F"], seed=meta["seed"])
    lists = dict(kps_left=LEFT, kps_right=RIGHT) if meta["Jout"] == 1 else H36M
    x = torch.from_numpy(z["x"]).to(cuda_device)
    chunks, K = _chunkings(meta["T"], m.receptive_field(), seed=3)["random"]
    got = _stream_all(m, x[None], chunks, K, lists)[0].cpu().numpy()
    y = z["y"].astype(np.float64)
    assert got.shape == y.shape
    assert float(np.abs(got - y).max() / np.abs(y).max()) <= tol


@pytest.mark.parametrize("causal", [False, True])
def test_slots_start_mid_stream(cuda_device, causal):
    """Slots begin (and one restarts) at different pushes under augment; every sequence equals its
    own offline TTA result and `frame` follows the logical bookkeeping."""
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=11)
    la = vp.streaming.lookahead(m)
    S, K, n_push = 3, 4, 16
    rng = np.random.RandomState(12)
    ks = [int(rng.randint(1, K + 1)) for _ in range(n_push)]
    starts = {0: [0], 1: [2], 2: [5, 9]}          # slot -> pushes that start a sequence there
    total = sum(ks)
    xs = orc.make_input(S, total, 17, 2, seed=13).to(cuda_device)
    sess = m.streaming(streams=S, max_frames=K, augment=True, **H36M)
    book = FrameBook(S, la)
    outs, t = [], 0
    seq_begin = {s: [] for s in range(S)}
    for i, k in enumerate(ks):
        mask = [i in starts[s] for s in range(S)]
        for s in range(S):
            if mask[s]:
                seq_begin[s].append(t)
        dev_mask = torch.tensor(mask, device=cuda_device) if i % 2 else mask
        y, frame = sess.push(xs[:, t:t + k], start=dev_mask)
        assert tuple(y.shape) == (S, k, 17, 3)
        assert np.array_equal(frame.cpu().numpy(), book.push(k, mask))
        outs.append((y, frame, t))
        t += k
    y, frame = sess.finish()
    assert np.array_equal(frame.cpu().numpy(), book.finish())
    outs.append((y, frame, t))
    for s in range(S):
        bounds = seq_begin[s] + [total]
        for j in range(len(seq_begin[s])):
            a, b = bounds[j], bounds[j + 1]
            finished = j == len(seq_begin[s]) - 1
            rows = {}
            for yy, fr, t0 in outs:
                fr = fr.cpu().numpy()
                for f in range(fr.shape[1]):
                    g = t0 + f
                    if fr[s, f] >= 0 and (a <= g < b + (la if finished else 0)):
                        rows[int(fr[s, f])] = yy[s, f]
            n_out = (b - a) if finished else (b - a - la)
            assert sorted(rows) == list(range(max(n_out, 0)))
            if n_out <= 0:
                continue
            ref = _offline_tta(m, xs[s, a:b], H36M)[:n_out]
            assert torch.equal(torch.stack([rows[f] for f in range(n_out)]), ref), (s, j)


def test_finish_of_a_non_causal_model(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, False, "bf16x3", seed=19)
    la = vp.streaming.lookahead(m)
    xs = orc.make_input(2, 20, 17, 2, seed=20).to(cuda_device)
    sess = m.streaming(streams=2, max_frames=5, augment=True, **H36M)
    outs = [sess.push(xs[:, t:t + 5], start=[True, True] if t == 0 else None) for t in range(0, 20, 5)]
    y, frame = sess.finish()
    assert tuple(y.shape) == (2, la, 17, 3) and frame[0].tolist() == list(range(20 - la, 20))
    got = _collect(outs + [(y, frame)], 2)
    for s in range(2):
        ref = _offline_tta(m, xs[s], H36M)
        assert torch.equal(torch.stack([got[s][f] for f in range(20 - la, 20)]), ref[20 - la:])


def test_identical_sessions_identical_bits(cuda_device):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, False, "fp16", seed=41)
    xs = orc.make_input(4, 20, 17, 2, seed=42).to(cuda_device)
    a = m.streaming(streams=4, max_frames=5, augment=True, **H36M)
    b = m.streaming(streams=4, max_frames=5, augment=True, **H36M)
    for t in range(0, 20, 5):
        st = [True] * 4 if t == 0 else None
        ya, fa = a.push(xs[:, t:t + 5], start=st)
        yb, fb = b.push(xs[:, t:t + 5], start=st)
        assert torch.equal(ya, yb) and torch.equal(fa, fb)


def test_interleaving_leaves_plain_sessions_and_forward_unchanged(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 100, False, "fp16", seed=51)
    xo = orc.make_input(3, 60, 17, 2, seed=52).to(cuda_device)
    xs = orc.make_input(2, 24, 17, 2, seed=53).to(cuda_device)
    with torch.no_grad():
        before = m(xo)
    plain_alone = m.streaming(streams=2, max_frames=6)
    plain = m.streaming(streams=2, max_frames=6)
    aug = m.streaming(streams=2, max_frames=6, augment=True, **H36M)
    outs = []
    for t in range(0, 24, 6):
        st = [True, True] if t == 0 else None
        want = plain_alone.push(xs[:, t:t + 6], start=st)
        outs.append(aug.push(xs[:, t:t + 6], start=st))
        got = plain.push(xs[:, t:t + 6], start=st)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        with torch.no_grad():
            assert torch.equal(m(xo), before)
    outs.append(aug.finish())
    got = _collect(outs, 2)
    for s in range(2):
        assert torch.equal(torch.stack([got[s][f] for f in range(24)]), _offline_tta(m, xs[s], H36M))


@pytest.mark.parametrize("S,k", [(1, 1), (3, 1), (1, 4), (3, 4)])
def test_launch_counts(cuda_device, S, k):
    """An augmented push makes the launches of a plain push over the same 2S physical rows, plus the
    output kernel where a plain push shrinks straight into y."""
    m = _model(cuda_device, [3, 3, 3, 3, 3], 64, False, "fp16", seed=61)
    x1, x2 = (orc.make_input(n, k, 17, 2, seed=62).to(cuda_device) for n in (S, 2 * S))
    aug = m.streaming(streams=S, max_frames=k, augment=True, **H36M)
    plain2 = m.streaming(streams=2 * S, max_frames=k)
    plain1 = m.streaming(streams=S, max_frames=k)
    for first in (True, False):
        # the count belongs to the model's plan, which the three sessions share: read it at once
        aug.push(x1, start=[True] * S if first else None)
        n_aug = aug.last_launch_count()
        plain2.push(x2, start=[True] * 2 * S if first else None)
        n_plain2 = plain2.last_launch_count()
        plain1.push(x1, start=[True] * S if first else None)
        n_plain1 = plain1.last_launch_count()
        assert n_aug == n_plain2 + (k == 1)
        assert n_aug == n_plain1 + (k == 1 or S == 1)
        if not first and k == 1:
            assert n_aug == 12   # input kernel, 10 GEMMs, output kernel at arc 3^5


def test_parameter_change_needs_reset(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, True, "fp16", seed=31)
    xs = orc.make_input(1, 12, 17, 2, seed=32).to(cuda_device)
    sess = m.streaming(streams=1, max_frames=4, augment=True, **H36M)
    sess.push(xs[:, :4], start=[True])
    with torch.no_grad():
        m.shrink.bias.add_(0.5)
    with pytest.raises(RuntimeError, match="reset"):
        sess.push(xs[:, 4:8])
    sess.reset()
    outs = [sess.push(xs[:, t:t + 4], start=[True] if t == 0 else None) for t in (0, 4, 8)]
    got = _collect(outs, 1)[0]
    assert torch.equal(torch.stack([got[f] for f in range(12)]), _offline_tta(m, xs[0], H36M))


def test_cabi_with_a_plan(cuda_device):
    """State sizes of both kinds of session, and the map checks that need the plan's joint counts."""
    lib = _capi.load()
    aug = _capi.VP3D_STREAM_AUGMENT
    m = _model(cuda_device, [3, 3], 64, False, "fp16", seed=71)
    sess = m.streaming(streams=2, max_frames=2, augment=True, **H36M)
    plan = sess._plan
    assert lib.vp3d_stream_state_bytes_ex(plan, 2, 2, 0) == lib.vp3d_stream_state_bytes(plan, 2, 2)
    assert lib.vp3d_stream_state_bytes_ex(plan, 2, 2, aug) == sess._state.numel()
    assert lib.vp3d_stream_state_bytes_ex(plan, 2, 2, aug) > lib.vp3d_stream_state_bytes(plan, 2, 2)
    assert lib.vp3d_stream_state_bytes_ex(plan, 2, 2, 2) == 0
    state = sess._state.data_ptr()
    n = sess._state.numel()
    bad = np.arange(17, dtype=np.int32)
    bad[3] = 17
    good = mirror_source(17, LEFT, RIGHT)
    assert lib.vp3d_stream_init_ex(plan, state, n, 2, 2, aug, bad.ctypes.data, None, None) == -1
    assert b"kps_src[3]" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(plan, state, n, 2, 2, aug, good.ctypes.data, bad.ctypes.data,
                                   None) == -1
    assert b"joints_src[3]" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(plan, state, n - 1, 2, 2, aug, good.ctypes.data, None,
                                   None) == -4
    assert b"too small" in lib.vp3d_last_error()
    sess.reset()   # the session is whole again
    x = orc.make_input(2, 2, 17, 2, seed=72).to(cuda_device)
    y, frame = sess.push(x, start=[True, True])
    assert tuple(y.shape) == (2, 2, 17, 3)
