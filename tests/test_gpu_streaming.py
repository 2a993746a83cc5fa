"""GPU: streaming sessions (videopose3d_b200.streaming) against the offline forward.

Per slot, the concatenated session output must equal ``model(edge_pad(x))`` -- the sequence padded
as run.py's UnchunkedGenerator pads it -- bit for bit: every layer runs the same GEMM kernel with
the same k-loop order on the same operands, and a fresh slot's history is the exact constant the
offline forward computes on the padded stretch.  The sequences here are longer than one frame, so
the offline forward takes its dilated schedule (one frame would take the dependency-cone schedule,
whose expand conv sums the taps in another order).
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200.streaming import FrameBook

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream")


def _model(dev, fw, C, causal, precision, dense=False, jout=17, F=2, seed=0):
    m = vp.TemporalModel(17, F, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(17, F, jout, fw, C, dense=dense, seed=seed))
    return m.to(dev).eval().set_precision(precision)


def _offline(m, x):
    """model(np.pad(x, (pad + shift, pad - shift), 'edge')) for one (T, J, F) sequence."""
    pad = (m.receptive_field() - 1) // 2
    shift = pad if m._causal else 0          # run.py:186-193
    xp = np.pad(x.cpu().numpy(), ((pad + shift, pad - shift), (0, 0), (0, 0)), "edge")
    with torch.no_grad():
        return m(torch.from_numpy(xp)[None].to(x.device))[0]


def _collect(outs, S):
    """{slot: {frame: y row}} from a list of (y, frame) pairs."""
    got = {s: {} for s in range(S)}
    for y, frame in outs:
        fr = frame.cpu().numpy()
        for s, f in zip(*np.nonzero(fr >= 0)):
            assert int(fr[s, f]) not in got[s], "frame returned twice"
            got[s][int(fr[s, f])] = y[s, f]
    return got


def _stream_all(m, xs, chunks, max_frames):
    """Every slot starts at the first push; the sequences are pushed in `chunks`, then finished."""
    S, T = xs.shape[0], xs.shape[1]
    sess = m.streaming(streams=S, max_frames=max_frames)
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
def test_session_equals_offline_bitwise(cuda_device, precision, causal, fw, C):
    m = _model(cuda_device, fw, C, causal, precision, seed=C)
    T = 40 if len(fw) == 3 else 30
    xs = orc.make_input(2, T, 17, 2, seed=C + 1).to(cuda_device)
    ref = [_offline(m, xs[s]) for s in range(2)]
    names = ["k1", "k7", "rf+5", "random"] if len(fw) == 3 else ["k1", "random", "rf+5"]
    for name in names:
        chunks, K = _chunkings(T, m.receptive_field(), seed=C)[name]
        got = _stream_all(m, xs, chunks, K)
        for s in range(2):
            assert torch.equal(got[s], ref[s]), (name, s, float((got[s] - ref[s]).abs().max()))


@pytest.mark.parametrize("dense,jout,F", [(True, 17, 2), (False, 1, 2), (False, 17, 3)])
def test_dense_trajectory_and_3d_inputs(cuda_device, dense, jout, F):
    fw = [3, 3] if dense else [3, 5, 3]
    m = _model(cuda_device, fw, 128, jout == 1, "fp16", dense=dense, jout=jout, F=F, seed=7)
    xs = orc.make_input(3, 33, 17, F, seed=8).to(cuda_device)
    for name in ("k1", "random"):
        chunks, K = _chunkings(33, m.receptive_field(), seed=9)[name]
        got = _stream_all(m, xs, chunks, K)
        for s in range(3):
            assert torch.equal(got[s], _offline(m, xs[s])), (name, s)


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
    chunks, K = _chunkings(meta["T"], m.receptive_field(), seed=3)["random"]
    got = _stream_all(m, x[None], chunks, K)[0].cpu().numpy()
    y = z["y"].astype(np.float64)
    assert got.shape == y.shape
    assert float(np.abs(got - y).max() / np.abs(y).max()) <= tol


@pytest.mark.parametrize("causal", [False, True])
def test_slots_start_mid_stream(cuda_device, causal):
    """Slots begin (and one restarts) at different pushes; every sequence still equals its own
    offline result, which makes the start-of-sequence history exact."""
    m = _model(cuda_device, [3, 3, 3], 64, causal, "fp16", seed=11)
    la = vp.streaming.lookahead(m)
    S, K, n_push = 3, 4, 16
    rng = np.random.RandomState(12)
    ks = [int(rng.randint(1, K + 1)) for _ in range(n_push)]
    starts = {0: [0], 1: [2], 2: [5, 9]}          # slot -> pushes that start a sequence there
    total = sum(ks)
    xs = orc.make_input(S, total, 17, 2, seed=13).to(cuda_device)
    sess = m.streaming(streams=S, max_frames=K)
    book = FrameBook(S, la)
    outs, t = [], 0
    seq_begin = {s: [] for s in range(S)}         # (push index, first global frame)
    for i, k in enumerate(ks):
        mask = [i in starts[s] for s in range(S)]
        for s in range(S):
            if mask[s]:
                seq_begin[s].append(t)
        dev_mask = torch.tensor(mask, device=cuda_device) if i % 2 else mask
        y, frame = sess.push(xs[:, t:t + k], start=dev_mask)
        assert np.array_equal(frame.cpu().numpy(), book.push(k, mask))
        outs.append((y, frame, t))
        t += k
    y, frame = sess.finish()
    assert np.array_equal(frame.cpu().numpy(), book.finish())
    outs.append((y, frame, t))
    # sequence boundaries in global frames
    for s in range(S):
        bounds = seq_begin[s] + [total]
        for j in range(len(seq_begin[s])):
            a, b = bounds[j], bounds[j + 1]
            finished = j == len(seq_begin[s]) - 1
            rows = {}
            for yy, fr, t0 in outs:
                fr = fr.cpu().numpy()
                for f in range(fr.shape[1]):
                    g = t0 + f        # global input frame that produced this row
                    if fr[s, f] >= 0 and (a <= g < b + (la if finished else 0)):
                        rows[int(fr[s, f])] = yy[s, f]
            n_out = (b - a) if finished else (b - a - la)
            assert sorted(rows) == list(range(max(n_out, 0)))
            if n_out <= 0:
                continue
            ref = _offline(m, xs[s, a:b])[:n_out]
            assert torch.equal(torch.stack([rows[f] for f in range(n_out)]), ref), (s, j)


def test_idle_slots_and_frame_tensor(cuda_device):
    m = _model(cuda_device, [3, 3], 64, False, "fp16", seed=21)
    sess = m.streaming(streams=2, max_frames=3)
    x = orc.make_input(2, 3, 17, 2, seed=22).to(cuda_device)
    y, frame = sess.push(x)                         # nothing started: every row is no frame
    assert frame.dtype == torch.int64 and tuple(frame.shape) == (2, 3)
    assert bool((frame == -1).all()) and tuple(y.shape) == (2, 3, 17, 3)
    _, frame = sess.push(x, start=[True, False])
    la = vp.streaming.lookahead(m)
    assert frame[0].tolist() == [f - la if f >= la else -1 for f in range(3)]
    assert frame[1].tolist() == [-1, -1, -1]
    _, frame = sess.finish()
    assert tuple(frame.shape) == (2, la)
    assert frame[0].tolist() == list(range(3 - la, 3)) and bool((frame[1] == -1).all())
    _, frame = sess.push(x)                         # finished slots are idle
    assert bool((frame == -1).all())


def test_parameter_change_needs_reset(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, True, "fp16", seed=31)
    xs = orc.make_input(1, 12, 17, 2, seed=32).to(cuda_device)
    sess = m.streaming(streams=1, max_frames=4)
    sess.push(xs[:, :4], start=[True])
    with torch.no_grad():
        m.shrink.bias.add_(0.5)
    with pytest.raises(RuntimeError, match="reset"):
        sess.push(xs[:, 4:8])
    m.load_state_dict(orc.make_state_dict(17, 2, 17, [3, 3, 3], 64, seed=33))
    with pytest.raises(RuntimeError, match="reset"):
        sess.push(xs[:, 4:8])
    sess.reset()
    outs = [sess.push(xs[:, t:t + 4], start=[True] if t == 0 else None) for t in (0, 4, 8)]
    got = _collect(outs, 1)[0]
    assert torch.equal(torch.stack([got[f] for f in range(12)]), _offline(m, xs[0]))


def test_identical_sessions_identical_bits(cuda_device):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, False, "fp16", seed=41)
    xs = orc.make_input(4, 20, 17, 2, seed=42).to(cuda_device)
    a = m.streaming(streams=4, max_frames=5)
    b = m.streaming(streams=4, max_frames=5)
    for t in range(0, 20, 5):
        st = [True] * 4 if t == 0 else None
        ya, fa = a.push(xs[:, t:t + 5], start=st)
        yb, fb = b.push(xs[:, t:t + 5], start=st)
        assert torch.equal(ya, yb) and torch.equal(fa, fb)


def test_push_leaves_offline_forward_unchanged(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 100, False, "fp16", seed=51)
    xo = orc.make_input(3, 60, 17, 2, seed=52).to(cuda_device)
    xs = orc.make_input(2, 24, 17, 2, seed=53).to(cuda_device)
    with torch.no_grad():
        before = m(xo)
    sess = m.streaming(streams=2, max_frames=6)
    outs = []
    for t in range(0, 24, 6):
        outs.append(sess.push(xs[:, t:t + 6], start=[True, True] if t == 0 else None))
        with torch.no_grad():
            assert torch.equal(m(xo), before)
    outs.append(sess.finish())
    got = _collect(outs, 2)
    for s in range(2):
        assert torch.equal(torch.stack([got[s][f] for f in range(24)]), _offline(m, xs[s]))


def test_validation(cuda_device):
    m = _model(cuda_device, [3, 3], 64, False, "fp16", seed=61)
    sess = m.streaming(streams=2, max_frames=4)
    ok = torch.zeros(2, 4, 17, 2, device=cuda_device)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sess.push(ok.cpu())
    with pytest.raises(TypeError):
        sess.push(ok.double())
    with pytest.raises(ValueError):
        sess.push(torch.zeros(2, 5, 17, 2, device=cuda_device))   # k > max_frames
    with pytest.raises(ValueError):
        sess.push(torch.zeros(2, 4, 16, 2, device=cuda_device))
    with pytest.raises(ValueError):
        sess.push(torch.zeros(3, 4, 17, 2, device=cuda_device))
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        sess.push(ok)
    with pytest.raises(RuntimeError, match="eval"):
        m.streaming(streams=2)
    m.eval().set_precision("mixed")
    with pytest.raises(NotImplementedError, match="mixed"):
        m.streaming(streams=2)
    opt = vp.TemporalModelOptimized1f(17, 2, 17, [3, 3], channels=64).to(cuda_device).eval()
    with pytest.raises(NotImplementedError, match="TemporalModel"):
        opt.streaming(streams=2)


def test_cabi_errors_with_a_plan(cuda_device):
    """k > max_frames and an unregistered state are reported by the library itself."""
    from videopose3d_b200 import _capi
    lib = _capi.load()
    m = _model(cuda_device, [3, 3], 64, False, "fp16", seed=71)
    sess = m.streaming(streams=2, max_frames=2)
    x = torch.zeros(2, 3, 17, 2, device=cuda_device)
    y = torch.empty(2, 3, 17, 3, device=cuda_device)
    fr = torch.empty(2, 3, dtype=torch.int64, device=cuda_device)
    assert lib.vp3d_stream_push(sess._plan, sess._state.data_ptr(), x.data_ptr(), 3, None,
                                y.data_ptr(), fr.data_ptr(), None) == -1
    assert b"exceeds max_frames" in lib.vp3d_last_error()
    assert lib.vp3d_stream_push(sess._plan, y.data_ptr(), x.data_ptr(), 1, None, y.data_ptr(),
                                fr.data_ptr(), None) == -5
    assert lib.vp3d_stream_state_bytes(sess._plan, 0, 2) == 0
    assert lib.vp3d_stream_lookahead(sess._plan) == vp.streaming.lookahead(m)
