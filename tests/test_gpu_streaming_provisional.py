"""GPU: provisional outputs of a push (push(..., provisional=True), vp3d_stream_push_provisional).

A provisional push also returns, for the frames still inside the look-ahead, what finish() would
return right after it, and leaves the session as a plain push leaves it.  Checked on every push of
random schedules (starts at different pushes, restarts, ends mid-push, draining and idle slots,
counts of 0, partial and full as host lists and device tensors, sequences shorter than the
look-ahead):
  * every provisional frame >= 0 is the offline forward on the sequence as pushed so far,
    ``model(np.pad(x[:c], (pad, pad), 'edge'))`` (the flip average with augment), bit for bit;
  * at chosen pushes, (y_prov, frame_prov) is finish() on a twin session fed identically;
  * y / frame of sessions asking on every push, and on every other push, equal a session without
    the flag, and the launches are its launches plus the output kernel where it shrinks into y.
A one-frame truncation is left to the finish() comparison: the offline forward of a one-frame
sequence takes the dependency-cone schedule, which sums the taps in another order.
"""
import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi, metrics
from videopose3d_b200.generators import UnchunkedGenerator
from videopose3d_b200.streaming import FrameBook, ring_history

pytestmark = pytest.mark.gpu

LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
H36M = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
TRAJ = dict(kps_left=LEFT, kps_right=RIGHT)

# name: (filter widths, channels, dense, num_joints_out)
ARCHS = {
    "333_c64": ([3, 3, 3], 64, False, 17),
    "337_c64": ([3, 3, 7], 64, False, 17),
    "33_dense": ([3, 3], 64, True, 17),
    "353_c128_traj": ([3, 5, 3], 128, False, 1),
}


def _model(dev, fw, C, precision, dense=False, jout=17, causal=False, seed=0):
    m = vp.TemporalModel(17, 2, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(17, 2, jout, fw, C, dense=dense, seed=seed))
    return m.to(dev).eval().set_precision(precision)


def _lists(m, augment):
    if not augment:
        return {}
    return TRAJ if m.num_joints_out == 1 else H36M


def _offline(m, x, augment=False):
    """run.py's evaluate(return_predictions=True) for one (T, J, F) sequence (non-causal)."""
    pad = (m.receptive_field() - 1) // 2
    if not augment:
        xp = np.pad(x.cpu().numpy(), ((pad, pad), (0, 0), (0, 0)), "edge")
        with torch.no_grad():
            return m(torch.from_numpy(xp)[None].to(x.device))[0]
    lists = _lists(m, True)
    gen = UnchunkedGenerator(None, None, [x.cpu().numpy()], pad=pad, causal_shift=0,
                             augment=True, kps_left=LEFT, kps_right=RIGHT, device=x.device)
    with torch.no_grad():
        for _, _, b in gen.next_epoch():
            return metrics.flip_average(m(b), lists.get("joints_left"), lists.get("joints_right"))[0]


def _session(m, S, K, augment, provisional):
    return m.streaming(streams=S, max_frames=K, augment=augment, provisional=provisional,
                       **_lists(m, augment))


def _schedule(S, K, la, n_push, T_range, seed, dev, J=17, F=2):
    """Random pushes: a list of dicts (k, x, start, end, count argument) and, per push and slot, the
    sequence the slot holds and its real frames so far (None: idle).  Pushes 0..K-1 have k = 1..K,
    later ones a random k; slots start after random idle gaps (slot 0 at once), restart now and then
    mid-sequence or while draining, take 0..k real frames per push (count), end with `end` once the
    rest fits, and drain.  count goes as a host list, a device tensor (full slots then sometimes
    out of range, read as k) or None (every open slot full)."""
    rng = np.random.RandomState(seed)
    seqs = []
    held = [-1] * S     # sequence each slot holds
    fed = [0] * S
    book = FrameBook(S, la)   # whether a slot holds a sequence (also while it drains)
    pushes = []
    for i in range(n_push):
        k = i + 1 if i < K else int(rng.randint(1, K + 1))
        mode = ("list", "tensor", None)[i % 3]
        start, end = [False] * S, [-1] * S
        count = [k] * S
        x = torch.rand(S, k, J, F, device=dev) * 2 - 1
        state = []
        busy = [bool(a) for a in book.active]
        for s in range(S):
            restart = busy[s] and rng.rand() < 0.04
            if (not busy[s] and (rng.rand() < 0.4 or (s == 0 and i == 0))) or restart:
                T = int(rng.randint(*T_range))
                seqs.append(orc.make_input(1, T, J, F, seed=seed * 1000 + len(seqs))[0].to(dev))
                held[s], fed[s], start[s], busy[s] = len(seqs) - 1, 0, True, True
            if not busy[s]:
                state.append(None)
                continue
            seq = seqs[held[s]]
            rest = len(seq) - fed[s]
            if rest > 0:
                n = k if mode is None else int(rng.randint(1 if start[s] else 0, k + 1))
                if rest <= n:
                    n = end[s] = rest
                else:
                    count[s] = n
                x[s, :n] = seq[fed[s]:fed[s] + n]
                x[s, n:] = float("nan")
                fed[s] += n
            else:
                x[s] = float("nan")   # draining: x is not read
            state.append((held[s], fed[s]))
        if mode == "tensor":
            arg = torch.tensor([c if c < k or rng.rand() < 0.5 else int(rng.choice([-7, k + 1]))
                                for c in count], dtype=torch.int32, device=dev)
        else:
            arg = count if mode == "list" else None
        pushes.append(dict(k=k, x=x, start=start, end=end, count=arg, host_count=count,
                           state=state))
        book.push(k, start, end, count)
    return seqs, pushes


def _run(m, S, K, augment, seqs, pushes, checkpoints=(), watch=None):
    """Drive a session that asks for provisional outputs on every push, one that asks on every
    other push, and one without the flag, and check everything the module docstring lists."""
    dev = m.expand_conv.weight.device
    la = vp.streaming.lookahead(m)
    watch = range(S) if watch is None else watch
    every = _session(m, S, K, augment, True)
    other = _session(m, S, K, augment, True)
    plain = _session(m, S, K, augment, False)
    book = FrameBook(S, la)
    offline = {}
    saved = {}
    n_checked = 0
    for i, p in enumerate(pushes):
        k = p["k"]
        kw = dict(start=p["start"] if any(p["start"]) else None,
                  end=p["end"] if max(p["end"]) >= 0 else None, count=p["count"])
        y0, f0 = plain.push(p["x"], **kw)
        n_plain = plain.last_launch_count()
        y1, f1, yp, fp = every.push(p["x"], provisional=True, **kw)
        n_prov = every.last_launch_count()
        if i % 2:
            y2, f2 = other.push(p["x"], **kw)
            assert other.last_launch_count() == n_plain, i
        else:
            y2, f2, yp2, fp2 = other.push(p["x"], provisional=True, **kw)
            assert torch.equal(fp2, fp), i
            assert torch.equal(yp2[fp >= 0], yp[fp >= 0]), i
        direct = not augment and (k == 1 or S == 1)
        assert n_prov == n_plain + int(direct), (i, n_prov, n_plain)
        want, want_prov = book.push(k, p["start"], p["end"], p["host_count"], provisional=True)
        assert np.array_equal(f0.cpu().numpy(), want), i
        assert torch.equal(y1, y0) and torch.equal(f1, f0), i
        assert torch.equal(y2, y0) and torch.equal(f2, f0), i
        fp_h = fp.cpu().numpy()
        assert np.array_equal(fp_h, want_prov), i
        assert tuple(yp.shape) == (S, la, m.num_joints_out, 3)
        for s in watch:
            st = p["state"][s]
            if st is None or not (fp_h[s] >= 0).any():
                continue
            seq, c = st
            if c < 2:
                continue
            if (seq, c) not in offline:
                offline[(seq, c)] = _offline(m, seqs[seq][:c], augment)
            ref = offline[(seq, c)]
            for j in np.nonzero(fp_h[s] >= 0)[0]:
                assert torch.equal(yp[s, j], ref[int(fp_h[s, j])]), (i, s, j)
                n_checked += 1
        if i in checkpoints:
            saved[i] = (yp.clone(), fp_h)
    assert n_checked > 0
    for c, (yp, fp_h) in saved.items():
        # finish() on a twin fed identically: with and without the flag (plain finish keeps its
        # bits on a flagged session)
        for flagged in (True, False):
            twin = _session(m, S, K, augment, flagged)
            for p in pushes[:c + 1]:
                twin.push(p["x"], start=p["start"] if any(p["start"]) else None,
                          end=p["end"] if max(p["end"]) >= 0 else None, count=p["count"])
            yf, ff = twin.finish()
            ff = ff.cpu().numpy()
            assert np.array_equal(ff, fp_h), (c, flagged)
            valid = torch.from_numpy(ff >= 0).to(dev)
            assert torch.equal(yf[valid], yp[valid]), (c, flagged)


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("precision", ["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("arch", list(ARCHS))
def test_provisional_pushes(cuda_device, arch, precision, K, augment):
    fw, C, dense, jout = ARCHS[arch]
    m = _model(cuda_device, fw, C, precision, dense=dense, jout=jout, seed=len(arch) + K)
    la = vp.streaming.lookahead(m)
    S = 4
    n_push = 30 if K == 1 else 16
    # sequences from one frame to a little longer than the look-ahead, so that most of them end
    # and drain within the pushes
    seqs, pushes = _schedule(S, K, la, n_push, (1, max(8, la + 5)), seed=K * 7 + augment,
                             dev=cuda_device)
    _run(m, S, K, augment, seqs, pushes, checkpoints=(K, n_push // 2, n_push - 1))


@pytest.mark.parametrize("augment", [False, True])
def test_provisional_pushes_beyond_one_wave(cuda_device, augment):
    """Arc 3,3,3,3,3 at C = 1024 (look-ahead 121): 24 slots compute k + 121 = 122 to 124 frame rows
    each, 2928 rows and more per GEMM (twice that with augment), at least 23 row tiles of 128 by 8
    channel tiles: more tiles than the 132 SMs, so the ping-pong schedule and its half-tile last
    wave run."""
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, "fp16", seed=211)
    S, K = 24, 3
    seqs, pushes = _schedule(S, K, vp.streaming.lookahead(m), 10, (2, 40), seed=212 + augment,
                             dev=cuda_device)
    _run(m, S, K, augment, seqs, pushes, checkpoints=(6,), watch=[0, 5, 23])


def _state_bytes(m, S, K, flags):
    """vp3d_stream_state_bytes_ex restated: the bookkeeping, every ring, h and xlast, the v-pass
    vectors, the shrink buffer and the augment maps, each 1 KiB-aligned, plus 1 KiB for alignment."""
    al = lambda n: -(-n // 1024) * 1024  # noqa: E731
    aug = bool(flags & _capi.VP3D_STREAM_AUGMENT)
    rows = K + (vp.streaming.lookahead(m) if flags & _capi.VP3D_STREAM_PROVISIONAL else 0)
    P = 2 * S if aug else S
    planes = 2 if m.precision == "bf16x3" else 1
    C = -(-m._channels // 64) * 64
    c_in = -(-m.num_joints_in * m.in_features // 64) * 64
    total = al(16 * S) + al(2 * S) + al(16 * S)
    for i, h in enumerate(ring_history(m.filter_widths)):
        total += al(2 * (h + rows + 1) * P * (c_in if i == 0 else C) * planes * 2)
    total += 2 * al(planes * rows * P * C * 2)
    total += (len(m.filter_widths) - 1) * al(planes * P * C * 2)
    total += al(rows * P * m.num_joints_out * 3 * 4)
    if aug:
        total += al(m.num_joints_in * 4) + al(m.num_joints_out * 4)
    return total + 1024


@pytest.mark.parametrize("precision", ["fp16", "bf16x3"])
def test_state_sizes_and_errors(cuda_device, precision):
    lib = _capi.load()
    prov, aug = _capi.VP3D_STREAM_PROVISIONAL, _capi.VP3D_STREAM_AUGMENT
    m = _model(cuda_device, [3, 3, 3], 64, precision, seed=213)
    sess = _session(m, 3, 2, True, True)
    plan = sess._plan
    assert sess._state.numel() == lib.vp3d_stream_state_bytes_ex(plan, 3, 2, aug | prov)
    for S, K, flags in [(1, 1, 0), (3, 2, aug), (5, 4, 0), (64, 1, aug), (7, 300, 0)]:
        with_tail = lib.vp3d_stream_state_bytes_ex(plan, S, K, flags | prov)
        assert with_tail == _state_bytes(m, S, K, flags | prov), (S, K, flags)
        assert lib.vp3d_stream_state_bytes_ex(plan, S, K, flags) == _state_bytes(m, S, K, flags)
        assert with_tail > lib.vp3d_stream_state_bytes_ex(plan, S, K, flags)
    for flags in (2, prov | 2, -1):
        assert lib.vp3d_stream_state_bytes_ex(plan, 3, 2, flags) == 0
    x = orc.make_input(3, 2, 17, 2, seed=214).to(cuda_device)

    # a session without the flag: refused before any device work, and by the C entry
    plain = _session(m, 3, 2, False, False)
    with pytest.raises(RuntimeError, match="provisional=True"):
        plain.push(x, provisional=True)
    y = torch.empty((3, 2, 17, 3), device=cuda_device)
    fr = torch.empty((3, 2), dtype=torch.int64, device=cuda_device)
    yp = torch.empty((3, 13, 17, 3), device=cuda_device)
    fp = torch.empty((3, 13), dtype=torch.int64, device=cuda_device)
    stream = plain._prepare()
    st = lib.vp3d_stream_push_provisional(plain._plan, plain._state.data_ptr(), x.data_ptr(), 2,
                                          None, None, None, y.data_ptr(), fr.data_ptr(),
                                          yp.data_ptr(), fp.data_ptr(), stream)
    assert st == -5 and b"VP3D_STREAM_PROVISIONAL" in lib.vp3d_last_error()
    st = lib.vp3d_stream_push_provisional(plan, sess._state.data_ptr(), x.data_ptr(), 3, None,
                                          None, None, y.data_ptr(), fr.data_ptr(), yp.data_ptr(),
                                          fp.data_ptr(), stream)
    assert st == -1 and b"exceeds max_frames" in lib.vp3d_last_error()
    torch.cuda.synchronize()

    # a causal plan: the flag is refused, and sized as 0
    causal = _model(cuda_device, [3, 3, 3], 64, precision, causal=True, seed=215)
    with pytest.raises(ValueError, match="non-causal"):
        _session(causal, 2, 1, False, True)
    cplan = causal._get_plan(cuda_device, causal.precision)
    assert lib.vp3d_stream_state_bytes_ex(cplan, 2, 1, prov) == 0
    assert lib.vp3d_stream_state_bytes_ex(cplan, 2, 1, 0) > 0
    buf = torch.empty(lib.vp3d_stream_state_bytes_ex(cplan, 2, 1, 0) * 2, dtype=torch.uint8,
                      device=cuda_device)
    st = lib.vp3d_stream_init_ex(cplan, buf.data_ptr(), buf.numel(), 2, 1, prov, None, None,
                                 stream)
    assert st == -1 and b"causal" in lib.vp3d_last_error()
