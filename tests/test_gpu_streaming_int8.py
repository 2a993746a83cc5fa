"""GPU: int8 streaming sessions (model.streaming(..., int8=True), VP3D_STREAM_INT8).

Every model is calibrated first.  Per slot, every returned frame must be the offline int8 forward
``model(np.pad(x, (pad + shift, pad - shift), 'edge'))`` (``metrics.flip_average`` of the
generator's batch with augment) bit for bit, under the random schedules of the counts and
provisional suites (starts at different pushes, restarts, ends mid-push, draining and idle slots,
counts as host lists and device tensors).  Those suites' drivers create sessions with
``m.streaming(...)``; the models here bind ``int8=True`` into that method, so the drivers run int8
sessions unchanged.  Also: provisional outputs, predict, block subsets and their launches, the
staleness rules and the state size.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.streaming import ring_history

import test_gpu_streaming_counts as counts
import test_gpu_streaming_provisional as prov

pytestmark = pytest.mark.gpu

VP3D_ERR_STATE = -5


def _model(dev, fw, C, causal=False, dense=False, jout=17, blocks=None, seed=0, int8=True):
    """A calibrated int8 TemporalModel whose streaming() makes int8 sessions (int8=False: the same
    weights in fp16)."""
    m = vp.TemporalModel(17, 2, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(17, 2, jout, fw, C, dense=dense, seed=seed))
    m = m.to(dev).eval()
    if not int8:
        return m.set_precision("fp16")
    m.calibrate_int8(orc.make_input(3, m.receptive_field() + 30, 17, 2, seed=seed + 1).to(dev))
    m.set_int8_blocks(blocks).set_precision("int8")
    m.streaming = functools.partial(type(m).streaming, m, int8=True)
    return m


# name: (filter widths, channels, causal, dense, num_joints_out)
ARCHS = {
    "333_c64": ([3, 3, 3], 64, False, False, 17),
    "333_c100": ([3, 3, 3], 100, False, False, 17),
    "337_c64": ([3, 3, 7], 64, False, False, 17),
    "33_dense": ([3, 3], 64, False, True, 17),
    "353_c128_traj": ([3, 5, 3], 128, False, False, 1),
    "333_c64_causal": ([3, 3, 3], 64, True, False, 17),
}


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("arch", list(ARCHS))
def test_int8_sessions_bit_identical(cuda_device, arch, augment):
    fw, C, causal, dense, jout = ARCHS[arch]
    m = _model(cuda_device, fw, C, causal, dense, jout, seed=len(arch) + 3 * augment)
    rng = np.random.RandomState(len(arch))
    S = 5
    out = counts._counted_session(m, S, 6, counts._lengths(rng, S, 3), seed=7 + augment,
                                  augment=augment)
    counts._check(m, out, augment)


@pytest.mark.parametrize("augment", [False, True])
def test_int8_row_addressed_with_skip_runs(cuda_device, augment):
    m = _model(cuda_device, [3, 3, 3], 64, seed=31)
    rng = np.random.RandomState(32)
    out = counts._counted_session(m, 4, 4, counts._lengths(rng, 4, 2, hi=50), seed=33,
                                  augment=augment, row_addressed=True, skip_runs=True)
    counts._check(m, out, augment)


def test_int8_bench_arc_bit_identical(cuda_device):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, seed=41)
    seqs = {0: [150, 2], 1: [40, 130], 2: [260]}
    counts._check(m, counts._counted_session(m, 3, 16, seqs, seed=42))


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("arch", ["333_c64", "33_dense", "353_c128_traj"])
def test_int8_provisional(cuda_device, arch, K, augment):
    """y_prov is the offline int8 forward on the sequence so far and finish() of a twin; y / frame
    and launches as an int8 session without the flag (prov._run)."""
    fw, C, causal, dense, jout = ARCHS[arch]
    m = _model(cuda_device, fw, C, causal, dense, jout, seed=51 + K)
    la = vp.streaming.lookahead(m)
    n_push = 24 if K == 1 else 14
    seqs, pushes = prov._schedule(4, K, la, n_push, (1, max(8, la + 5)), seed=K * 5 + augment,
                                  dev=cuda_device)
    prov._run(m, 4, K, augment, seqs, pushes, checkpoints=(K, n_push - 1))


@pytest.mark.parametrize("augment", [False, True])
def test_int8_session_predict(cuda_device, augment):
    m = _model(cuda_device, [3, 3, 3], 64, seed=61)
    lists = prov._lists(m, augment)
    clips = [orc.make_input(1, T, 17, 2, seed=62 + T)[0].to(cuda_device)
             for T in (2, 40, 7, 90, 26)]
    sess = m.streaming(streams=3, max_frames=8, augment=augment, **lists)
    got = sess.predict(clips)
    with torch.no_grad():
        want = m.predict(clips, augment=augment, **lists)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), i


def _transitions(blocks):
    """fp16 -> int8 block transitions a push quantises in a pass of its own (block 1 reads the
    expand's Q_0, written in its epilogue)."""
    return sum(1 for b in blocks if b >= 2 and b - 1 not in blocks)


@pytest.mark.parametrize("blocks", [None, (1,), (2,), (2, 3), ()])
def test_int8_block_sets_and_launches(cuda_device, blocks):
    """A 4-block arc with every block, {1}, {2}, {2, 3} and none in int8: bit identity, and the
    launches of an fp16 session of the same weights plus one per transition in the push and one
    in the start pass.  No int8 block: the fp16 session's bits too."""
    fw = [3, 3, 3, 3, 3]
    m = _model(cuda_device, fw, 64, blocks=blocks, seed=71)
    f = _model(cuda_device, fw, 64, seed=71, int8=False)
    rng = np.random.RandomState(72)
    counts._check(m, counts._counted_session(m, 4, 5, counts._lengths(rng, 4, 2, hi=140),
                                             seed=73))
    t = _transitions(m.int8_blocks)
    S, K = 3, 4
    a = m.streaming(streams=S, max_frames=K)
    b = f.streaming(streams=S, max_frames=K)
    x = orc.make_input(S, 40, 17, 2, seed=74).to(cuda_device)
    for i, (k, start, cnt) in enumerate([(4, [True] * S, None), (2, None, None),
                                         (3, [False, True, False], None), (4, None, [4, 1, 0]),
                                         (1, None, None)]):
        xk = x[:, 4 * i:4 * i + k]
        ya, fa = a.push(xk, start=start, count=cnt)
        yb, fb = b.push(xk, start=start, count=cnt)
        assert torch.equal(fa, fb), i
        assert a.last_launch_count() == b.last_launch_count() + t * (2 if start else 1), i
        if not m.int8_blocks:
            assert torch.equal(ya, yb), i
    ya, fa = a.finish()
    yb, fb = b.finish()
    assert torch.equal(fa, fb)
    assert a.last_launch_count() == b.last_launch_count() + t * -(-vp.streaming.lookahead(m) // K)
    if not m.int8_blocks:
        assert torch.equal(ya, yb)


def _push_all(sess, x, start=False):
    return sess.push(x, start=[True] * sess.streams if start else None)


def test_int8_staleness(cuda_device):
    """Each of calibrate_int8, load_int8_calibration (other values), set_int8_blocks and a
    parameter change under a session with history makes its next push raise; after reset() the
    session equals a fresh one with the new settings."""
    dev = cuda_device
    m = _model(dev, [3, 3, 3, 3], 64, seed=81)
    x = orc.make_input(2, 12, 17, 2, seed=82).to(dev)
    cal = orc.make_input(2, m.receptive_field() + 20, 17, 2, seed=83).to(dev)
    changes = [
        lambda: m.calibrate_int8(cal),
        lambda: m.load_int8_calibration(m.int8_calibration() * 1.25),
        lambda: m.set_int8_blocks([2, 3]),
        lambda: m.set_int8_blocks(None),
    ]

    def edit_params():
        with torch.no_grad():
            m.layers_bn[1].running_mean.add_(0.01)
        m.calibrate_int8(cal)   # (the old calibration is stale after a parameter change)

    for i, change in enumerate(changes + [edit_params]):
        sess = m.streaming(streams=2, max_frames=3)
        _push_all(sess, x[:, :3], start=True)
        _push_all(sess, x[:, 3:6])
        change()
        with pytest.raises(RuntimeError, match="reset"):
            _push_all(sess, x[:, 6:9])
        sess.reset()
        fresh = m.streaming(streams=2, max_frames=3)
        for j in range(3):
            ya, fa = _push_all(sess, x[:, 3 * j:3 * j + 3], start=j == 0)
            yb, fb = _push_all(fresh, x[:, 3 * j:3 * j + 3], start=j == 0)
            assert torch.equal(ya, yb) and torch.equal(fa, fb), (i, j)


def test_int8_c_abi_state_rules(cuda_device):
    """vp3d_set_int8_blocks between two pushes: VP3D_ERR_STATE (stale packs, and once re-packed
    and folded the changed mask); a push on an unfolded plan: VP3D_ERR_STATE."""
    dev = cuda_device
    lib = _capi.load()
    m = _model(dev, [3, 3, 3, 3], 64, seed=91)
    S = 2
    sess = m.streaming(streams=S, max_frames=1)
    x = orc.make_input(S, 1, 17, 2, seed=92).to(dev)
    y = torch.empty((S, 1, 17, 3), device=dev)
    fr = torch.empty((S, 1), dtype=torch.int64, device=dev)
    mask = torch.ones(S, dtype=torch.uint8, device=dev)

    def push(start=None):
        stream = torch.cuda.current_stream().cuda_stream
        return lib.vp3d_stream_push(sess._plan, sess._state.data_ptr(), x.data_ptr(), 1,
                                    None if start is None else start.data_ptr(), y.data_ptr(),
                                    fr.data_ptr(), stream)

    _push_all(sess, x, start=True)   # syncs and folds, records the session's mask and scales
    assert push() == 0
    # the mask changes on the plan: stale packs first, then (re-packed and folded) a different mask
    _capi.check(lib.vp3d_set_int8_blocks(sess._plan, 0b0101), "vp3d_set_int8_blocks")
    assert push() == VP3D_ERR_STATE
    m.set_int8_blocks([1, 3])
    m._sync_weights(m._get_plan(dev, "int8"), torch.cuda.current_stream().cuda_stream)
    assert push() == VP3D_ERR_STATE and b"changed" in lib.vp3d_last_error()
    # a new init takes the new mask
    sess.reset()
    assert push(mask) == 0 and push() == 0
    # new scales on the plan, not folded yet
    vals = (_capi.ctypes.c_float * 6)(*([1.0] * 6))
    _capi.check(lib.vp3d_set_int8_scales(sess._plan, vals, 6), "vp3d_set_int8_scales")
    assert push() == VP3D_ERR_STATE and b"folded" in lib.vp3d_last_error()
    torch.cuda.synchronize()


def _state_bytes_int8(m, S, K, flags):
    """prov._state_bytes (the 16-bit layout) plus, per residual block, its u8 ring plane and u8
    v-pass vector, each 1 KiB-aligned."""
    al = lambda n: -(-n // 1024) * 1024  # noqa: E731
    base = prov._state_bytes(m, S, K, flags & ~_capi.VP3D_STREAM_INT8)
    rows = K + (vp.streaming.lookahead(m) if flags & _capi.VP3D_STREAM_PROVISIONAL else 0)
    P = 2 * S if flags & _capi.VP3D_STREAM_AUGMENT else S
    C = -(-m._channels // 64) * 64
    for h in ring_history(m.filter_widths)[1:]:
        base += al(2 * (h + rows + 1) * P * C) + al(P * C)
    return base


def test_int8_state_sizes(cuda_device):
    lib = _capi.load()
    i8, aug, pv = _capi.VP3D_STREAM_INT8, _capi.VP3D_STREAM_AUGMENT, _capi.VP3D_STREAM_PROVISIONAL
    for fw, C in (([3, 3, 3], 64), ([3, 5, 3], 100), ([3, 3, 3, 3, 3], 1024)):
        m = _model(cuda_device, fw, C, seed=101)
        plan = m._get_plan(cuda_device, "int8")
        for S, K in ((1, 1), (3, 2), (64, 1), (7, 300)):
            for flags in (0, aug, pv, aug | pv):
                got = lib.vp3d_stream_state_bytes_ex(plan, S, K, flags | i8)
                assert got == _state_bytes_int8(m, S, K, flags | i8), (fw, S, K, flags)
                # without the flag: the 16-bit layout, as before int8 sessions existed
                assert lib.vp3d_stream_state_bytes_ex(plan, S, K, flags) == \
                    prov._state_bytes(m, S, K, flags)
        sess = m.streaming(streams=3, max_frames=2, augment=True, provisional=True,
                           **prov._lists(m, True))
        assert sess._state.numel() == lib.vp3d_stream_state_bytes_ex(plan, 3, 2, aug | pv | i8)
        f = _model(cuda_device, fw, C, seed=101, int8=False)
        fplan = f._get_plan(cuda_device, "fp16")
        for flags in (0, aug, pv, aug | pv):
            assert lib.vp3d_stream_state_bytes_ex(fplan, 3, 2, flags | i8) == 0
        buf = torch.empty(1 << 20, dtype=torch.uint8, device=cuda_device)
        st = lib.vp3d_stream_init_ex(fplan, buf.data_ptr(), buf.numel(), 1, 1, i8, None, None,
                                     None)
        assert st == -1 and b"needs an int8 plan" in lib.vp3d_last_error()
        # an int8 plan without the flag: still refused, naming it
        st = lib.vp3d_stream_init_ex(plan, buf.data_ptr(), buf.numel(), 1, 1, 0, None, None, None)
        assert st != 0 and b"int8" in lib.vp3d_last_error() and \
            b"VP3D_STREAM_INT8" in lib.vp3d_last_error()
    torch.cuda.synchronize()
