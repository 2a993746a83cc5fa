"""GPU: TemporalModel.predict, offline inference on a list of clips as a few long GEMM chains.

Every clip of T >= 2 frames must come out bit for bit as the per-clip forward on the clip
edge-padded as UnchunkedGenerator pads it, ``model(np.pad(x, (pad + shift, pad - shift), 'edge'))``,
or ``metrics.flip_average(model(b))[0]`` with test-time augmentation: every GEMM of the dilated
schedule sums each output row in the same order wherever the row sits in a tile, and the chain's
output row t reads input rows [t, t + RF - 1] only.  A 1-frame clip pads to exactly one receptive
field, where model(x) takes the dependency-cone schedule and sums the taps in another order; such
clips are checked against a streaming session (whose flat ring windows give the chain's bits) and,
in int8, against tests/int8_oracle.py.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
import int8_oracle as io
import videopose3d_b200 as vp
from videopose3d_b200 import metrics
from videopose3d_b200.clips import clip_chains
from videopose3d_b200.generators import UnchunkedGenerator

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_seq")
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
H36M = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
TRAJ = dict(kps_left=LEFT, kps_right=RIGHT)
INT8_GATE, INT8_ORACLE_TOL = 1e-2, 2e-3   # as tests/test_gpu_int8.py


def _model(dev, fw, C, causal, precision, dense=False, jout=17, F=2, seed=0, calib=None):
    m = vp.TemporalModel(17, F, jout, filter_widths=fw, causal=causal, dropout=0.0, channels=C,
                         dense=dense)
    m.load_state_dict(orc.make_state_dict(17, F, jout, fw, C, dense=dense, seed=seed))
    m = m.to(dev).eval()
    if precision == "int8":
        m.calibrate_int8(calib)
    return m.set_precision(precision)


def _lists(m, augment):
    if not augment:
        return {}
    return TRAJ if m.num_joints_out == 1 else H36M


def _pad(m):
    pad = (m.receptive_field() - 1) // 2
    return pad, (pad if m._causal else 0)          # run.py:186-193


def _offline(m, x, augment=False):
    """run.py's evaluate(return_predictions=True) for one (T, J, F) clip."""
    pad, shift = _pad(m)
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


def _clips(dev, n, J, F, seed, hi=300):
    rng = np.random.RandomState(seed)
    lengths = [1, 2, 3] + [int(v) for v in rng.randint(1, hi, n - 3)]
    return [orc.make_input(1, T, J, F, seed=seed * 100 + i)[0].to(dev) for i, T in enumerate(lengths)]


def _predict(m, clips, augment, **kw):
    with torch.no_grad():
        return m.predict(clips, augment=augment, **_lists(m, augment), **kw)


CASES = [
    # fw, C, causal, precision, dense, jout, F
    ([3, 3, 3], 64, False, "fp16", False, 17, 2),
    ([3, 3, 3], 64, True, "fp16", False, 17, 2),
    ([3, 3, 3, 3, 3], 64, False, "bf16x3", False, 17, 2),
    ([3, 3, 3, 3, 3], 128, True, "bf16", False, 17, 2),
    ([3, 3], 128, False, "bf16", True, 17, 2),
    ([3, 5, 3], 128, False, "fp16", False, 1, 2),
    ([3, 3, 3], 64, False, "fp16", False, 17, 3),
    ([3, 3, 3], 128, False, "int8", False, 17, 2),
    ([3, 3, 3, 3, 3], 128, True, "int8", False, 17, 2),
]


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("fw,C,causal,precision,dense,jout,F", CASES)
def test_every_clip_equals_its_own_forward(cuda_device, fw, C, causal, precision, dense, jout, F,
                                           augment):
    calib = orc.make_input(4, 300, 17, F, seed=7).to(cuda_device)
    m = _model(cuda_device, fw, C, causal, precision, dense, jout, F, seed=11, calib=calib)
    clips = _clips(cuda_device, 24, 17, F, seed=12)
    ys = _predict(m, clips, augment)
    B = len(fw) - 1
    assert m.last_predict_launches == 2 * B + 4   # one chain
    assert len(ys) == len(clips)
    for x, y in zip(clips, ys):
        assert tuple(y.shape) == (len(x), jout, 3)
        if len(x) >= 2:
            assert torch.equal(y, _offline(m, x, augment)), len(x)
    if precision != "int8":
        # every clip, 1-frame ones included: a streaming session computes the same bits
        sess = m.streaming(streams=3, max_frames=4, augment=augment, **_lists(m, augment))
        for a, b in zip(ys, sess.predict(clips)):
            assert torch.equal(a, b)


@pytest.mark.parametrize("causal", [False, True])
def test_int8_one_frame_clip_against_the_oracle(cuda_device, causal):
    fw, C = [3, 3, 3], 128
    sd = orc.make_state_dict(17, 2, 17, fw, C, seed=13)
    m = vp.TemporalModel(17, 2, 17, filter_widths=fw, causal=causal, dropout=0.0, channels=C)
    m.load_state_dict(sd)
    m = m.to(cuda_device).eval()
    m.calibrate_int8(orc.make_input(4, 200, 17, 2, seed=14).to(cuda_device)).set_precision("int8")
    amax = m.int8_calibration().numpy()
    clips = [orc.make_input(1, 1, 17, 2, seed=15 + i)[0].to(cuda_device) for i in range(3)]
    ys = _predict(m, clips, False)
    pad, shift = _pad(m)
    for x, y in zip(clips, ys):
        xp = np.pad(x.cpu().numpy(), ((pad + shift, pad - shift), (0, 0), (0, 0)), "edge")[None]
        ref = orc.forward_numpy(sd, xp, fw, causal=causal)[0]
        y_or = io.forward_int8(sd, xp, fw, amax, causal=causal)[0]
        scale = np.abs(ref).max()
        yn = y.cpu().numpy()
        assert float(np.abs(yn - y_or).max() / scale) <= INT8_ORACLE_TOL
        assert float(np.abs(yn - ref).max() / scale) <= INT8_GATE


def _golden_names():
    return sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))


@pytest.mark.parametrize("precision,tol", [("fp16", 1e-3), ("bf16x3", 1e-3), ("bf16", 3e-2)])
@pytest.mark.parametrize("name", _golden_names())
def test_against_reference_goldens(cuda_device, name, precision, tol):
    """The reference's evaluate() outputs (tests/golden/stream_seq, with 1-frame clips and clips
    shorter than the receptive field), within the tolerance the streaming tests apply to them."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    m = _model(cuda_device, meta["fw"], meta["C"], meta["causal"], precision, dense=meta["dense"],
               jout=meta["Jout"], F=meta["F"], seed=meta["seed"])
    x = torch.from_numpy(z["x"]).to(cuda_device)
    got = torch.cat(_predict(m, list(torch.split(x, meta["lengths"])), meta["augment"]))
    got = got.cpu().numpy()
    y = z["y"].astype(np.float64)
    assert got.shape == y.shape
    off = np.concatenate([[0], np.cumsum(meta["lengths"])])
    for i in range(len(meta["lengths"])):
        a, b = off[i], off[i + 1]
        assert float(np.abs(got[a:b] - y[a:b]).max() / np.abs(y[a:b]).max()) <= tol, i


@pytest.mark.parametrize("augment", [False, True])
def test_grouping_never_changes_bits(cuda_device, augment):
    m = _model(cuda_device, [3, 3, 3, 3, 3], 64, False, "fp16", seed=16)
    clips = _clips(cuda_device, 30, 17, 2, seed=17)
    rf, B = m.receptive_field(), 4
    one = _predict(m, clips, augment)
    assert m.last_predict_launches == 2 * B + 4
    alone = _predict(m, clips, augment, max_rows=1)            # every clip its own chain
    assert m.last_predict_launches == len(clips) * (2 * B + 4)
    some = _predict(m, clips, augment, max_rows=3000)
    n = len(clip_chains([len(x) for x in clips], rf, augment, 3000))
    assert 1 < n < len(clips) and m.last_predict_launches == n * (2 * B + 4)
    perm = np.random.RandomState(18).permutation(len(clips))
    shuffled = _predict(m, [clips[i] for i in perm], augment, max_rows=3000)
    for i, (a, b, c) in enumerate(zip(one, alone, some)):
        assert torch.equal(a, b) and torch.equal(a, c), i
    for k, i in enumerate(perm):
        assert torch.equal(shuffled[k], one[i])


def test_default_chain_at_channels_1024(cuda_device):
    """The bench model (arc 3^5, C = 1024) with augmentation, in one chain of the default size."""
    m = _model(cuda_device, [3, 3, 3, 3, 3], 1024, False, "fp16", seed=19)
    clips = _clips(cuda_device, 10, 17, 2, seed=20, hi=600)
    ys = _predict(m, clips, True)
    assert m.last_predict_launches == 12
    for x, y in zip(clips, ys):
        if len(x) >= 2:
            assert torch.equal(y, _offline(m, x, True)), len(x)


def test_predict_makes_no_synchronisation(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=21)
    clips = _clips(cuda_device, 12, 17, 2, seed=22)
    _predict(m, clips, True, max_rows=500)   # workspace and weights in place
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ys = _predict(m, clips, True, max_rows=500)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for x, y in zip(clips, ys):
        if len(x) >= 2:
            assert torch.equal(y, _offline(m, x, True))


def test_weight_and_calibration_changes(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, True, "fp16", seed=23)
    clips = _clips(cuda_device, 8, 17, 2, seed=24)[3:]
    before = _predict(m, clips, False)
    with torch.no_grad():
        m.shrink.bias.add_(0.5)
    after = _predict(m, clips, False)
    for x, a, b in zip(clips, before, after):
        assert not torch.equal(a, b)
        assert torch.equal(b, _offline(m, x))
    # int8: the calibration checks of model(x)
    m.calibrate_int8(orc.make_input(2, 100, 17, 2, seed=25).to(cuda_device)).set_precision("int8")
    _predict(m, clips, False)
    with torch.no_grad():
        m.layers_conv[0].weight.mul_(1.01)
    with pytest.raises(RuntimeError, match="stale"):
        _predict(m, clips, False)


def test_autograd_is_refused(cuda_device):
    m = _model(cuda_device, [3, 3, 3], 64, False, "fp16", seed=26)
    x = orc.make_input(1, 40, 17, 2, seed=27)[0].to(cuda_device)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.predict([x])
    with pytest.raises(RuntimeError, match="inference-only"):
        with torch.enable_grad():
            for p in m.parameters():
                p.requires_grad_(False)
            m.predict([x.clone().requires_grad_()])
