"""GPU: int8 calibration from exact activation histograms (vp3d_calibrate_int8_hist) and its
clipping thresholds (vp3d_int8_thresholds) behind TemporalModel.calibrate_int8(method=...).

1. The device histogram of every quantised activation equals np.bincount of the fp16 bit patterns
   the fp16 forward stores (the fp16 replay of eval_replay, tied to model(x) bit for bit), over the
   real channels only, in both schedules.
2. Batches accumulate; a device generator gives what the list of its batches gives.
3-5. amax, percentile and mse against vp3d_calibrate_int8 and the NumPy restatement
   (int8_calib_ref.py); 6. repeat bit for bit; 7. the outlier scenario with the bounds fixed by
   tests/test_int8_calibration_cpu.py; 8. saved and loaded calibrations; 9. refusals.
"""
import ctypes

import numpy as np
import pytest
import torch

import eval_replay as er
import int8_calib_ref as cr
import int8_oracle as io
from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.generators import UnchunkedGenerator

pytestmark = pytest.mark.gpu

TM = "TemporalModel"


def _cfg(fw, C, causal=False):
    return dict(cls=TM, fw=list(fw), C=C, J=17, F=2, Jout=17, causal=causal, dense=False)


def _build(cfg, sd, dev):
    m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], filter_widths=cfg["fw"],
                         causal=cfg["causal"], dropout=0.0, channels=cfg["C"])
    m.load_state_dict(sd)
    return m.to(dev).eval()


def _hist(m, xs):
    """(counts [2B][BINS], invalid [2B]) of vp3d_calibrate_int8_hist over the batches xs."""
    lib = _capi.load()
    dev = m.expand_conv.weight.device
    plan = m._get_plan(dev, "fp16")
    stream = torch.cuda.current_stream(dev).cuda_stream
    m._sync_weights(plan, stream)
    hist = torch.zeros(lib.vp3d_int8_hist_bytes(plan) // 8, dtype=torch.int64, device=dev)
    for x in xs:
        N, T = int(x.shape[0]), int(x.shape[1])
        ws = torch.empty(lib.vp3d_workspace_bytes(plan, N, T), dtype=torch.uint8, device=dev)
        _capi.check(lib.vp3d_calibrate_int8_hist(plan, x.data_ptr(), N, T, ws.data_ptr(),
                                                 ws.numel(), hist.data_ptr(), stream),
                    "vp3d_calibrate_int8_hist")
    h = hist.cpu().numpy()
    L = len(m.layers_conv)
    return h[:L * cr.BINS].reshape(L, cr.BINS), h[L * cr.BINS:]


def _thresholds(h, method, param=0.0):
    """vp3d_int8_thresholds on a downloaded histogram (uploaded again)."""
    lib = _capi.load()
    L = h.shape[0]
    hd = torch.from_numpy(np.concatenate([h.ravel(), np.zeros(L, np.int64)])).cuda()
    out = torch.empty(L, dtype=torch.float32, device="cuda")
    scratch = torch.empty(lib.vp3d_int8_thresholds_scratch_bytes(L), dtype=torch.uint8, device="cuda")
    _capi.check(lib.vp3d_int8_thresholds(hd.data_ptr(), L, method, param, out.data_ptr(),
                                         scratch.data_ptr(), scratch.numel(),
                                         torch.cuda.current_stream().cuda_stream),
                "vp3d_int8_thresholds")
    return out.cpu().numpy()


def _calib(m, x, method, **kw):
    return m.calibrate_int8(x, method=method, **kw).int8_calibration().numpy()


# ------------------------------------------------------------------------------ 1. histograms
HIST_CASES = [  # (id, cfg, N)
    ("tm_53_c129", _cfg([5, 3], 129), 6),
    ("tm_333_causal", _cfg([3, 3, 3], 64, causal=True), 6),
    ("bench_c1024", _cfg([3, 3, 3, 3, 3], 1024), 2),
]


@pytest.mark.parametrize("extra", [0, 30], ids=["strided_t_rf", "dilated_t_gt_rf"])
@pytest.mark.parametrize("case,cfg,N", HIST_CASES, ids=[c[0] for c in HIST_CASES])
def test_histogram_exact(cuda_device, case, cfg, N, extra):
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], cfg["C"], seed=0)
    T = orc.arch(cfg["fw"])["receptive_field"] + extra
    x = orc.make_input(N, T, seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device)
    h, bad = _hist(m, [x])
    acts = []
    with torch.no_grad():
        er.replay(sd, cfg, x, "fp16", er.gpu_gemm, collect=acts)
    L = len(m.layers_conv)
    assert len(acts) == L + 1   # X_0, H_1, X_1, ..., X_B; X_B is not quantised
    for l in range(L):
        exp, exp_bad = cr.histogram(acts[l])
        assert acts[l].shape[-1] == cfg["C"]
        assert exp_bad == 0 and bad[l] == 0
        assert np.array_equal(h[l], exp), f"{case} T={T}: layer {l} differs in " \
            f"{int((h[l] != exp).sum())} bins"
    # the histogram's largest bin is the calibration maximum
    assert np.array_equal(_thresholds(h, _capi.VP3D_INT8_CALIB_AMAX).view(np.int32),
                          _calib(m, x, "amax").view(np.int32))


# ------------------------------------------------------------------------------ 2. accumulation
def test_batches_accumulate_and_generator_matches_list(cuda_device):
    cfg = _cfg([5, 3], 129)
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], cfg["C"], seed=0)
    m = _build(cfg, sd, cuda_device)
    x1 = orc.make_input(3, 60, seed=2).to(cuda_device)
    x2 = orc.make_input(4, 60, seed=3).to(cuda_device)
    h12, _ = _hist(m, [torch.cat([x1, x2])])
    h1, _ = _hist(m, [x1])
    h2, _ = _hist(m, [x2])
    assert np.array_equal(_hist(m, [x1, x2])[0], h12)
    assert np.array_equal(h1 + h2, h12)
    # a device generator (one padded sequence per batch) against the list of its batches
    rf = m.receptive_field()
    seqs = [np.random.RandomState(s).uniform(-1, 1, (n, 17, 2)).astype(np.float32)
            for s, n in ((4, 50), (5, 80), (6, 33))]
    gen = UnchunkedGenerator(None, None, seqs, pad=(rf - 1) // 2, device=cuda_device)
    batches = [b[-1] for b in gen.next_epoch()]
    for method in ("percentile", "mse"):
        a = _calib(m, gen, method)
        b = _calib(m, batches, method)
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), method


# ------------------------------------------------------------------------------ 3-6. selection
SEL_CASES = [("tm_53_c129", _cfg([5, 3], 129), 8, 80),
             ("tm_333_causal", _cfg([3, 3, 3], 64, causal=True), 8, 27)]


@pytest.mark.parametrize("case,cfg,N,T", SEL_CASES, ids=[c[0] for c in SEL_CASES])
def test_amax_percentile_mse_and_determinism(cuda_device, case, cfg, N, T):
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], cfg["C"], seed=0)
    x = orc.make_input(N, T, seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device)
    h, _ = _hist(m, [x])
    # 3. amax: the histogram path equals the maximum path; percentile 100 is amax; "amax" is the
    # default and unchanged
    amax = _calib(m, x, "amax")
    assert np.array_equal(m.calibrate_int8(x).int8_calibration().numpy().view(np.int32),
                          amax.view(np.int32))
    assert np.array_equal(_thresholds(h, _capi.VP3D_INT8_CALIB_AMAX).view(np.int32),
                          amax.view(np.int32))
    assert np.array_equal(cr.thresholds(h, "amax"), amax)
    assert np.array_equal(_calib(m, x, "percentile", percentile=100).view(np.int32),
                          amax.view(np.int32))
    # 4. percentile: integer arithmetic, so exactly the restatement
    for p in (1.0, 50.0, 99.0, 99.99):
        got = _calib(m, x, "percentile", percentile=p)
        assert np.array_equal(got, cr.thresholds(h, "percentile", p)), p
    # 5. mse: the device's choice is NumPy's optimum up to fp64 summation order
    got = _calib(m, x, "mse")
    for l in range(h.shape[0]):
        cand = cr.candidates(h[l])
        e = cr.mse_errors(h[l], cand)
        k = int(np.flatnonzero(cr.BIN_VALUES[cand] == got[l])[0])
        assert e[k] <= (1 + 1e-12) * e.min(), (l, e[k], e.min())
        order = np.sort(e)
        if len(order) > 1 and order[1] > order[0] * (1 + 1e-9):
            assert got[l] == cr.mse(h[l]), l
    print(f"\n{case}: amax {amax.tolist()}\n  mse {got.tolist()}")
    # 6. the same bits again
    for method in ("percentile", "mse"):
        a = _calib(_build(cfg, sd, cuda_device), x, method)
        b = _calib(_build(cfg, sd, cuda_device), x, method)
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), method


# ------------------------------------------------------------------------------ 7. outliers
def test_outlier_robustness(cuda_device):
    sd, xc, xg, xe = cr.scenario_inputs()
    arc, p = cr.SCENARIO["arc"], cr.SCENARIO["percentile"]
    cfg = _cfg(arc, cr.SCENARIO["C"])
    m = _build(cfg, sd, cuda_device).set_precision("int8")
    ref = orc.forward_numpy(sd, xe, arc, strided=True)
    xe_d = torch.from_numpy(xe).to(cuda_device)
    joint = {}
    for name, xcal in (("clean", xc), ("glitch", xg)):
        for method in cr.METHODS:
            m.calibrate_int8(torch.from_numpy(xcal).to(cuda_device), method=method, percentile=p)
            with torch.no_grad():
                y = m(xe_d).cpu().numpy()
            e_max, joint[name, method] = cr.int8_errors(y, ref)
            print(f"\n{name} {method}: thresholds "
                  f"{np.round(m.int8_calibration().numpy(), 3).tolist()}, max|d|/max|ref| "
                  f"{e_max:.3e}, mean joint distance {joint[name, method]:.3e}", end="")
    for method, bound in cr.GPU_MARGINS.items():
        assert joint["glitch", method] < bound * joint["glitch", "amax"], method
    assert joint["clean", "mse"] < cr.CLEAN_MSE_TOL * joint["clean", "amax"]


# ------------------------------------------------------------------------------ 8-9. API
def test_round_trip_and_staleness(cuda_device):
    cfg = _cfg([3, 3, 3], 128)
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], 128, seed=0)
    x = orc.make_input(12, 60, seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device).set_precision("int8")
    m.calibrate_int8(x, method="percentile", percentile=99.9)
    saved = m.int8_calibration()
    assert not torch.equal(saved, _build(cfg, sd, cuda_device).calibrate_int8(x).int8_calibration())
    with torch.no_grad():
        y = m(x)
    m2 = _build(cfg, sd, cuda_device).set_precision("int8").load_int8_calibration(saved)
    with torch.no_grad():
        assert torch.equal(m2(x), y)
    with torch.no_grad():
        m.layers_conv[0].weight.mul_(1.01)
    with pytest.raises(RuntimeError, match="stale"):
        with torch.no_grad():
            m(x)


def test_refusals(cuda_device):
    cfg = _cfg([3, 3, 3], 64)
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], 64, seed=0)
    x = orc.make_input(4, 40, seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device).calibrate_int8(x, method="mse")
    before = m.int8_calibration()
    bad = x.clone()
    bad[1, 7, 3, 0] = float("nan")
    for method in ("percentile", "mse"):
        with pytest.raises(ValueError, match="NaN"):
            m.calibrate_int8([x, bad], method=method)
    for kw in (dict(method="entropy"), dict(method="percentile", percentile=0.0),
               dict(method="percentile", percentile=101.0)):
        with pytest.raises(ValueError):
            m.calibrate_int8(x, **kw)
    assert torch.equal(m.int8_calibration(), before)
    # the NaN thresholds a refused histogram gives would not be accepted by an int8 plan either
    h, invalid = _hist(m, [bad])
    assert invalid[0] >= 1   # the NaN input (the input pack makes it finite for the chain)
    lib = _capi.load()
    L = len(m.layers_conv)
    hd = torch.from_numpy(np.concatenate([h.ravel(), invalid])).to(cuda_device)
    out = torch.empty(L, dtype=torch.float32, device=cuda_device)
    scratch = torch.empty(lib.vp3d_int8_thresholds_scratch_bytes(L), dtype=torch.uint8,
                          device=cuda_device)
    _capi.check(lib.vp3d_int8_thresholds(hd.data_ptr(), L, _capi.VP3D_INT8_CALIB_MSE, 0.0,
                                         out.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                         torch.cuda.current_stream().cuda_stream),
                "vp3d_int8_thresholds")
    out = out.cpu()
    assert torch.isnan(out[0])
    with pytest.raises(ValueError, match="finite"):
        m.load_int8_calibration(out)
    # a plan without residual blocks has no histogram
    assert lib.vp3d_int8_hist_bytes(ctypes.c_void_p(None)) == 0
