"""CPU: the int8 calibration thresholds (percentile, mse) of int8_calib_ref.py against brute force,
the outlier scenario that motivates them on the float64 restatement of the int8 forward, and the
argument checks of the new C entries and of TemporalModel.calibrate_int8.

The outlier scenario (TemporalModel 3,3,3, C = 256, one receptive field per sample; 128 calibration
sequences, 128 held-out clean ones): with about 1 % of the calibration frames scaled by 20 to 50,
the mean joint distance of the int8 output from the float64 one is 1.05e-2 with amax, 3.9e-3 with
the 99.9th percentile (0.37x) and 9.8e-3 with mse (0.93x; the outliers, a few percent of the deeper
layers' values, dominate the squared error, so mse clips little).  On clean calibration data mse
gives 0.97x amax's mean joint distance.  int8_calib_ref.GPU_MARGINS and CLEAN_MSE_TOL, the bounds
the GPU test applies to the same scenario run by the model, are fixed from these figures."""
import ctypes
import math

import numpy as np
import pytest

import int8_calib_ref as cr
import int8_oracle as io
from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi

# ---------------------------------------------------------------------- selection rules
def _expand(h):
    return np.repeat(cr.BIN_VALUES, h)


def _random_hist(rng, bins, top):
    h = np.zeros(cr.BINS, np.int64)
    idx = rng.choice(np.arange(1, top + 1), size=bins, replace=False)
    h[idx] = rng.randint(1, 50, size=bins)
    h[0] = rng.randint(0, 200)
    return h


@pytest.mark.parametrize("seed", range(6))
def test_percentile_against_sorted_values(seed):
    rng = np.random.RandomState(seed)
    h = _random_hist(rng, 40, int(rng.choice([0x1000, 0x3C00, 0x7BFF])))
    v = np.sort(_expand(h))
    for p in (0.001, 1.0, 50.0, 99.0, 99.99, 100.0):
        c = math.ceil(p / 100.0 * len(v))
        assert cr.percentile(h, p) == v[c - 1], p
    assert cr.percentile(h, 100.0) == cr.amax(h) == v[-1]


@pytest.mark.parametrize("seed", range(4))
def test_mse_against_brute_force(seed):
    rng = np.random.RandomState(10 + seed)
    h = _random_hist(rng, 25, int(rng.choice([0x0300, 0x2A00, 0x4C00])))
    v = _expand(h)
    cand = cr.candidates(h)
    top = cr.amax(h)
    # every fp16 value in [amax / 256, amax], found by scanning all patterns
    in_range = np.flatnonzero((cr.BIN_VALUES >= np.float64(top) / 256) & (cr.BIN_VALUES <= top))
    assert np.array_equal(cand, in_range)
    # E(t) per element with int8_oracle's quantiser and scales
    brute = []
    for t in cr.BIN_VALUES[cand]:
        s, inv = io.act_scales([t])
        q = io.quant_act(v, inv[0])
        brute.append(float(((v.astype(np.float64) - np.float64(s[0]) * q) ** 2).sum()))
    brute = np.array(brute)
    e = cr.mse_errors(h)
    assert np.allclose(e, brute, rtol=1e-12, atol=0)
    best = cr.mse(h)
    k = int(np.flatnonzero(cr.BIN_VALUES[cand] == best)[0])
    assert brute[k] <= brute.min() * (1 + 1e-12)
    assert e[-1] >= e[k]   # amax is a candidate: mse never loses to it


def test_mse_tie_rule_prefers_the_larger_threshold():
    cand = np.array([10, 11, 12, 13])
    assert cr.pick(cand, np.array([3.0, 1.0, 2.0, 1.0])) == 13
    assert cr.pick(cand, np.array([1.0, 1.0, 2.0, 1.5])) == 11
    assert cr.pick(cand, np.array([0.5, 1.0, 2.0, 1.5])) == 10


def test_all_zero_and_empty_layers():
    h = np.zeros(cr.BINS, np.int64)
    for m in cr.METHODS:
        assert cr.threshold(h, m) == 0
    h[0] = 1000
    for m in cr.METHODS:
        assert cr.threshold(h, m, 50.0) == 0


def test_histogram_bins():
    vals = np.array([0.0, -0.0, -3.0, 1.0, 1.0, 65504.0, np.inf, np.nan, 2.0 ** -24])
    h, bad = cr.histogram(vals)
    assert bad == 2 and h[0] == 3 and h[0x3C00] == 2 and h[0x7BFF] == 1 and h[1] == 1
    assert h.sum() == 7


# ---------------------------------------------------------------------- outlier scenario
def test_outlier_scenario_on_the_int8_restatement():
    sd, xc, xg, xe = cr.scenario_inputs()
    arc, p = cr.SCENARIO["arc"], cr.SCENARIO["percentile"]
    ref = orc.forward_numpy(sd, xe, arc, strided=True)
    joint = {}
    for name, xcal in (("clean", xc), ("glitch", xg)):
        hists = cr.calibration_histograms(sd, xcal, arc, strided=True)
        for m in cr.METHODS:
            t = cr.thresholds(hists, m, p)
            y = io.forward_int8(sd, xe, arc, t, strided=True)
            e_max, joint[name, m] = cr.int8_errors(y, ref)
            print(f"\n{name} {m}: thresholds {np.round(t, 3).tolist()}, max|d|/max|ref| "
                  f"{e_max:.3e}, mean joint distance {joint[name, m]:.3e}", end="")
        assert np.array_equal(cr.thresholds(hists, "amax"),
                              io.calibrate(sd, xcal, arc, strided=True))
    for m, bound in cr.GPU_MARGINS.items():
        ratio = joint["glitch", m] / joint["glitch", "amax"]
        # the GPU test's bound, with room for the kernels' fp32 roundings
        assert ratio < bound - 0.02, (m, ratio)
    assert joint["clean", "mse"] / joint["clean", "amax"] < cr.CLEAN_MSE_TOL - 0.05


# ---------------------------------------------------------------------- argument checks
def test_c_entries_check_arguments_without_gpu():
    lib = _capi.load()
    fake = ctypes.c_void_p(0x10000)
    out = ctypes.c_void_p(0x20000)
    assert lib.vp3d_int8_hist_bytes(None) == 0
    assert lib.vp3d_int8_thresholds_scratch_bytes(0) == 0
    assert lib.vp3d_int8_thresholds_scratch_bytes(_capi.VP3D_MAX_LAYERS + 1) == 0
    need = lib.vp3d_int8_thresholds_scratch_bytes(8)
    assert need > 8 * cr.BINS * 20
    assert lib.vp3d_calibrate_int8_hist(None, fake, 1, 27, fake, 1 << 20, fake, None) == -1
    ok = dict(hist=fake, layers=8, method=_capi.VP3D_INT8_CALIB_MSE, param=99.9, out=out,
              scratch=fake, nbytes=need)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.vp3d_int8_thresholds(a["hist"], a["layers"], a["method"], a["param"], a["out"],
                                        a["scratch"], a["nbytes"], None)

    assert call(hist=None) == -1
    assert call(out=None) == -1
    assert call(layers=0) == -1
    assert call(layers=_capi.VP3D_MAX_LAYERS + 1) == -1
    assert call(method=3) == -1 and call(method=-1) == -1
    pct = _capi.VP3D_INT8_CALIB_PERCENTILE
    for bad in (0.0, -1.0, 100.001, float("nan"), float("inf")):
        assert call(method=pct, param=bad) == -1, bad
    assert "percentile" in lib.vp3d_last_error().decode()
    assert call(hist=ctypes.c_void_p(0x10004)) == -1
    assert call(scratch=None) == -4
    assert call(nbytes=need - 1) == -4


def test_python_arguments_are_checked_first():
    m = vp.TemporalModel(17, 2, 17, [3, 3, 3], channels=64).eval()
    x = orc.make_input(2, 27, seed=1)
    for kw in (dict(method="kl"), dict(method="max"), dict(method="percentile", percentile=0),
               dict(method="percentile", percentile=100.5),
               dict(method="percentile", percentile=float("nan"))):
        with pytest.raises(ValueError):
            m.calibrate_int8(x, **kw)
    # valid arguments get as far as the device requirement
    for method in cr.METHODS:
        with pytest.raises(RuntimeError, match="CUDA"):
            m.calibrate_int8(x, method=method, percentile=100)
    assert m.int8_calibration() is None
