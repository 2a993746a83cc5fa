"""NumPy restatement of the int8 calibration thresholds (vp3d_int8_thresholds) and of the histograms
they are chosen from (vp3d_calibrate_int8_hist).

A histogram has one bin per fp16 bit pattern 0x0000 .. 0x7BFF of a stored activation (patterns with
the sign bit in bin 0, inf / NaN counted apart as invalid), so every rule below is exact:
    amax        the largest non-empty bin
    percentile  the smallest bin whose cumulative count reaches c = ceil(p / 100 * n) (fp64)
    mse         the fp16 value t in [amax / 256, amax] minimising
                E(t) = sum_b n_b (x_b - s q_b)^2 (fp64), s = fp32(t / 255), inv = fp32(1 / s),
                q_b = min(255, rint(fp32(x_b * inv))); the larger t on an exact tie
An all-zero layer gives 0.
"""
import math

import numpy as np

import int8_oracle as io
from oracle import temporal_model_oracle as orc

BINS = 0x7C00
F32 = np.float32
BIN_VALUES = np.arange(BINS, dtype=np.uint16).view(np.float16).astype(F32)
METHODS = ("amax", "percentile", "mse")

# The outlier scenario of tests/test_int8_calibration_cpu.py (where its figures are) and of the GPU
# test: TemporalModel 3,3,3, C = 256, one receptive field per sample, about 1 % of the calibration
# frames scaled by 20 to 50, evaluation on held-out clean sequences.
SCENARIO = dict(arc=[3, 3, 3], C=256, n_cal=128, n_eval=128, percentile=99.9)
# method -> bound on (its mean joint distance from float64) / (amax's), glitched calibration data
GPU_MARGINS = {"percentile": 0.5, "mse": 0.96}
CLEAN_MSE_TOL = 1.05   # the same ratio for mse, clean calibration data


def histogram(values):
    """(counts [BINS] int64, invalid count) of values that are fp16 values (any float array)."""
    b = np.asarray(values, np.float64).astype(np.float16).view(np.uint16).ravel()
    b = np.where(b & 0x8000, 0, b)
    bad = b >= BINS
    return np.bincount(b[~bad], minlength=BINS).astype(np.int64), int(bad.sum())


def amax_bits(h):
    nz = np.flatnonzero(h)
    return int(nz[-1]) if nz.size else 0


def amax(h):
    return F32(BIN_VALUES[amax_bits(h)])


def percentile(h, p):
    if amax_bits(h) == 0:
        return F32(0)
    c = math.ceil(p / 100.0 * float(h.sum()))
    cum = np.cumsum(h).astype(np.float64)
    return F32(BIN_VALUES[int(np.argmax(cum >= c))])


def candidates(h):
    """fp16 bit patterns of the mse candidates: the smallest fp16 >= amax / 256 .. amax."""
    top = amax_bits(h)
    if top == 0:
        return np.zeros(0, np.int64)
    lo_val = BIN_VALUES[top] / F32(256)
    lo = int(np.float16(lo_val).view(np.uint16))
    if BIN_VALUES[lo] < lo_val:
        lo += 1
    return np.arange(lo, top + 1)


def mse_errors(h, cand=None, chunk=256):
    """E(t) of each candidate pattern (default: all of them), float64."""
    cand = candidates(h) if cand is None else np.asarray(cand)
    nz = np.flatnonzero(h)
    x = BIN_VALUES[nz]
    n = h[nz].astype(np.float64)
    out = np.empty(len(cand))
    for k0 in range(0, len(cand), chunk):
        t = BIN_VALUES[cand[k0:k0 + chunk]]
        s = (t / F32(255)).astype(F32)
        inv = (F32(1) / s).astype(F32)
        q = np.minimum(np.rint((x[None, :] * inv[:, None]).astype(F32)), F32(255))
        d = x.astype(np.float64)[None, :] - s.astype(np.float64)[:, None] * q.astype(np.float64)
        out[k0:k0 + chunk] = (n[None, :] * d * d).sum(axis=1)
    return out


def pick(cand, e):
    """The candidate of smallest error; of exactly equal errors the last (larger t)."""
    return cand[np.flatnonzero(e == e.min())[-1]]


def mse(h):
    cand = candidates(h)
    if not cand.size:
        return F32(0)
    return F32(BIN_VALUES[pick(cand, mse_errors(h, cand))])


def threshold(h, method, p=99.99):
    if method == "amax":
        return amax(h)
    if method == "percentile":
        return percentile(h, p)
    return mse(h)


def thresholds(hists, method, p=99.99):
    return np.array([threshold(h, method, p) for h in hists], F32)


def calibration_histograms(sd, x, filter_widths, causal=False, dense=False, strided=False):
    """The 2B histograms (X_{i-1}, H_i per block) of the fp16 forward's stored activations, float64
    restated as int8_oracle.calibrate restates their maxima."""
    sd = orc.state_dict_to_numpy(sd, np.float32)
    a = orc.arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    x = np.asarray(x, np.float64)
    N, T = x.shape[:2]
    f16 = io.f16
    bs, bt = io.bn_fold(sd, "expand_bn")
    X = f16(np.maximum(orc._conv_cl(f16(x.reshape(N, T, -1)), f16(sd["expand_conv.weight"]),
                                    stride=fw[0] if strided else 1) * bs + bt, 0))
    hists = []
    for i in range(len(fw) - 1):
        w = fw[i + 1]
        hists.append(histogram(X)[0])
        s1, t1 = io.bn_fold(sd, f"layers_bn.{2 * i}")
        s2, t2 = io.bn_fold(sd, f"layers_bn.{2 * i + 1}")
        if strided:
            res = X[:, a["shift"][i + 1] + w // 2:: w, :]
            z = orc._conv_cl(X, f16(sd[f"layers_conv.{2 * i}.weight"]), stride=w)
            res = res[:, :z.shape[1], :]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = X[:, pad + sh: X.shape[1] - pad + sh, :]
            z = orc._conv_cl(X, f16(sd[f"layers_conv.{2 * i}.weight"]), dilation=a["dilation"][i + 1])
        H = f16(np.maximum(z * s1 + t1, 0))
        hists.append(histogram(H)[0])
        X = f16(np.maximum(orc._conv_cl(H, f16(sd[f"layers_conv.{2 * i + 1}.weight"])) * s2 + t2, 0)
                + res)
    return hists


def scenario_inputs():
    """(state_dict, clean calibration x, glitched calibration x, held-out x), numpy float32."""
    rf = orc.arch(SCENARIO["arc"])["receptive_field"]
    sd = orc.make_state_dict(17, 2, 17, SCENARIO["arc"], SCENARIO["C"], seed=0)
    xc = orc.make_input(SCENARIO["n_cal"], rf, seed=5).numpy()
    return sd, xc, inject_glitches(xc, seed=6), orc.make_input(SCENARIO["n_eval"], rf, seed=78).numpy()


def inject_glitches(x, seed, rate=0.01, lo=20.0, hi=50.0):
    """x (N, T, J, F) with about `rate` of its frames scaled by a factor in [lo, hi], like the
    glitch frames of a 2-D detector."""
    x = np.array(x, np.float32, copy=True)
    rng = np.random.RandomState(seed)
    hit = rng.rand(*x.shape[:2]) < rate
    x[hit] *= rng.uniform(lo, hi, int(hit.sum())).astype(np.float32)[:, None, None]
    return x


def int8_errors(y, ref):
    """(max |y - ref| / max |ref|, mean joint distance) of outputs (N, T, J, 3)."""
    return (float(np.abs(y - ref).max() / np.abs(ref).max()),
            float(np.linalg.norm(y - ref, axis=-1).mean()))
