"""The Adam / AMSGrad update of csrc/step_ops.cu restated exactly, in numpy float32.

``adam_update`` spells out every rounding (``__fmaf_rn``, ``__fsub_rn``, ``__fmul_rn``,
``__fdiv_rn``, ``__fsqrt_rn``, ``__fadd_rn``), so its result is fixed by IEEE 754 alone and a
CPU can reproduce it bit for bit: float32 add, subtract, multiply, divide and square root in numpy
are correctly rounded, and ``fma32`` supplies the fused multiply-add numpy lacks.  The library is
built without flush-to-zero, so subnormals take part as IEEE defines them.

``hyper`` is ``adam_hyper``: the bias corrections in double with ``pow``, each value then cast to
float32 once.  ``update`` is ``adam_update``, operation for operation, on whole arrays.
"""
import math

import numpy as np

F32 = np.float32


def fma32(a, b, c):
    """a * b + c with one rounding to float32 (round to nearest, ties to even), elementwise.

    a * b is exact in float64 (24 + 24 significant bits).  s = fl64(a b + c) rounds once more, and
    TwoSum gives its error e exactly, so a b + c = s + e.  Rounding s to float32 is right unless s
    lies exactly on a float32 midpoint while e != 0: then the exact value lies on e's side of the
    midpoint, so s moves one float64 ulp toward e first.  That keeps it on the same side of the
    midpoint as the exact value and strictly inside the same float32 rounding interval."""
    a = np.asarray(a, F32).astype(np.float64)
    b = np.asarray(b, F32).astype(np.float64)
    c = np.asarray(c, F32).astype(np.float64)
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        # candidates: in the normal float32 range a midpoint has the low 29 of the 52 float64
        # fraction bits equal to 1 << 28; outside it every nonzero sum is checked
        low = s.view(np.uint64) & np.uint64((1 << 29) - 1)
        mag = np.abs(s)
        cand = (low == np.uint64(1 << 28)) | ~((mag >= 2.0 ** -126) & (mag < 2.0 ** 127))
        idx = np.flatnonzero(cand & np.isfinite(e) & (e != 0))
        if idx.size:
            si, ei = s.flat[idx], e.flat[idx]
            # a midpoint is the float64 whose two neighbours round to different float32 values
            up, down = np.nextafter(si, np.inf), np.nextafter(si, -np.inf)
            mid = up.astype(F32) != down.astype(F32)
            s = s.copy()
            s.flat[idx] = np.where(mid, np.where(ei > 0, up, down), si)
        return s.astype(F32)


class Hyper:
    __slots__ = ("one_minus_beta1", "beta2", "one_minus_beta2", "eps", "weight_decay",
                 "step_size", "bc2_sqrt")


def hyper(step, lr, beta1, beta2, eps, wd):
    """adam_hyper (csrc/step_ops.cu): every value one float32 rounding of a double."""
    bc1 = 1.0 - math.pow(beta1, float(step))
    bc2 = 1.0 - math.pow(beta2, float(step))
    h = Hyper()
    h.one_minus_beta1 = F32(1.0 - beta1)
    h.beta2 = F32(beta2)
    h.one_minus_beta2 = F32(1.0 - beta2)
    h.eps = F32(eps)
    h.weight_decay = F32(wd)
    h.step_size = F32(lr / bc1)
    h.bc2_sqrt = F32(math.sqrt(bc2))
    return h


def nan_max(a, b):
    """max(a, b) that returns NaN when either is NaN, as torch.maximum does."""
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(a) | np.isnan(b), F32(np.nan), np.maximum(a, b)).astype(F32)


def update(p, g, m, v, vmax, amsgrad, h):
    """adam_update on float32 arrays; returns the new (p, m, v, vmax) (vmax None without amsgrad)."""
    p, g, m, v = (np.asarray(t, F32) for t in (p, g, m, v))
    with np.errstate(all="ignore"):
        if h.weight_decay != 0:
            g = fma32(h.weight_decay, p, g)
        m = fma32(h.one_minus_beta1, g - m, m)
        v = fma32(h.one_minus_beta2 * g, g, v * h.beta2)
        second = v
        if amsgrad:
            vmax = nan_max(np.asarray(vmax, F32), v)
            second = vmax
        denom = np.sqrt(second) / h.bc2_sqrt + h.eps
        p = p - h.step_size * (m / denom)
    return p.astype(F32), m.astype(F32), v.astype(F32), (vmax if amsgrad else None)


class State:
    """One tensor's fp32 master and Adam moments, stepped with ``update``."""

    def __init__(self, p, amsgrad):
        self.p = np.array(p, F32)
        self.m = np.zeros_like(self.p)
        self.v = np.zeros_like(self.p)
        self.vmax = np.zeros_like(self.p) if amsgrad else None
        self.amsgrad = amsgrad

    def step(self, g, h):
        self.p, self.m, self.v, self.vmax = update(self.p, g, self.m, self.v, self.vmax,
                                                   self.amsgrad, h)
