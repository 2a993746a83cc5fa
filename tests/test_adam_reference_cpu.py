"""No GPU: adam_reference.py is exact where it claims to be and is the algorithm torch.optim.Adam
runs.  fma32 against exact rational arithmetic; the restated update against torch.optim.Adam within
float32 round-off (torch orders the operations differently); one step worked out by hand."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import adam_reference as ar

F32 = np.float32


def _round_f32(x):
    """The float32 nearest to the rational x, ties to even (IEEE round to nearest), as a float."""
    if x == 0:
        return 0.0
    neg, x = x < 0, abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    # now 2^e <= x < 2^(e+1); below 2^-126 the spacing stays 2^-149 (subnormals)
    q = max(e, -126) - 23
    n = round(x / Fraction(2) ** q)        # Fraction rounds half to even
    v = Fraction(n) * Fraction(2) ** q
    r = math.inf if v >= Fraction(2) ** 128 else float(v)
    return -r if neg else r


def _exact_fma(a, b, c):
    return _round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _check_fma(a, b, c):
    got = ar.fma32(a, b, c)
    for i in range(a.size):
        want = _exact_fma(a[i], b[i], c[i])
        assert float(got[i]) == want, (float(a[i]), float(b[i]), float(c[i]), float(got[i]), want)


def test_fma32_random_triples_are_exact():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.uniform(1, 2, n) * np.exp2(rng.integers(-75, 64, n)) * rng.choice([-1, 1], n))
    b = (rng.uniform(1, 2, n) * np.exp2(rng.integers(-75, 64, n)) * rng.choice([-1, 1], n))
    a, b = a.astype(F32), b.astype(F32)
    c = (rng.uniform(1, 2, n) * np.exp2(rng.integers(-149, 127, n)) * rng.choice([-1, 1], n))
    c = c.astype(F32)
    # a quarter of the addends cancel the product to within its float32 rounding, a few are zero
    k = n // 4
    c[:k] = -(a[:k].astype(np.float64) * b[:k]).astype(F32)
    c[k:k + 50] = 0
    a[k + 50:k + 60] = 0
    _check_fma(a, b, c)


def test_fma32_midpoints_and_double_rounding():
    """s = fl64(a b + c) lands exactly on a float32 midpoint while the exact sum lies beside it:
    rounding s to float32 directly (ties to even) gives the wrong neighbour, fma32 must not."""
    a0 = 1 + 2.0 ** -15
    b0 = 2.0 ** -24 * (1 - 2.0 ** -15)          # a0 b0 = 2^-24 - 2^-54
    rows = []
    for k in (0, -40, 30, 100):                  # several binades
        s = 2.0 ** k
        c_odd = (1 + 2.0 ** -23) * s             # c + a0 b0 just below the midpoint above c
        rows += [(a0, b0 * s, c_odd), (a0, -b0 * s, c_odd),   # just above the midpoint below c
                 (-a0, b0 * s, -c_odd), (-a0, -b0 * s, -c_odd)]
    a, b, c = (np.array(col, F32) for col in zip(*rows))
    assert all(float(t) == v for t, v in zip(np.concatenate([a, b, c]),
                                             [r[i] for i in range(3) for r in rows]))
    _check_fma(a, b, c)
    naive = (a.astype(np.float64) * b + c).astype(F32)
    assert (naive != ar.fma32(a, b, c)).all()    # every row is a double-rounding case
    # the overflow threshold: max float32 + half an ulp, approached from either side
    big = F32(np.finfo(F32).max)
    half = 2.0 ** 103
    a1 = np.array([1 + 2.0 ** -15, 1 + 2.0 ** -15], F32)
    b1 = np.array([half * (1 - 2.0 ** -15), -half * (1 - 2.0 ** -15)], F32)
    c1 = np.array([big, big], F32)
    _check_fma(a1, b1, c1)


def _torch_run(params, grads, kw, lrs, foreach):
    ps = [torch.nn.Parameter(torch.from_numpy(p.copy())) for p in params]
    opt = torch.optim.Adam(ps, foreach=foreach, **kw)
    for step, lr in enumerate(lrs):
        for group in opt.param_groups:
            group["lr"] = lr
        for p, g in zip(ps, grads[step]):
            p.grad = torch.from_numpy(g.copy())
        opt.step()
    return ps, opt


@pytest.mark.parametrize("amsgrad,wd", [(True, 0.0), (False, 0.0), (True, 0.01), (False, 0.01)])
def test_restatement_follows_torch_adam(amsgrad, wd):
    """8 steps, lr decayed after the fourth: parameters within 2e-6 relative + 2e-7 absolute, first
    moments 2e-6 + 2e-6, second moments 5e-6 relative (the tolerances of test_gpu_step_ops)."""
    rng = np.random.default_rng(1)
    shapes = [(300,), (7, 5, 3), (1,)]
    params = [rng.standard_normal(s).astype(F32) for s in shapes]
    grads = [[(rng.standard_normal(s) * (0.1 + k)).astype(F32) for s in shapes] for k in range(8)]
    lrs = [1e-3] * 4 + [0.95e-3] * 4
    kw = dict(betas=(0.9, 0.999), eps=1e-8, weight_decay=wd, amsgrad=amsgrad)
    ps, opt = _torch_run(params, grads, dict(kw, lr=lrs[0]), lrs, foreach=False)
    moved = 0.0
    for i, p0 in enumerate(params):
        st = ar.State(p0, amsgrad)
        for k in range(8):
            st.step(grads[k][i], ar.hyper(k + 1, lrs[k], 0.9, 0.999, 1e-8, wd))
        ref = opt.state[ps[i]]
        np.testing.assert_allclose(st.p, ps[i].detach().numpy(), rtol=2e-6, atol=2e-7)
        np.testing.assert_allclose(st.m, ref["exp_avg"].numpy(), rtol=2e-6, atol=2e-6)
        np.testing.assert_allclose(st.v, ref["exp_avg_sq"].numpy(), rtol=5e-6, atol=1e-12)
        if amsgrad:
            np.testing.assert_allclose(st.vmax, ref["max_exp_avg_sq"].numpy(), rtol=5e-6, atol=1e-12)
        moved = max(moved, float(np.abs(st.p - p0).max()))
    assert moved > 1e-3   # not the identity: some parameter moved by about lr per step


def test_one_step_by_hand():
    """p = 1, g = 0.5, zero moments, step 1, lr 1e-3, betas (0.9, 0.999), eps 1e-8.
    m = fl(0.1) * 0.5 = fl(0.05) and v = fl(0.001) * 0.25 = fl(0.00025) (halving is exact);
    sqrt(v) / fl(sqrt(0.001)) = 0.5000000119 rounds to 0.5, and eps is below half its ulp;
    step_size = fl(0.01), m / denom = fl(0.1), their product rounds to about 1e-3, and
    1 - 1e-3 rounds to fl(0.999)."""
    h = ar.hyper(1, 1e-3, 0.9, 0.999, 1e-8, 0.0)
    assert h.step_size == F32(0.01) and h.bc2_sqrt == F32(math.sqrt(0.001))
    one = np.ones(1, F32)
    zero = np.zeros(1, F32)
    p, m, v, vmax = ar.update(one, one * F32(0.5), zero, zero, zero, True, h)
    assert m[0] == F32(0.05) and v[0] == F32(0.00025) and vmax[0] == v[0]
    assert p[0] == F32(0.999)
    # the same with weight decay 0.5: g' = fma(0.5, 1, 0.5) = 1, m = fl(0.1), v = fl(0.001)
    h = ar.hyper(1, 1e-3, 0.9, 0.999, 1e-8, 0.5)
    p, m, v, _ = ar.update(one, one * F32(0.5), zero, zero, None, False, h)
    assert m[0] == F32(0.1) and v[0] == F32(0.001) and p[0] == F32(0.999)


@pytest.mark.parametrize("foreach", [False, True])
def test_amsgrad_maximum_propagates_nan_like_torch(foreach):
    """torch.maximum keeps a NaN of either operand, so after a NaN gradient torch's AMSGrad state
    holds NaN in max_exp_avg_sq; the restatement (and csrc/step_ops.cu) follow it."""
    p0 = np.array([1.0, -2.0, 0.5, 3.0], F32)
    grads = [np.array([0.1, np.nan, np.inf, -np.inf], F32), np.array([0.2, 0.3, 0.4, 0.5], F32)]
    ps, opt = _torch_run([p0], [[g] for g in grads], dict(lr=1e-3, amsgrad=True), [1e-3, 1e-3],
                         foreach)
    st = ar.State(p0, True)
    for k, g in enumerate(grads):
        st.step(g, ar.hyper(k + 1, 1e-3, 0.9, 0.999, 1e-8, 0.0))
    ref = opt.state[ps[0]]
    for ours, theirs in ((st.p, ps[0].detach()), (st.m, ref["exp_avg"]), (st.v, ref["exp_avg_sq"]),
                         (st.vmax, ref["max_exp_avg_sq"])):
        theirs = theirs.numpy()
        assert np.array_equal(np.isnan(ours), np.isnan(theirs)), (ours, theirs)
        assert np.array_equal(np.isposinf(ours), np.isposinf(theirs)), (ours, theirs)
        assert np.array_equal(np.isneginf(ours), np.isneginf(theirs)), (ours, theirs)
    assert np.isnan(st.vmax[1]) and not np.isnan(st.vmax[0])
