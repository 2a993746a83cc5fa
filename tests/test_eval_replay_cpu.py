"""CPU: the Python restatement of the eval launch schedule (eval_replay.py), pinned without a GPU.

With the float64 fake GEMM and float64 operands the replay is the model's algorithm in the plan's
row order and per-layer layout, so it must equal the oracle's forward_numpy to rounding, output
and every intermediate activation, in every precision's schedule (planes, lo-row ranges, split
layers).  A lo plane the schedule does not write stays NaN, so a residual or split-bf16 GEMM that
reads one outside its range fails here too."""
import numpy as np
import pytest
import torch

import eval_replay as er
from oracle import temporal_model_oracle as orc

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


# (id, cfg, N, T): the architectures of the GPU matrix (tests/test_gpu_eval_layers.py)
ARCHS = [
    ("bench_cone", _cfg(TM, [3, 3, 3, 3, 3], 1024), 2, 243),
    ("bench_dilated", _cfg(TM, [3, 3, 3, 3, 3], 1024), 1, 250),
    ("wave_c640", _cfg(TM, [3, 3, 3], 640), 3, 27),
    ("opt_333_c64_t27", _cfg(OPT, [3, 3, 3], 64), 3, 27),
    ("opt_333_c64_t30", _cfg(OPT, [3, 3, 3], 64), 3, 30),
    ("opt_35_c128_causal", _cfg(OPT, [3, 5], 128, causal=True), 3, 15),
    ("tm_333_causal_cone", _cfg(TM, [3, 3, 3], 64, causal=True), 3, 27),
    ("tm_333_causal_dilated", _cfg(TM, [3, 3, 3], 64, causal=True), 2, 40),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 2, 20),
    ("tm_353_c96_cone", _cfg(TM, [3, 5, 3], 96), 2, 45),
    ("tm_53_c129_dilated", _cfg(TM, [5, 3], 129), 2, 30),
    ("tm_333_j15_f3", _cfg(TM, [3, 3, 3], 64, J=15, F=3, Jout=15), 3, 27),
    ("tm_353_traj", _cfg(TM, [3, 5, 3], 128, Jout=1), 2, 60),
    ("tm_333333_c64_split", _cfg(TM, [3, 3, 3, 3, 3, 3], 64), 1, 729),
]


def _sd(cfg):
    return orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"],
                               dense=cfg["dense"], seed=0)


@pytest.mark.parametrize("precision", er.PRECISIONS)
@pytest.mark.parametrize("name,cfg,N,T", ARCHS, ids=[a[0] for a in ARCHS])
def test_exact_replay_equals_forward_numpy(name, cfg, N, T, precision):
    sd = _sd(cfg)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1)
    acts = []
    rep = er.replay(sd, cfg, x, precision, er.fake_gemm, exact=True, collect=acts)
    ref_acts = []
    ref = orc.forward_numpy(sd, x.numpy(), cfg["fw"], causal=cfg["causal"], dense=cfg["dense"],
                            strided=rep.plan.strided, collect=ref_acts)
    # one output frame per sample on the strided schedule, all of them on the dilated one
    assert rep.plan.strided == (cfg["cls"] == OPT or (not cfg["dense"] and T == rep.plan.receptive_field))
    y = rep.y.numpy()
    assert y.shape == ref.shape
    assert np.abs(y - ref).max() <= 1e-12 * np.abs(ref).max()
    assert len(acts) == len(ref_acts) == 1 + 2 * rep.plan.nb
    names = [a[0] for a in rep.acts]
    for k, (got, exp) in enumerate(zip(acts, ref_acts)):
        exp = exp[:, :got.shape[1]]   # rows the strided output depends on (strided_trim)
        assert got.shape == exp.shape, names[k]
        assert not np.isnan(got).any(), names[k]
        assert np.abs(got - exp).max() <= 1e-12 * max(np.abs(exp).max(), 1e-30), names[k]
    for lc in rep.launches:   # padding channels of every activation are exactly zero
        if lc.out is not None:
            assert (lc.out[0][:, rep.plan.c_real:] == 0).all(), lc.name
    assert rep.launch_count == 3 + 2 * rep.plan.nb


def _peel(r, n, perm_regions, perm_widths, last_rows):
    """pack_input_kernel's row map (pack.cu), one row at a time."""
    t, row = r, 0
    for region, w in zip(perm_regions, perm_widths):
        q = t // w
        row += (t - q * w) * region
        t = q
    return row + n * last_rows + t


@pytest.mark.parametrize("fw,N", [([3, 3, 3, 3, 3], 5), ([3, 5, 3], 4), ([5, 3], 3), ([3, 7], 2)])
def test_tap_major_permutation(fw, N):
    cfg = _cfg(OPT, fw, 64)
    p = er.Plan(cfg, "fp16", N, 1 + 2 * sum(orc.arch(fw)["pad"]))
    L, R = p.L, p.R
    pos0 = p.region_rows(0)
    regions, widths = R[1:], fw[1:]
    for n in range(N):
        for r in range(L[0]):
            assert int(pos0[n, r]) == _peel(r, n, regions, widths, L[-1])
    for lv in range(p.nb + 1):
        pos = p.region_rows(lv)
        assert torch.equal(pos.flatten().sort().values, torch.arange(N * L[lv]))   # bijection
        if lv < p.nb:
            # tap k of output row (n, t) of block lv + 1 is row k * R[lv + 1] + that row's position
            w = fw[lv + 1]
            nxt = p.region_rows(lv + 1)
            for k in range(w):
                assert torch.equal(pos[:, k::w][:, :L[lv + 1]], k * R[lv + 1] + nxt)


def test_mixed_flop_rule():
    # benchmark architecture: every residual block is far above 0.5 % of the FLOPs
    p = er.Plan(_cfg(TM, [3, 3, 3, 3, 3], 1024), "mixed", 1024, 243)
    assert p.x3 == [True, False, False, False, False, True]
    assert p.lo_range(0) == (1 * p.R[1], 2 * p.R[1])   # expand writes lo on block 1's centre only
    assert p.lo_range(p.nb) == (0, 0)
    # 3,3,3,3,3,3 at C = 64: the last block holds 16384 of 3572032 FLOP units (0.46 %)
    p = er.Plan(_cfg(TM, [3, 3, 3, 3, 3, 3], 64), "mixed", 7, 729)
    assert p.x3 == [True, False, False, False, False, True, True]
    assert p.lo_range(4) == (0, 0)                       # its input keeps lo on every row
    assert p.lo_range(3) == (p.R[4], 2 * p.R[4])
    # causal: the residual is the last tap region
    p = er.Plan(_cfg(OPT, [3, 5], 128, causal=True), "mixed", 3, 15)
    assert p.lo_range(0) == (4 * p.R[1], 5 * p.R[1])
    for prec in ("fp16", "bf16", "bf16x3"):
        q = er.Plan(_cfg(TM, [3, 3, 3, 3, 3], 1024), prec, 4, 243)
        assert q.x3 == [prec == "bf16x3"] * 6
        assert all(q.lo_range(i) == (0, 0) for i in range(q.nb + 1))


def test_bn_fold_fused_shift():
    """shift = fmaf(-mean, scale, beta): one rounding of the exact value, ties settled exactly."""
    g = torch.Generator().manual_seed(3)
    a = torch.randn(4096, generator=g)
    b = torch.randn(4096, generator=g)
    c = torch.randn(4096, generator=g)
    r = er.fma_f32(a, b, c)
    from fractions import Fraction
    for i in range(0, 4096, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(r[i]))
        nb = [np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
        assert all(abs(Fraction(float(lo)) - exact) <= abs(Fraction(float(v)) - exact) for v in nb)
    # a double-rounding case: 13325 * 80581 = 2^30 + 1, so a*b + 1 = 1 + 2^-24 + 2^-54, which
    # float64 rounds onto the fp32 midpoint 1 + 2^-24 (and then to even, 1.0); fmaf gives 1 + 2^-23
    a = torch.tensor([13325 * 2.0 ** -27])
    b = torch.tensor([80581 * 2.0 ** -27])
    c = torch.tensor([1.0])
    assert float((a.double() * b.double() + c.double()).float()) == 1.0
    assert float(er.fma_f32(a, b, c)[0]) == 1.0 + 2.0 ** -23
