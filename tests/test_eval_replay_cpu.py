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
import int8_oracle as io
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
    # widths other than 3 and 5, and the 32-joint skeleton (tests/test_gpu_architectures.py)
    ("a337_cone", _cfg(TM, [3, 3, 7], 1024), 2, 63),
    ("a337_dilated", _cfg(TM, [3, 3, 7], 1024), 1, 90),
    ("a337_opt", _cfg(OPT, [3, 3, 7], 1024), 2, 63),
    ("a355c_cone", _cfg(TM, [3, 5, 5], 100, causal=True), 2, 75),
    ("a355c_dilated", _cfg(TM, [3, 5, 5], 100, causal=True), 1, 100),
    ("a733_opt", _cfg(OPT, [7, 3, 3], 256), 2, 63),
    ("a733_dilated", _cfg(TM, [7, 3, 3], 256), 1, 80),
    ("a313_cone", _cfg(TM, [3, 1, 3], 128), 3, 9),
    ("a313_dilated", _cfg(TM, [3, 1, 3], 128), 2, 20),
    ("a133_opt", _cfg(OPT, [1, 3, 3], 128), 3, 9),
    ("a133_dilated", _cfg(TM, [1, 3, 3], 128), 2, 20),
    ("j32_cone", _cfg(TM, [3, 3, 3], 256, J=32, F=3, Jout=32), 2, 27),
    ("j32_dilated", _cfg(TM, [3, 3, 3], 256, J=32, F=3, Jout=32), 1, 40),
    ("d337_dense", _cfg(TM, [3, 3, 7], 128, dense=True), 1, 80),
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


@pytest.mark.parametrize("name,cfg,N,T", ARCHS, ids=[a[0] for a in ARCHS])
def test_int8_replay_equals_forward_int8(name, cfg, N, T):
    """The int8 schedule with the fake GEMM (exact integer sums, the kernels' fp32 epilogue and
    quantisation) against int8_oracle's float64 restatement of the same forward: they differ by
    the fp32 fmaf BatchNorm shift and epilogue versus float64 ones, which move single codes by one
    and values by an fp16 rounding.  Plus the descriptors of every launch of the chain."""
    sd = _sd(cfg)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1)
    kw = dict(causal=cfg["causal"], dense=cfg["dense"],
              strided=er.Plan(cfg, er.INT8, N, T).strided)
    # the calibration maxima, made distinct (fp16 maxima of two layers can coincide) so that a
    # launch quantising with another layer's scale shows in its descriptor
    amax = io.calibrate(sd, x.numpy(), cfg["fw"], **kw)
    amax = (amax * (1 + np.arange(amax.size) / 64)).astype(np.float32)
    acts = []
    rep = er.replay(sd, cfg, x, er.INT8, er.fake_gemm, amax=amax, collect=acts)
    ref_acts = []
    ref = io.forward_int8(sd, x.numpy(), cfg["fw"], amax, collect=ref_acts, **kw)
    ref_acts = [a for a in ref_acts if a is not None]   # (the last block writes no Q)
    y = rep.y.numpy()
    assert y.shape == ref.shape
    print(f"\n{name}: int8 replay vs forward_int8 {np.abs(y - ref).max() / np.abs(ref).max():.2e}")
    assert np.abs(y - ref).max() <= 1e-3 * np.abs(ref).max()
    names = [a[0] for a in rep.acts]
    assert len(acts) == len(ref_acts) == 2 + 3 * rep.plan.nb - 1
    for k, (got, exp) in enumerate(zip(acts, ref_acts)):
        exp = exp[:, :got.shape[1]]
        assert got.shape == exp.shape, names[k]
        if names[k][0] in "QH":   # u8 codes
            assert np.abs(got - exp).max() <= 1, names[k]
        else:   # fp16 roundings, and the codes one apart in earlier layers: a few fp16 ulps
            assert np.abs(got - exp).max() <= 3e-3 * np.abs(exp).max(), names[k]

    # the launches of run_infer_chain in an int8 plan
    p, ls = rep.plan, rep.launches
    _, inv = io.act_scales(amax)
    assert len(set(inv.tolist())) == len(inv)
    assert rep.launch_count == 3 + 2 * p.nb == 1 + len(ls)
    expand, shrink = ls[0], ls[-1]
    assert expand.desc["precision"] == shrink.desc["precision"] == er.K_FP16
    assert expand.inv_s == float(inv[0]) and expand.out_u8 is not None
    assert shrink.out_u8 is None and shrink.out_f32 is not None
    q_prev, x_prev = expand.out_u8, expand.out
    for i in range(1, p.nb + 1):
        c1, c2 = ls[2 * i - 1], ls[2 * i]
        assert (c1.name, c2.name) == (f"block {i} conv 1", f"block {i} conv 2")
        for lc in (c1, c2):
            d = lc.desc
            assert d["precision"] == er.K_INT8 and d["a_planes"] == 1 and d["a_ld"] == p.C
            assert d["k_per_tap"] == er.round_up(p.C, 128) and lc.w.shape[-1] == d["k_per_tap"]
            assert lc.a.dtype == torch.uint8 and lc.w.dtype == torch.int8
        # conv 1: Q_{i-1} -> H, u8 alone
        assert c1.a is q_prev and c1.out is None and c1.res is None
        assert c1.inv_s == float(inv[2 * (i - 1) + 1])
        # conv 2: H -> X_i in fp16 over the residual X_{i-1}, and Q_i except in the last block
        assert c2.a is c1.out_u8 and c2.res is x_prev and c2.out.dtype == torch.float16
        if i < p.nb:
            assert c2.out_u8 is not None and c2.inv_s == float(inv[2 * i])
        else:
            assert c2.out_u8 is None and c2.inv_s is None
        q_prev, x_prev = c2.out_u8, c2.out
    assert shrink.a is x_prev


def test_int8_epilogue_rounding():
    """The restated int8 epilogue on hand-picked values: fmaf rounds once, codes round half to
    even and saturate, fp16 saturates to 65504."""
    desc = er.new_desc(a_planes=1, samples=1, a_rows=4, a_ld=64, taps=1, k_per_tap=128,
                       n_pad=64, out_rows=4, precision=er.K_INT8, relu=1, res_planes=1,
                       res_row_step=1)
    a = torch.zeros(1, 4, 64, dtype=torch.uint8)
    a[0, :, 0] = torch.tensor([1, 2, 3, 255], dtype=torch.uint8)
    w = torch.zeros(1, 64, 128, dtype=torch.int8)
    w[0, 0, 0], w[0, 1, 0], w[0, 2, 0] = 1, -1, 127
    # col 0: 0.5 acc + 1 + residual; col 1: negative -> ReLU 0; col 2: 127 acc * 1e3 saturates
    # (K runs to 128 past the row of 64: A reads as zero there)
    scale = torch.zeros(64)
    scale[0], scale[1], scale[2] = 0.5, 1.0, 1e3
    shift = torch.zeros(64)
    shift[0] = 1.0
    res = torch.zeros(1, 4, 64, dtype=torch.float16)
    res[0, :, 0] = torch.tensor([0.25, 0.0, 0.5, 0.0], dtype=torch.float16)
    lc = er.Launch("t", desc, a, w, scale, shift, res=res,
                   out=torch.empty(1, 4, 64, dtype=torch.float16),
                   out_u8=torch.empty(1, 4, 64, dtype=torch.uint8), inv_s=1.0)
    er.fake_gemm(lc)
    # col 0: 0.5 a + 1 + res = 1.75, 2.0, 3.0, 128.5  ->  codes 2, 2, 3, 128 (half to even)
    assert lc.out[0, :, 0].tolist() == [1.75, 2.0, 3.0, 128.5]
    assert lc.out_u8[0, :, 0].tolist() == [2, 2, 3, 128]
    assert lc.out[0, :, 1].tolist() == [0.0] * 4 and lc.out_u8[0, :, 1].tolist() == [0] * 4
    assert lc.out[0, 3, 2].item() == 65504.0 and lc.out_u8[0, 3, 2].item() == 255
    assert (lc.out[0, :, 3:] == 0).all() and (lc.out_u8[0, :, 3:] == 0).all()


def _peel(r, n, perm_regions, perm_widths, last_rows):
    """pack_input_kernel's row map (pack.cu), one row at a time."""
    t, row = r, 0
    for region, w in zip(perm_regions, perm_widths):
        q = t // w
        row += (t - q * w) * region
        t = q
    return row + n * last_rows + t


@pytest.mark.parametrize("fw,N", [([3, 3, 3, 3, 3], 5), ([3, 5, 3], 4), ([5, 3], 3), ([3, 7], 2),
                                  ([3, 3, 7], 2), ([7, 3, 3], 2), ([3, 1, 3], 3), ([1, 3, 3], 3)])
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
