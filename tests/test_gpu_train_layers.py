"""GPU: the training step launch by launch against float64, in both training precisions, and the
schedule restated in Python (train_replay.py) tied to the model bit for bit.

Each case runs one step on the model -- ``torch.manual_seed(s)``, ``y = m(x)``,
``(y * gy).sum().backward()`` -- then replays the same step through the operator-level C entries
(``train_replay.GpuOps``; the dropout seed is ``train_emulation.step_seed(s)``, the draw the model
makes) and asserts:

1. every launch against float64 on that launch's own kernel-made inputs (u = 2^-24):
   * conv GEMMs (forward Z, shrink, every data gradient with its skip term, dx): the float64 product
     of the stored operand planes plus the skip term; the fp32 accumulation error is
     eval_replay.fake_conv's acc_err = 2^-20 sum|a||w| + steps 2^-23 |acc| (summation order, and
     the tensor cores truncating at each of the k16 steps), then one rounding to the output format:
     2^-8 |exp| (bf16), 2^-16 |exp| (hi + lo, bf16x3), 2^-23 |exp| (fp32 y and dx).  The skip
     term is added in fp32 plane by plane (a few u |exp|, inside those roundings).
   * per-slab statistics of the forward GEMMs (sum, sum of squares of the fp32 accumulator over
     each 32-row slab) against float64 sums of the stored Z: the stored Z is one rounding of the
     accumulator, so |sum - ref| <= r sum|Z| + 64 u sum|Z| and |sumsq - ref| <= (2 r + 64 u)
     sum Z^2, r = 2^-8 (bf16) or 2^-16 (hi + lo); 64 u covers the 32 fp32 additions.
   * finalize (mean, invstd, scale, shift, running statistics): the gates of
     test_gpu_bn_train_ops._stats_ok, k = 8 sqrt(slabs) + 32, against float64 moments of the
     launch's own slab partials.
   * bn_apply, bn_bwd_reduce, ordered_col_sums, bn_bwd_apply: the gates of test_gpu_bn_train_ops
     (one bf16 rounding of the float64 value plus 8 u of the fp32 terms; 32 u sum|terms| for
     the ordered sums; dgamma / dbeta equal to the sums bit for bit).
   * the fused BatchNorm-backward slab sums of the data-gradient GEMMs (bf16): float64 sums of
     dY = G * mask * [Z scale + shift > 0] over each slab of the stored G, 64 u sum|terms|.
   * every weight gradient: test_gpu_wgrad_gemm's gate, k = 4 sqrt(K) + 64, against float64 over
     the stored dZ and X planes.
   * the shrink-bias gradient (launch_col_sum_f32): the model's value within (64 + chunks) u
     sum|dY| of the float64 sum (64-row chunk sums, then the chunks in order).
   * padding channels [c_real, C) exactly zero, no output left NaN, no launch reading a NaN.
   Each gate is shown to reject a plausible wrong answer in the same test: a weight gradient
   without one 64-row chunk, and a BatchNorm output whose skip term is read one row off.
2. the replay is the model bit for bit: y, every parameter gradient but shrink.bias, the running
   statistics, dx, and the forward's and the backward's launch counts.
"""
import functools
import math

import pytest
import torch

import eval_replay as er
import train_replay as tr
from oracle import temporal_model_oracle as orc
from oracle import train_emulation as emu
from test_gpu_bn_train_ops import (_apply_ref, _apply_tol, _bwd_apply_ref, _bwd_sums_ref,
                                   _stats_ok, _stats_ref_moments)
from test_gpu_eval_layers import _wave_case, _wave_tiles
from test_gpu_wgrad_gemm import _dw, _products
import videopose3d_b200 as vp

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TM, OPT = "TemporalModel", "TemporalModelOptimized1f"
P = 0.25
WORST = {}   # launch kind -> (ratio to its bound, case, launch)


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


# (id, cfg | wave kind, N, T, options)
CASES = [
    ("opt_333_c64_n512", _cfg(OPT, [3, 3, 3], 64), 512, 27, {}),
    ("opt_333_c128_n600", _cfg(OPT, [3, 3, 3], 128), 600, 27, {}),
    ("opt_333_c256_n512", _cfg(OPT, [3, 3, 3], 256), 512, 27, {}),
    ("opt_35_c128_causal", _cfg(OPT, [3, 5], 128, causal=True), 200, 15, {}),
    ("opt_333_c40", _cfg(OPT, [3, 3, 3], 40), 300, 27, {}),
    ("opt_33_c100", _cfg(OPT, [3, 3], 100), 300, 9, {}),
    ("opt_333_j15_f3", _cfg(OPT, [3, 3, 3], 64, J=15, F=3, Jout=15), 300, 27, {}),
    ("opt_333_jout1", _cfg(OPT, [3, 3, 3], 64, Jout=1), 300, 27, {}),
    ("tm_333_dilated_t40", _cfg(TM, [3, 3, 3], 64), 24, 40, {}),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 24, 30, {}),
    ("tm_35_causal", _cfg(TM, [3, 5], 128, causal=True), 16, 40, {}),
    ("opt_33333_c1024", _cfg(OPT, [3, 3, 3, 3, 3], 1024), 48, 243, {}),
    ("wave_full", "full", None, 27, {}),
    ("wave_plus1", "plus1", None, 27, {}),
    ("wave_narrow", "narrow", None, 27, {}),
    ("opt_333_dx_t29", _cfg(OPT, [3, 3, 3], 64), 300, 29, dict(dx=True)),
    ("tm_333_dx", _cfg(TM, [3, 3, 3], 64), 24, 40, dict(dx=True)),
    ("opt_333_frozen_dx", _cfg(OPT, [3, 3, 3], 64), 300, 27, dict(dx=True, frozen=True)),
    ("tm_35_frozen_dx", _cfg(TM, [3, 5], 64, causal=True), 16, 40, dict(dx=True, frozen=True)),
]
PARAMS = [pytest.param(c[0], c[1], c[2], c[3], c[4], prec, p, id=f"{c[0]}-{prec}-p{p}")
          for c in CASES for prec in ("bf16", "bf16x3")
          for p in ((0.0,) if c[4].get("frozen") else (0.0, P))]


def _resolve(cfg, N):
    """Wave edges: the block-1 first conv of the strided 3,3,3 model at T = 27 has the tiles of
    test_gpu_eval_layers' block-1 conv (3 rows per window), so _wave_case's (C, N) apply."""
    if isinstance(cfg, str):
        C, N = _wave_case(cfg)
        return _cfg(OPT, [3, 3, 3], C), N
    return cfg, N


@functools.lru_cache(maxsize=2)
def _state_dict(key):
    cfg = dict(key)
    return orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], list(cfg["fw"]), cfg["C"],
                               dense=cfg["dense"], seed=0)


def _key(cfg):
    return tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in cfg.items()))


def _build(cfg, sd, dev, precision, p):
    kw = dict(filter_widths=cfg["fw"], causal=cfg["causal"], dropout=p, channels=cfg["C"])
    if cfg["cls"] == TM:
        m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], dense=cfg["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(cfg["J"], cfg["F"], cfg["Jout"], **kw)
    m.load_state_dict(sd)
    return m.to(dev).train().set_train_precision(precision)


# --------------------------------------------------------------------------------------- gates
def _note(kind, ratio, where):
    prev = WORST.get(kind, (0.0, None))
    if ratio > prev[0]:
        WORST[kind] = (ratio, where)
    return ratio


def _ratio(diff, bound):
    return float(torch.where(bound > 0, diff / bound.clamp_min(1e-300),
                             torch.where(diff > 0, torch.full_like(diff, math.inf),
                                         torch.zeros_like(diff))).max())


def _gate(kind, got, ref, bound, where):
    diff = (got - ref).abs()
    r = _ratio(diff, bound)
    assert r <= 1.0, f"{where}: {kind} off by {r:.2f} of its bound"
    return _note(kind, r, where)


def _no_nan(t, where):
    assert not torch.isnan(t).any(), f"{where}: NaN left in the output"


def _pad_zero(buf, c_real, C, where):
    cols = torch.arange(buf.shape[-1], device=buf.device) % C >= c_real
    assert (buf[..., cols] == 0).all(), f"{where}: padding channels not zero"


def _check_conv(lc, plan, where, demos):
    """demos: the set of gates already shown to reject a wrong answer in this case."""
    d = lc.desc
    base = er.Launch(lc.name, d, lc.a, lc.w,
                     lc.scale if lc.scale is not None else tr._ones(lc),
                     lc.shift if lc.shift is not None else tr._zeros(lc))
    exp, err = er.fake_conv(base, with_err=True)
    assert not torch.isnan(exp).any(), f"{where}: reads a NaN"
    exp = lc.skip_value(exp)
    assert not torch.isnan(exp).any(), f"{where}: skip term reads a NaN"
    if lc.out_f32 is not None:
        nv = d["n_valid"]
        got = lc.out_f32.double()
        _no_nan(got, where)
        _gate("conv f32", got, exp[:, :nv], 2.0 ** -23 * exp[:, :nv].abs() + err[:, :nv], where)
    else:
        _no_nan(lc.out, where)
        _pad_zero(lc.out, plan.c_real, plan.C, where)
        got = er.stored_value(lc.out)
        rel = 2.0 ** -8 if lc.out.shape[0] == 1 else 2.0 ** -16
        _gate("conv " + ("bf16" if rel > 1e-3 else "hi+lo"), got, exp, rel * exp.abs() + err, where)
    if lc.stats is not None:    # per-slab sums of the fp32 accumulator vs the stored Z
        z = er.stored_value(lc.out)
        r = 2.0 ** -8 if lc.out.shape[0] == 1 else 2.0 ** -16
        s = lc.stats.double()
        _no_nan(s, where)
        _gate("stats sum", s[:, 0], lc.per_slab(z), (r + 64 * U) * lc.per_slab(z.abs()), where)
        _gate("stats sumsq", s[:, 1], lc.per_slab(z * z), (2 * r + 64 * U) * lc.per_slab(z * z),
              where)
        if "stats" not in demos:   # rejects the sums of Z with every row read one row off
            zs = z.roll(1, 0)
            assert not bool(((s[:, 0] - lc.per_slab(zs)).abs()
                             <= (r + 64 * U) * lc.per_slab(zs.abs())).all()), \
                f"{where}: stats gate misses a shifted row"
            demos.add("stats")
    if lc.bnb is not None:      # fused BatchNorm-backward slab sums over the stored G
        dy, zc = lc.bnb_dy(er.stored_value(lc.out))
        s = lc.bnb["sums"].double()
        _no_nan(s, where)
        _gate("bnb sums", s[:, 0], lc.per_slab(dy), 64 * U * lc.per_slab(dy.abs()), where)
        _gate("bnb sums", s[:, 1], lc.per_slab(dy * zc), 64 * U * lc.per_slab((dy * zc).abs()),
              where)
        if "bnb" not in demos:     # rejects the sums of G read one row off
            dys, _ = lc.bnb_dy(er.stored_value(lc.out).roll(1, 0))
            assert not bool(((s[:, 0] - lc.per_slab(dys)).abs()
                             <= 64 * U * lc.per_slab(dys.abs())).all()), \
                f"{where}: fused sums gate misses a shifted row"
            demos.add("bnb")


def _check_finalize(rec, plan, where):
    """Against float64 moments of the launch's own slab partials (their sums treated as exact)."""
    lc = rec.ins["lc"]
    cr = plan.c_real
    s = lc.stats.double().sum(0)
    n = lc.total_rows()
    mean = s[0, :cr] / n
    var = (s[1, :cr] / n - mean * mean).clamp_min(0.0)
    m = float(torch.tensor(tr.MOMENTUM, dtype=torch.float32))
    ref = _stats_ref_moments(mean, var, n, rec.ins["gamma"], rec.ins["beta"], rec.ins["rm"],
                             rec.ins["rv"], cr, m)
    ref["momentum"] = m
    out = {k: rec.outs[k] for k in ("scale", "shift", "mean", "invstd", "rm", "rv")}
    k = 8 * math.sqrt(lc.slabs()) + 32
    ok, checks = _stats_ok(out, ref, k, cr)
    assert ok, f"{where}: finalize {checks}"
    for key in ("scale", "shift", "mean", "invstd"):
        assert torch.all(out[key][cr:] == 0), f"{where}: padding of {key}"
    dm = float(((out["mean"][:cr].double() - mean).abs()
                / (U * (var + mean ** 2).sqrt()).clamp_min(1e-300)).max())
    _note("finalize mean (of k u rms)", dm / k, where)


def _mask(seed, layer, rows, C, p, dev):
    return emu.dropout_mask(seed, layer, rows, C, C, p).to(dev) if p > 0 else 1.0


def _check_bn_apply(rec, plan, p, seed, where, shift_rows=0):
    """Returns True when the gate holds (shift_rows != 0: the skip term read that many rows off)."""
    z = er.stored_value(rec.ins["z"])
    rows, C = z.shape
    sc, sh = rec.ins["scale"], rec.ins["shift"]
    res = rec.ins["res"]
    rv = er.stored_value(res) if res is not None else None
    ref = _apply_ref(z, sc, sh, _mask(seed, rec.layer, rows, C, p, z.device), rv,
                     rec.desc["rmap"], shift_rows)
    x = rec.outs["out"]
    got = er.stored_value(x)
    bound = _apply_tol(ref, z, sc, sh, rv, p, x.shape[0])
    if shift_rows:
        return bool(((got - ref).abs() <= bound).all())
    _no_nan(got, where)
    _pad_zero(x, plan.c_real, plan.C, where)
    _gate("bn_apply", got, ref, bound, where)
    return True


def _dy_terms(rec, p, seed):
    """(dY, s1, s2, tol1, tol2, z) of a BatchNorm backward from the stored G and Z."""
    v = rec.ins["v"]
    gv, zv = er.stored_value(rec.ins["g"]), er.stored_value(rec.ins["z"])
    rows, C = zv.shape
    return _bwd_sums_ref(gv, zv, v["scale"], v["shift"], v["mean"], v["invstd"],
                         _mask(seed, rec.layer, rows, C, p, gv.device)) + (zv,)


def _check_sums(rec, p, seed, where):
    sums = rec.outs["sums"].double()
    _no_nan(sums, where)
    if rec.kind == "bn_bwd_reduce":
        _, s1, s2, t1, t2, zv = _dy_terms(rec, p, seed)
        C = zv.shape[1]
    else:   # ordered_col_sums over the fused slab partials, column blocks folded per channel
        lc = rec.ins["lc"]
        C = sums.shape[0] // 2
        part = lc.bnb["sums"].double()
        pd = part.reshape(part.shape[0], 2, part.shape[-1] // C, C)
        inv = rec.ins["invstd"].double()
        s1, s2 = pd[:, 0].sum((0, 1)), pd[:, 1].sum((0, 1)) * inv
        t1 = 32 * U * pd[:, 0].abs().sum((0, 1))
        t2 = 32 * U * pd[:, 1].abs().sum((0, 1)) * inv + 2 * U * s2.abs()
    _gate(rec.kind, sums[:C], s1, t1, where)
    _gate(rec.kind, sums[C:], s2, t2, where)


def _check_bwd_apply(rec, plan, frozen, p, seed, where):
    v = rec.ins["v"]
    dy, _, _, _, _, zv = _dy_terms(rec, p, seed)
    rows, C = zv.shape
    ref, fp32 = _bwd_apply_ref(dy, zv, v["scale"], v["mean"], v["invstd"], rec.ins["sums"], rows,
                               frozen)
    dz = rec.outs["dz"]
    got = er.stored_value(dz)
    _no_nan(got, where)
    _pad_zero(dz, plan.c_real, plan.C, where)
    _gate("bn_bwd_apply", got, ref, (2.0 ** -8 if dz.shape[0] == 1 else 2.0 ** -16) * ref.abs()
          + fp32, where)
    cr = plan.c_real
    s = rec.ins["sums"]
    assert torch.equal(rec.outs["dbeta"], s[:cr]) and torch.equal(rec.outs["dgamma"], s[C:C + cr]), \
        f"{where}: dgamma / dbeta are not the sums"


def _check_wgrad(rec, where, demo=False):
    g = tr.wgrad_geo(rec.desc)
    dz, x = rec.ins["dz"], rec.ins["x"]
    dzp = dz.reshape(dz.shape[0], g.s, g.rows, g.dz_ld)
    xp = x.reshape(x.shape[0], g.s, g.xr, g.x_ld)
    pairs = _products(dzp, xp)
    ref = sum(_dw(g, a, b) for a, b in pairs)
    mag = sum(_dw(g, a.abs(), b.abs()) for a, b in pairs)
    assert not torch.isnan(ref).any(), f"{where}: reads a NaN"
    got = rec.outs["grad"].double()
    _no_nan(got, where)
    k = 4 * math.sqrt(g.rows * g.s) + 64
    _gate("wgrad (of k)", got, ref, k * U * mag, where)
    if demo:   # the gate rejects the gradient without one 64-row chunk of one sample
        r0 = (g.rows // 2) // 64 * 64
        lost = sum(_dw(g, a[:1], b[:1], r0=r0, r1=min(r0 + 64, g.rows)) for a, b in pairs)
        assert not bool(((got - (ref - lost)).abs() <= k * U * mag).all()), \
            f"{where}: wgrad gate misses a lost chunk"


# ---------------------------------------------------------------------------------------- test
@pytest.mark.parametrize("case,cfg,N,T,opt,precision,p", PARAMS)
def test_train_layers(cuda_device, case, cfg, N, T, opt, precision, p):
    dev = cuda_device
    cfg, N = _resolve(cfg, N)
    frozen, want_dx = opt.get("frozen", False), opt.get("dx", False)
    sd = _state_dict(_key(cfg))
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(dev)
    m = _build(cfg, sd, dev, precision, p)
    if frozen:
        m.eval()
    torch_seed = 11
    xin = x.clone().requires_grad_(want_dx)
    torch.manual_seed(torch_seed)
    y = m(xin)
    fwd_launches = m.last_launch_count()
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(5)).to(dev)
    (y * gy).sum().backward()
    torch.cuda.synchronize()
    bwd_launches = m.last_launch_count()
    seed = 0 if frozen else emu.step_seed(torch_seed)
    with torch.no_grad():
        rep = tr.replay(sd, cfg, x, gy, precision, tr.GpuOps(dev), p_drop=p, seed=seed,
                        frozen=frozen, want_dx=want_dx)
    plan = rep.plan
    if case.startswith("wave_"):
        conv1 = next(r.outs["lc"] for r in rep.recs if r.kind == "conv" and r.layer == 1)
        tiles, bn = _wave_tiles(N, cfg["C"])
        assert (conv1.block_n, conv1.tiles) == (bn, tiles)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert {"wave_full": tiles % sms == 0 and bn == 128,
                "wave_plus1": tiles % sms == 1 and bn == 128, "wave_narrow": bn == 64}[case]

    # 1. every launch against float64 on its own inputs
    tag = f"{case}-{precision}-p{p}"
    demos = set()
    demo_wgrad = demo_skip = True
    for rec in rep.recs:
        where = f"{tag}: {rec.kind} {rec.name}"
        if rec.kind in ("conv", "dgrad"):
            _check_conv(rec.outs["lc"], plan, where, demos)
        elif rec.kind == "stats_finalize":
            _check_finalize(rec, plan, where)
        elif rec.kind == "bn_apply":
            _check_bn_apply(rec, plan, p, seed, where)
            if demo_skip and rec.ins["res"] is not None:
                assert not _check_bn_apply(rec, plan, p, seed, where, shift_rows=1), \
                    f"{where}: gate misses a skip row one off"
                demo_skip = False
        elif rec.kind in ("bn_bwd_reduce", "ordered_col_sums"):
            _check_sums(rec, p, seed, where)
        elif rec.kind == "bn_bwd_apply":
            _check_bwd_apply(rec, plan, frozen, p, seed, where)
        elif rec.kind == "wgrad":
            _check_wgrad(rec, where, demo=demo_wgrad and rec.desc["rows"] >= 128)
            demo_wgrad = demo_wgrad and rec.desc["rows"] < 128
        elif rec.kind == "dx_tail":
            assert torch.all(rec.outs["dx"][:, plan.fw[0] * plan.L[0]:] == 0)
    assert not demo_wgrad and not demo_skip and demos == ({"bnb"} if plan.planes == 1 else set()) \
        | ({"stats"} if not frozen else set()), "a gate was not shown to reject a wrong answer"
    # shrink bias: the model's ordered fp32 sum against float64
    dyv = gy.reshape(-1, plan.c_out_raw).double()
    chunks = -(-dyv.shape[0] // 64)
    _gate("shrink bias", m.shrink.bias.grad.double(), dyv.sum(0),
          (64 + chunks) * U * dyv.abs().sum(0), f"{tag}: shrink bias")
    print(f"\n{tag}: N={N} T={T} launches {rep.fwd_launches}+{rep.bwd_launches}; worst ratio per "
          f"launch kind so far: " + ", ".join(f"{k} {v[0]:.3f} ({v[1]})" for k, v in
                                               sorted(WORST.items())))

    # 2. the replay is the model, bit for bit
    same = lambda a, b: torch.equal(a.detach().float().view(torch.int32),
                                    b.detach().float().reshape(a.shape).view(torch.int32))
    if not frozen:    # (frozen: y is the eval forward's; the replay's y is the recompute's)
        assert same(rep.y, y), f"replay y differs in {int((rep.y != y).sum())} of {y.numel()}"
        assert rep.fwd_launches == fwd_launches
    assert rep.bwd_launches == bwd_launches
    for name, prm in m.named_parameters():
        if name == "shrink.bias":
            continue
        assert same(rep.grads[name], prm.grad), (
            f"{name}: replay differs from the model in "
            f"{int((rep.grads[name] != prm.grad.reshape(rep.grads[name].shape)).sum())} entries")
    sd_new = m.state_dict()
    for name, v in rep.stats.items():
        assert same(v, sd_new[name]), f"{name} differs from the model's"
    if want_dx:
        assert same(rep.dx, xin.grad), "dx differs from the model's"
