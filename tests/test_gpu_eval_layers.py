"""GPU: the eval forward layer by layer, in every precision, against float64 -- and the schedule
restated in Python (eval_replay.py) tied to the model bit for bit.

Each case runs ``y = model(x)``, then replays the same launch schedule through ``vp3d_conv_gemm``
and asserts:
1. per layer: every GEMM's stored output against the float64 fake of the same descriptor applied
   to that GEMM's own kernel-produced inputs.  What remains is the fp32 accumulation, bounded by
   acc_err = (2^-20 * sum|a||w| + steps * 2^-23 * |acc|) * |scale| (summation order, and the
   tensor cores truncating at each of the layer's k16 steps: eval_replay.fake_conv), and one
   rounding to the output format:
       fp16 out         2^-11 |exp| + acc_err + 2^-24
       bf16 out         2^-8  |exp| + acc_err
       hi + lo out      2^-16 |exp| + acc_err  (lo written exactly on the tiles of its lo range)
       fp32 shrink      2^-23 |exp| + acc_err
   padding channels [c_real, C) exactly zero, and no NaN read or written (buffers start as NaN);
2. the replay's output equals model(x) bit for bit, with as many launches (both run the same
   descriptors through the same kernel instances, every tile accumulated by one CTA in a fixed k
   order -- a difference means the replay is wrong about the plan);
3. the replay's activations, mapped back from the plan's row order to (N, L, C), against
   forward_numpy's on a few windows: O(1) for a layout error, so loose gates suffice.
"""
import functools

import numpy as np
import pytest
import torch

import eval_replay as er
from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp

pytestmark = pytest.mark.gpu

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"
ALL = er.PRECISIONS
# (`mixed` runs the residual blocks' GEMMs in plain bf16 and stores their inner activations as
# bf16: its activations carry ~3e-3 of their scale, above the 3e-3 of its model-level gate)
LAYOUT_TOL = {"fp16": 2e-3, "mixed": 1e-2, "bf16": 3e-2, "bf16x3": 1e-4}
WORST = {}   # precision -> (fraction of the per-layer bound, case, layer)


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wave_tiles(N, C):
    """(tiles, tile width) of the block-1 conv of TemporalModel 3,3,3 at T = 27 (3 rows/window)."""
    m_tiles = -(-3 * N // er.BLOCK_M)
    n_pad = er.round_up(C, 64)
    if n_pad % 128 == 0 and m_tiles * (n_pad // 128) * 2 >= _num_sms():
        return m_tiles * (n_pad // 128), 128
    return m_tiles * (n_pad // 64), 64


@functools.lru_cache(maxsize=None)
def _wave_case(kind):
    """(C, N) of a block-1 conv with exactly k * num_sms 128-wide tiles, k * num_sms + 1 of them,
    or as many tiles as still select the 64-wide tile."""
    sms = _num_sms()
    for N in range(1, 12000):
        for C in (1024, 640, 896, 384, 1152, 768):
            tiles, bn = _wave_tiles(N, C)
            if kind == "full" and bn == 128 and tiles % sms == 0:
                return C, N
            if kind == "plus1" and bn == 128 and tiles % sms == 1 and tiles > sms:
                return C, N
            if kind == "narrow" and bn == 64 and _wave_tiles(N + 1, C)[1] == 128:
                return C, N
    raise AssertionError(f"no wave-edge shape for {kind} on {sms} SMs")


BENCH = _cfg(TM, [3, 3, 3, 3, 3], 1024)
# (id, cfg | wave kind, N, T, precisions)
CASES = [
    ("bench_n1024", BENCH, 1024, 243, ("fp16", "mixed")),
    ("bench_n256", BENCH, 256, 243, ("bf16", "bf16x3")),
    ("bench_dilated_t250", BENCH, 32, 250, ALL),
    ("wave_full", "full", None, 27, ALL),
    ("wave_plus1", "plus1", None, 27, ALL),
    ("wave_narrow", "narrow", None, 27, ALL),
    ("opt_333_c64_t27", _cfg(OPT, [3, 3, 3], 64), 300, 27, ALL),
    ("opt_333_c64_t30", _cfg(OPT, [3, 3, 3], 64), 300, 30, ALL),
    ("opt_35_c128_causal", _cfg(OPT, [3, 5], 128, causal=True), 200, 15, ALL),
    ("tm_333_causal_cone", _cfg(TM, [3, 3, 3], 64, causal=True), 300, 27, ALL),
    ("tm_333_causal_dilated", _cfg(TM, [3, 3, 3], 64, causal=True), 24, 90, ALL),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 24, 60, ALL),
    ("tm_353_c96_cone", _cfg(TM, [3, 5, 3], 96), 200, 45, ALL),
    ("tm_53_c129_dilated", _cfg(TM, [5, 3], 129), 16, 100, ALL),
    ("tm_333_j15_f3", _cfg(TM, [3, 3, 3], 64, J=15, F=3, Jout=15), 300, 27, ALL),
    ("tm_353_traj", _cfg(TM, [3, 5, 3], 128, Jout=1), 16, 120, ALL),
    ("tm_333333_c64_split", _cfg(TM, [3, 3, 3, 3, 3, 3], 64), 40, 729, ALL),
]
PARAMS = [pytest.param(c[0], c[1], c[2], c[3], p, id=f"{c[0]}-{p}") for c in CASES for p in c[4]]


def _resolve(cfg, N):
    if isinstance(cfg, str):
        C, N = _wave_case(cfg)
        return _cfg(TM, [3, 3, 3], C), N
    return cfg, N


def _build(cfg, sd, dev, precision):
    kw = dict(filter_widths=cfg["fw"], causal=cfg["causal"], dropout=0.0, channels=cfg["C"])
    if cfg["cls"] == TM:
        m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], dense=cfg["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(cfg["J"], cfg["F"], cfg["Jout"], **kw)
    m.load_state_dict(sd)
    return m.to(dev).eval().set_precision(precision)


def _check_launch(lc, plan, case):
    """Assertion 1 for one GEMM; returns its worst |got - exp| / bound."""
    d = lc.desc
    where = f"{case}: {lc.name} (block_n={lc.block_n}, {d['out_rows']} rows x {d['n_pad']})"
    exp, err = er.fake_conv(lc, with_err=True)
    assert not torch.isnan(exp).any(), f"{where}: reads a NaN (a row or lo plane nobody wrote)"
    if lc.out_f32 is not None:
        nv = d["n_valid"]
        exp, err = exp[:, :nv], err[:, :nv]
        got = lc.out_f32.double()
        bound = 2.0 ** -23 * exp.abs() + err
    else:
        out = lc.out
        hi = out[0].double()
        assert not torch.isnan(hi).any(), f"{where}: rows left unwritten"
        pad_cols = out[:, :, plan.c_real:]
        assert (pad_cols[0] == 0).all(), f"{where}: padding channels not zero"
        if out.dtype == torch.float16:
            got = hi
            bound = 2.0 ** -11 * exp.abs() + err + 2.0 ** -24
        elif out.shape[0] == 1:
            got = hi
            bound = 2.0 ** -8 * exp.abs() + err
        else:
            lo_rows = lc.lo_mask().to(hi.device)
            lo = out[1].double()
            assert not torch.isnan(lo[lo_rows]).any(), f"{where}: lo plane missing inside its range"
            assert torch.isnan(lo[~lo_rows]).all(), f"{where}: lo plane written outside its range"
            assert (pad_cols[1][lo_rows] == 0).all(), f"{where}: padding channels not zero (lo)"
            got = hi.clone()
            got[lo_rows] += lo[lo_rows]
            rel = torch.where(lo_rows, 2.0 ** -16, 2.0 ** -8).to(hi.device, torch.float64)
            bound = rel[:, None] * exp.abs() + err
    diff = (got - exp).abs()
    excess = diff - bound
    k = int(torch.argmax(excess))
    r, c = divmod(k, exp.shape[1])
    assert float(excess.flatten()[k]) <= 0, (
        f"{where}: row {r} col {c}: got {float(got[r, c])!r}, float64 {float(exp[r, c])!r}, "
        f"|diff| {float(diff[r, c]):.3e} > bound {float(bound[r, c]):.3e}")
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.zeros_like(diff))
    return float(ratio.max())


@functools.lru_cache(maxsize=8)
def _reference(cfg_key, N, T):
    """forward_numpy's activations on a few windows (first, last, spread)."""
    cfg = dict(cfg_key)
    cfg["fw"] = list(cfg["fw"])
    sd = _state_dict(cfg_key)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1)
    idx = sorted(set([0, N - 1] + list(range(0, N, max(1, N // 3)))))[:6]
    strided = cfg["cls"] == OPT or (not cfg["dense"] and T == orc.arch(cfg["fw"])["receptive_field"])
    acts = []
    orc.forward_numpy(sd, x[idx].numpy(), cfg["fw"], causal=cfg["causal"], dense=cfg["dense"],
                      strided=strided, collect=acts)
    return idx, acts


@functools.lru_cache(maxsize=4)
def _state_dict(cfg_key):
    cfg = dict(cfg_key)
    return orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], list(cfg["fw"]), cfg["C"],
                               dense=cfg["dense"], seed=0)


def _key(cfg):
    return tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in cfg.items()))


@pytest.mark.parametrize("case,cfg,N,T,precision", PARAMS)
def test_eval_layers(cuda_device, case, cfg, N, T, precision):
    cfg, N = _resolve(cfg, N)
    sd = _state_dict(_key(cfg))
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device, precision)
    with torch.no_grad():
        y = m(x)
        torch.cuda.synchronize()
        launches = m.last_launch_count()
        rep = er.replay(sd, cfg, x, precision, er.gpu_gemm)
    plan = rep.plan
    if case.startswith("wave_"):
        conv1 = rep.launches[1]
        assert conv1.name == "block 1 conv 1"
        tiles = -(-conv1.desc["out_rows"] // er.BLOCK_M) * (plan.C // conv1.block_n)
        sms = _num_sms()
        assert {"wave_full": tiles % sms == 0 and conv1.block_n == 128,
                "wave_plus1": tiles % sms == 1 and conv1.block_n == 128,
                "wave_narrow": conv1.block_n == 64}[case]

    # 1. per layer, against float64 on the layer's own inputs
    worst = (0.0, None)
    for lc in rep.launches:
        ratio = _check_launch(lc, plan, f"{case}-{precision}")
        worst = max(worst, (ratio, lc.name))
    prev = WORST.get(precision, (0.0, None, None))
    if worst[0] > prev[0]:
        WORST[precision] = (worst[0], case, worst[1])
    print(f"\n{case}-{precision}: N={N} T={T} strided={plan.strided} x3={plan.x3} "
          f"worst per-layer error {worst[0]:.3f} of its bound ({worst[1]}); "
          f"worst so far for {precision}: {WORST[precision]}")

    # 2. the replay is the plan: same bits, same launch count
    assert rep.launch_count == launches
    assert rep.y.shape == y.shape
    assert torch.equal(rep.y.view(torch.int32), y.view(torch.int32)), (
        f"replay differs from model(x) in {int((rep.y != y).sum())} of {y.numel()} outputs")

    # 3. layout against the reference algorithm
    idx, ref_acts = _reference(_key(cfg), N, T)
    for k, ref in enumerate(ref_acts):
        got = rep.activation(k)[idx].cpu().numpy()
        ref = ref[:, :got.shape[1]]
        scale = max(float(np.abs(ref).max()), 1e-30)
        err = float(np.abs(got - ref).max()) / scale
        assert err <= LAYOUT_TOL[precision], f"{case}-{precision}: {rep.acts[k][0]} {err:.2e} of scale"
