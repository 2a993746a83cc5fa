"""GPU: the 'int8' eval forward layer by layer -- every u8 x s8 GEMM bit for bit against exact integer
sums, and the schedule restated in Python (eval_replay.py, precision "int8") tied to model(x).

Each case calibrates the model (``calibrate_int8``), runs ``y = model(x)`` in int8, then replays the
same launch schedule through ``vp3d_conv_gemm`` and asserts:
1. the replay's s8 packs and folded scales are the plan's (``vp3d_int8_packs``);
2. per int8 GEMM (both convs of every block): H, X_i and Q_i equal, bit for bit, the exact
   restatement on the layer's own kernel-produced u8 input and fp16 residual -- int32 sums, exact in
   float64, then the kernel's fp32 chain fmaxf(fmaf(fp32(acc), scale', shift), 0) [+ residual],
   cvt.rn.satfinite to fp16 and cvt.rni.sat.u8(v * inv_s).  Padding channels [c_real, C) are 0 in
   fp16 and u8; every row is written: the GEMM is run again into a buffer prefilled with 0x00
   instead of 0xFF (u8 has no NaN) and must give the same bytes;
3. the fp16 expand: X_0 within the bound of test_gpu_eval_layers, and Q_0 between the codes of the
   two ends of X_0's fp16 rounding interval (the kernel's fp32 value itself is not observable);
   the shrink within its fp32 bound;
4. the replay's output equals model(x) bit for bit, with as many launches (3 + 2 B);
5. the replay's activations, mapped back to (N, L, C), against int8_oracle.forward_int8 on a few
   windows: a gate that only a layout error exceeds.
The count of non-identical elements of each int8 GEMM is printed before anything is asserted.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

import eval_replay as er
import int8_oracle as io
from oracle import temporal_model_oracle as orc
from test_gpu_eval_layers import _check_launch, _num_sms, _wave_case
import videopose3d_b200 as vp
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"
LAYOUT_TOL = 2e-2    # of each activation's scale: codes 5 apart, a layout error is O(1)


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


BENCH = _cfg(TM, [3, 3, 3, 3, 3], 1024)
# (id, cfg | wave kind, N, T, kind): kind "saturate" calibrates on 0.5 x and runs on x; "zero"
# drives block 1's H to zero (layers_bn.0's bias far below its pre-activations: amax 0, s = 1)
CASES = [
    ("bench_cone_n256", BENCH, 256, 243, None),
    ("bench_dilated_t250", BENCH, 16, 250, None),
    ("wave_full", "full", None, 27, None),
    ("wave_plus1", "plus1", None, 27, None),
    ("wave_narrow", "narrow", None, 27, None),
    ("opt_333_c64_t27", _cfg(OPT, [3, 3, 3], 64), 300, 27, None),
    ("opt_35_c128_causal", _cfg(OPT, [3, 5], 128, causal=True), 200, 15, None),
    ("tm_333_causal_dilated", _cfg(TM, [3, 3, 3], 64, causal=True), 24, 90, None),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 24, 60, None),
    ("tm_353_c96_cone", _cfg(TM, [3, 5, 3], 96), 200, 45, None),
    ("tm_53_c129_dilated", _cfg(TM, [5, 3], 129), 16, 100, None),
    ("tm_333_c129_cone", _cfg(TM, [3, 3, 3], 129), 200, 27, None),
    ("tm_333_j15_f3", _cfg(TM, [3, 3, 3], 64, J=15, F=3, Jout=15), 300, 27, None),
    ("tm_353_traj", _cfg(TM, [3, 5, 3], 128, Jout=1), 16, 120, None),
    ("tm_333333_c64", _cfg(TM, [3, 3, 3, 3, 3, 3], 64), 8, 729, None),
    ("tm_333_c320_dilated", _cfg(TM, [3, 3, 3], 320), 16, 300, None),
    ("tm_333_c128_saturate", _cfg(TM, [3, 3, 3], 128), 24, 60, "saturate"),
    ("tm_333_c128_zero_layer", _cfg(TM, [3, 3, 3], 128), 24, 60, "zero"),
]


def _resolve(cfg, N):
    if isinstance(cfg, str):
        C, N = _wave_case(cfg)
        return _cfg(TM, [3, 3, 3], C), N
    return cfg, N


def _key(cfg):
    return tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in cfg.items()))


@functools.lru_cache(maxsize=2)
def _state_dict(cfg_key, kind):
    cfg = dict(cfg_key)
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], list(cfg["fw"]), cfg["C"],
                             dense=cfg["dense"], seed=0)
    if kind == "zero":
        sd["layers_bn.0.bias"] = torch.full_like(sd["layers_bn.0.bias"], -1e3)
    return sd


def _build(cfg, sd, dev):
    kw = dict(filter_widths=cfg["fw"], causal=cfg["causal"], dropout=0.0, channels=cfg["C"])
    if cfg["cls"] == TM:
        m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], dense=cfg["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(cfg["J"], cfg["F"], cfg["Jout"], **kw)
    m.load_state_dict(sd)
    return m.to(dev).eval()


def _check_packs(m, rep, case):
    """The replay's s8 packs and scale' (int8_oracle's formulas) are the plan's own."""
    lib = _capi.load()
    stream = torch.cuda.current_stream().cuda_stream
    int8_launches = [lc for lc in rep.launches if lc.desc["precision"] == er.K_INT8]
    assert len(int8_launches) == 2 * rep.plan.nb
    for layer, lc in enumerate(int8_launches):
        w8 = torch.empty_like(lc.w)
        qs = torch.empty_like(lc.scale)
        _capi.check(lib.vp3d_int8_packs(m._plan, layer, w8.data_ptr(), None, qs.data_ptr(),
                                        stream), "vp3d_int8_packs")
        torch.cuda.synchronize()
        assert torch.equal(w8, lc.w), f"{case}: s8 pack of layer {layer} ({lc.name})"
        assert torch.equal(qs.view(torch.int32), lc.scale.view(torch.int32)), \
            f"{case}: scale' of layer {layer} ({lc.name})"


def _rerun_zero_filled(lc):
    """Launch lc again into fresh outputs, the u8 one prefilled with 0x00; returns (out, out_u8)."""
    again = er.Launch(lc.name, lc.desc, lc.a, lc.w, lc.scale, lc.shift, res=lc.res,
                      out=None if lc.out is None else torch.empty_like(lc.out),
                      out_u8=torch.zeros_like(lc.out_u8), inv_s=lc.inv_s)
    er.gpu_gemm(again)
    return again.out, again.out_u8


def _check_u8_rows(lc, where):
    """Every row of the u8 output (and the fp16 one) is written: a second run into a 0x00-filled
    buffer gives the bytes of the first run, which started from 0xFF."""
    out0, q0 = _rerun_zero_filled(lc)
    assert torch.equal(q0, lc.out_u8), \
        f"{where}: u8 bytes depend on the buffer's fill ({int((q0 != lc.out_u8).sum())} differ)"
    if lc.out is not None:
        assert torch.equal(out0.view(torch.int16), lc.out.view(torch.int16)), \
            f"{where}: fp16 output differs between two runs"


def _check_int8(lc, plan, where):
    """Assertion 2 for one int8 launch; returns the count of codes that saturate (v inv_s > 255.5)."""
    v, _ = er.fake_conv(lc)
    assert not torch.isnan(v).any(), f"{where}: reads a NaN (a residual row nobody wrote)"
    v32 = v.float()
    report = [where]
    bad = []
    if lc.out is not None:
        exp = v32.clamp(-er.FP16_MAX, er.FP16_MAX).half()
        got = lc.out[0]
        n = int((got.view(torch.int16) != exp.view(torch.int16)).sum())
        report.append(f"fp16 {n}/{got.numel()} not bit-identical")
        bad.append(("fp16", n, got, exp))
    if lc.out_u8 is not None:
        exp = er.quant_u8(v32, lc.inv_s)
        got = lc.out_u8[0]
        n = int((got != exp).sum())
        report.append(f"u8 {n}/{got.numel()} not bit-identical")
        bad.append(("u8", n, got, exp))
    print(", ".join(report))
    for fmt, n, got, exp in bad:
        if n:
            k = int(torch.nonzero((got != exp).flatten())[0])
            r, c = divmod(k, got.shape[1])
            pytest.fail(f"{where}: {n} {fmt} elements differ from the exact restatement; first at "
                        f"row {r} col {c}: got {got[r, c].item()!r}, exact {exp[r, c].item()!r} "
                        f"(fp32 value {float(v32[r, c])!r}, inv_s {lc.inv_s!r})")
    for _, _, got, _ in bad:
        assert (got[:, plan.c_real:] == 0).all(), f"{where}: padding channels not zero"
    if lc.out_u8 is None:   # (an fp16 row nobody wrote is NaN, which the comparison caught)
        return 0
    _check_u8_rows(lc, where)
    return int((v32 * torch.tensor(lc.inv_s, device=v32.device) > 255.5).sum())


def _check_q0(lc, plan, where):
    """Q_0 of the fp16 expand against X_0: the kernel rounds one fp32 value v to both, so v lies in
    X_0's fp16 rounding interval [midpoint below, midpoint above] (closed: ties go to even) and
    Q_0 between the codes of its two ends (the product and the rounding are monotonic)."""
    xh = lc.out[0].cpu().numpy()
    x64 = xh.astype(np.float64)
    lo = (x64 + np.nextafter(xh, np.float16(-np.inf)).astype(np.float64)) / 2
    hi = (x64 + np.nextafter(xh, np.float16(np.inf)).astype(np.float64)) / 2   # (65504: inf)
    q_lo = er.quant_u8(torch.from_numpy(np.maximum(lo, 0.0)).float(), lc.inv_s)
    q_hi = er.quant_u8(torch.from_numpy(hi).float(), lc.inv_s)
    q = lc.out_u8[0].cpu()
    n = int(((q < q_lo) | (q > q_hi)).sum())
    print(f"{where}: u8 {n}/{q.numel()} outside the codes of X_0's rounding interval, "
          f"{int((q_lo != q_hi).sum())} intervals span two codes")
    assert n == 0, f"{where}: Q_0 inconsistent with X_0 in {n} elements"
    assert (q[:, plan.c_real:] == 0).all(), f"{where}: padding channels of Q_0 not zero"
    _check_u8_rows(lc, where)


@functools.lru_cache(maxsize=4)
def _reference(cfg_key, kind, N, T, amax_bytes, strided):
    """int8_oracle.forward_int8's activations on a few windows (first, middle, last)."""
    cfg = dict(cfg_key)
    sd = _state_dict(cfg_key, kind)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1)
    idx = sorted({0, N // 2, N - 1})
    acts = []
    io.forward_int8(sd, x[idx].numpy(), list(cfg["fw"]), np.frombuffer(amax_bytes, np.float32),
                    causal=cfg["causal"], dense=cfg["dense"], strided=strided, collect=acts)
    return idx, [a for a in acts if a is not None]


@pytest.mark.parametrize("case,cfg,N,T,kind", CASES, ids=[c[0] for c in CASES])
def test_eval_layers_int8(cuda_device, case, cfg, N, T, kind):
    cfg, N = _resolve(cfg, N)
    sd = _state_dict(_key(cfg), kind)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(0.5 * x if kind == "saturate" else x)
    amax = m.int8_calibration()
    m.set_precision("int8")
    with torch.no_grad():
        y = m(x)
        torch.cuda.synchronize()
        launches = m.last_launch_count()
        rep = er.replay(sd, cfg, x, er.INT8, er.gpu_gemm, amax=amax.numpy())
    plan = rep.plan
    _check_packs(m, rep, case)

    sms = _num_sms()
    if case.startswith("wave_"):
        conv1 = rep.launches[1]
        assert conv1.name == "block 1 conv 1"
        assert {"wave_full": conv1.tiles % sms == 0 and conv1.block_n == 128,
                "wave_plus1": conv1.tiles % sms == 1 and conv1.block_n == 128 and conv1.pingpong,
                "wave_narrow": conv1.block_n == 64}[case]
    if "c320" in case:   # five 64-wide N blocks over the two ping-pong warpgroups
        assert all(lc.block_n == 64 and lc.pingpong for lc in rep.launches[1:-1])
    if kind == "zero":
        assert float(amax[1]) == 0.0 and rep.launches[1].inv_s == 1.0
        assert not rep.launches[1].out_u8.any(), f"{case}: block 1's H is not all zero"

    # 2-3. per layer
    saturated = 0
    for lc in rep.launches:
        int8 = lc.desc["precision"] == er.K_INT8
        sched = ("ping-pong, " if lc.pingpong else "cooperative, ") \
            if int8 or lc.out_u8 is not None else ""
        where = (f"{case}: {lc.name} (block_n={lc.block_n}, {sched}{lc.desc['out_rows']} rows x "
                 f"{lc.desc['n_pad']}, k_per_tap {lc.desc['k_per_tap']})")
        if int8:
            saturated += _check_int8(lc, plan, where)
        else:
            _check_launch(lc, plan, case)
            if lc.out_u8 is not None:
                _check_q0(lc, plan, where)
    print(f"{case}: N={N} T={T} strided={plan.strided} amax={amax.tolist()} "
          f"saturated codes {saturated}")
    if kind == "saturate":
        assert saturated > 0, f"{case}: no code saturates"

    # 4. the replay is the plan: same bits, same launch count
    assert rep.launch_count == launches == 3 + 2 * plan.nb
    assert rep.y.shape == y.shape
    assert torch.equal(rep.y.view(torch.int32), y.view(torch.int32)), (
        f"replay differs from model(x) in {int((rep.y != y).sum())} of {y.numel()} outputs")

    # 5. layout against the restatement of the algorithm
    idx, ref_acts = _reference(_key(cfg), kind, N, T, amax.numpy().tobytes(), plan.strided)
    assert len(ref_acts) == len(rep.acts)
    for k, ref in enumerate(ref_acts):
        got = rep.activation(k)[idx].cpu().numpy()
        ref = ref[:, :got.shape[1]]
        scale = max(float(np.abs(ref).max()), 1e-30)
        err = float(np.abs(got - ref).max()) / scale
        assert err <= LAYOUT_TOL, f"{case}: {rep.acts[k][0]} {err:.2e} of scale"
