"""GPU: the 'int8' eval precision -- u8 activations times s8 weights on the integer tensor cores.

1. GEMM: vp3d_conv_gemm with precision INT8 on random u8 / s8 operands, both geometries, both tile
   widths, both schedules (cooperative / ping-pong), with and without the residual, writing u8 alone
   or fp16 [+ u8]; and the fp16 GEMM with a u8 second output.  The int32 sums are exact and the int8
   epilogue a fixed chain of fp32 operations (eval_replay.int8_epilogue), so the int8 launches
   equal its restatement bit for bit; the fp16 GEMM, whose fp32 accumulation order is not
   restated, stays within one fp16 rounding and one code.  The number of elements that are not
   bit-identical is printed.
2. Calibration: amax equals, exactly, the maximum of every fp16 activation the fp16 forward stores
   (the fp16 replay of eval_replay, tied to model(x) bit for bit), and repeats bit for bit.
3. Model: model(x) in int8 against int8_oracle.forward_int8 (same calibration) and against the
   float64 forward within int8_oracle's gate; repeated runs are bit-identical.
4. Persistence, staleness, the int32 bound of the dense ablation, eval autograd and streaming.
"""
import ctypes

import numpy as np
import pytest
import torch

import eval_replay as er
import int8_oracle as io
from gpu_utils import expected_conv
from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"
GATE = 1e-2          # int8_oracle vs float64 (tests/test_int8_cpu.py)
ORACLE_TOL = 2e-3    # model vs int8_oracle: fp32 vs float64 epilogues flip single codes


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


def _build(cfg, sd, dev):
    kw = dict(filter_widths=cfg["fw"], causal=cfg["causal"], dropout=0.0, channels=cfg["C"])
    if cfg["cls"] == TM:
        m = vp.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], dense=cfg["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(cfg["J"], cfg["F"], cfg["Jout"], **kw)
    m.load_state_dict(sd)
    return m.to(dev).eval()


# ------------------------------------------------------------------------------ 1. GEMM
def _launch(a, samples, a_rows, a_ld, w, taps, k_pad, n_pad, *, per_sample, tap_row_step, out_rows,
            precision, scale, shift, res=None, res_rows_per_sample=0, res_row_off=0, out=None,
            out_u8=None, inv_s=1.0):
    d = _capi.ConvDesc()
    d.a = a.data_ptr(); d.a_planes = 1; d.samples = samples; d.a_rows = a_rows; d.a_ld = a_ld
    d.w = w.data_ptr(); d.taps = taps; d.k_per_tap = k_pad; d.n_pad = n_pad
    d.per_sample_tiles = int(per_sample); d.tap_row_step = tap_row_step; d.out_rows = out_rows
    d.precision = precision; d.scale = scale.data_ptr(); d.shift = shift.data_ptr(); d.relu = 1
    if res is not None:
        d.res = res.data_ptr(); d.res_planes = 1; d.res_ld = res.shape[-1]
        d.res_plane_stride = res.numel(); d.res_rows_per_sample = res_rows_per_sample
        d.res_row_step = 1; d.res_row_off = res_row_off
    if out is not None:
        d.out = out.data_ptr(); d.out_planes = 1; d.out_ld = out.shape[-1]
        d.out_plane_stride = out.numel()
    if out_u8 is not None:
        d.out_u8 = out_u8.data_ptr(); d.out_u8_ld = out_u8.shape[-1]; d.out_u8_inv_scale = inv_s
    _capi.check(_capi.load().vp3d_conv_gemm(ctypes.byref(d), torch.cuda.current_stream().cuda_stream),
                "vp3d_conv_gemm")
    torch.cuda.synchronize()


def _epilogue(acc, scale, shift):
    """fp32 epilogue of the fp16 GEMM on its float64 sums: max(fp32(acc) * scale + shift, 0)."""
    return (acc.float().double() * scale.double() + shift.double()).float().clamp_min(0)


# (id, per_sample, samples, a_rows, out_rows, taps, step, c_in, n_pad, res, u8, int8)
GEMMS = [
    ("dil_h_c129_n64", True, 6, 150, 140, 3, 5, 129, 192, False, True, True),
    ("dil_x_q_n128", True, 40, 130, 128, 1, 0, 256, 256, True, True, True),
    ("dil_x_last", True, 7, 90, 90, 1, 0, 96, 128, True, False, True),
    ("flat_h_pp", False, 1, 3 * 17000, 17000, 3, 17000, 1024, 1024, False, True, True),
    ("flat_x_q_pp", False, 1, 17000, 17000, 1, 0, 1024, 1024, True, True, True),
    ("flat_x_pp_c192", False, 1, 30000, 30000, 1, 0, 192, 192, True, False, True),
    ("expand_fp16_u8", True, 5, 120, 118, 3, 1, 64, 128, False, True, False),
    ("expand_fp16_u8_pp", False, 1, 20000, 20000, 1, 0, 128, 1024, False, True, False),
]


@pytest.mark.parametrize("g", GEMMS, ids=[g[0] for g in GEMMS])
def test_int8_gemm(cuda_device, g):
    name, per_sample, S, a_rows, out_rows, taps, step, c_in, n_pad, has_res, u8, int8 = g
    dev = cuda_device
    gen = torch.Generator(device="cpu").manual_seed(sum(map(ord, name)))
    a_ld = -(-c_in // 64) * 64
    rows_out = S * out_rows if per_sample else out_rows
    if int8:
        k_pad = -(-a_ld // 128) * 128
        a = torch.randint(0, 256, (S * a_rows, a_ld), generator=gen, dtype=torch.uint8)
        a[:, c_in:] = 0
        w = torch.randint(-127, 128, (taps, n_pad, k_pad), generator=gen, dtype=torch.int8)
        w[:, :, c_in:] = 0
        scale = torch.rand(n_pad, generator=gen) * 2e-5
        precision = _capi.VP3D_PRECISION_INT8
    else:
        k_pad = a_ld
        a = (torch.rand(S * a_rows, a_ld, generator=gen) * 2 - 1).half()
        w = (torch.randn(taps, n_pad, k_pad, generator=gen) * 0.1).half()
        a_val, w_val = a.double(), w.double()
        scale = torch.rand(n_pad, generator=gen) + 0.5
        precision = _capi.VP3D_PRECISION_FP16
    shift = torch.randn(n_pad, generator=gen) * 0.3
    res = None
    if has_res:   # residual rows 1.. of a sample (per-sample tiles) / the rows themselves (flat)
        res_rows = out_rows + (2 if per_sample else 0)
        res = (torch.rand(S * res_rows, n_pad, generator=gen) * 2).half().to(dev)
    a, w, scale, shift = a.to(dev), w.to(dev), scale.to(dev).float(), shift.to(dev).float()
    if int8:   # the exact restatement: integer sums, then the kernel's fp32 operations
        desc = er.new_desc(a_planes=1, samples=S, a_rows=a_rows, a_ld=a_ld, taps=taps,
                           k_per_tap=k_pad, n_pad=n_pad, per_sample_tiles=int(per_sample),
                           tap_row_step=step, out_rows=out_rows, precision=er.K_INT8, relu=1,
                           res_planes=1, res_rows_per_sample=out_rows + 2 if per_sample else 0,
                           res_row_step=1, res_row_off=1 if per_sample else 0)
        lc = er.Launch(name, desc, a.unsqueeze(0), w, scale, shift,
                       res=res.unsqueeze(0) if has_res else None)
        v = er.fake_conv(lc)[0].float()
    else:
        acc = expected_conv(a_val.to(dev), w_val.to(dev), samples=S, a_rows=a_rows, taps=taps,
                            k_per_tap=a_ld, per_sample_tiles=per_sample, tap_row_step=step,
                            tap_col_step=0, out_rows=out_rows)
        v = _epilogue(acc, scale, shift)
    inv_s = float(np.float32(255.0) / np.float32(float(v.max()) * 0.9))
    out = torch.full((rows_out, n_pad), float("nan"), dtype=torch.float16, device=dev) \
        if (has_res or not int8) else None
    q = torch.full((rows_out, n_pad), 7, dtype=torch.uint8, device=dev) if u8 else None
    _launch(a, S, a_rows, a_ld, w, taps, k_pad, n_pad, per_sample=per_sample, tap_row_step=step,
            out_rows=out_rows, precision=precision, scale=scale, shift=shift, res=res,
            res_rows_per_sample=out_rows + 2 if per_sample else 0,
            res_row_off=1 if per_sample else 0, out=out, out_u8=q, inv_s=inv_s)
    report = [name]
    if int8:
        exact = []
        if out is not None:
            exp = v.clamp(-er.FP16_MAX, er.FP16_MAX).half()
            exact.append(("fp16", out.view(torch.int16), exp.view(torch.int16)))
        if q is not None:
            exact.append(("u8", q, er.quant_u8(v, np.float32(inv_s))))
        for fmt, got, exp in exact:
            report.append(f"{fmt} {int((got != exp).sum())}/{got.numel()} not bit-identical")
        print("\n" + ", ".join(report))
        for fmt, got, exp in exact:
            assert torch.equal(got, exp), \
                f"{name}: {fmt} output differs from the exact int8 epilogue in {int((got != exp).sum())}"
        return
    if out is not None:
        exp = v.half()
        # one fp16 rounding (of a value the kernel may round differently in its last fp32 bit);
        # the fp16 GEMM also accumulates in fp32: up to K * 2^-24 of sum |a| |w|, scaled
        bound = 2.0 ** -11 * (v.abs().double() + exp.abs().double()) + 2.0 ** -24
        acc_abs = expected_conv(a_val.abs().to(dev), w_val.abs().to(dev), samples=S,
                                a_rows=a_rows, taps=taps, k_per_tap=a_ld,
                                per_sample_tiles=per_sample, tap_row_step=step,
                                tap_col_step=0, out_rows=out_rows)
        bound = bound + taps * a_ld * 2.0 ** -24 * acc_abs * scale.double()
        diff = (out.double() - exp.double()).abs()
        assert not torch.isnan(out).any(), f"{name}: rows left unwritten"
        assert bool((diff <= bound).all()), \
            f"{name}: fp16 output off by more than one rounding (max {float(diff.max()):.3e})"
        report.append(f"fp16 {int((out != exp).sum())}/{out.numel()} not bit-identical")
    if q is not None:
        qe = (v * np.float32(inv_s)).float().round().clamp(0, 255)
        dq = (q.double() - qe.double()).abs()
        assert float(dq.max()) <= 1, f"{name}: u8 output off by {float(dq.max())} codes"
        report.append(f"u8 {int((dq > 0).sum())}/{q.numel()} not bit-identical")
    print("\n" + ", ".join(report))


# ------------------------------------------------------------------------------ 2-3. model
BENCH = _cfg(TM, [3, 3, 3, 3, 3], 1024)
MODELS = [  # (id, cfg, N, T)
    ("bench_cone_n256", BENCH, 256, 243),
    ("bench_dilated_t250", BENCH, 16, 250),
    ("opt_333_c64", _cfg(OPT, [3, 3, 3], 64), 300, 27),
    ("opt_35_c128_causal", _cfg(OPT, [3, 5], 128, causal=True), 200, 15),
    ("tm_333_causal_dilated", _cfg(TM, [3, 3, 3], 64, causal=True), 24, 90),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 24, 60),
    ("tm_353_c96_cone", _cfg(TM, [3, 5, 3], 96), 200, 45),
    ("tm_53_c129_dilated", _cfg(TM, [5, 3], 129), 16, 100),
    ("tm_333_j15_f3", _cfg(TM, [3, 3, 3], 64, J=15, F=3, Jout=15), 300, 27),
    ("tm_353_traj", _cfg(TM, [3, 5, 3], 128, Jout=1), 16, 120),
    ("tm_333333_c64", _cfg(TM, [3, 3, 3, 3, 3, 3], 64), 8, 729),
]


def _strided(cfg, T):
    return cfg["cls"] == OPT or (not cfg["dense"] and T == orc.arch(cfg["fw"])["receptive_field"])


@pytest.mark.parametrize("case,cfg,N,T", MODELS, ids=[c[0] for c in MODELS])
def test_int8_model(cuda_device, case, cfg, N, T):
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"],
                             dense=cfg["dense"], seed=0)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    amax = m.int8_calibration()
    assert amax.shape == (2 * (len(cfg["fw"]) - 1),)
    # 2. exactly the maxima of the fp16 forward's stored activations, reproducibly
    with torch.no_grad():
        rep = er.replay(sd, cfg, x, "fp16", er.gpu_gemm)
    exp = torch.tensor([float(buf[0].float().max()) for _, _, buf in rep.acts[:len(amax)]])
    assert torch.equal(amax, exp), f"{case}: amax {amax.tolist()} != {exp.tolist()}"
    assert torch.equal(_build(cfg, sd, cuda_device).calibrate_int8([x[: N // 2], x[N // 2:]])
                       .int8_calibration().view(torch.int32), amax.view(torch.int32))
    # 3. the model against the restatement and the float64 forward; run to run bit-identical
    m.set_precision("int8")
    with torch.no_grad():
        y = m(x)
        y2 = m(x)
    assert torch.equal(y.view(torch.int32), y2.view(torch.int32))
    kw = dict(causal=cfg["causal"], dense=cfg["dense"], strided=_strided(cfg, T))
    xn = x.cpu().numpy()
    ref = orc.forward_numpy(sd, xn, cfg["fw"], **kw)
    y_or = io.forward_int8(sd, xn, cfg["fw"], amax.numpy(), **kw)
    yn = y.cpu().numpy()
    scale = np.abs(ref).max()
    e_or = float(np.abs(yn - y_or).max() / scale)
    e_ref = float(np.abs(yn - ref).max() / scale)
    print(f"\n{case}: int8 vs restatement {e_or:.2e}, vs float64 {e_ref:.2e} "
          f"({m.last_launch_count()} launches)")
    assert e_or <= ORACLE_TOL and e_ref <= GATE


# ------------------------------------------------------------------------------ 4. API
def _small(dev):
    cfg = _cfg(TM, [3, 3, 3], 128)
    sd = orc.make_state_dict(17, 2, 17, cfg["fw"], 128, seed=0)
    return cfg, sd, orc.make_input(12, 60, seed=1).to(dev)


def test_int8_persistence_and_staleness(cuda_device):
    cfg, sd, x = _small(cuda_device)
    m = _build(cfg, sd, cuda_device).set_precision("int8")
    with pytest.raises(RuntimeError, match="calibrate_int8"):
        m(x)
    m.calibrate_int8(x)
    with torch.no_grad():
        y = m(x)
    saved = m.int8_calibration()
    m2 = _build(cfg, sd, cuda_device).set_precision("int8").load_int8_calibration(saved)
    with torch.no_grad():
        assert torch.equal(m2(x), y)
    # an optimizer step changes the parameters: the calibration is stale until renewed
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    for p in m.parameters():
        p.grad = torch.full_like(p, 1e-3)
    opt.step()
    with pytest.raises(RuntimeError, match="stale"):
        with torch.no_grad():
            m(x)
    m.calibrate_int8(x)
    with torch.no_grad():
        y3 = m(x)
    assert torch.isfinite(y3).all() and not torch.equal(y3, y)
    m2.load_state_dict(m.state_dict())
    with pytest.raises(RuntimeError, match="stale"):
        with torch.no_grad():
            m2(x)
    m2.load_int8_calibration(m.int8_calibration())
    with torch.no_grad():
        assert torch.equal(m2(x), y3)
    m2.invalidate()
    with pytest.raises(RuntimeError, match="stale"):
        with torch.no_grad():
            m2(x)


def test_int8_dense_overflow_bound(cuda_device):
    m = vp.TemporalModel(17, 2, 17, [3, 3, 3, 3, 3], dense=True, channels=1024).to(cuda_device).eval()
    m.set_precision("int8").load_int8_calibration(torch.ones(8))
    with pytest.raises(NotImplementedError, match="overflow"):
        with torch.no_grad():
            m(orc.make_input(1, 243, seed=1).to(cuda_device))


def test_int8_eval_autograd_and_streaming(cuda_device):
    cfg, sd, x = _small(cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    grads = {}
    for precision in ("fp16", "int8"):
        m.set_precision(precision)
        with torch.no_grad():
            y_ng = m(x)
        xg = x.clone().requires_grad_(True)
        y = m(xg)
        assert torch.equal(y, y_ng)
        y.backward(torch.ones_like(y))
        grads[precision] = xg.grad
    assert torch.equal(grads["fp16"], grads["int8"])
    with pytest.raises(NotImplementedError, match="int8"):
        m.streaming(2)


# ------------------------------------------------------------------------------ 1b. packs
PACKS = [  # (id, cfg, N, T)
    ("tm_53_c129", _cfg(TM, [5, 3], 129), 4, 100),
    ("tm_33_dense_c64", _cfg(TM, [3, 3], 64, dense=True), 4, 60),
    ("bench_c1024", BENCH, 4, 243),
]


@pytest.mark.parametrize("case,cfg,N,T", PACKS, ids=[c[0] for c in PACKS])
def test_int8_packs_exact(cuda_device, case, cfg, N, T):
    """The s8 weights, their scales and every layer's folded scale' read back from the plan equal
    int8_oracle's fp32 formulas bit for bit, with the layer's own input scale."""
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"],
                             dense=cfg["dense"], seed=0)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x).set_precision("int8")
    with torch.no_grad():
        m(x)
    torch.cuda.synchronize()
    s_act, _ = io.act_scales(m.int8_calibration().numpy())
    C = cfg["C"]
    n_pad = -(-C // 64) * 64
    k_pad = -(-n_pad // 128) * 128
    lib = _capi.load()
    stream = torch.cuda.current_stream().cuda_stream
    for layer in range(2 * (len(cfg["fw"]) - 1)):
        taps = sd[f"layers_conv.{layer}.weight"].shape[2]
        w8 = torch.empty(taps, n_pad, k_pad, dtype=torch.int8, device=cuda_device)
        ws = torch.empty(n_pad, dtype=torch.float32, device=cuda_device)
        qs = torch.empty(n_pad, dtype=torch.float32, device=cuda_device)
        _capi.check(lib.vp3d_int8_packs(m._plan, layer, w8.data_ptr(), ws.data_ptr(),
                                        qs.data_ptr(), stream), "vp3d_int8_packs")
        torch.cuda.synchronize()
        sc, _, wq = io.int8_affine(sd, layer, s_act[layer])
        _, ws_exp = io.quant_weight(sd[f"layers_conv.{layer}.weight"].numpy())
        w_exp = np.zeros((taps, n_pad, k_pad), np.int8)
        w_exp[:, :C, :C] = wq.transpose(2, 0, 1).astype(np.int8)
        ws_full = np.ones(n_pad, np.float32)
        ws_full[:C] = ws_exp
        qs_full = np.zeros(n_pad, np.float32)
        qs_full[:C] = sc
        assert np.array_equal(w8.cpu().numpy(), w_exp), f"{case}: s8 pack of layer {layer}"
        assert np.array_equal(ws.cpu().numpy().view(np.int32), ws_full.view(np.int32)), \
            f"{case}: weight scales of layer {layer}"
        assert np.array_equal(qs.cpu().numpy().view(np.int32), qs_full.view(np.int32)), \
            f"{case}: scale' of layer {layer}"
