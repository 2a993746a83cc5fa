"""GPU: int8 on a chosen set of residual blocks (``set_int8_blocks``), the other blocks in fp16.

1. No int8 block is the fp16 precision, bit for bit; None and the full list are the default int8.
2. Per block set, layer by layer against the replay of the mixed schedule (int8_blocks_replay): every u8 x s8 GEMM bit for bit against the exact integer restatement, every
   fp16 GEMM within the fp16 bound of test_gpu_eval_layers, the plan's s8 packs and scales (and the
   refusal of vp3d_int8_packs for an fp16 block's layer), the quantise pass's Q_i bit for bit against
   NumPy on the model's stored fp16 X_i, and the model's output equal to the replay's with as many
   launches.
3. Changing the set after a forward equals a fresh model built with that set; predict() and the
   eval autograd forward inherit the set.
4. vp3d_set_int8_blocks refusals and the stale-pack state after a change.
"""
import ctypes

import numpy as np
import pytest
import torch

import eval_replay as er
from int8_blocks_replay import replay_blocks
from oracle import temporal_model_oracle as orc
from test_gpu_eval_layers import _check_launch
from test_gpu_eval_layers_int8 import TM, OPT, _build, _cfg, _check_int8, _check_q0
from test_gpu_predict import _clips, _offline, _predict
import videopose3d_b200 as vp
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

# (id, cfg, N, T): C = 64 is the K-padding case (u8 x s8 K per tap 128, fp16 64)
CASES = [
    ("tm_3333_c64_dilated", _cfg(TM, [3, 3, 3, 3], 64), 8, 120),
    ("opt_3333_c100_causal", _cfg(OPT, [3, 3, 3, 3], 100, causal=True), 64, 81),
    ("tm_3333_c1024_causal", _cfg(TM, [3, 3, 3, 3], 1024, causal=True), 4, 100),
]
# every single block and two mixed sets
SETS = [[1], [2], [3], [1, 3], [2, 3]]


def _data(cfg, N, T, dev):
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"], seed=0)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).to(dev)
    return sd, x


def _run(m, x):
    with torch.no_grad():
        y = m(x)
    torch.cuda.synchronize()
    return y


def _bits(y):
    return y.view(torch.int32)


@pytest.mark.parametrize("case,cfg,N,T", CASES, ids=[c[0] for c in CASES])
def test_no_block_is_fp16_and_all_is_int8(cuda_device, case, cfg, N, T):
    sd, x = _data(cfg, N, T, cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    y16 = _run(m.set_precision("fp16"), x)
    n16 = m.last_launch_count()
    y8 = _run(m.set_precision("int8"), x)
    assert not torch.equal(y8, y16)
    nb = len(cfg["fw"]) - 1
    for blocks in (None, list(range(1, nb + 1))):
        assert torch.equal(_bits(_run(m.set_int8_blocks(blocks), x)), _bits(y8)), blocks
    y = _run(m.set_int8_blocks([]), x)
    assert torch.equal(_bits(y), _bits(y16)), \
        f"{case}: no int8 block differs from fp16 in {int((y != y16).sum())} outputs"
    assert m.last_launch_count() == n16


def _workspace_q(m, rep):
    """The Q buffer of the model's eval workspace (api.cu ws_layout: a0, X0, X1, H, Q, each
    1024-byte aligned from the 1024-aligned base) over the rows of the replay's last Q."""
    p = rep.plan
    align = lambda v: -(-v // 1024) * 1024   # noqa: E731
    a0 = p.N * p.L[0] * p.k0_pad if p.strided else p.N * p.T * p.c_in_pad
    x0 = align(2 * a0)
    x1 = align(x0 + 2 * p.N * p.L[0] * p.C)
    h = align(x1 + 2 * p.N * p.L[1] * p.C)
    q = align(h + 2 * p.N * p.L[1] * p.C)
    ws = m._engine.workspace
    base = (-ws.data_ptr()) % 1024
    last = [buf for name, _, buf in rep.acts if name.startswith("Q")][-1]
    return ws[base + q: base + q + last[0].numel()].view(last[0].shape), last[0]


@pytest.mark.parametrize("blocks", SETS, ids=["b" + "".join(map(str, s)) for s in SETS])
@pytest.mark.parametrize("case,cfg,N,T", CASES, ids=[c[0] for c in CASES])
def test_layers(cuda_device, case, cfg, N, T, blocks):
    sd, x = _data(cfg, N, T, cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    amax = m.int8_calibration()
    m.set_precision("int8").set_int8_blocks(blocks)
    y = _run(m, x)
    launches = m.last_launch_count()
    with torch.no_grad():
        rep = replay_blocks(sd, cfg, x, er.gpu_gemm, amax.numpy(), blocks)
    plan = rep.plan
    nb = plan.nb
    int8 = [b in blocks for b in range(1, nb + 1)]
    transitions = sum(1 for i in range(1, nb) if not int8[i - 1] and int8[i])
    assert len(rep.quants) == transitions

    # packs: the int8 layers' s8 packs and scale' are the replay's; an fp16 layer has none
    lib = _capi.load()
    stream = torch.cuda.current_stream().cuda_stream
    blocks_launches = rep.launches[1:-1]
    for layer, lc in enumerate(blocks_launches):
        if int8[layer // 2]:
            assert lc.desc["precision"] == er.K_INT8
            w8, qs = torch.empty_like(lc.w), torch.empty_like(lc.scale)
            _capi.check(lib.vp3d_int8_packs(m._plan, layer, w8.data_ptr(), None, qs.data_ptr(),
                                            stream), "vp3d_int8_packs")
            torch.cuda.synchronize()
            assert torch.equal(w8, lc.w), f"{case}: s8 pack of layer {layer}"
            assert torch.equal(qs.view(torch.int32), lc.scale.view(torch.int32)), \
                f"{case}: scale' of layer {layer}"
        else:
            assert lc.desc["precision"] == er.K_FP16 and lc.desc["k_per_tap"] == plan.C
            assert lib.vp3d_int8_packs(m._plan, layer, None, None, None, stream) == -1
            assert b"runs fp16" in lib.vp3d_last_error()

    # every GEMM
    for lc in rep.launches:
        where = f"{case} {blocks}: {lc.name} ({lc.desc['out_rows']} rows x {lc.desc['n_pad']})"
        if lc.desc["precision"] == er.K_INT8:
            _check_int8(lc, plan, where)
        else:
            _check_launch(lc, plan, f"{case} {blocks}")
            if lc.out_u8 is not None:
                assert lc.name == "expand" and int8[0]
                _check_q0(lc, plan, where)

    # the quantise pass: the replay's Q_i is NumPy's formula on the stored X_i, and the model's
    # last Q buffer is the replay's (the quantise pass wrote it when the last int8 block follows an
    # fp16 one)
    for i, xs, q, inv_s in rep.quants:
        xh = xs[0].cpu().numpy().astype(np.float32)
        exp = np.clip(np.rint(xh * np.float32(inv_s)), 0, 255).astype(np.uint8)
        assert np.array_equal(q[0].cpu().numpy(), exp), f"{case} {blocks}: Q_{i}"
    if any(int8):
        got, exp = _workspace_q(m, rep)
        n = int((got != exp).sum())
        assert n == 0, f"{case} {blocks}: {n} of {got.numel()} codes of the model's last Q differ"

    # the replay is the plan
    assert rep.launch_count == launches == 3 + 2 * nb + transitions
    assert torch.equal(_bits(rep.y), _bits(y)), (
        f"{case} {blocks}: replay differs from model(x) in {int((rep.y != y).sum())} outputs")


@pytest.mark.parametrize("case,cfg,N,T", CASES, ids=[c[0] for c in CASES])
def test_changing_the_set_equals_a_fresh_model(cuda_device, case, cfg, N, T):
    sd, x = _data(cfg, N, T, cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    amax = m.int8_calibration()
    m.set_precision("int8")
    first = _run(m, x)
    for blocks in ([2], [1, 3], [], None):
        got = _run(m.set_int8_blocks(blocks), x)
        fresh = _build(cfg, sd, cuda_device).set_int8_blocks(blocks).set_precision("int8")
        fresh.load_int8_calibration(amax)
        assert torch.equal(_bits(got), _bits(_run(fresh, x))), f"{case}: {blocks}"
    assert torch.equal(_bits(got), _bits(first))


def test_predict_and_eval_autograd_inherit_the_set(cuda_device):
    fw, C = [3, 3, 3, 3], 128
    m = vp.TemporalModel(17, 2, 17, filter_widths=fw, dropout=0.0, channels=C)
    m.load_state_dict(orc.make_state_dict(17, 2, 17, fw, C, seed=11))
    m = m.to(cuda_device).eval()
    m.calibrate_int8(orc.make_input(4, 300, 17, 2, seed=7).to(cuda_device))
    m.set_precision("int8").set_int8_blocks([1, 3])
    clips = _clips(cuda_device, 12, 17, 2, seed=12)
    ys = _predict(m, clips, True)
    assert m.last_predict_launches == 2 * 3 + 4 + 1   # one chain, one quantise pass
    for x, y in zip(clips, ys):
        if len(x) >= 2:
            assert torch.equal(y, _offline(m, x, True)), len(x)
    x = orc.make_input(2, 120, 17, 2, seed=3).to(cuda_device)
    y_ng = _run(m, x)
    y = m(x.clone().requires_grad_(True))
    assert y.requires_grad and torch.equal(y.detach(), y_ng)
    assert not torch.equal(y_ng, _run(m.set_int8_blocks(None), x))


def test_c_entry_refusals_and_stale_packs(cuda_device):
    cfg = _cfg(TM, [3, 3, 3], 64)
    sd, x = _data(cfg, 2, 60, cuda_device)
    m = _build(cfg, sd, cuda_device)
    m.calibrate_int8(x)
    lib = _capi.load()
    fp16 = m._get_plan(x.device, "fp16")
    assert lib.vp3d_set_int8_blocks(fp16, 1) == -1
    assert b"not an int8 plan" in lib.vp3d_last_error()
    m.set_precision("int8")
    y = _run(m, x)
    plan = m._get_plan(x.device, "int8")
    assert lib.vp3d_set_int8_blocks(plan, 0b100) == -1 and lib.vp3d_set_int8_blocks(plan, 1 << 31) == -1
    assert lib.vp3d_set_int8_blocks(None, 1) == -1
    assert lib.vp3d_set_int8_blocks(plan, 0b11) == 0          # the current mask: nothing changes
    ws = m._engine.workspace
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.empty_like(y)
    assert lib.vp3d_forward_eval(plan, x.data_ptr(), out.data_ptr(), 2, 60, ws.data_ptr(),
                                 ws.numel(), stream) == 0
    assert lib.vp3d_set_int8_blocks(plan, 0b10) == 0          # a change: the packs are stale
    assert lib.vp3d_forward_eval(plan, x.data_ptr(), out.data_ptr(), 2, 60, ws.data_ptr(),
                                 ws.numel(), stream) == -5
    assert lib.vp3d_int8_packs(plan, 0, None, None, None, stream) == -1
    w = m._weights_struct()
    _capi.check(lib.vp3d_set_weights(plan, ctypes.byref(w), _capi.VP3D_PACK_CONV, stream),
                "vp3d_set_weights")
    assert lib.vp3d_forward_eval(plan, x.data_ptr(), out.data_ptr(), 2, 60, ws.data_ptr(),
                                 ws.numel(), stream) == 0
    torch.cuda.synchronize()
    fresh = _build(cfg, sd, cuda_device).set_precision("int8").set_int8_blocks([2])
    fresh.load_int8_calibration(m.int8_calibration())
    assert torch.equal(_bits(out), _bits(_run(fresh, x)))
