"""CPU: int8 on a chosen set of residual blocks (``set_int8_blocks``), the rest in fp16.

The float64 restatement of the mixed chain (int8_blocks_oracle) is checked against the
restatements it generalises -- int8_oracle's all-int8 forward and, with no int8 block, the fp16
launch schedule of eval_replay -- and against the kernels' own formats (int8_blocks_replay with
fake_gemm, including the quantise pass that makes Q_i from a stored fp16 X_i).  The mixed replay
with every block, and with none, is eval_replay's int8 and fp16 replay.  Then the Python API's
validation and state, and the C entry's refusals that need no GPU."""
import copy
import pickle

import numpy as np
import pytest
import torch

import eval_replay as er
import int8_blocks_oracle as ibo
import int8_oracle as io
from int8_blocks_replay import replay_blocks
import videopose3d_b200 as vp
from oracle import temporal_model_oracle as orc
from videopose3d_b200 import _capi

# (id, cfg, N, T, strided)
CASES = [
    ("tm_3333_c64_dilated", dict(cls="TemporalModel", J=17, F=2, Jout=17, fw=[3, 3, 3, 3], C=64),
     4, 100, False),
    ("opt_3333_c100_causal", dict(cls="TemporalModelOptimized1f", J=17, F=2, Jout=17,
                                  fw=[3, 3, 3, 3], C=100, causal=True), 16, 81, True),
]
# the fp16 schedule restated in the kernels' formats against the float64 restatement: both store
# fp16 activations, they differ in where fp32 rounds (BatchNorm shift, accumulation); measured
# below 5e-5 of max|y| on these cases
FP16_TOL = 2e-4
# the mixed chain in the kernels' formats against float64: an fp16 rounding on the other side of a
# code boundary moves one u8 code; measured below 2e-4, a tenth of the int8 forward's own error
MIXED_TOL = 1e-3


def _data(cfg, N, T):
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"], seed=0)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=1).numpy()
    return sd, x


def _kw(cfg, strided):
    return dict(causal=cfg.get("causal", False), strided=strided)


@pytest.mark.parametrize("case,cfg,N,T,strided", CASES, ids=[c[0] for c in CASES])
def test_all_blocks_is_the_int8_forward(case, cfg, N, T, strided):
    sd, x = _data(cfg, N, T)
    amax = io.calibrate(sd, x, cfg["fw"], **_kw(cfg, strided))
    y = io.forward_int8(sd, x, cfg["fw"], amax, **_kw(cfg, strided))
    nb = len(cfg["fw"]) - 1
    for blocks in (None, list(range(1, nb + 1)), range(nb, 0, -1)):
        yb = ibo.forward_int8_blocks(sd, x, cfg["fw"], amax, blocks, **_kw(cfg, strided))
        assert np.array_equal(yb, y), f"{case}: int8_blocks={blocks}"


@pytest.mark.parametrize("case,cfg,N,T,strided", CASES, ids=[c[0] for c in CASES])
def test_no_block_is_the_fp16_forward(case, cfg, N, T, strided):
    sd, x = _data(cfg, N, T)
    amax = io.calibrate(sd, x, cfg["fw"], **_kw(cfg, strided))
    acts = []
    y = ibo.forward_int8_blocks(sd, x, cfg["fw"], amax, [], collect=acts, **_kw(cfg, strided))
    assert all(a is None for a in acts[1::3]), "a Q without an int8 block to read it"
    rep = er.replay(sd, cfg, torch.from_numpy(x).float(), "fp16", er.fake_gemm)
    assert rep.plan.strided == strided
    ref = rep.y.double().numpy()
    err = float(np.abs(y - ref).max() / np.abs(ref).max())
    assert err < FP16_TOL, f"{case}: {err:.2e}"
    # and it is not the int8 forward
    y8 = io.forward_int8(sd, x, cfg["fw"], amax, **_kw(cfg, strided))
    assert float(np.abs(y8 - ref).max()) > 2 * float(np.abs(y - ref).max())


@pytest.mark.parametrize("blocks", [[1], [2], [3], [1, 3], [2, 3], []])
@pytest.mark.parametrize("case,cfg,N,T,strided", CASES, ids=[c[0] for c in CASES])
def test_mixed_chain_in_kernel_formats(case, cfg, N, T, strided, blocks):
    """The replay of the mixed schedule (fake GEMMs, exact int8 epilogues, the quantise pass in
    quant_u8) against the float64 restatement; the quantise pass against the formula."""
    sd, x = _data(cfg, N, T)
    amax = io.calibrate(sd, x, cfg["fw"], **_kw(cfg, strided))
    y = ibo.forward_int8_blocks(sd, x, cfg["fw"], amax, blocks, **_kw(cfg, strided))
    rep = replay_blocks(sd, cfg, torch.from_numpy(x).float(), er.fake_gemm, amax, blocks)
    nb = len(cfg["fw"]) - 1
    int8 = [b in blocks for b in range(1, nb + 1)]
    # launches: pack, expand, 2 per block, shrink, one quantise pass per fp16 -> int8 transition
    transitions = sum(1 for i in range(1, nb) if not int8[i - 1] and int8[i])
    assert len(rep.quants) == transitions
    assert rep.launch_count == 3 + 2 * nb + transitions
    assert [lc.desc["precision"] == er.K_INT8 for lc in rep.launches[1:-1]] == \
        [b for b in int8 for _ in range(2)]
    _, inv = io.act_scales(amax)
    for i, xs, q, inv_s in rep.quants:
        assert inv_s == float(inv[2 * i])
        xh = xs[0].numpy().astype(np.float32)
        exp = np.clip(np.rint(xh * np.float32(inv_s)), 0, 255).astype(np.uint8)
        assert np.array_equal(q[0].numpy(), exp)
        assert not q[0, :, cfg["C"]:].any()
    ref = rep.y.double().numpy()
    err = float(np.abs(y - ref).max() / np.abs(ref).max())
    assert err < MIXED_TOL, f"{case} blocks={blocks}: {err:.2e}"


@pytest.mark.parametrize("case,cfg,N,T,strided", CASES, ids=[c[0] for c in CASES])
def test_mixed_replay_generalises_the_int8_and_fp16_replays(case, cfg, N, T, strided):
    sd, x = _data(cfg, N, T)
    amax = io.calibrate(sd, x, cfg["fw"], **_kw(cfg, strided))
    xt = torch.from_numpy(x).float()
    nb = len(cfg["fw"]) - 1
    ref8 = er.replay(sd, cfg, xt, er.INT8, er.fake_gemm, amax=amax)
    ref16 = er.replay(sd, cfg, xt, "fp16", er.fake_gemm)
    for blocks, ref in ((None, ref8), (list(range(1, nb + 1)), ref8), ([], ref16)):
        rep = replay_blocks(sd, cfg, xt, er.fake_gemm, amax, blocks)
        assert rep.launch_count == ref.launch_count and not rep.quants
        assert torch.equal(rep.y, ref.y), f"{case}: {blocks}"
        assert [n for n, _, _ in rep.acts] == [n for n, _, _ in ref.acts]


def _model(cls=vp.TemporalModel, fw=(3, 3, 3)):
    return cls(17, 2, 17, filter_widths=list(fw), channels=64)


@pytest.mark.parametrize("cls", [vp.TemporalModel, vp.TemporalModelOptimized1f])
def test_set_int8_blocks_api(cls):
    m = _model(cls)
    assert m.int8_blocks == (1, 2)
    assert m.set_int8_blocks([2]) is m and m.int8_blocks == (2,)
    assert m.set_int8_blocks((2, 1, 2)).int8_blocks == (1, 2)
    assert m.set_int8_blocks([]).int8_blocks == ()
    assert m.set_int8_blocks(None).int8_blocks == (1, 2)
    m.set_int8_blocks([1])
    for bad in ([0], [3], [-1], [1.0], ["1"], [True], [None]):
        with pytest.raises(ValueError):
            m.set_int8_blocks(bad)
        assert m.int8_blocks == (1,), f"{bad} changed the selection"
    # outside the state_dict; carried by copies and pickles; untouched by loads and invalidate()
    assert not any("int8" in k for k in m.state_dict())
    for other in (copy.deepcopy(m), pickle.loads(pickle.dumps(m))):
        assert other.int8_blocks == (1,)
    m.load_state_dict(_model(cls).state_dict())
    m.invalidate()
    assert m.int8_blocks == (1,)


def test_set_int8_blocks_c_refusals_without_gpu():
    lib = _capi.load()
    assert lib.vp3d_set_int8_blocks(None, 1) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert lib.vp3d_set_int8_blocks(None, 0) == -1
