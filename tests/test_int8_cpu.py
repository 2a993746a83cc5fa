"""CPU: the float64 restatement of the int8 eval forward (int8_oracle.py) against the float64
reference forward.

On the bench model (TemporalModel 3,3,3,3,3, C = 1024, one receptive field per sample), calibrated
on 128 sequences and tested on 256 others, u8 x s8 with one activation scale per tensor lands at
5.4e-3 of max|ref| and a mean joint distance of 3.5e-3 of the mean joint norm.  (An emulation that
quantised in float64 -- no fp32 fold of the scales, no fp32 v * 1/s -- and measured against its own
fp32 forward put the first figure at 4.2e-3 and the second at the same 3.5e-3: the maximum is one
worst output and moves with such details, the mean does not.)  Every other model shape the eval
forward supports stays below GATE."""
import numpy as np
import pytest

import int8_oracle as io
from oracle import temporal_model_oracle as orc

GATE = 1e-2


def test_bench_model_error():
    arc = [3, 3, 3, 3, 3]
    sd = orc.make_state_dict(17, 2, 17, arc, 1024, seed=0)
    amax = io.calibrate(sd, orc.make_input(128, 243, seed=5).numpy(), arc, strided=True)
    x = orc.make_input(256, 243, seed=78).numpy()
    ref = orc.forward_numpy(sd, x, arc, strided=True)
    y = io.forward_int8(sd, x, arc, amax, strided=True)
    rel_max = float(np.abs(y - ref).max() / np.abs(ref).max())
    rel_joint = float(np.linalg.norm(y - ref, axis=-1).mean() / np.linalg.norm(ref, axis=-1).mean())
    print(f"\nbench model int8: max|d|/max|ref| {rel_max:.2e}, mean joint distance / norm "
          f"{rel_joint:.2e}")
    assert 5.0e-3 < rel_max < 6.0e-3
    assert 3.2e-3 < rel_joint < 3.8e-3


CASES = [  # (id, widths, C, J, F, J_out, causal, dense, N, T, strided)
    ("tm_333_c64", [3, 3, 3], 64, 17, 2, 17, False, False, 8, 60, False),
    ("tm_333_causal", [3, 3, 3], 64, 17, 2, 17, True, False, 8, 90, False),
    ("tm_33_dense", [3, 3], 64, 17, 2, 17, False, True, 8, 60, False),
    ("tm_353_c96_cone", [3, 5, 3], 96, 17, 2, 17, False, False, 16, 45, True),
    ("tm_53_c129", [5, 3], 129, 17, 2, 17, False, False, 8, 100, False),
    ("j15_f3", [3, 3, 3], 64, 15, 3, 15, False, False, 16, 27, True),
    ("traj_jout1", [3, 5, 3], 128, 17, 2, 1, False, False, 8, 120, False),
    ("opt_35_causal", [3, 5], 128, 17, 2, 17, True, False, 32, 15, True),
    ("six_blocks", [3, 3, 3, 3, 3, 3], 64, 17, 2, 17, False, False, 2, 729, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_model_shapes_gate(case):
    _, fw, C, J, F, Jo, causal, dense, N, T, strided = case
    sd = orc.make_state_dict(J, F, Jo, fw, C, dense=dense, seed=0)
    x = orc.make_input(N, T, J, F, seed=1).numpy()
    kw = dict(causal=causal, dense=dense, strided=strided)
    amax = io.calibrate(sd, x, fw, **kw)
    assert amax.shape == (2 * (len(fw) - 1),) and (amax > 0).all()
    ref = orc.forward_numpy(sd, x, fw, **kw)
    y = io.forward_int8(sd, x, fw, amax, **kw)
    assert y.shape == ref.shape
    assert np.abs(y - ref).max() / np.abs(ref).max() < GATE


def test_quantisation_formulas():
    # zero amax -> scale 1; codes round half to even and saturate
    s, inv = io.act_scales([0.0, 255.0, 25.5])
    assert s.tolist() == [1.0, 1.0, np.float32(0.1)] and inv.dtype == np.float32
    assert io.quant_act([0.5, 1.5, 2.5, 300.0, -3.0], 1.0).tolist() == [0, 2, 2, 255, 0]
    w = np.array([[[1.0, -2.0], [0.5, 0.0]], [[0.0, 0.0], [0.0, 0.0]]], np.float32)
    q, ws = io.quant_weight(w)
    assert ws.tolist() == [np.float32(2.0) / np.float32(127), 1.0]
    assert q[0].tolist() == [[64, -127], [32, 0]] and not q[1].any()
