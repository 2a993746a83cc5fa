"""GPU: the ping-pong lean instances of conv_gemm_kernel (each consumer warpgroup computes whole
tiles, the CTA's tiles alternating between the two) must match the general epilogue BIT FOR BIT,
in fp16 and bf16, on the shapes where the schedule's bookkeeping changes:

* C = 320: five 64-wide N blocks, so with 132 CTAs the two warpgroups of a CTA hold different N
  blocks (and affines);
* layers with at most 1, 2 and 3 tiles per CTA (arc 3,3,3, C = 1024, T = 27: N = 1400 gives the
  block-1 convs 264 tiles, N = 2090 gives them 392 and the block-2 convs 136);
* a grid smaller than the SM count (VP3D_SM_LIMIT), where every layer runs several tiles per CTA.

VP3D_LEAN and VP3D_SM_LIMIT are read once per process, so every configuration runs in a child."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, %(root)r)
import videopose3d_b200 as vp
from oracle import temporal_model_oracle as orc
out = {}
dev = torch.device("cuda:0")
cases = %(cases)r
for name, arc, ch, n, t in cases:
    sd = orc.make_state_dict(17, 2, 17, arc, ch, seed=7)
    m = vp.TemporalModel(17, 2, 17, filter_widths=arc, channels=ch)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = orc.make_input(n, t, 17, 2, seed=8).to(dev)
    for prec in ("fp16", "bf16"):
        m.set_precision(prec)
        with torch.no_grad():
            out[name + "_" + prec] = m(x).float().cpu().numpy()
np.savez(sys.argv[1], **out)
"""

FULL_GRID = [
    ("c320", [3, 3, 3], 320, 2000, 27),
    ("c1024_two", [3, 3, 3], 1024, 1400, 27),
    ("c1024_three", [3, 3, 3], 1024, 2090, 27),
]
SMALL_GRID = [
    ("c320", [3, 3, 3], 320, 300, 27),
    ("c512", [3, 3, 3], 512, 200, 27),
]


def _run(cases, lean, path, sm_limit=None):
    env = dict(os.environ, VP3D_LEAN=lean)
    if sm_limit is not None:
        env["VP3D_SM_LIMIT"] = str(sm_limit)
    r = subprocess.run([sys.executable, "-c", CHILD % {"root": ROOT, "cases": cases}, path],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return np.load(path)


@pytest.mark.parametrize("cases,sm_limit", [(FULL_GRID, None), (SMALL_GRID, 20)],
                         ids=["full_grid", "sm_limit_20"])
def test_pingpong_matches_general_epilogue_bitwise(tmp_path, cases, sm_limit):
    a = _run(cases, "1", str(tmp_path / "lean.npz"), sm_limit)
    b = _run(cases, "0", str(tmp_path / "general.npz"), sm_limit)
    assert set(a.files) == set(b.files) and len(a.files) == 2 * len(cases)
    for k in a.files:
        assert a[k].shape == b[k].shape
        assert np.isfinite(a[k]).all()
        assert np.array_equal(a[k], b[k]), (k, float(np.abs(a[k] - b[k]).max()))
