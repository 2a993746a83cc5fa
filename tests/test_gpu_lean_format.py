"""GPU: the lean inference instances of conv_gemm_kernel fix the operand format (fp16 or bf16) at
compile time.  Their outputs must match the general epilogue, which reads the format at run time,
BIT FOR BIT in both formats, on the shapes where the k-loop length or the tile width changes: a
one-k-block 1x1 conv (64 channels), the expand (K = 128, two k-blocks), residual layers at 64- and
128-wide tiles, grids where some CTAs get one tile and others several, and the flagship shape
(arc 3,3,3,3,3, C = 1024, N = 1024).  VP3D_LEAN is read once per process, so both run in children."""
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
cases = [
    ("c64", [3, 3, 3], 64, 96, 27),           # 1x1 convs of one k-block
    ("c128", [3, 3, 3], 128, 200, 27),        # residual layers, few tiles per CTA
    ("c256_small", [3, 3], 256, 5, 9),        # fewer tiles than SMs: one tile per CTA
    ("c512", [3, 3, 3], 512, 300, 27),        # odd and even tile counts per CTA
    ("flagship", [3, 3, 3, 3, 3], 1024, 1024, 243),
]
for name, arc, ch, n, t in cases:
    sd = orc.make_state_dict(17, 2, 17, arc, ch, seed=5)
    m = vp.TemporalModel(17, 2, 17, filter_widths=arc, channels=ch)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = orc.make_input(n, t, 17, 2, seed=6).to(dev)
    for prec in ("fp16", "bf16"):
        m.set_precision(prec)
        with torch.no_grad():
            out[name + "_" + prec] = m(x).float().cpu().numpy()
np.savez(sys.argv[1], **out)
"""


def _run(lean, path):
    env = dict(os.environ, VP3D_LEAN=lean)
    r = subprocess.run([sys.executable, "-c", CHILD % {"root": ROOT}, path], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return np.load(path)


def test_lean_compile_time_format_matches_general_epilogue_bitwise(tmp_path):
    a = _run("1", str(tmp_path / "lean.npz"))
    b = _run("0", str(tmp_path / "general.npz"))
    assert set(a.files) == set(b.files) and len(a.files) == 10
    for k in a.files:
        assert a[k].shape == b[k].shape
        assert np.isfinite(a[k]).all()
        assert np.array_equal(a[k], b[k]), (k, float(np.abs(a[k] - b[k]).max()))
