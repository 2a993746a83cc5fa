"""GPU: the lean inference instances of conv_gemm_kernel must reproduce the general epilogue BIT FOR
BIT.  The lean instances resolve affine + ReLU [+ one-plane TMA residual] into one 16-bit plane, and
the operand format (fp16 or bf16), at compile time; with more tiles than CTAs they run the ping-pong
schedule (each consumer warpgroup computes whole tiles, the CTA's tiles alternating between the
two).  The general epilogue reads all of that at run time.  Cases:

* "cone" / "seq": random modules with non-trivial running statistics, strided and dilated eval
  schedules, padded channels (C = 100);
* "format": the shapes where the k-loop length or the tile width changes: a one-k-block 1x1 conv
  (64 channels), the expand (K = 128, two k-blocks), residual layers at 64- and 128-wide tiles,
  grids where some CTAs get one tile and others several, and the flagship shape (arc 3,3,3,3,3,
  C = 1024, N = 1024);
* "pingpong": C = 320 (five 64-wide N blocks, so the two warpgroups of a CTA hold different N blocks
  and affines), and layers with at most 1, 2 and 3 tiles per CTA (arc 3,3,3, C = 1024, T = 27:
  N = 1400 gives the block-1 convs 264 tiles, N = 2090 gives them 392 and the block-2 convs 136);
* a grid smaller than the SM count (VP3D_SM_LIMIT=20), where every layer runs several tiles per CTA.

VP3D_LEAN and VP3D_SM_LIMIT are read once per process, so each (VP3D_LEAN, VP3D_SM_LIMIT) pair runs
all its cases in one child."""
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
g = torch.Generator().manual_seed(11)
for name, cls, arc, ch, n, t, prec in %(random)r:
    torch.manual_seed(3)
    m = getattr(vp, cls)(17, 2, 17, filter_widths=arc, channels=ch).to(dev).eval().set_precision(prec)
    with torch.no_grad():
        for bn in [m.expand_bn] + list(m.layers_bn):     # non-trivial running statistics
            bn.running_mean.uniform_(-0.2, 0.2, generator=None)
            bn.running_var.uniform_(0.5, 1.5)
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.3, 0.3)
        x = (torch.rand(n, t, 17, 2, generator=g) * 2 - 1).to(dev)
        out[name] = m(x).float().cpu().numpy()
for name, arc, ch, n, t, seed in %(seeded)r:
    sd = orc.make_state_dict(17, 2, 17, arc, ch, seed=seed)
    m = vp.TemporalModel(17, 2, 17, filter_widths=arc, channels=ch)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = orc.make_input(n, t, 17, 2, seed=seed + 1).to(dev)
    for prec in ("fp16", "bf16"):
        m.set_precision(prec)
        with torch.no_grad():
            out[name + "_" + prec] = m(x).float().cpu().numpy()
np.savez(sys.argv[1], **out)
"""

# (name, class, filter widths, channels, N, T, precision): random modules, one input each
RANDOM = [
    ("tm_cone_fp16", "TemporalModel", [3, 3, 3], 128, 96, 27, "fp16"),      # strided eval schedule
    ("tm_cone_bf16", "TemporalModel", [3, 3, 3], 128, 96, 27, "bf16"),
    ("tm_seq_fp16", "TemporalModel", [3, 3, 3], 128, 3, 300, "fp16"),       # dilated schedule
    ("opt_fp16", "TemporalModelOptimized1f", [3, 3, 3], 256, 640, 27, "fp16"),
    ("tm_c100_fp16", "TemporalModel", [3, 5], 100, 64, 15, "fp16"),         # padded channels
]
# (name, filter widths, channels, N, T, seed): the oracle's seeded parameters, fp16 and bf16
SEEDED = [
    ("format_c64", [3, 3, 3], 64, 96, 27, 5),           # 1x1 convs of one k-block
    ("format_c128", [3, 3, 3], 128, 200, 27, 5),        # residual layers, few tiles per CTA
    ("format_c256_small", [3, 3], 256, 5, 9, 5),        # fewer tiles than SMs: one tile per CTA
    ("format_c512", [3, 3, 3], 512, 300, 27, 5),        # odd and even tile counts per CTA
    ("format_flagship", [3, 3, 3, 3, 3], 1024, 1024, 243, 5),
    ("pingpong_c320", [3, 3, 3], 320, 2000, 27, 7),
    ("pingpong_c1024_two", [3, 3, 3], 1024, 1400, 27, 7),
    ("pingpong_c1024_three", [3, 3, 3], 1024, 2090, 27, 7),
]
SEEDED_SM_LIMIT = [
    ("c320", [3, 3, 3], 320, 300, 27, 7),
    ("c512", [3, 3, 3], 512, 200, 27, 7),
]


def _run(random, seeded, lean, path, sm_limit):
    env = dict(os.environ, VP3D_LEAN=lean)
    if sm_limit is not None:
        env["VP3D_SM_LIMIT"] = str(sm_limit)
    src = CHILD % {"root": ROOT, "random": random, "seeded": seeded}
    r = subprocess.run([sys.executable, "-c", src, path], env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    return np.load(path)


@pytest.mark.parametrize("random,seeded,sm_limit", [(RANDOM, SEEDED, None),
                                                    ([], SEEDED_SM_LIMIT, 20)],
                         ids=["full_grid", "sm_limit_20"])
def test_lean_matches_general_epilogue_bitwise(tmp_path, random, seeded, sm_limit):
    a = _run(random, seeded, "1", str(tmp_path / "lean.npz"), sm_limit)
    b = _run(random, seeded, "0", str(tmp_path / "general.npz"), sm_limit)
    n = len(random) + 2 * len(seeded)
    assert set(a.files) == set(b.files) and len(a.files) == n
    for k in a.files:
        assert a[k].shape == b[k].shape
        assert np.isfinite(a[k]).all()
        assert np.array_equal(a[k], b[k]), (k, float(np.abs(a[k] - b[k]).max()))
