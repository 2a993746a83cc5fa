"""GPU: the last partial wave of the 128-wide ping-pong conv GEMM instances as 128 x 64 half tiles.

A ping-pong launch of T tiles on a grid of S CTAs leaves L = T mod S tiles for its last wave.  When
0 < L <= S / 2 the launch runs them as 2L half tiles of 64 columns instead (one per CTA), so that the
last wave takes about half a tile.  Each case below launches one descriptor through vp3d_conv_gemm
under an SM limit that makes L equal to 1, S / 2 or S / 2 + 1 (the last keeps whole tiles), in
fp16, bf16 and int8, with and without the residual, on flat and per-sample (dilated) tiles, and
checks it three ways:
1. float64: the same bound as test_gpu_conv_gemm_instances (int8 bit for bit against the exact
   integer epilogue);
2. the same descriptor under an SM limit that divides T (no partial wave) stores the same bits;
3. the guard zones around the outputs (NaN, or a fixed byte for u8; 64 columns past n_pad, so past
   the second half of the last N block) are untouched.
"""
import numpy as np
import pytest
import torch

import test_gpu_conv_gemm_instances as gi
from test_gpu_conv_gemm_instances import sm_limit  # noqa: F401  (the fixture)

S = 8   # SM limit of the partial-wave launches: L = 1, S / 2 and S / 2 + 1
N_PAD = 384   # three 128-wide N blocks: halves of the first, middle and last block all occur
# L -> (row tiles, an SM limit with no partial wave); T = row tiles x 3 N blocks
WAVES = {1: (3, 3), S // 2: (4, 6), S // 2 + 1: (7, 7)}

# (format, residual) -> the 128-wide ping-pong instance, for the flat and the dilated geometry
INSTANCES = {
    ("fp16", False): ("128 lean fp16 pp", "128 lean fp16 pp u8beside"),
    ("fp16", True): ("128 lean fp16 pp res", "128 lean fp16 pp res"),
    ("bf16", False): ("128 lean bf16 pp", "128 lean bf16 pp"),
    ("bf16", True): ("128 lean bf16 pp res", "128 lean bf16 pp res"),
    ("int8", False): ("128 lean int8 pp u8alone", "128 lean int8 pp u8alone"),
    ("int8", True): ("128 lean int8 pp res", "128 lean int8 pp res u8beside"),
}


def _case(fmt, res, geo, left):
    m_tiles, _ = WAVES[left]
    inst = INSTANCES[(fmt, res)][geo == "dilated"]
    flags = inst.split()[4:]
    u8 = "alone" if "u8alone" in flags else "beside" if "u8beside" in flags else None
    k = 128 if fmt == "int8" else 64
    name = f"{fmt}_{'res' if res else 'nores'}_{geo}_L{left}"
    if geo == "flat":
        # ragged last row tile; the 1x1 convs of the model (taps as one K row for 16-bit, as row
        # regions for int8, whose taps must step rows)
        return gi.case(name, inst, S, fmt=fmt, geo="regions" if fmt == "int8" else "flat",
                       taps=3 if fmt == "int8" else 2, out_rows=m_tiles * 128 - 27, n_pad=N_PAD,
                       k=k, res=gi.R(off=1) if res else None,
                       out=None if u8 == "alone" else "16", u8=u8)
    # one ragged tile per sample, taps two frames apart
    return gi.case(name, inst, S, fmt=fmt, geo="dilated", samples=m_tiles, a_rows=110, out_rows=100,
                   taps=3, step=5, n_pad=N_PAD, k=k,
                   res=gi.R(rps=104, off=2) if res else None,
                   out=None if u8 == "alone" else "16", u8=u8)


CASES = [(_case(fmt, res, geo, left), left)
         for fmt in ("fp16", "bf16", "int8") for res in (False, True)
         for geo in ("flat", "dilated") for left in WAVES]


def _run(c, d, outs, lim, set_limit):
    set_limit(lim)
    got = gi.query_key(d)
    assert got == c["key"], f"{c['name']} at {lim} SMs selects [{gi.key_text(got)}]"
    outs.reset()
    gi.launch(d)
    return outs.bits()


@pytest.mark.gpu
@pytest.mark.parametrize("c,left", CASES, ids=[c["name"] for c, _ in CASES])
def test_last_wave(cuda_device, sm_limit, c, left):
    m_tiles, whole = WAVES[left]
    assert (m_tiles * N_PAD // 128) % S == left and (m_tiles * N_PAD // 128) % whole == 0
    ops = gi.Operands(c, cuda_device)
    v, err = gi.reference(c, ops)
    outs = gi.Outputs(c, cuda_device)
    outs.inv_s = 1.0
    if c["u8"]:
        outs.inv_s = float(np.float32(255.0) / np.float32(float(v.max()) * 0.9))
    d = gi._desc(c, ops, outs)
    tag = f"{c['name']} [{gi.key_text(c['key'])}] at {S} SMs"
    bits = _run(c, d, outs, S, sm_limit)
    gi._check_guards(outs, tag)
    gi._check_values(c, outs, v, err, tag)
    ref = _run(c, d, outs, whole, sm_limit)
    for n in bits:
        assert torch.equal(bits[n], ref[n]), f"{tag}: {n} differs from the launch at {whole} SMs"
