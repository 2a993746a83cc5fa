"""GPU: the weight-gradient GEMM (vp3d_wgrad_gemm = wgrad_gemm_kernel + wgrad_reduce_kernel, the
launches vp3d_backward makes for every conv layer) against float64, operator by operator.

Reference.  dW[co][ci][tap] = sum_row dZ[row, co] * X[map(row, tap), ci], evaluated in float64 from
the index definition (one einsum per tap over all rows of all samples, nothing of the kernel's
tiling or splitting) on the SAME bf16 operands the kernel reads.  With two planes the kernel forms
three products per pair of entries, hi*hi + lo*hi + hi*lo, and so does the reference.

Gate.  Per entry |got - ref| <= k * 2^-24 * A, A = sum_row |dZ| |X| over the same terms (for two
planes the sum of the three products' magnitudes), k = 4 sqrt(K) + 64, K = the number of rows the
entry sums over.  Where it comes from: the kernel accumulates in fp32 -- each split runs one
accumulator through 4 k16 MMA steps per 64-row chunk and operand pair, then the <= 16 split
partials are added left to right -- and every accumulator update errs by at most about 2^-24 of the
running sum (the tensor core may truncate rather than round, so the errors need not cancel).  The
operands here have random signs: the running sum stays within a few sqrt(K) times the rms term while
A grows like K times the mean term, so n updates cost about n / sqrt(K) units of 2^-24 A.  Flat
layouts make n ~ K / 16 per split, i.e. ~sqrt(K) / 16; per-sample layouts with short rows pay 4
updates per pair for every chunk however few of its rows are real (one row per sample: 12 updates
per row with two planes), which is what the 4 sqrt(K) term has to cover.  Measured on an H100, the
worst ratio over the cases below is 74 units (two planes, one row per sample, K = 1024, gate 192);
every other case stays under 25 with gates of 136 to 561.  The worst-case (deterministic) bound
K * 2^-24 A would be far too loose to see a lost chunk.

Each gate is shown to reject plausible wrong answers in the same test: the reference with one
64-row chunk removed at a split boundary, with one tap read one row / column off, and (per-sample
layouts) with one sample's dZ paired with its neighbour's X.

Dispatch.  A Python mirror of run_wgrad (videopose3d_b200/csrc/train_api.cu) gives each shape's tile
width and split count; with the 132 SMs of an H100 SXM the table below asserts which case every
shape hits, and the test checks it on the kernel's own output: the split partials in `partial` are
exactly the first `splits` slabs (the rest stay NaN) and the gradient is their left-to-right fp32
sum, bit for bit.  Cases: tile width 64 and 128; 1 split (many items), 2, 5 (= the chunk count),
7, 11, 15, 16 (few items, many chunks; chunk counts 16 does not divide), splits reduced by a small
partial buffer, and a buffer too small for one split (VP3D_ERR_WORKSPACE, nothing written).

Output properties: the gradient is NaN-filled before the call and every entry must be written;
the padding columns of dZ and X (beyond c_out / c_in) hold NaN and must not reach a real entry;
two calls are bit-identical."""
import ctypes
import math
from dataclasses import dataclass

import pytest
import torch

from gpu_utils import split_planes
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
REFERENCE_SMS = 132   # H100 SXM: the split counts in CASES hold for this SM count


@dataclass
class Geo:
    c_out: int
    dz_ld: int
    c_in: int
    x_ld: int
    rows: int               # per sample when per_sample
    taps: int = 1           # gradient taps (taps_out)
    per_sample: int = 0
    samples: int = 1
    x_rows: int = 0         # per sample (per_sample only)
    tap_row_step: int = 0
    tap_col_step: int = 0
    merged: int = 0

    @property
    def gemm_taps(self):
        return 1 if self.merged else self.taps

    @property
    def c_in_cols(self):
        return self.taps * self.c_in if self.merged else self.c_in

    @property
    def s(self):
        return self.samples if self.per_sample else 1

    @property
    def xr(self):
        return self.x_rows if self.per_sample else self.rows


def _rup(v, m):
    return (v + m - 1) // m * m


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan(g, partial_bytes):
    """Mirror of run_wgrad: (tile width, split count, bytes of one split's partial)."""
    n64 = _rup(g.c_in_cols, 64)
    block_n = 128 if n64 % 128 == 0 else 64
    m_pad, n_pad = _rup(g.c_out, 128), _rup(g.c_in_cols, block_n)
    items = g.gemm_taps * (m_pad // 128) * (n_pad // block_n)
    total_kb = -(-g.rows // 64) * g.s
    splits = max(1, min(-(-2 * _num_sms() // items), 16, total_kb))
    slab = g.gemm_taps * m_pad * n_pad * 4
    while splits > 1 and splits * slab > partial_bytes:
        splits -= 1
    return block_n, splits, slab, m_pad, n_pad


def _strided(C, c_real, w, rows):
    return Geo(c_out=c_real, dz_ld=C, c_in=c_real, x_ld=w * C, rows=rows, taps=w, tap_col_step=C)


def _dilated(C, c_real, w, d, N, L):
    return Geo(c_out=c_real, dz_ld=C, c_in=c_real, x_ld=C, rows=L, taps=w, per_sample=1, samples=N,
               x_rows=L + (w - 1) * d, tap_row_step=d)


def _merged(C, c_real, jf, w, rows):
    return Geo(c_out=c_real, dz_ld=C, c_in=jf, x_ld=_rup(w * jf, 64), rows=rows, taps=w, merged=1)


def _dil_expand(C, c_real, jf, w, N, T):
    return Geo(c_out=c_real, dz_ld=C, c_in=jf, x_ld=_rup(jf, 64), rows=T - w + 1, taps=w,
               per_sample=1, samples=N, x_rows=T, tap_row_step=1)


def _flat(C, c_real, rows, c_out=None, dz_ld=None):
    return Geo(c_out=c_out or c_real, dz_ld=dz_ld or C, c_in=c_real, x_ld=C, rows=rows)


# name -> (geometry, tile width, splits) -- the call sites of vp3d_backward:
#   shrink (c_out = 3 J_out on a 128-padded dZ), block 1x1 (flat), strided first conv (column taps,
#   tap_col_step = C), dilated first conv (per-sample rows, tap_row_step = dilation), strided expand
#   (tap-merged, width w0 * J * F), dilated expand (tap_row_step = 1 over the raw input)
CASES = {
    "shrink_c51_c256": (_flat(256, 256, 64 * 37 + 5, c_out=51, dz_ld=128), 128, 16),
    "shrink_c153_c100on128": (_flat(128, 100, 5000, c_out=153, dz_ld=256), 128, 16),
    "1x1_c64_5chunks": (_flat(64, 64, 320), 64, 5),
    "1x1_c192": (_flat(192, 192, 3000), 64, 16),
    "1x1_c1024": (_flat(1024, 1024, 8192 + 17), 128, 5),
    "strided_c256_w3": (_strided(256, 256, 3, 4000), 128, 16),
    "strided_c100on128_w5": (_strided(128, 100, 5, 1500), 128, 16),
    "strided_c1024_w5": (_strided(1024, 1024, 5, 2000), 128, 1),
    "strided_c1024_w3": (_strided(1024, 1024, 3, 64 * 200), 128, 2),
    "strided_c192_w7": (_strided(192, 192, 7, 700), 64, 7),
    "dilated_c256_w3_d9": (_dilated(256, 256, 3, 9, 40, 200), 128, 16),
    "dilated_c192_w3_d27_L64": (_dilated(192, 192, 3, 27, 64, 64), 64, 15),
    "dilated_c1024_w3_d81_L1_n1024": (_dilated(1024, 1024, 3, 81, 1024, 1), 128, 2),
    "dilated_c100on128_w5_d3_L37": (_dilated(128, 100, 5, 3, 30, 37), 128, 16),
    "dilated_c64_w7_d1": (_dilated(64, 64, 7, 1, 8, 300), 64, 16),
    "merged_jf34_w3_c256": (_merged(256, 256, 34, 3, 3000), 128, 16),
    "merged_jf45_w5_c1024": (_merged(1024, 1024, 45, 5, 4096 + 3), 128, 16),
    "merged_jf34_w7_c192": (_merged(192, 192, 34, 7, 1000), 128, 16),
    "merged_jf45_w3_c100on128": (_merged(128, 100, 45, 3, 2000), 64, 16),
    "dil_expand_jf34_w3_c1024": (_dil_expand(1024, 1024, 34, 3, 64, 243), 64, 11),
    "dil_expand_jf45_w5_c256": (_dil_expand(256, 256, 45, 5, 16, 100), 64, 16),
}


def _rand(shape, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.rand(shape, generator=g, device=dev) * 2 - 1


def _operands(g, planes, dev, seed):
    """dZ [planes][S][rows][dz_ld], X [planes][S][x_rows][x_ld] with NaN in every padding column."""
    dz = _rand((g.s, g.rows, g.dz_ld), seed, dev)
    dz[..., g.c_out:] = float("nan")
    x = _rand((g.s, g.xr, g.x_ld), seed + 1, dev)
    col = torch.arange(g.x_ld, device=dev)
    if g.merged:
        pad = col >= g.taps * g.c_in
    elif g.tap_col_step:
        pad = (col % g.tap_col_step >= g.c_in) | (col >= g.taps * g.tap_col_step)
    else:
        pad = col >= g.c_in
    x[..., pad] = float("nan")
    return split_planes(dz, planes), split_planes(x, planes)


def _dw(g, dz, x, r0=0, r1=None, shift=None):
    """float64 sum_{rows [r0, r1) of every given sample} dz[n, r, co] * x[n, xrow(r, tap), xcol(tap, ci)]
    straight from the index definition.  dz: [S, R, >= c_out], x: [S, x_rows, x_ld] (same S).
    shift = (tap, d_row, d_col) reads that tap one row / column off (clamped to the tap's own range:
    a plausible indexing slip, never a padding column)."""
    r1 = g.rows if r1 is None else r1
    dev = dz.device
    out = torch.zeros(g.c_out, g.c_in, g.taps, dtype=torch.float64, device=dev)
    d = dz[:, r0:r1, :g.c_out]
    for t in range(g.taps):
        c0 = t * g.c_in if g.merged else t * g.tap_col_step
        ro = 0 if g.merged else t * g.tap_row_step
        dr = dc = 0
        if shift is not None and shift[0] == t:
            dr, dc = shift[1], shift[2]
        rows = torch.arange(r0, r1, device=dev) + ro
        rows = (rows + dr).clamp(0, x.shape[1] - 1) if dr else rows
        cols = (torch.arange(g.c_in, device=dev) + dc).clamp(0, g.c_in - 1) + c0
        out[:, :, t] = torch.einsum("nrc,nrd->cd", d, x[:, rows][:, :, cols])
    return out


def _products(dzp, xp):
    """(dZ, X) fp64 operand pairs of the products the kernel forms."""
    dh, xh = dzp[0].double(), xp[0].double()
    if dzp.shape[0] == 1:
        return [(dh, xh)]
    return [(dh, xh), (dzp[1].double(), xh), (dh, xp[1].double())]


def _ref(g, pairs, **kw):
    return sum(_dw(g, a, b, **kw) for a, b in pairs)


def _call(g, dzp, xp, grad, partial):
    lib = _capi.load()
    d = _capi.WgradDesc()
    d.dz, d.dz_ld, d.x, d.x_ld = dzp.data_ptr(), g.dz_ld, xp.data_ptr(), g.x_ld
    d.planes, d.rows, d.per_sample, d.samples = dzp.shape[0], g.rows, g.per_sample, g.samples
    d.x_rows, d.taps, d.tap_row_step, d.tap_col_step = g.x_rows, g.gemm_taps, g.tap_row_step, g.tap_col_step
    d.c_out, d.c_in_cols, d.c_in, d.taps_out, d.merged = g.c_out, g.c_in_cols, g.c_in, g.taps, g.merged
    d.grad, d.partial, d.partial_bytes = grad.data_ptr(), partial.data_ptr(), partial.numel() * 4
    st = lib.vp3d_wgrad_gemm(ctypes.byref(d), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return st


def _partials_real(g, partial, splits_seen, m_pad, n_pad):
    """The real entries of every split slab as [slab, c_out, c_in, taps]."""
    p = partial[:splits_seen * g.gemm_taps * m_pad * n_pad].reshape(splits_seen, g.gemm_taps, m_pad, n_pad)
    if g.merged:
        p = p[:, 0, :g.c_out, :g.taps * g.c_in].reshape(splits_seen, g.c_out, g.taps, g.c_in)
        return p.permute(0, 1, 3, 2)
    return p[:, :, :g.c_out, :g.c_in].permute(0, 2, 3, 1)


def _gate(got, ref, mag, k):
    return bool(((got.double() - ref).abs() <= k * U * mag).all())


def _run_case(dev, g, planes, block_n, splits, partial_slabs=None, seed=11):
    slab = _plan(g, 1 << 62)[2]
    partial_bytes = (partial_slabs if partial_slabs is not None else 17) * slab
    bn, sp, _, m_pad, n_pad = _plan(g, partial_bytes)
    if _num_sms() == REFERENCE_SMS:
        assert (bn, sp) == (block_n, splits), "the shape no longer hits the case it stands for"
    dzp, xp = _operands(g, planes, dev, seed)
    runs = []
    for _ in range(2):
        grad = torch.full((g.c_out, g.c_in, g.taps), float("nan"), dtype=torch.float32, device=dev)
        partial = torch.full((partial_bytes // 4,), float("nan"), dtype=torch.float32, device=dev)
        assert _call(g, dzp, xp, grad, partial) == 0, _capi.load().vp3d_last_error()
        runs.append((grad, partial))
    (grad, partial), (grad2, partial2) = runs
    assert torch.equal(grad, grad2), "second call differs"
    assert not torch.isnan(grad).any(), "every gradient entry is written, no padding NaN reaches it"

    # the kernel's own split count: slabs [0, sp) written, the next one untouched; the gradient is
    # their left-to-right fp32 sum
    slabs_seen = min(sp + 1, partial_bytes // slab)
    parts = _partials_real(g, partial, slabs_seen, m_pad, n_pad)
    assert not torch.isnan(parts[:sp]).any()
    if slabs_seen > sp:
        assert torch.isnan(parts[sp]).all(), "more splits than the mirror predicts"
    acc = parts[0].clone()
    for s in range(1, sp):
        acc = acc + parts[s]
    assert torch.equal(acc, grad), "gradient is not the ordered sum of the split partials"

    pairs = _products(dzp, xp)
    ref = _ref(g, pairs)
    mag = sum(_dw(g, a.abs(), b.abs()) for a, b in pairs)
    K = g.rows * g.s
    k = 4 * math.sqrt(K) + 64
    worst = float(((grad.double() - ref).abs() / (U * mag).clamp_min(1e-300)).max())
    print(f"planes {planes} tile {bn} splits {sp} K {K}: max |err| = {worst:.1f} x 2^-24 A (gate {k:.0f})")
    assert _gate(grad, ref, mag, k), worst

    # the gate rejects: one 64-row chunk lost at a split boundary (or in the middle)
    kchunks = -(-g.rows // 64)
    kb = (g.s * kchunks) // sp if sp > 1 else (g.s * kchunks) // 2
    n, r0 = kb // kchunks, (kb % kchunks) * 64
    r1 = min(r0 + 64, g.rows)
    lost = sum(_dw(g, a[n:n + 1], b[n:n + 1], r0=r0, r1=r1) for a, b in pairs)
    assert not _gate(grad, ref - lost, mag, k), "gate misses a lost chunk"
    # ... one tap read one row (row taps) or one column (column taps / merged / 1x1) off
    t = min(1, g.taps - 1)
    shift = (t, 1, 0) if g.tap_row_step else (t, 0, 1)
    assert not _gate(grad, _ref(g, pairs, shift=shift), mag, k), "gate misses a shifted tap"
    # ... one sample's dZ paired with its neighbour's X
    if g.per_sample and g.samples > 1:
        swap = sum(_dw(g, a[:1], b[1:2]) - _dw(g, a[:1], b[:1]) for a, b in pairs)
        assert not _gate(grad, ref + swap, mag, k), "gate misses a sample mix-up"
    return sp


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_matches_fp64(cuda_device, name, planes):
    g, block_n, splits = CASES[name]
    _run_case(cuda_device, g, planes, block_n, splits)


@pytest.mark.parametrize("planes", [1, 2])
def test_small_partial_buffer_forces_fewer_splits(cuda_device, planes):
    """Room for 5 split slabs (and a little more): 1x1_c192 runs 5 splits instead of 16."""
    g, _, _ = CASES["1x1_c192"]
    assert _run_case(cuda_device, g, planes, 64, 5, partial_slabs=5) == 5


def test_partial_buffer_below_one_split_is_an_error(cuda_device):
    g, _, _ = CASES["strided_c256_w3"]
    slab = _plan(g, 1 << 62)[2]
    dzp, xp = _operands(g, 2, cuda_device, 5)
    grad = torch.full((g.c_out, g.c_in, g.taps), float("nan"), dtype=torch.float32, device=cuda_device)
    partial = torch.full((slab // 4 - 1,), float("nan"), dtype=torch.float32, device=cuda_device)
    assert _call(g, dzp, xp, grad, partial) == -4   # VP3D_ERR_WORKSPACE
    assert b"partial buffer too small" in _capi.load().vp3d_last_error()
    assert torch.isnan(grad).all() and torch.isnan(partial).all(), "nothing may be written"
