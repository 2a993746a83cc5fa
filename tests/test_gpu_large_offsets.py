"""GPU: the inference paths at sizes where a 32-bit element or byte offset would wrap.

Every other GPU suite stays below 2^31 elements per buffer.  The offset arithmetic is 64-bit
throughout (the conv GEMM epilogue's rows and plane strides, the input pack's rows, the clip
kernels' row scan, the histogram's floor on its block count), and users reach these sizes: a long
recording through ``predict``, a large batch through ``model(x)`` or ``calibrate_int8``, a large
training batch from ``ChunkedGenerator``.  If an ``int`` slipped into one of those offsets only the
rows past the boundary would come out wrong, so each case below compares exactly those rows:

1. ``test_conv_gemm_launch_past_2_31``: one ``vp3d_conv_gemm`` launch per epilogue, against
   float64 (gpu_utils.expected_conv / expected_residual, the gates of
   test_gpu_conv_gemm_instances) on the 128-row tiles on both sides of every element boundary
   k 2^31 and byte boundary k 2^32 of each output plane, the last tile and a few random tiles;
   the guard rows around the output stay untouched.
2. ``test_offline_forward_planes_past_2_31``: TemporalModel 3,3,3,3,3 at C = 1024 on the dilated
   schedule; the samples past the boundary run alone give the same bits (every GEMM of the
   dilated schedule sums a row in the same order wherever the row sits), two of them within
   test_gpu_parity's 1e-3 of oracle.temporal_model_oracle.forward_numpy in float64.
3. ``test_clip_chain_past_2_31``: ``predict([long_clip, short_clip])``, the long clip one chain
   whose activation planes pass 2^31 elements; frames at the boundary and at the end equal, bit
   for bit, ``predict`` on a window of the clip that holds their receptive fields (fp16 with and
   without augment, int8).
4. ``test_int8_calibration_past_2_31``: the device histograms and maxima of a batch whose
   activations pass 2^31 elements equal the sums and maxima of its halves calibrated alone; the
   int8 forward of that batch (blocks 2 and 4 on u8 x s8, so a quantize_u8 pass reads X_1) gives
   the far samples' bits.
5. ``test_chunked_generator_past_2_31``: one ``ChunkedGenerator`` batch of 2^31 + elements
   (2^33 + bytes), bit for bit against oracle.generator_oracle on windows at every boundary, the
   last window and random ones, 2-D, 3-D and cameras.

Every gate is shown, in the same test, to reject the answer a wrapped offset would give: the
compared rows are replaced by the rows their offset modulo 2^31 elements (or 2^32 bytes)
addresses, and the gate must fail on them.  No kernel is ever run with a truncated index.

Each case states the device bytes it needs (the sizing entry points vp3d_workspace_bytes,
vp3d_clips_workspace_bytes, vp3d_int8_hist_bytes plus its own tensors), skips when
torch.cuda.mem_get_info() shows less free, frees everything before the next case, and stays under
MAX_BYTES (the machines are shared).  Peak torch.cuda.max_memory_allocated() and wall time of
the test body per case, measured on an H100 80GB HBM3 at a 700 W power limit (19 s for the file):

    conv GEMM  lean_fp16_tma_res                8.30 GiB  0.7 s
               general_bf16x3_res_sample_div   12.62 GiB  0.1 s
               general_f32_shrink               9.07 GiB  0.0 s
    forward    fp16 N = 5800                   12.84 GiB  1.3 s
               bf16x3 N = 2900                 12.64 GiB  1.0 s
    clips      fp16                            13.70 GiB  0.4 s
               fp16 augment                    13.26 GiB  0.8 s
               int8                            15.70 GiB  0.3 s
    int8 calibration                           14.88 GiB  1.2 s
    chunked generator                           8.21 GiB  0.3 s

Out of scope: the pose loss and metric kernels (inputs past 2^31 floats need over 17 GB for
prediction and target together), streaming sessions (their buffers scale with streams x receptive
field, not with sequence length) and data-parallel training.
"""
import ctypes
import gc
import time

import numpy as np
import pytest
import torch

import eval_replay as er
from gpu_utils import expected_conv, expected_residual
from oracle import generator_oracle as gorc
from oracle import temporal_model_oracle as orc
import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200 import generators as G

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MAX_BYTES = 24 * GiB
E31, B32 = 1 << 31, 1 << 32     # the element and byte boundaries a 32-bit offset wraps at
BLOCK_M = 128
GUARD_TOP, GUARD_BOTTOM = 8, 128
FW, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
RF = 243
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


# ------------------------------------------------------------------------------ budget
@pytest.fixture
def budget(cuda_device):
    """Starts a case with nothing cached, reports its peak and wall time, frees it all."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n  peak {torch.cuda.max_memory_allocated() / GiB:.2f} GiB, "
          f"{time.perf_counter() - t0:.1f} s")
    gc.collect()
    torch.cuda.empty_cache()


def _require(need, what):
    """Skips (never retries) when the device has less than `need` bytes free."""
    assert need <= MAX_BYTES, f"{what}: needs {need / GiB:.1f} GiB, more than the case may take"
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{what}: needs {need / GiB:.1f} GiB, {free / GiB:.1f} GiB free")


def _wrapped(offsets, modulus):
    """The offsets a 32-bit wrap at `modulus` leaves of them."""
    return offsets % modulus


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


# ------------------------------------------------------------------------------ 1. conv GEMM
# (epilogue, operand format, auxiliary TMA tiles, two planes) the launch must select
CONV = [
    # fp16 X plane of 2^21 + 1000 rows x 1024: elements pass 2^31, bytes pass 2^32; the
    # residual (one row on) comes through TMA
    dict(name="lean_fp16_tma_res", fmt="fp16", rows=(1 << 21) + 1000, n_pad=1024, k=64,
         out="16", planes=1, res="tma", key=(2, 2, 1, 0)),
    # split-bf16 hi + lo planes: the lo plane starts (rows + guard) x 1024 > 2^31 elements in and
    # ends past 2^32; the residual map splits rows per 128-row sample (register path)
    dict(name="general_bf16x3_res_sample_div", fmt="bf16x3", rows=(1 << 21) + 1000, n_pad=1024,
         k=64, out="16", planes=2, res="div", key=(1, 0, 0, 1)),
    # the shrink's shape: fp32 rows of 51 channels, bytes pass 2^32 (elements stay below 2^31)
    dict(name="general_f32_shrink", fmt="fp16", rows=21_100_000, n_pad=64, k=128, out="f32",
         planes=1, res=None, key=(1, 0, 0, 0)),
]
RES_RPS, RES_OFF, RES_DIV = 130, 1, 128
PRECISION = {"bf16": 0, "bf16x3": 1, "fp16": 3}


def _uniform(shape, dt, lo, hi, gen):
    t = torch.empty(shape, dtype=dt, device="cuda")
    return t.uniform_(lo, hi, generator=gen)


class ConvCase:
    def __init__(self, c):
        self.c = c
        R, n_pad, k = c["rows"], c["n_pad"], c["k"]
        gen = torch.Generator(device="cuda").manual_seed(sum(map(ord, c["name"])))
        dt = torch.float16 if c["fmt"] == "fp16" else torch.bfloat16
        self.dt = dt
        if c["fmt"] == "bf16x3":
            a32 = _uniform((R, k), torch.float32, -1, 1, gen)
            self.a = torch.stack([a32.bfloat16(), (a32 - a32.bfloat16().float()).bfloat16()])
            del a32
            w32 = _uniform((1, n_pad, k), torch.float32, -1, 1, gen) / k ** 0.5
            self.w = torch.stack([w32.bfloat16(), (w32 - w32.bfloat16().float()).bfloat16()])
        else:
            self.a = _uniform((1, R, k), dt, -1, 1, gen)
            self.w = (_uniform((1, n_pad, k), torch.float32, -1, 1, gen) / k ** 0.5).to(dt)
            self.w = self.w.unsqueeze(0)
        self.w = self.w.contiguous()   # [planes][taps = 1][n_pad][k]
        self.scale = _uniform((n_pad,), torch.float32, 0.5, 1.5, gen)
        self.shift = _uniform((n_pad,), torch.float32, -0.5, 0.5, gen)
        self.res = None
        if c["res"] == "tma":
            self.res = _uniform((1, R + RES_OFF, n_pad), dt, -2, 2, gen)
        elif c["res"] == "div":
            self.res = _uniform((1, (R // RES_DIV + 1) * RES_RPS, n_pad), dt, -2, 2, gen)
        if c["out"] == "16":
            self.ld = n_pad
            self.out = torch.full((c["planes"], GUARD_TOP + R + GUARD_BOTTOM, self.ld),
                                  float("nan"), dtype=dt, device="cuda")
        else:
            self.ld = 51
            self.out = torch.full((1, GUARD_TOP + R + GUARD_BOTTOM, self.ld), float("nan"),
                                  dtype=torch.float32, device="cuda")
        self.plane = self.out[0].numel()   # elements between the planes

    @staticmethod
    def bytes_needed(c):
        R, n_pad, k = c["rows"], c["n_pad"], c["k"]
        a_planes = 2 if c["fmt"] == "bf16x3" else 1
        need = a_planes * R * k * 2 + (R * k * 4 if a_planes == 2 else 0)   # A (+ its fp32 source)
        if c["res"] == "tma":
            need += (R + RES_OFF) * n_pad * 2
        elif c["res"] == "div":
            need += (R // RES_DIV + 1) * RES_RPS * n_pad * 2
        rows = GUARD_TOP + R + GUARD_BOTTOM
        need += c["planes"] * rows * n_pad * 2 if c["out"] == "16" else rows * 51 * 4
        return need + GiB   # the reference tiles, the guard checks, the allocator's slack

    def desc(self):
        c = self.c
        d = _capi.ConvDesc()
        d.a = self.a.data_ptr(); d.a_planes = self.a.shape[0]
        d.samples = 1; d.a_rows = c["rows"]; d.a_ld = c["k"]
        d.w = self.w.data_ptr(); d.taps = 1; d.k_per_tap = c["k"]; d.n_pad = c["n_pad"]
        d.per_sample_tiles = 0; d.tap_row_step = 0; d.tap_col_step = 0
        d.out_rows = c["rows"]; d.precision = PRECISION[c["fmt"]]
        d.scale = self.scale.data_ptr(); d.shift = self.shift.data_ptr()
        d.relu = int(c["out"] == "16")
        if self.res is not None:
            d.res = self.res.data_ptr(); d.res_planes = 1
            d.res_plane_stride = self.res[0].numel(); d.res_ld = c["n_pad"]
            d.res_row_step = 1; d.res_row_off = RES_OFF
            if c["res"] == "div":
                d.res_rows_per_sample = RES_RPS; d.res_sample_div = RES_DIV
        body = self.out[0, GUARD_TOP:].data_ptr()
        if c["out"] == "16":
            d.out = body; d.out_planes = c["planes"]
            d.out_plane_stride = self.plane; d.out_ld = self.ld
        else:
            d.out_f32 = body; d.out_f32_ld = self.ld; d.n_valid = 51
        return d

    def reference(self, r0, r1):
        """(v, err) of rows [r0, r1): the float64 epilogue value and its accumulation bound
        (test_gpu_conv_gemm_instances.reference on these rows)."""
        c = self.c
        n = r1 - r0
        geo = dict(samples=1, a_rows=n, taps=1, k_per_tap=c["k"], per_sample_tiles=False,
                   tap_row_step=0, tap_col_step=0, out_rows=n)
        a, w = self.a[:, r0:r1].double(), self.w.double()
        if self.a.shape[0] == 2:
            acc = expected_conv(a[0], w[0] + w[1], **geo) + expected_conv(a[1], w[0], **geo)
            mag = expected_conv((a[0] + a[1]).abs(), (w[0] + w[1]).abs(), **geo)
            pairs = 3
        else:
            acc = expected_conv(a[0], w[0], **geo)
            mag = expected_conv(a[0].abs(), w[0].abs(), **geo)
            pairs = 1
        scale, shift = self.scale.double(), self.shift.double()
        v = acc * scale + shift
        if c["out"] == "16":
            v = v.clamp_min(0.0)
        res_abs = 0.0
        if self.res is not None:
            if c["res"] == "tma":
                src = self.res[:, r0 + RES_OFF:r1 + RES_OFF].double()
                rm = dict(samples=1, out_rows=n, per_sample_tiles=False)
            else:   # a tile is one sample of RES_DIV rows
                s = r0 // RES_DIV
                src = self.res[:, s * RES_RPS:(s + 1) * RES_RPS].double()
                rm = dict(samples=1, out_rows=n, per_sample_tiles=False,
                          res_rows_per_sample=RES_RPS, res_row_off=RES_OFF,
                          res_sample_div=RES_DIV)
            v = v + expected_residual(src, c["n_pad"], **rm)
            res_abs = expected_residual(src.abs(), c["n_pad"], **rm)
        steps = pairs * c["k"] // 16
        err = (mag * 2.0 ** -20 + acc.abs() * (steps * 2.0 ** -23)) * scale.abs()
        err = err + 2.0 ** -23 * ((acc * scale).abs() + shift.abs() + res_abs)
        return v, err

    def rows_of(self, plane, r0, r1, modulus=None):
        """Rows [r0, r1) of an output plane, read at their element offsets from the output
        pointer, or at those offsets modulo `modulus` (what a wrapped offset addresses)."""
        flat = self.out.view(-1)
        cols = self.c["n_pad"] if self.c["out"] == "16" else 51
        off = (plane * self.plane + torch.arange(r0, r1, device="cuda")[:, None] * self.ld
               + torch.arange(cols, device="cuda")[None, :])
        if modulus is not None:
            off = _wrapped(off, modulus)
        return flat[GUARD_TOP * self.ld + off]

    def check_tile(self, got, v, err):
        """The instance suite's gates; got: [planes][rows][cols].  Returns a failure or None."""
        c = self.c
        if c["out"] == "f32":
            g = got[0].double()
            bad = ~((g - v[:, :51]).abs() <= 2.0 ** -23 * v[:, :51].abs() + err[:, :51])
            return f"{int(bad.sum())} fp32 outputs out of bound" if bad.any() else None
        hi = got[0].double()
        if c["fmt"] == "fp16":
            exp = v.clamp(-er.FP16_MAX, er.FP16_MAX)
            bad = ~((hi - exp).abs() <= 2.0 ** -11 * exp.abs() + err + 2.0 ** -24)
        else:
            bad = ~((hi - v).abs() <= 2.0 ** -8 * v.abs() + err)
        if bad.any():
            return f"{int(bad.sum())} 16-bit outputs out of bound"
        if c["planes"] == 2:
            two = hi + got[1].double()
            bad = ~((two - v).abs() <= 2.0 ** -16 * v.abs() + err)
            if bad.any():
                return f"{int(bad.sum())} hi + lo outputs out of bound"
        return None


def _boundary_tiles(R, ld, plane_offsets, esize, rng, extra=6):
    """First rows of the 128-row tiles on both sides of every k 2^31-element and k 2^32-byte
    offset of every plane, the last tile and `extra` random ones."""
    tiles = {(R - 1) // BLOCK_M}
    for base in plane_offsets:
        end = base + R * ld
        for step in (E31, B32 // esize):
            for b in range((base // step + 1) * step, end, step):
                row = (b - base) // ld
                tiles.update(t for t in (row // BLOCK_M - 1, row // BLOCK_M, row // BLOCK_M + 1)
                             if 0 <= t * BLOCK_M < R)
    tiles.update(int(t) for t in rng.integers(0, (R - 1) // BLOCK_M + 1, extra))
    return sorted(t * BLOCK_M for t in tiles)


def _guard_untouched(case):
    """Every guard row (above and below the output, each plane) still holds its NaN bits."""
    nan = _bits(torch.full((1,), float("nan"), dtype=case.out.dtype, device="cuda"))[0]
    R = case.c["rows"]
    for p in range(case.out.shape[0]):
        for rows in (slice(0, GUARD_TOP), slice(GUARD_TOP + R, None)):
            g = _bits(case.out[p, rows])
            assert bool((g == nan).all()), \
                f"{case.c['name']}: {int((g != nan).sum())} stores into the guard rows of plane {p}"


@pytest.mark.parametrize("c", CONV, ids=[c["name"] for c in CONV])
def test_conv_gemm_launch_past_2_31(budget, c):
    """One launch whose output plane passes 2^31 elements (lean fp16, general bf16x3 with its
    lo plane wholly past 2^31) or 2^32 bytes (fp32 shrink shape), K of one or two k-blocks."""
    _require(ConvCase.bytes_needed(c), c["name"])
    case = ConvCase(c)
    R, esize = c["rows"], case.out.element_size()
    assert case.plane * (c["planes"] - 1) + R * case.ld > (E31 if c["out"] == "16" else B32 // 4)
    d = case.desc()
    key = (ctypes.c_int * 7)()
    lib = _capi.load()
    _capi.check(lib.vp3d_conv_gemm_instance(ctypes.byref(d), key), "vp3d_conv_gemm_instance")
    assert (key[1], key[2], key[4], key[5]) == c["key"], f"{c['name']} selects {tuple(key)}"
    _capi.check(lib.vp3d_conv_gemm(ctypes.byref(d), torch.cuda.current_stream().cuda_stream),
                "vp3d_conv_gemm")
    torch.cuda.synchronize()
    _guard_untouched(case)
    rng = np.random.default_rng(7)
    planes = [p * case.plane for p in range(c["planes"])]
    tiles = _boundary_tiles(R, case.ld, planes, esize, rng)
    for r0 in tiles:
        r1 = min(r0 + BLOCK_M, R)
        v, err = case.reference(r0, r1)
        got = torch.stack([case.rows_of(p, r0, r1) for p in range(c["planes"])])
        bad = case.check_tile(got, v, err)
        assert bad is None, f"{c['name']}: tile at row {r0}: {bad}"
    # the gate rejects the last tile read where a wrapped offset points: 2^31 elements for the
    # 16-bit planes, 2^32 bytes for fp32
    modulus = E31 if c["out"] == "16" else B32 // esize
    r0 = tiles[-1]
    r1 = min(r0 + BLOCK_M, R)
    assert (c["planes"] - 1) * case.plane + r0 * case.ld >= modulus
    v, err = case.reference(r0, r1)
    wrong = torch.stack([case.rows_of(p, r0, r1, modulus) for p in range(c["planes"])])
    assert case.check_tile(wrong, v, err) is not None, \
        f"{c['name']}: the gate accepts the rows a wrapped offset reads"
    print(f"  {c['name']}: key {tuple(key)}, {len(tiles)} tiles checked")


# ------------------------------------------------------------------------------ 2. offline forward
def _model(dev, precision="fp16", seed=0):
    """TemporalModel 3,3,3,3,3 at C = 1024 (an int8 model stays fp16 until calibrated)."""
    m = vp.TemporalModel(J, F, J, filter_widths=FW, dropout=0.0, channels=C)
    m.load_state_dict(orc.make_state_dict(J, F, J, FW, C, seed=seed))
    m = m.to(dev).eval()
    return m if precision == "int8" else m.set_precision(precision)


def _input(N, T, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return _uniform((N, T, J, F), torch.float32, -1, 1, g)


def _layer_rows(T):
    """Rows per sample out of every stage of the dilated 3,3,3,3,3 schedule."""
    L, d = [], 1
    for w in FW:
        T -= (w - 1) * d
        L.append(T)
        d *= w
    return L


def _far_samples(N, L0, planes):
    """(straddling sample, first sample wholly past 2^31) of the X_0 planes: the lo plane of
    bf16x3 starts N L0 C elements in."""
    lo0 = (planes - 1) * N * L0 * C
    s = (E31 - lo0) // (L0 * C)
    return s, s + 1


def _wrapped_sample(n, N, L0, planes):
    """The sample whose X_0 rows an offset of sample n's wrapped at 2^31 would read."""
    off = (planes - 1) * N * L0 * C + n * L0 * C
    w = _wrapped(off, E31) // (L0 * C)
    return int(w % N)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


T_FWD = 370   # L = 368, 362, 344, 290, 128 rows per sample


@pytest.mark.parametrize("precision,N", [("fp16", 5800), ("bf16x3", 2900)])
def test_offline_forward_planes_past_2_31(budget, cuda_device, precision, N):
    """fp16: X_0 and H_1 / X_1 hold N L C = 5800 x 368 x 1024 = 2.19e9 and 5800 x 362 x 1024 =
    2.15e9 > 2^31 elements.  bf16x3: the lo plane starts N L C = 2900 x 368 x 1024 = 1.09e9
    elements past the hi plane, so the lo rows of samples >= 2799 sit past 2^31."""
    dev = cuda_device
    planes = 2 if precision == "bf16x3" else 1
    L = _layer_rows(T_FWD)
    assert (planes * N * L[0] * C > E31) and (planes * N * L[1] * C > E31)
    m = _model(dev, precision)
    lib = _capi.load()
    ws = lib.vp3d_workspace_bytes(m._get_plan(dev, precision), N, T_FWD)
    need = ws + N * T_FWD * J * F * 4 + N * L[-1] * J * 3 * 4 + GiB
    _require(need, f"forward {precision} N={N}")
    x = _input(N, T_FWD, dev, seed=11)
    with torch.no_grad():
        y = m(x)
    straddle, first_far = _far_samples(N, L[0], planes)
    idx = [0, straddle, first_far, (first_far + N) // 2, N - 2, N - 1]
    with torch.no_grad():
        alone = m(x[idx].contiguous())
    for i, n in enumerate(idx):
        assert _same_bits(y[n], alone[i]), f"sample {n} differs from the same sample run alone"
    # two far samples against float64 within test_gpu_parity's model-level gate
    sd = orc.make_state_dict(J, F, J, FW, C, seed=0)
    far = [first_far, N - 1]
    ref = orc.forward_numpy(sd, x[far].cpu().numpy(), FW, dtype=np.float64)
    err = _rel(y[far].cpu().numpy(), ref)
    assert err <= 1e-3, f"far samples {far}: rel err {err:.2e} against float64"
    # both gates reject the far samples' outputs replaced by those of the samples a wrapped
    # offset reads
    wrong = torch.stack([y[_wrapped_sample(n, N, L[0], planes)] for n in idx[2:]])
    assert not _same_bits(wrong, alone[2:]), "the bit gate accepts wrapped samples"
    wrong_far = np.stack([y[_wrapped_sample(n, N, L[0], planes)].cpu().numpy() for n in far])
    assert _rel(wrong_far, ref) > 1e-3, "the float64 gate accepts wrapped samples"
    print(f"  {precision} N={N}: workspace {ws / GiB:.2f} GiB, far samples {idx}, "
          f"rel err {err:.2e}")


# ------------------------------------------------------------------------------ 3. clip chains
def _predict(m, clips, augment):
    kw = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT) if augment \
        else {}
    with torch.no_grad():
        return m.predict(clips, augment=augment, **kw)


@pytest.mark.parametrize("precision,augment", [("fp16", False), ("fp16", True),
                                               ("int8", False)])
def test_clip_chain_past_2_31(budget, cuda_device, precision, augment):
    """The long clip's chain has rows = copies (T + 242) rows: T = 2^21 + 4000 (2^20 + 4000
    with augment) gives X_0 (rows - 2) x 1024 > 2^31 elements, X_1 and H_1 (rows - 8) x 1024
    too.  Frame f of copy 0 sits at chain row f, of the mirrored copy at row P + f, P = T + 242."""
    dev = cuda_device
    copies = 2 if augment else 1
    T = (1 << (21 if copies == 1 else 20)) + 4000
    P = T + RF - 1
    rows = copies * P
    assert (rows - 8) * C > E31
    m = _model(dev, precision)
    if precision == "int8":
        m.calibrate_int8(_input(4, 600, dev, seed=3))
        m.set_precision("int8")
    lib = _capi.load()
    flags = _capi.VP3D_CLIPS_AUGMENT if augment else 0
    ws = lib.vp3d_clips_workspace_bytes(m._get_plan(dev, precision), rows, flags)
    assert ws > 0
    # the clips, their concatenation inside predict, and the poses
    need = ws + 2 * (T + 300) * J * F * 4 + (T + 300) * J * 3 * 4 + GiB
    _require(need, f"clip chain {precision} augment={augment}")
    x = _input(T, 1, dev, seed=21).view(T, J, F)
    short = _input(300, 1, dev, seed=22).view(300, J, F)
    y_long, y_short = _predict(m, [x, short], augment)
    K = 64
    # frames at the 2^31-element row of X_0 (the mirrored copy's, with augment) and at the end
    f_b = (E31 // C) - (copies - 1) * P - RF // 2
    windows = [f_b - K // 2, T - K]
    demos = 0
    for f0 in windows:
        lo = f0 - (RF - 1)
        win = x[lo:min(T, f0 + K + RF - 1)].contiguous()
        y_win = _predict(m, [win], augment)[0]
        got, exp = y_long[f0:f0 + K], y_win[RF - 1:RF - 1 + K]
        assert _same_bits(got, exp), \
            f"frames [{f0}, {f0 + K}) differ from predict on the window from frame {lo}"
        # the gate rejects, for frames whose X_0 rows lie past 2^31 elements, the frames their
        # wrapped row offsets read (row r' < P: frame r' of the clip; else the mirrored copy's)
        if (f0 + (copies - 1) * P) * C >= E31:
            wrapped = [int(_wrapped((f + (copies - 1) * P) * C, E31) // C)
                       for f in range(f0, f0 + K)]
            fw = [r - P if r >= P else r for r in wrapped]
            assert not _same_bits(y_long[fw], exp), "the bit gate accepts wrapped frames"
            demos += 1
    assert demos > 0, "no compared frame lies past the boundary"
    assert y_short.shape == (300, J, 3) and bool(torch.isfinite(y_short).all())
    print(f"  {precision} augment={augment}: chain of {rows} rows, workspace {ws / GiB:.2f} GiB")


# ------------------------------------------------------------------------------ 4. int8 calibration
N_CAL = 5800


def _calibrate(m, x, hist):
    """vp3d_calibrate_int8_hist (hist=True: [2B][BINS] counts, then the invalid counts) or
    vp3d_calibrate_int8 (the 2B maxima) of batch x on its own."""
    lib = _capi.load()
    dev = x.device
    plan = m._get_plan(dev, "fp16")
    stream = torch.cuda.current_stream(dev).cuda_stream
    m._sync_weights(plan, stream)
    N, T = int(x.shape[0]), int(x.shape[1])
    ws = torch.empty(lib.vp3d_workspace_bytes(plan, N, T), dtype=torch.uint8, device=dev)
    if hist:
        out = torch.zeros(lib.vp3d_int8_hist_bytes(plan) // 8, dtype=torch.int64, device=dev)
        _capi.check(lib.vp3d_calibrate_int8_hist(plan, x.data_ptr(), N, T, ws.data_ptr(),
                                                 ws.numel(), out.data_ptr(), stream),
                    "vp3d_calibrate_int8_hist")
    else:
        out = torch.zeros(2 * (len(FW) - 1), dtype=torch.float32, device=dev)
        _capi.check(lib.vp3d_calibrate_int8(plan, x.data_ptr(), N, T, ws.data_ptr(), ws.numel(),
                                            out.data_ptr(), stream), "vp3d_calibrate_int8")
    torch.cuda.synchronize()
    del ws
    return out.cpu()


def test_int8_calibration_past_2_31(budget, cuda_device):
    """Activations of N = 5800 samples of T = 370 frames: X_0 holds 5800 x 368 x 1024 = 2.19e9
    and H_1 / X_1 5800 x 362 x 1024 = 2.15e9 elements, past 2^31 (hist_f16_kernel, amax_f16_kernel
    over them; in the int8 forward quantize_u8 over X_1); each half alone stays below."""
    dev = cuda_device
    N, T = N_CAL, T_FWD
    L = _layer_rows(T)
    assert N * L[0] * C > E31 and N * L[1] * C > E31 and (N // 2) * L[0] * C < E31
    m = _model(dev, "fp16")
    lib = _capi.load()
    fp16 = m._get_plan(dev, "fp16")
    ws16 = lib.vp3d_workspace_bytes(fp16, N, T)
    ws8 = lib.vp3d_workspace_bytes(m._get_plan(dev, "int8"), N, T)
    x_bytes = N * T * J * F * 4
    need = max(ws16 + lib.vp3d_int8_hist_bytes(fp16), ws8) + 2 * x_bytes + GiB
    _require(need, "int8 calibration")
    x = _input(N, T, dev, seed=31)
    x[N - 1] *= 4   # the largest activations in the last sample, wholly past 2^31
    x[N - 1, T - 1, 0, 0] = float("nan")
    x[N - 2, 5, 3, 1] = float("inf")
    halves = [x[:N // 2], x[N // 2:]]
    hist = _calibrate(m, x, True)
    parts = [_calibrate(m, h, True) for h in halves]
    assert torch.equal(hist, parts[0] + parts[1]), \
        f"{int((hist != parts[0] + parts[1]).sum())} histogram bins differ from the halves' sum"
    invalid0 = 2 * (len(FW) - 1) * 0x7C00   # X_0's invalid count, after every layer's bins
    assert int(hist[invalid0]) >= 2, "the two non-finite inputs are not counted"
    amax = _calibrate(m, x, False)
    amax_parts = torch.maximum(*[_calibrate(m, h, False) for h in halves])
    assert torch.equal(amax, amax_parts), f"amax {amax.tolist()} != halves' {amax_parts.tolist()}"
    # both gates reject the far samples counted where a wrapped offset reads
    straddle, first_far = _far_samples(N, L[0], 1)
    wrapped = [_wrapped_sample(n, N, L[0], 1) for n in range(first_far, N)]
    near, wrap_x = x[:first_far], x[wrapped].contiguous()
    assert not torch.equal(hist, _calibrate(m, near, True) + _calibrate(m, wrap_x, True)), \
        "the histogram gate accepts wrapped samples"
    assert not torch.equal(amax, torch.maximum(_calibrate(m, near, False),
                                               _calibrate(m, wrap_x, False))), \
        "the amax gate accepts wrapped samples"
    del near, wrap_x, halves
    # the int8 forward of the same batch: blocks 1 and 3 fp16, so quantize_u8 reads X_1 and X_3
    m.load_int8_calibration(amax)
    m.set_int8_blocks([2, 4]).set_precision("int8")
    with torch.no_grad():
        y = m(x)
        idx = [0, straddle, first_far, N - 2, N - 1]
        alone = m(x[idx].contiguous())
    for i, n in enumerate(idx):
        assert _same_bits(y[n], alone[i]), f"int8: sample {n} differs from the sample alone"
    wrong = torch.stack([y[_wrapped_sample(n, N, L[0], 1)] for n in idx[2:]])
    assert not _same_bits(wrong, alone[2:]), "the int8 bit gate accepts wrapped samples"
    print(f"  workspaces fp16 {ws16 / GiB:.2f} GiB, int8 {ws8 / GiB:.2f} GiB; "
          f"amax {[round(float(a), 3) for a in amax]}")


# ------------------------------------------------------------------------------ 5. generators
def test_chunked_generator_past_2_31(budget, cuda_device):
    """One batch of 262144 windows of 1 + 2 x 121 frames x 17 x 2 floats: 2,165,833,728 elements
    (> 2^31) and 8.66e9 bytes (> 2 x 2^32) in the 2-D output."""
    dev = cuda_device
    bs, chunk, pad = 262144, 1, 121
    frames = chunk + 2 * pad
    per_window = frames * J * F
    assert bs * per_window > E31 and bs * per_window * 4 > 2 * B32
    lengths = [50000, 60000, 30000]   # 280000 mirrored-augmented windows: batch 0 is full
    need = bs * per_window * 4 + bs * chunk * J * 3 * 4 + bs * 9 * 4 + GiB
    _require(need, "chunked generator")
    rng = np.random.RandomState(5)
    p2 = [rng.uniform(-1, 1, (n, J, F)).astype(np.float32) for n in lengths]
    p3 = [rng.uniform(-1, 1, (n, J, 3)).astype(np.float32) for n in lengths]
    cams = [rng.uniform(-1, 1, 9).astype(np.float32) for _ in lengths]
    kw = dict(pad=pad, causal_shift=0, shuffle=True, random_seed=9, augment=True,
              kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
    gen = G.ChunkedGenerator(bs, cams, p3, p2, chunk, device=dev, **kw)
    cam, b3, b2 = next(gen.next_epoch())
    torch.cuda.synchronize()
    assert b2.shape == (bs, frames, J, F)
    orc_gen = gorc.ChunkedGeneratorOracle(bs, cams, p3, p2, chunk, **kw)
    _, order = orc_gen.epoch_order()
    # windows at every element boundary k 2^31 and byte boundary k 2^32, the last, random ones
    sample = {bs - 1}
    for step in (E31, B32 // 4):
        for b in range(step, bs * per_window, step):
            sample.update(range(b // per_window - 1, b // per_window + 2))
    sample.update(int(w) for w in np.random.default_rng(3).integers(0, bs, 16))
    sample = sorted(sample)
    cam_o, b3_o, b2_o = orc_gen.batch(order[sample])

    def same(dev_t, oracle):
        return np.array_equal(dev_t.cpu().numpy().view(np.uint32),
                              oracle.astype(np.float32).view(np.uint32))
    assert same(b2[sample], b2_o), "2-D windows differ from the oracle"
    assert same(b3[sample], b3_o), "3-D windows differ from the oracle"
    assert same(cam[sample], cam_o), "cameras differ from the oracle"
    # the gate rejects the windows past each boundary read at their wrapped offsets
    flat = b2.view(-1)
    for modulus in (E31, B32 // 4):
        far = [w for w in sample if w * per_window >= modulus]
        off = torch.tensor(far, device=dev)[:, None] * per_window + \
            torch.arange(per_window, device=dev)[None, :]
        wrong = flat[_wrapped(off, modulus)].view(len(far), frames, J, F)
        _, _, b2_far = orc_gen.batch(order[far])
        assert not same(wrong, b2_far), f"the gate accepts windows wrapped at {modulus}"
    print(f"  {len(sample)} windows checked, output {b2.numel() * 4 / GiB:.2f} GiB")
