"""GPU: every compiled conv GEMM kernel instance, at its tile, pipeline and store edges.

Each case of CASES is one vp3d_conv_gemm launch -- descriptor, operands and an SM limit (set with
vp3d_set_sm_limit, restored afterwards) -- and the instance key it must select.  For every case:
1. instance: vp3d_conv_gemm_instance returns that key (block_n, epilogue, format, schedule,
   auxiliary TMA tiles, two planes, u8 output);
2. float64: the output against the index definition of the operation (gpu_utils.expected_conv and
   expected_residual) on the exact 16-bit values the kernel reads.  What remains is the fp32
   accumulation, acc_err = (2^-20 sum|a||w| + steps 2^-23 |acc|) |scale| (summation order and the
   truncating k16 steps, eval_replay.fake_conv), the epilogue's own fp32 roundings
   (2^-23 (|acc scale| + |shift| + |res|)), and one rounding to the output format:
       fp16   2^-11 |exp| + acc_err + 2^-24   (exp clamped to +-65504: the store saturates)
       bf16   2^-8 |exp| + acc_err
       hi+lo  2^-16 |exp| + acc_err           (on the tiles that meet the lo window)
       fp32   2^-23 |exp| + acc_err
   int8 launches bit for bit against eval_replay.int8_epilogue (exact integer sums, the kernel's
   fp32 chain); the u8 copy of an fp16 launch within one code.  Training launches: every slab of
   the batch-statistics partials written, each within the sum of its rows' bounds;
3. guard zones: the outputs are views into larger buffers (rows above and 128 below, columns past
   n_pad / n_valid) filled with NaN, or a fixed byte for u8; after the launch every element
   outside the region the launch may write is untouched, bit for bit.  The region: rows <
   out_rows, columns < n_pad (< n_valid for fp32), the lo plane only on tiles that meet
   [lo_row_begin, lo_row_end), stats slabs [0, 4 row tiles);
4. a second launch gives the same bits.

The schedule-invariance test runs fixed descriptors under every SM limit that changes their
(block_n, schedule) and asserts bit-identical outputs: predict and streaming promise the offline
forward's bits while launching the same GEMM over other row counts.
"""
import ctypes

import numpy as np
import pytest
import torch

import eval_replay as er
from gpu_utils import expected_conv, expected_residual
from videopose3d_b200 import _capi

BLOCK_M = 128
GUARD_TOP, GUARD_BOTTOM = 8, 128   # guard rows around every output (a whole ragged tile below)
U8_FILL = 0xA5

EPI = {"train": 0, "general": 1, "lean": 2}
FMT = {"runtime": 0, "bf16": 1, "fp16": 2, "int8": 3}
SCHED = {"coop": 0, "pp": 1}
U8 = {"u8beside": 1, "u8alone": 2}


def key(text):
    """'128 lean fp16 pp res' -> the 7 ints of vp3d_conv_gemm_instance."""
    t = text.split()
    flags = set(t[4:])
    assert flags <= {"res", "out2", "u8beside", "u8alone"}, text
    u8 = [U8[f] for f in flags if f in U8]
    return (int(t[0]), EPI[t[1]], FMT[t[2]], SCHED[t[3]], int("res" in flags),
            int("out2" in flags), u8[0] if u8 else 0)


def key_text(k):
    names = [str(k[0]), *(next(n for n, v in m.items() if v == x)
                          for m, x in ((EPI, k[1]), (FMT, k[2]), (SCHED, k[3])))]
    names += ["res"] * k[4] + ["out2"] * k[5] + [n for n, v in U8.items() if v == k[6]]
    return " ".join(names)


PRECISION = {"bf16": 0, "bf16x3": 1, "fp16": 3, "int8": 4}


def case(name, inst, sm, *, fmt="bf16", geo="flat", samples=1, a_rows=None, out_rows=128, taps=1,
         step=0, k=64, n_pad=128, affine=True, relu=True, res=None, out="16", out_planes=1,
         n_valid=None, u8=None, stats=False, lo=None, amp=1.0):
    """geo: 'flat' (1x1, or taps > 1 as column blocks of one row), 'regions' (taps as tap-major
    row regions of out_rows rows), 'dilated' (per-sample tiles, taps `step` rows apart).
    res: None or dict(planes, step, off, rps (rows per sample), div, check, col_begin, cols)."""
    return dict(name=name, key=key(inst), sm=sm, fmt=fmt, geo=geo, samples=samples,
                a_rows=a_rows, out_rows=out_rows, taps=taps, step=step, k=k, n_pad=n_pad,
                affine=affine, relu=relu, res=res, out=out, out_planes=out_planes,
                n_valid=n_valid, u8=u8, stats=stats, lo=lo, amp=amp)


def R(**kw):
    d = dict(planes=1, step=1, off=0, rps=0, div=0, check=0, col_begin=0, cols=0)
    d.update(kw)
    return d


CASES = [
    # ---- training epilogue (batch statistics of the stored value): cooperative only
    case("train_one_kblock_r127", "128 train runtime coop", 4, out_rows=127, n_pad=256,
         stats=True, affine=False, relu=False),
    case("train_two_planes_r129_lo", "64 train runtime coop out2", 5, out_rows=129, n_pad=192,
         out_planes=2, stats=True, lo=(100, 120), affine=False, relu=False, k=192),
    case("train_regions_two_planes", "128 train runtime coop out2", 2, geo="regions", taps=3,
         out_rows=256, n_pad=128, out_planes=2, stats=True, lo=(0, 1), relu=False),
    case("train_dilated_neg_step", "64 train runtime coop", 3, geo="dilated", samples=3,
         a_rows=90, out_rows=90, taps=3, step=-7, n_pad=64, stats=True, relu=False),
    case("train_dilated_tma_res_ragged", "128 train runtime coop res", 3, geo="dilated",
         samples=3, a_rows=104, out_rows=100, taps=3, step=2, n_pad=128, stats=True,
         res=R(rps=104, off=2)),
    case("train_res_strided_view", "64 train runtime coop res", 5, out_rows=300, n_pad=192,
         k=128, stats=True, res=R(step=3, off=2)),
    case("train_res_step2_two_planes", "64 train runtime coop res out2", 4, out_rows=200,
         n_pad=64, stats=True, out_planes=2, res=R(step=2, off=1), lo=(130, 131)),
    case("train_bf16x3_res_two_planes", "128 train runtime coop res out2", 2, fmt="bf16x3",
         out_rows=257, n_pad=256, k=128, stats=True, out_planes=2, res=R(off=5, planes=2)),
    # ---- general epilogue: launches the lean instances do not serve
    case("general_f32_nvalid_fp16", "128 general runtime coop", 2, fmt="fp16", out_rows=129,
         n_pad=256, out="f32", n_valid=200, relu=False),
    case("general_f32_sample_div_res", "64 general runtime coop", 3, out_rows=5 * 44, n_pad=64,
         out="f32", n_valid=51, relu=False, res=R(rps=50, off=3, div=44)),
    case("general_fp16_saturates", "64 general runtime coop", 4, fmt="fp16", out_rows=64,
         n_pad=64, relu=False, amp=4e5),
    case("general_bf16x3_lo_window", "128 general runtime coop out2", 2, fmt="bf16x3",
         out_rows=3 * 128 + 5, n_pad=128, out_planes=2, lo=(130, 300), k=256),
    case("general_check_rows_two_planes", "64 general runtime coop out2", 5, out_rows=9 * 30,
         n_pad=192, out_planes=2, res=R(rps=28, off=-1, div=30, check=1), lo=(0, 200)),
    case("general_col_window_tma_res", "128 general runtime coop res", 2, out_rows=129,
         n_pad=256, res=R(col_begin=128, cols=128, off=7)),
    case("general_two_res_planes_norelu", "64 general runtime coop res", 3, geo="dilated",
         samples=2, a_rows=70, out_rows=70, taps=2, step=5, n_pad=64, relu=False,
         res=R(planes=2, rps=72, off=2)),
    case("general_bf16x3_res_step_two_planes", "128 general runtime coop res out2", 3,
         fmt="bf16x3", out_rows=130, n_pad=128, out_planes=2, res=R(step=2, off=1)),
    case("general_dilated_res_two_planes", "64 general runtime coop res out2", 5, geo="dilated",
         samples=2, a_rows=150, out_rows=140, taps=3, step=5, n_pad=64, out_planes=2,
         res=R(rps=150, off=5)),
    # ---- lean bf16
    case("lean_bf16_one_tile_per_cta", "128 lean bf16 coop", 4, out_rows=256, n_pad=256),
    case("lean_bf16_res_exact_tiles", "128 lean bf16 coop res", 2, geo="dilated", samples=2,
         a_rows=130, out_rows=128, taps=3, step=1, n_pad=128, res=R(rps=130, off=1)),
    case("lean_bf16_pp_idle_warpgroup", "128 lean bf16 pp", 3, out_rows=200, n_pad=256, k=128),
    case("lean_bf16_pp_res_odd_tiles", "128 lean bf16 pp res", 2, geo="dilated", samples=5,
         a_rows=64, out_rows=64, taps=3, step=3, n_pad=128, res=R(rps=128, step=2, off=1)),
    case("lean_bf16_r640_wide_ld", "64 lean bf16 coop", 5, out_rows=640, n_pad=64, taps=3,
         k=64, geo="regions"),
    case("lean_bf16_res_one_row", "64 lean bf16 coop res", 3, out_rows=1, n_pad=192,
         res=R(off=2)),
    case("lean_bf16_pp_n_blocks", "64 lean bf16 pp", 5, out_rows=257, n_pad=192, taps=3, k=64),
    case("lean_bf16_pp_res_ragged_samples", "64 lean bf16 pp res", 2, geo="dilated", samples=3,
         a_rows=129, out_rows=127, taps=3, step=1, n_pad=64, res=R(rps=129, off=1)),
    # ---- lean fp16
    case("lean_fp16_both_ends_saturates", "128 lean fp16 coop", 5, fmt="fp16", geo="dilated",
         samples=2, a_rows=120, out_rows=129, taps=3, step=-50, n_pad=128, amp=1e5),
    case("lean_fp16_res_strided_view", "128 lean fp16 coop res", 2, fmt="fp16", out_rows=128,
         n_pad=128, res=R(step=3, off=1)),
    case("lean_fp16_pp_deep_k", "128 lean fp16 pp", 5, fmt="fp16", geo="dilated", samples=11,
         a_rows=110, out_rows=100, taps=3, step=4, k=512, n_pad=128),
    case("lean_fp16_pp_res_two_kblocks", "128 lean fp16 pp res", 4, fmt="fp16", out_rows=5,
         n_pad=896, k=128, res=R(off=3)),
    case("lean_fp16_col_taps", "64 lean fp16 coop", 5, fmt="fp16", out_rows=100, n_pad=320,
         taps=3, k=64),
    case("lean_fp16_res_past_sample", "64 lean fp16 coop res", 4, fmt="fp16", geo="dilated",
         samples=4, a_rows=66, out_rows=64, taps=3, step=1, n_pad=64,
         res=R(rps=66, off=4, check=1)),
    case("lean_fp16_pp_one_kblock", "64 lean fp16 pp", 2, fmt="fp16", geo="regions", taps=1,
         out_rows=127, n_pad=192, k=64),
    case("lean_fp16_pp_res_step3", "64 lean fp16 pp res", 3, fmt="fp16", geo="dilated",
         samples=7, a_rows=32, out_rows=30, taps=3, step=1, n_pad=64, res=R(rps=90, step=3, off=2)),
    # ---- int8 chain (u8 x s8) and the fp16 expand with its u8 copy, 128 wide
    case("i8_u8_alone_coop", "128 lean int8 coop u8alone", 4, fmt="int8", geo="regions",
         taps=3, out_rows=300, n_pad=128, k=128, out=None, u8="alone"),
    case("i8_res_coop", "128 lean int8 coop res", 2, fmt="int8", geo="dilated", samples=2,
         a_rows=128, out_rows=128, taps=1, n_pad=128, k=256, res=R(rps=130, off=1)),
    case("i8_res_u8_coop", "128 lean int8 coop res u8beside", 5, fmt="int8", out_rows=129,
         n_pad=256, k=128, res=R(off=1), u8="beside"),
    case("fp16_u8_coop", "128 lean fp16 coop u8beside", 3, fmt="fp16", geo="dilated", samples=2,
         a_rows=120, out_rows=118, taps=3, step=1, n_pad=128, u8="beside"),
    case("i8_u8_alone_pp", "128 lean int8 pp u8alone", 2, fmt="int8", geo="dilated", samples=3,
         a_rows=150, out_rows=140, taps=3, step=5, n_pad=128, k=128, out=None, u8="alone"),
    case("i8_res_pp_n_blocks", "128 lean int8 pp res", 3, fmt="int8", out_rows=200,
         n_pad=256, k=128, res=R(off=2)),
    case("i8_res_u8_pp", "128 lean int8 pp res u8beside", 4, fmt="int8", geo="dilated",
         samples=9, a_rows=40, out_rows=40, taps=1, n_pad=128, k=384, res=R(rps=42, off=1),
         u8="beside"),
    case("fp16_u8_pp", "128 lean fp16 pp u8beside", 2, fmt="fp16", out_rows=129 + 128,
         n_pad=128, k=128, u8="beside"),
    # ---- the same at 64 wide
    case("i8_u8_alone_coop_64", "64 lean int8 coop u8alone", 3, fmt="int8", geo="dilated",
         samples=1, a_rows=70, out_rows=64, taps=3, step=3, n_pad=192, k=128, out=None,
         u8="alone"),
    case("i8_res_coop_64", "64 lean int8 coop res", 5, fmt="int8", out_rows=1, n_pad=64, k=128,
         res=R(step=2, off=1)),
    case("i8_res_u8_coop_64", "64 lean int8 coop res u8beside", 5, fmt="int8", out_rows=129,
         n_pad=128, k=128, res=R(off=3), u8="beside"),
    case("fp16_u8_coop_64", "64 lean fp16 coop u8beside", 5, fmt="fp16", out_rows=64,
         n_pad=320, k=64, u8="beside"),
    case("i8_u8_alone_pp_64", "64 lean int8 pp u8alone", 4, fmt="int8", geo="regions", taps=3,
         out_rows=3 * 128, n_pad=192, k=128, out=None, u8="alone"),
    case("i8_res_pp_64", "64 lean int8 pp res", 2, fmt="int8", geo="dilated", samples=5,
         a_rows=50, out_rows=50, taps=3, step=2, n_pad=64, k=128, res=R(rps=52, off=1)),
    case("i8_res_u8_pp_64", "64 lean int8 pp res u8beside", 3, fmt="int8", out_rows=2 * 128,
         n_pad=192, k=256, res=R(off=1), u8="beside"),
    case("fp16_u8_pp_64", "64 lean fp16 pp u8beside", 5, fmt="fp16", geo="dilated", samples=11,
         a_rows=20, out_rows=20, taps=3, step=-1, n_pad=64, u8="beside"),
    # ---- more row / grid / pipeline edges on instances covered above
    case("lean_bf16_r64_pp_2l_minus_1", "64 lean bf16 pp", 2, out_rows=64, n_pad=192),
    case("lean_bf16_r129_pp_2l_plus_1", "128 lean bf16 pp", 2, out_rows=5 * 128 - 100,
         n_pad=128),
    case("lean_fp16_r128_coop_halfwave", "128 lean fp16 coop", 4, fmt="fp16", out_rows=128,
         n_pad=256),
    case("lean_fp16_pp_many_tiles_per_cta", "128 lean fp16 pp res", 3, fmt="fp16",
         out_rows=20 * 128 + 1, n_pad=256, k=64, res=R(off=1)),
    case("lean_bf16_dilated_pp_n_blocks", "64 lean bf16 pp res", 4, geo="dilated", samples=2,
         a_rows=200, out_rows=190, taps=3, step=5, n_pad=320, k=128, res=R(rps=200, off=5)),
    case("i8_pp_deep_k_wraps", "128 lean int8 pp res u8beside", 2, fmt="int8", geo="dilated",
         samples=3, a_rows=110, out_rows=100, taps=3, step=5, n_pad=128, k=512,
         res=R(rps=110, off=5), u8="beside"),
]


@pytest.fixture
def sm_limit():
    """Caps the GEMM grids at n SMs; always restores the default."""
    lib = _capi.load()

    def set_limit(n):
        _capi.check(lib.vp3d_set_sm_limit(n), "vp3d_set_sm_limit")
    try:
        yield set_limit
    finally:
        _capi.check(lib.vp3d_set_sm_limit(0), "vp3d_set_sm_limit")


# ------------------------------------------------------------------------------ operands
def _geometry(c):
    """(a_rows, a_ld, tap_row_step, tap_col_step, per_sample) of a case."""
    taps, k, out_rows = c["taps"], c["k"], c["out_rows"]
    if c["geo"] == "dilated":
        return c["a_rows"], k, c["step"], 0, True
    if c["geo"] == "regions":
        return taps * out_rows, k, out_rows, 0, False
    return out_rows, taps * k, 0, (k if taps > 1 else 0), False


def _total_rows(c):
    return c["samples"] * c["out_rows"] if c["geo"] == "dilated" else c["out_rows"]


def _res_rows(c, r):
    """Rows of the residual source: every row the map reads, and the view its TMA map spans."""
    if c["geo"] == "dilated":
        return c["samples"] * r["rps"]
    if r["div"]:
        return (c["out_rows"] // r["div"] + 1) * r["rps"]
    return c["out_rows"] * r["step"] + abs(r["off"]) + 1


class Operands:
    def __init__(self, c, dev):
        gen = torch.Generator().manual_seed(sum(map(ord, c["name"])))
        a_rows, a_ld, _, _, _ = _geometry(c)
        rows = c["samples"] * a_rows
        n_pad, K = c["n_pad"], c["taps"] * c["k"]
        self.c = c
        if c["fmt"] == "int8":
            self.a = torch.randint(0, 256, (1, rows, a_ld), generator=gen, dtype=torch.uint8)
            self.w = torch.randint(-127, 128, (c["taps"], n_pad, c["k"]), generator=gen,
                                   dtype=torch.int8)
            self.scale = torch.rand(n_pad, generator=gen) * 2e-5 * (1024 / K) ** 0.5
        else:
            dt = torch.float16 if c["fmt"] == "fp16" else torch.bfloat16
            a32 = torch.rand(rows, a_ld, generator=gen) * 2 - 1
            w32 = (torch.rand(c["taps"], n_pad, c["k"], generator=gen) * 2 - 1) / K ** 0.5
            if c["fmt"] == "bf16x3":
                self.a = torch.stack([a32.bfloat16(), (a32 - a32.bfloat16().float()).bfloat16()])
                self.w = torch.stack([w32.bfloat16(), (w32 - w32.bfloat16().float()).bfloat16()])
            else:
                self.a, self.w = a32.to(dt).unsqueeze(0), w32.to(dt).unsqueeze(0)
            self.scale = (torch.rand(n_pad, generator=gen) + 0.5) * c["amp"]
        self.shift = torch.randn(n_pad, generator=gen) * 0.3
        self.res = None
        r = c["res"]
        if r is not None:
            ld = n_pad - r["col_begin"] if r["cols"] else n_pad
            dt = torch.float16 if c["fmt"] in ("fp16", "int8") else torch.bfloat16
            v = torch.rand(r["planes"], _res_rows(c, r), ld, generator=gen) * 4 - 2
            if r["planes"] == 2:   # a split-bf16 residual: hi and its lo
                v[1] = v[0] - v[0].bfloat16().float()
            self.res = v.to(dt)
        dev_all = ("a", "w", "scale", "shift", "res")
        for n in dev_all:
            t = getattr(self, n)
            if t is not None:
                setattr(self, n, t.to(dev).contiguous())
        self.scale, self.shift = self.scale.float(), self.shift.float()


class Outputs:
    """The case's outputs as views into guarded buffers, and the mask of what a launch may write."""

    def __init__(self, c, dev):
        self.c = c
        total, n_pad = _total_rows(c), c["n_pad"]
        rows = GUARD_TOP + total + GUARD_BOTTOM
        body = slice(GUARD_TOP, GUARD_TOP + total)
        self.bufs, self.masks = {}, {}
        if c["out"] == "16":
            dt = torch.float16 if c["fmt"] in ("fp16", "int8") else torch.bfloat16
            buf = torch.full((c["out_planes"], rows, n_pad + 64), float("nan"), dtype=dt,
                             device=dev)
            m = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
            m[0, body, :n_pad] = True
            if c["out_planes"] == 2:
                m[1, body, :n_pad] = self.lo_rows()[:, None].to(dev)
            self.bufs["out"], self.masks["out"] = buf, m
        elif c["out"] == "f32":
            buf = torch.full((rows, n_pad + 8), float("nan"), dtype=torch.float32, device=dev)
            m = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
            m[body, :c["n_valid"]] = True
            self.bufs["out_f32"], self.masks["out_f32"] = buf, m
        if c["u8"]:
            buf = torch.full((rows, n_pad + 64), U8_FILL, dtype=torch.uint8, device=dev)
            m = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
            m[body, :n_pad] = True
            self.bufs["out_u8"], self.masks["out_u8"] = buf, m
        if c["stats"]:
            slabs = 4 * self.m_tiles()
            buf = torch.full((8 + slabs + 8, 2, n_pad), float("nan"), dtype=torch.float32,
                             device=dev)
            m = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
            m[8:8 + slabs] = True
            self.bufs["stats"], self.masks["stats"] = buf, m
        self.fresh = {n: b.clone() for n, b in self.bufs.items()}

    def m_tiles(self):
        c = self.c
        t = -(-c["out_rows"] // BLOCK_M)
        return c["samples"] * t if c["geo"] == "dilated" else t

    def lo_rows(self):
        """Rows whose lo plane the launch writes: all (per-sample tiles), else the rows of the
        tiles that meet [lo_row_begin, lo_row_end)."""
        c = self.c
        rows = torch.arange(_total_rows(c))
        if c["geo"] == "dilated" or c["lo"] is None:
            return torch.ones_like(rows, dtype=torch.bool)
        row0 = rows // BLOCK_M * BLOCK_M
        return (row0 < c["lo"][1]) & (row0 + BLOCK_M > c["lo"][0])

    def reset(self):
        for n, b in self.bufs.items():
            b.copy_(self.fresh[n])

    def view(self, n):
        """The region of buffer n a launch addresses (rows from the first output row on)."""
        b = self.bufs[n]
        total = _total_rows(self.c)
        if n == "out":
            return b[:, GUARD_TOP:GUARD_TOP + total, :self.c["n_pad"]]
        if n == "stats":
            return b[8:8 + 4 * self.m_tiles()]
        return b[GUARD_TOP:GUARD_TOP + total]

    def bits(self):
        return {n: b.view(torch.uint8).clone() for n, b in self.bufs.items()}


def _desc(c, ops, outs):
    a_rows, a_ld, rstep, cstep, per_sample = _geometry(c)
    d = _capi.ConvDesc()
    d.a = ops.a.data_ptr(); d.a_planes = ops.a.shape[0]
    d.samples = c["samples"] if per_sample else 1
    d.a_rows = a_rows; d.a_ld = a_ld
    d.w = ops.w.data_ptr(); d.taps = c["taps"]; d.k_per_tap = c["k"]; d.n_pad = c["n_pad"]
    d.per_sample_tiles = int(per_sample); d.tap_row_step = rstep; d.tap_col_step = cstep
    d.out_rows = c["out_rows"]; d.precision = PRECISION[c["fmt"]]
    if c["affine"]:
        d.scale = ops.scale.data_ptr(); d.shift = ops.shift.data_ptr()
    d.relu = int(c["relu"])
    r = c["res"]
    if r is not None:
        d.res = ops.res.data_ptr(); d.res_planes = r["planes"]
        d.res_plane_stride = ops.res[0].numel(); d.res_ld = ops.res.shape[-1]
        d.res_rows_per_sample = r["rps"]; d.res_row_step = r["step"]; d.res_row_off = r["off"]
        d.res_sample_div = r["div"]; d.res_check_rows = r["check"]
        d.res_col_begin = r["col_begin"]; d.res_cols = r["cols"]
    if "out" in outs.bufs:
        b = outs.bufs["out"]
        d.out = outs.view("out").data_ptr(); d.out_planes = b.shape[0]
        d.out_plane_stride = b[0].numel(); d.out_ld = b.shape[-1]
    if "out_f32" in outs.bufs:
        d.out_f32 = outs.view("out_f32").data_ptr()
        d.out_f32_ld = outs.bufs["out_f32"].shape[-1]; d.n_valid = c["n_valid"]
    if "out_u8" in outs.bufs:
        d.out_u8 = outs.view("out_u8").data_ptr(); d.out_u8_ld = outs.bufs["out_u8"].shape[-1]
        d.out_u8_inv_scale = outs.inv_s
    if "stats" in outs.bufs:
        d.stats = outs.view("stats").data_ptr()
    if c["lo"] is not None:
        d.lo_row_begin, d.lo_row_end = c["lo"]
    return d


def query_key(d):
    k = (ctypes.c_int * 7)()
    _capi.check(_capi.load().vp3d_conv_gemm_instance(ctypes.byref(d), k), "vp3d_conv_gemm_instance")
    return tuple(k)


def launch(d):
    _capi.check(_capi.load().vp3d_conv_gemm(ctypes.byref(d), torch.cuda.current_stream().cuda_stream),
                "vp3d_conv_gemm")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------ references
def reference(c, ops):
    """(v, err): the epilogue's value before the output rounding, float64 [total_rows, n_pad],
    and its bound without that rounding (zero for int8, restated exactly)."""
    a_rows, _, rstep, cstep, per_sample = _geometry(c)
    geo = dict(samples=c["samples"] if per_sample else 1, a_rows=a_rows, taps=c["taps"],
               k_per_tap=c["k"], per_sample_tiles=per_sample, tap_row_step=rstep,
               tap_col_step=cstep, out_rows=c["out_rows"])
    r = c["res"]
    if c["fmt"] == "int8":
        desc = er.new_desc(a_planes=1, samples=geo["samples"], a_rows=a_rows,
                           a_ld=ops.a.shape[-1], taps=c["taps"], k_per_tap=c["k"],
                           n_pad=c["n_pad"], per_sample_tiles=int(per_sample),
                           tap_row_step=rstep, out_rows=c["out_rows"], precision=er.K_INT8,
                           relu=1, res_planes=1 if r else 0,
                           res_rows_per_sample=r["rps"] if r else 0,
                           res_row_step=r["step"] if r else 1, res_row_off=r["off"] if r else 0)
        lc = er.Launch(c["name"], desc, ops.a, ops.w, ops.scale, ops.shift, res=ops.res)
        v = er.int8_epilogue(lc, geo)
        return v, torch.zeros_like(v)
    a, w = ops.a.double(), ops.w.double()
    if c["fmt"] == "bf16x3":   # hi*hi + lo*hi + hi*lo
        acc = expected_conv(a[0], w[0] + w[1], **geo) + expected_conv(a[1], w[0], **geo)
        mag = expected_conv((a[0] + a[1]).abs(), (w[0] + w[1]).abs(), **geo)
        pairs = 3
    else:
        acc = expected_conv(a[0], w[0], **geo)
        mag = expected_conv(a[0].abs(), w[0].abs(), **geo)
        pairs = 1
    scale = ops.scale.double() if c["affine"] else torch.ones_like(ops.scale, dtype=torch.float64)
    shift = ops.shift.double() if c["affine"] else torch.zeros_like(ops.shift, dtype=torch.float64)
    v = acc * scale + shift
    if c["relu"]:
        v = v.clamp_min(0.0)
    res_abs = 0.0
    if r is not None:
        rm = dict(samples=geo["samples"], out_rows=c["out_rows"], per_sample_tiles=per_sample,
                  res_rows_per_sample=r["rps"], res_row_step=r["step"], res_row_off=r["off"],
                  res_sample_div=r["div"], res_check_rows=r["check"],
                  res_col_begin=r["col_begin"], res_cols=r["cols"])
        v = v + expected_residual(ops.res.double(), c["n_pad"], **rm)
        res_abs = expected_residual(ops.res.double().abs(), c["n_pad"], **rm)
    steps = pairs * c["taps"] * c["k"] // 16
    err = (mag * 2.0 ** -20 + acc.abs() * (steps * 2.0 ** -23)) * scale.abs()
    err = err + 2.0 ** -23 * ((acc * scale).abs() + shift.abs() + res_abs)
    return v, err


def _check_values(c, outs, v, err, tag):
    n_pad = c["n_pad"]
    if c["fmt"] == "int8":
        v32 = v.float()
        if "out" in outs.bufs:
            got = outs.view("out")[0]
            exp = v32.clamp(-er.FP16_MAX, er.FP16_MAX).half()
            bad = int((got.view(torch.int16) != exp.view(torch.int16)).sum())
            assert bad == 0, f"{tag}: {bad} fp16 outputs differ from the exact int8 epilogue"
        if "out_u8" in outs.bufs:
            got = outs.view("out_u8")[:, :n_pad]
            exp = er.quant_u8(v32, np.float32(outs.inv_s))
            bad = int((got != exp).sum())
            assert bad == 0, f"{tag}: {bad} u8 outputs differ from the exact int8 epilogue"
        return
    if "out" in outs.bufs:
        got = outs.view("out")
        if c["fmt"] == "fp16":
            exp = v.clamp(-er.FP16_MAX, er.FP16_MAX)
            bound = 2.0 ** -11 * exp.abs() + err + 2.0 ** -24
            diff = (got[0].double() - exp).abs()
            assert torch.isfinite(got[0]).all(), f"{tag}: fp16 output not finite (no saturation)"
            if c["amp"] > 1:   # the case is meant to saturate
                assert bool((got[0] == er.FP16_MAX).any()), f"{tag}: nothing saturated"
        else:
            exp = v
            bound = 2.0 ** -8 * exp.abs() + err
            diff = (got[0].double() - exp).abs()
        bad = ~(diff <= bound)
        assert not bad.any(), \
            f"{tag}: {int(bad.sum())} 16-bit outputs out of bound, first at (row, col) " \
            f"{tuple(torch.nonzero(bad)[0].tolist())}, max excess {float((diff - bound).max()):.3e}"
        if c["out_planes"] == 2:
            lo = outs.lo_rows().to(v.device)
            two = (got[0].double() + got[1].double())[lo]
            diff = (two - v[lo]).abs()
            bad = ~(diff <= 2.0 ** -16 * v[lo].abs() + err[lo])
            assert not bad.any(), f"{tag}: {int(bad.sum())} hi + lo outputs out of bound"
    if "out_f32" in outs.bufs:
        nv = c["n_valid"]
        got = outs.view("out_f32")[:, :nv].double()
        diff = (got - v[:, :nv]).abs()
        bad = ~(diff <= 2.0 ** -23 * v[:, :nv].abs() + err[:, :nv])
        assert not bad.any(), f"{tag}: {int(bad.sum())} fp32 outputs out of bound"
    if "out_u8" in outs.bufs:   # (fp16 launch: its fp32 sum order is not restated)
        got = outs.view("out_u8")[:, :n_pad].double()
        qe = (v.float() * np.float32(outs.inv_s)).round().clamp(0, 255).double()
        assert float((got - qe).abs().max()) <= 1, f"{tag}: u8 copy off by more than one code"
    if c["stats"]:
        _check_stats(c, outs, v, err, tag)


def _check_stats(c, outs, v, err, tag):
    """Per 32-row slab of every row tile: sum and sum of squares of the stored fp32 values."""
    n_pad, out_rows = c["n_pad"], c["out_rows"]
    tiles_per_sample = -(-out_rows // BLOCK_M)
    samples = c["samples"] if c["geo"] == "dilated" else 1
    pad = torch.zeros(samples, tiles_per_sample * BLOCK_M, n_pad, dtype=torch.float64,
                      device=v.device)

    def slabs(x):
        p = pad.clone()
        p[:, :out_rows] = x.reshape(samples, out_rows, n_pad)
        return p.reshape(-1, 32, n_pad).sum(1)
    got = outs.view("stats")
    assert not torch.isnan(got).any(), f"{tag}: stats slabs left unwritten"
    # (the slab sums: 32 fp32 additions, and one product per square)
    s_bound = slabs(err) + 2.0 ** -18 * slabs(v.abs())
    q_bound = slabs(2 * v.abs() * err + err * err) + 2.0 ** -18 * slabs(v * v)
    for i, (exp, bound, what) in enumerate(((slabs(v), s_bound, "sum"),
                                            (slabs(v * v), q_bound, "sum of squares"))):
        bad = ~((got[:, i].double() - exp).abs() <= bound)
        assert not bad.any(), f"{tag}: {int(bad.sum())} slab {what} partials out of bound"


def _check_guards(outs, tag):
    for n, b in outs.bufs.items():
        m = outs.masks[n]
        same = b.view(torch.uint8) == outs.fresh[n].view(torch.uint8)
        el = b.element_size()
        same = same.reshape(*b.shape[:-1], b.shape[-1], el).all(-1)
        bad = ~same & ~m
        if bad.any():
            first = tuple(torch.nonzero(bad)[0].tolist())
            raise AssertionError(f"{tag}: {int(bad.sum())} stores outside the region of "
                                 f"{n}, first at buffer index {first}")


# ------------------------------------------------------------------------------ tests
@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_instance_case(cuda_device, sm_limit, c):
    dev = cuda_device
    ops = Operands(c, dev)
    v, err = reference(c, ops)
    outs = Outputs(c, dev)
    outs.inv_s = 1.0
    if c["u8"]:
        outs.inv_s = float(np.float32(255.0) / np.float32(float(v.max()) * 0.9))
    d = _desc(c, ops, outs)
    sm_limit(c["sm"])
    tag = f"{c['name']} [{key_text(c['key'])}]"
    got_key = query_key(d)
    assert got_key == c["key"], f"{tag}: selects [{key_text(got_key)}]"
    launch(d)
    _check_guards(outs, tag)
    _check_values(c, outs, v, err, tag)
    first = outs.bits()
    outs.reset()
    launch(d)
    again = outs.bits()
    for n in first:
        assert torch.equal(first[n], again[n]), f"{tag}: {n} differs on a second launch"


def test_cases_cover_every_compiled_instance():
    """Every instance the library compiles has a case above (and no case names one it lacks)."""
    lib = _capi.load()
    n = lib.vp3d_conv_gemm_instances(None, 0)
    keys = (ctypes.c_int * (7 * n))()
    assert lib.vp3d_conv_gemm_instances(keys, n) == n
    compiled = {tuple(keys[7 * i:7 * i + 7]) for i in range(n)}
    assert len(compiled) == n == 48
    covered = {c["key"] for c in CASES}
    missing = sorted(key_text(k) for k in compiled - covered)
    unknown = sorted(key_text(k) for k in covered - compiled)
    assert not missing and not unknown, f"no case for {missing}; not compiled: {unknown}"


# (id, case) -- fixed descriptors run under every SM limit that changes (block_n, schedule)
INVARIANT = [
    case("inv_lean_fp16_res", "128 lean fp16 pp res", 0, fmt="fp16", out_rows=3 * 128 + 9,
         n_pad=256, k=128, res=R(off=1)),
    case("inv_lean_bf16_dilated", "128 lean bf16 pp", 0, geo="dilated", samples=3, a_rows=110,
         out_rows=100, taps=3, step=4, n_pad=128),
    case("inv_int8_res_u8", "128 lean int8 pp res u8beside", 0, fmt="int8", out_rows=2 * 128 + 1,
         n_pad=256, k=128, res=R(off=2), u8="beside"),
    case("inv_fp16_u8_expand", "128 lean fp16 pp u8beside", 0, fmt="fp16", geo="dilated",
         samples=3, a_rows=120, out_rows=118, taps=3, step=1, n_pad=128, u8="beside"),
    case("inv_general_f32", "128 general runtime coop", 0, fmt="fp16", out_rows=300,
         n_pad=256, out="f32", n_valid=200, relu=False),
    case("inv_lean_fp16_n192", "64 lean fp16 pp", 0, fmt="fp16", out_rows=2 * 128 + 3,
         n_pad=192, taps=3, k=64),
]
SM_LIMITS = (2, 3, 4, 5, 6, 8, 9, 12, 16, 17, 24, 33, 64, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("c", INVARIANT, ids=[c["name"] for c in INVARIANT])
def test_schedule_invariance(cuda_device, sm_limit, c):
    """For a fixed descriptor, every (block_n, schedule) the selection reaches stores the same
    bits."""
    dev = cuda_device
    ops = Operands(c, dev)
    outs = Outputs(c, dev)
    outs.inv_s = 1.0
    if c["u8"]:
        v, _ = reference(c, ops)
        outs.inv_s = float(np.float32(255.0) / np.float32(float(v.max()) * 0.9))
    d = _desc(c, ops, outs)
    runs = {}
    for lim in SM_LIMITS:
        sm_limit(lim)
        k = query_key(d)
        if k in runs:
            continue
        outs.reset()
        launch(d)
        runs[k] = (lim, outs.bits())
    keys = list(runs)
    lean_128 = c["n_pad"] % 128 == 0 and key_text(keys[0]).split()[1] == "lean"
    assert len(keys) >= (3 if lean_128 else 2), \
        f"{c['name']}: only reached {[key_text(k) for k in keys]}"
    k0 = keys[0]
    for k in keys[1:]:
        for n, b in runs[k][1].items():
            assert torch.equal(b, runs[k0][1][n]), \
                f"{c['name']}: {n} differs between [{key_text(k0)}] (SM limit {runs[k0][0]}) " \
                f"and [{key_text(k)}] (SM limit {runs[k][0]})"
