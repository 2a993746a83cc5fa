"""Python restatement of the eval-mode launch schedule of ``vp3d_forward_eval`` (api.cu).

``replay(sd, cfg, x, precision, gemm)`` rebuilds, in torch, the operations the eval forward
runs -- input pack, expand, the two convs of every residual block, shrink -- with the same conv
GEMM descriptors (the fields of ``vp3d_conv_desc``) and operand bits, and hands every GEMM to
``gemm``:

* ``gpu_gemm``  launches the kernel through ``vp3d_conv_gemm`` (the op-level C entry).  Every GEMM
  then computes exactly what the model's own launch of the same descriptor computes, so the
  replay's output equals ``model(x)`` bit for bit, and every layer's stored output can be checked
  against a float64 evaluation of the same GEMM on that layer's own kernel-produced inputs.
* ``fake_gemm``  a float64 restatement of the same descriptor on the tensors' device: the products
  of the stored planes the kernel forms, affine, ReLU, residual, then the store in the output's
  format (fp16 with saturation, bf16 hi [+ lo on the tiles of the lo range]).  With ``exact=True``
  the replay keeps float64 operands and activations, so the result is the model's algorithm in
  float64 in the plan's row order -- the replay can be checked without a GPU.

Both schedules: the strided one (tap-major row order, ``use_strided``) and the dilated one
(per-sample tiles).  Per-layer precision as ``vp3d_forward_eval`` picks it, including the FLOP rule
of ``mixed``.  Buffers that the kernel writes are prefilled with NaN, so a lo plane outside its lo
range (or any row nobody wrote) poisons whatever reads it.

``"int8"`` (``replay(..., "int8", gemm, amax=...)``) restates ``run_infer_chain`` for an int8 plan:
the expand in fp16, also writing the u8 codes Q_0; per block a u8 x s8 conv Q_{i-1} -> H (u8
alone) and a u8 x s8 1x1 conv H -> X_i (fp16, residual X_{i-1}) [+ Q_i]; the shrink in fp16.  Its
int8 GEMMs have exact int32 sums and a fixed fp32 epilogue, so ``fake_conv`` restates them bit for
bit.  It is not in PRECISIONS: its output is not the float64 forward's (int8_oracle restates it).
"""
from fractions import Fraction

import numpy as np
import torch
import torch.nn.functional as F

import int8_oracle as io
from gpu_utils import conv_gemm, expected_conv

PRECISIONS = ("fp16", "bf16", "mixed", "bf16x3")
INT8 = "int8"
K_BF16, K_BF16X3, K_FP16, K_INT8 = 0, 1, 3, 4   # VP3D_PRECISION_* of a conv descriptor
BLOCK_K8 = 128                           # K per k-block of the int8 GEMM (k_per_tap padded to it)
FP16_MAX = 65504.0
BLOCK_M = 128                            # rows per output tile of the conv GEMM
EPS = 1e-5                               # nn.BatchNorm1d default (model.py:32)

DESC_FIELDS = ("a_planes", "samples", "a_rows", "a_ld", "a_plane_stride", "taps", "k_per_tap",
               "n_pad", "per_sample_tiles", "tap_row_step", "tap_col_step", "out_rows",
               "precision", "relu", "res_planes", "res_rows_per_sample", "res_row_step",
               "res_row_off", "res_sample_div", "out_planes", "out_plane_stride", "out_ld",
               "out_f32_ld", "n_valid", "lo_row_begin", "lo_row_end")


def round_up(v, m):
    return (v + m - 1) // m * m


class Plan:
    """What ``vp3d_plan_create`` and the head of ``vp3d_forward_eval`` derive from a configuration
    and an input shape.  cfg: dict(cls="TemporalModel" | "TemporalModelOptimized1f", J, F, Jout,
    fw, C, causal=False, dense=False) -- the keys of the golden fixtures' meta."""

    def __init__(self, cfg, precision, N, T):
        if precision not in PRECISIONS + (INT8,):
            raise ValueError(f"unknown precision {precision!r}")
        fw = [int(w) for w in cfg["fw"]]
        causal, dense = bool(cfg.get("causal", False)), bool(cfg.get("dense", False))
        self.fw, self.nb, self.N, self.T = fw, len(fw) - 1, N, T
        self.precision = precision
        self.c_real = cfg["C"]
        self.C = round_up(cfg["C"], 64)
        self.c_in_raw = cfg["J"] * cfg["F"]
        self.c_out_raw = cfg["Jout"] * 3
        self.c_in_pad = round_up(self.c_in_raw, 64)
        self.k0_pad = round_up(self.c_in_raw * fw[0], 64)
        self.c_out_pad = round_up(self.c_out_raw, 64)
        self.int8 = precision == INT8
        self.f16 = precision in ("fp16", INT8)     # (int8: fp16 expand, residual stream, shrink)
        self.planes = 2 if precision in ("mixed", "bf16x3") else 1
        self.k_conv = round_up(self.C, BLOCK_K8) if self.int8 else self.C   # K per tap, block convs
        # api.cu plan_create: pad / causal shifts / dilation / taps per stage
        self.pad, self.shift_dil, self.shift_str = [fw[0] // 2], [0], [0]
        self.shift_dil[0] = self.shift_str[0] = fw[0] // 2 if causal else 0
        self.dilation, self.taps = [1], [fw[0]]
        nd = fw[0]
        for w in fw[1:]:
            p = (w - 1) * nd // 2
            self.pad.append(p)
            self.shift_dil.append((w // 2) * nd if causal else 0)
            self.shift_str.append(w // 2 if causal else 0)
            self.dilation.append(1 if dense else nd)
            self.taps.append(2 * p + 1 if dense else w)
            nd *= w
        self.receptive_field = 1 + 2 * sum(self.pad)
        strided_variant = cfg["cls"] != "TemporalModel"
        if strided_variant and dense:
            raise ValueError("dense=True only exists for TemporalModel")
        self.strided = strided_variant or (not dense and T == self.receptive_field)
        if self.strided:
            L = [T // fw[0]]
            for i in range(1, self.nb + 1):
                L.append(L[-1] // fw[i])
        else:
            L = [T - (fw[0] - 1)]
            for i in range(1, self.nb + 1):
                L.append(L[-1] - 2 * self.pad[i])
        if min(L) < 1:
            raise ValueError(f"sequence of {T} frames is shorter than the receptive field "
                             f"({self.receptive_field})")
        if self.strided:   # strided_trim: the rows the output depends on
            for i in range(1, self.nb + 1):
                first = self.shift_str[i] + fw[i] // 2
                res_len = (L[i - 1] - first + fw[i] - 1) // fw[i] if L[i - 1] > first else 0
                if res_len != L[i]:
                    raise ValueError(f"residual slice of block {i} has {res_len} rows, the conv {L[i]}")
            for i in range(self.nb, 0, -1):
                L[i - 1] = fw[i] * L[i]
        self.L = L
        self.R = [N * l for l in L]
        self.x3 = mixed_layers(self) if precision == "mixed" else \
            [precision == "bf16x3"] * (self.nb + 2)

    def region_rows(self, level):
        """Buffer row of every (sample, frame) of the activation after stage `level` (0 = expand,
        i = block i): (N, L[level]) int64.  Strided schedule: tap-major order (pack.cuh), where the
        taps of the next block's conv are contiguous regions of R[level + 1] rows; dilated: n*L + t."""
        L, N = self.L, self.N
        t = torch.arange(L[level])
        n = torch.arange(N)
        if not self.strided:
            return n[:, None] * L[level] + t[None, :]
        pos = torch.zeros(L[level], dtype=torch.int64)
        for lv in range(level + 1, self.nb + 1):
            w = self.fw[lv]
            pos += (t % w) * self.R[lv]
            t = t // w
        return pos[None, :] + n[:, None] * L[self.nb] + t[None, :]

    def lo_range(self, i):
        """lo_rows() of api.cu for the GEMM producing X_i: (begin, end), (0, 0) = every row."""
        if not self.strided or self.planes != 2 or i >= self.nb or self.x3[i + 1]:
            return 0, 0
        c = self.fw[i + 1] // 2 + self.shift_str[i + 1]
        return c * self.R[i + 1], (c + 1) * self.R[i + 1]


def mixed_layers(p):
    """Which GEMMs of `mixed` run split-bf16: index 0 = expand, 1..nb = residual blocks, nb + 1 =
    shrink.  Expand and shrink always; a block when it holds < 0.5 % of the forward's FLOPs."""
    N, L, C = p.N, p.L, p.C
    fl = [N * L[0] * p.c_in_raw * p.fw[0] * C]
    fl += [N * L[i] * (p.taps[i] + 1.0) * C * C for i in range(1, p.nb + 1)]
    fl.append(N * L[p.nb] * C * p.c_out_raw)
    total = sum(fl)
    return [i == 0 or i == p.nb + 1 or fl[i] < 0.005 * total for i in range(p.nb + 2)]


# ---------------------------------------------------------------------------- operand formats
def fma_f32(a, b, c):
    """fp32 fmaf(a, b, c) elementwise (one rounding of the exact a*b + c).  The product of two fp32
    values is exact in float64; the float64 sum rounds once more, which can only change the fp32
    result when it lands exactly on a midpoint between two fp32 values -- those are settled
    with exact rationals."""
    a, b, c = (t.detach().cpu().float().flatten() for t in (a, b, c))
    r64 = a.double() * b.double() + c.double()
    r = r64.float()
    # r64 is a midpoint exactly when its mirror image about r64 is another fp32 value
    other = 2.0 * r64 - r.double()
    mid = (r64 != r.double()) & (other.float().double() == other)
    for i in torch.nonzero(mid).flatten().tolist():
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        m = Fraction(float(r64[i]))
        if exact != m:   # (a true tie keeps the round-to-even choice of r)
            pick = max if exact > m else min
            r[i] = pick(float(r[i]), float(other[i]))
    return r


def bn_fold(bn, c_pad, exact):
    """bn_fold_kernel: scale = gamma / sqrtf(var + eps), shift = fmaf(-mean, scale, beta) in
    fp32 (IEEE sqrt and division), zero padded; float64 in exact mode."""
    g, b, m, v = (bn[k].detach().cpu() for k in ("weight", "bias", "running_mean", "running_var"))
    dt = torch.float64 if exact else torch.float32
    scale = torch.zeros(c_pad, dtype=dt)
    shift = torch.zeros(c_pad, dtype=dt)
    c = g.numel()
    if exact:
        scale[:c] = g.double() / torch.sqrt(v.double() + EPS)
        shift[:c] = b.double() - m.double() * scale[:c]
    else:
        # each fp32 operation as float64 then one rounding to fp32: correctly rounded for + / sqrt
        # (53 >= 2 * 24 + 2), as the device's IEEE ops are; torch's own fp32 CPU sqrt is not
        # always correctly rounded
        eps = float(torch.tensor(EPS, dtype=torch.float32))
        var_eps = (v.double() + eps).float()
        scale[:c] = (g.double() / torch.sqrt(var_eps.double()).float().double()).float()
        shift[:c] = fma_f32(-m.float(), scale[:c], b.float())
    return scale, shift


class Storage:
    """The 16-bit operand / activation formats of one precision (or float64 in exact mode)."""

    def __init__(self, p, exact, device):
        self.p, self.exact, self.device = p, exact, device
        self.dtype = torch.float64 if exact else (torch.float16 if p.f16 else torch.bfloat16)

    def planes_of(self, v, planes):
        """fp32 values -> [planes, ...] stored planes: bf16 RNE hi + RNE(v - hi) lo; fp16 clamps
        to +-65504 then rounds; exact: the value and a zero lo plane."""
        if self.exact:
            out = torch.zeros((planes,) + tuple(v.shape), dtype=torch.float64, device=v.device)
            out[0] = v.double()
            return out
        v = v.float()
        if self.p.f16:
            assert planes == 1
            return v.clamp(-FP16_MAX, FP16_MAX).half().unsqueeze(0)
        hi = v.bfloat16()
        if planes == 1:
            return hi.unsqueeze(0)
        return torch.stack([hi, (v - hi.float()).bfloat16()])

    def empty(self, planes, rows, ld):
        return torch.full((planes, rows, ld), float("nan"), dtype=self.dtype, device=self.device)


def pack_weights(sd, p, st):
    """plan weight packs [planes][taps][n_pad][k_pad] (launch_pack_conv_weight), affine vectors."""
    dev = st.device
    src = torch.float64 if st.exact else torch.float32

    def w_of(name):
        return sd[name].detach().to(device=dev, dtype=src)

    def pack(w, n_pad, k_pad, merged):
        co, ci, k = w.shape
        if merged:
            buf = torch.zeros(1, n_pad, k_pad, dtype=src, device=dev)
            buf[0, :co, :k * ci] = w.permute(0, 2, 1).reshape(co, k * ci)
        else:
            buf = torch.zeros(k, n_pad, k_pad, dtype=src, device=dev)
            buf[:, :co, :ci] = w.permute(2, 0, 1)
        return st.planes_of(buf, p.planes).contiguous()

    def bn(prefix, c_pad):
        s, t = bn_fold({k: sd[f"{prefix}.{k}"] for k in
                        ("weight", "bias", "running_mean", "running_var")}, c_pad, st.exact)
        return s.to(dev), t.to(dev)

    ew = w_of("expand_conv.weight")
    pk = {"expand_flat": pack(ew, p.C, p.k0_pad, True),
          "expand_dil": pack(ew, p.C, p.c_in_pad, False),
          "expand_aff": bn("expand_bn", p.C)}
    for j in range(2 * p.nb):
        pk[f"aff{j}"] = bn(f"layers_bn.{j}", p.C)
        if not p.int8:   # (int8: the s8 packs of pack_int8)
            pk[f"conv{j}"] = pack(w_of(f"layers_conv.{j}.weight"), p.C, p.C, False)
    pk["shrink"] = pack(w_of("shrink.weight"), p.c_out_pad, p.C, False)
    dt = torch.float64 if st.exact else torch.float32
    scale = torch.zeros(p.c_out_pad, dtype=dt, device=dev)
    shift = torch.zeros(p.c_out_pad, dtype=dt, device=dev)
    scale[:p.c_out_raw] = 1.0
    shift[:p.c_out_raw] = sd["shrink.bias"].detach().to(device=dev, dtype=dt)
    pk["shrink_aff"] = (scale, shift)
    return pk


def pack_int8(sd, p, amax, pk, device):
    """The int8 plan's block-conv operands, into pk: per layer j the s8 pack [taps][C][k_conv]
    (int8_oracle.quant_weight, zero past c_real and in the K padding) and the folded affine
    scale' = fp32(bn_s * fp32(s_w * s_in)) (int8_oracle.int8_affine) with the kernel's fp32 fmaf
    BatchNorm shift (bn_fold, not int8_oracle's float64 one); pk["inv_s"]: the fp32 reciprocals
    of the activation scales of the 2B calibration maxima amax."""
    s_act, inv = io.act_scales(np.asarray(amax, np.float32))
    cr = p.c_real
    sdn = {k: v.detach().cpu().numpy() for k, v in sd.items()}
    for j in range(2 * p.nb):
        sc, _, wq = io.int8_affine(sdn, j, s_act[j])
        w8 = torch.zeros(wq.shape[2], p.C, p.k_conv, dtype=torch.int8)
        w8[:, :cr, :cr] = torch.from_numpy(wq.transpose(2, 0, 1).astype(np.int8))
        scale = torch.zeros(p.C, dtype=torch.float32)
        scale[:cr] = torch.from_numpy(sc)
        pk[f"conv{j}"] = w8.to(device)
        pk[f"aff{j}"] = (scale.to(device), pk[f"aff{j}"][1])
    pk["inv_s"] = [float(v) for v in inv]


# ---------------------------------------------------------------------------- launches
class Launch:
    """One conv GEMM: descriptor fields + operand tensors (16-bit planes [planes][rows][ld]; an
    int8 launch: u8 A [1][rows][ld] and s8 W).  out_u8 [1][rows][C]: the u8 codes of the stored
    values times inv_s (an fp32 value), beside `out` or alone."""

    def __init__(self, name, desc, a, w, scale, shift, res=None, out=None, out_f32=None,
                 out_u8=None, inv_s=None):
        self.name, self.desc = name, desc
        self.a, self.w, self.scale, self.shift = a, w, scale, shift
        self.res, self.out, self.out_f32 = res, out, out_f32
        self.out_u8, self.inv_s = out_u8, inv_s

    def _m_tiles(self):
        d = self.desc
        return d["samples"] * -(-d["out_rows"] // BLOCK_M) if d["per_sample_tiles"] \
            else -(-d["out_rows"] // BLOCK_M)

    @property
    def block_n(self):
        """The N tile width run_conv picks for this launch."""
        d = self.desc
        return 128 if d["n_pad"] % 128 == 0 and self._m_tiles() * (d["n_pad"] // 128) * 2 >= \
            num_sms() else 64

    @property
    def tiles(self):
        """Output tiles of the launch (m tiles x n_pad / block_n)."""
        return self._m_tiles() * (self.desc["n_pad"] // self.block_n)

    @property
    def pingpong(self):
        """Whether select_instance gives an int8 / u8-output launch (always a lean instance) the
        ping-pong schedule: when some CTA gets a second tile."""
        assert self.desc["precision"] == K_INT8 or self.out_u8 is not None, self.name
        return self.tiles > num_sms()

    def total_rows(self):
        d = self.desc
        return d["samples"] * d["out_rows"] if d["per_sample_tiles"] else d["out_rows"]

    def lo_mask(self):
        """Output rows whose lo plane the kernel writes: every row of a per-sample-tile launch,
        else the rows of the 128-row tiles that intersect [lo_row_begin, lo_row_end)."""
        d = self.desc
        rows = torch.arange(self.total_rows())
        if d["per_sample_tiles"] or d["lo_row_end"] <= 0:
            return torch.ones_like(rows, dtype=torch.bool)
        row0 = rows // BLOCK_M * BLOCK_M
        return (row0 < d["lo_row_end"]) & (row0 + BLOCK_M > d["lo_row_begin"])

    def residual_rows(self):
        d = self.desc
        t = torch.arange(d["out_rows"])
        if d["per_sample_tiles"]:
            s = torch.arange(d["samples"])
            return (s[:, None] * d["res_rows_per_sample"] + t[None, :] * d["res_row_step"]
                    + d["res_row_off"]).flatten()
        assert d["res_sample_div"] == 0
        return t * d["res_row_step"] + d["res_row_off"]


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count \
        if torch.cuda.is_available() else 132


def new_desc(**kw):
    d = dict.fromkeys(DESC_FIELDS, 0)
    for k, v in kw.items():
        assert k in d, k
        d[k] = int(v)
    return d


def fake_conv(lc, with_err=False):
    """float64 restatement of one launch on the operands' device.  Returns (exp, err): the
    epilogue's value before its output rounding, [total_rows, n_pad], and (with_err) the bound of
    the fp32 accumulation, times |scale| (None otherwise):
        2^-20 * sum|a||w|  +  steps * 2^-23 * |acc|
    The first term is the order-of-summation error; the second is the tensor cores' own: each of
    the `steps` k16 wgmma steps (pairs * taps * k_per_tap / 16) adds into the fp32 accumulator
    truncating, not rounding to nearest -- a bias toward zero of up to one ulp of the partial sum
    per step, which dominates the split-bf16 layers' error.
    An int8 launch is restated exactly (int8_epilogue); its err is zero."""
    d = lc.desc
    geo = dict(samples=d["samples"], a_rows=d["a_rows"], taps=d["taps"], k_per_tap=d["k_per_tap"],
               per_sample_tiles=bool(d["per_sample_tiles"]), tap_row_step=d["tap_row_step"],
               tap_col_step=d["tap_col_step"], out_rows=d["out_rows"])
    if d["precision"] == K_INT8:
        v = int8_epilogue(lc, geo)
        return v, (torch.zeros_like(v) if with_err else None)
    a = lc.a[:d["a_planes"]].double()
    w = lc.w.double()
    if d["precision"] == K_BF16X3:   # hi*hi + lo*hi + hi*lo (pairs 0, 1, 2 of the kernel)
        assert d["a_planes"] == 2 and w.shape[0] == 2
        acc = expected_conv(a[0], w[0] + w[1], **geo) + expected_conv(a[1], w[0], **geo)
        mag = expected_conv((a[0] + a[1]).abs(), (w[0] + w[1]).abs(), **geo) if with_err else None
    else:                            # one MMA on the hi planes (A may carry a lo plane it ignores)
        acc = expected_conv(a[0], w[0], **geo)
        mag = expected_conv(a[0].abs(), w[0].abs(), **geo) if with_err else None
    scale, shift = lc.scale.double(), lc.shift.double()
    v = acc * scale + shift
    if d["relu"]:
        v = v.clamp_min(0.0)
    if lc.res is not None:
        rows = lc.residual_rows().to(v.device)
        for pl in range(d["res_planes"]):
            v = v + lc.res[pl].double()[rows]
    err = None
    if with_err:
        steps = (3 if d["precision"] == K_BF16X3 else 1) * d["taps"] * d["k_per_tap"] // 16
        err = (mag * 2.0 ** -20 + acc.abs() * (steps * 2.0 ** -23)) * scale.abs()
    return v, err


def int8_epilogue(lc, geo):
    """The value an int8 launch stores, before its output rounding: fp32 values (as float64).
    The sums of u8 x s8 products are integers below 2^53, so float64 adds them exactly in any
    order: they are the kernel's int32 sums.  Then the kernel's fp32 chain, operation by operation:
        fmaxf(fmaf(fp32(acc), scale', shift), 0)   [+ residual, an fp32 add of the fp16 value].
    A reads as zero past its row (a_ld) up to the K padding k_per_tap: TMA fills it so."""
    d = lc.desc
    assert lc.a.dtype == torch.uint8 and lc.w.dtype == torch.int8 and d["a_planes"] == 1
    a = lc.a[0].double()
    a = F.pad(a, (0, d["k_per_tap"] - a.shape[-1]))
    acc = expected_conv(a, lc.w.double(), **geo)
    assert float(acc.abs().max()) < 2.0 ** 31, f"{lc.name}: int32 sums overflow"
    n = acc.shape[1]
    v = fma_f32(acc.float(), lc.scale.float().expand(acc.shape[0], n),
                lc.shift.float().expand(acc.shape[0], n)).view(acc.shape).to(acc.device)
    v = v.clamp_min(0.0)
    if lc.res is not None:
        assert d["res_planes"] == 1 and lc.res.dtype == torch.float16
        v = v + lc.res[0].float()[lc.residual_rows().to(v.device)]
    return v.double()


def quant_u8(v32, inv_s):
    """cvt.rni.sat.u8.f32(v * inv_s): the fp32 product, rounded half to even, clamped to [0, 255]."""
    q = (v32 * torch.tensor(inv_s, dtype=torch.float32, device=v32.device)).round()
    return q.clamp(0, 255).to(torch.uint8)


def store(lc, v):
    """Write the epilogue value v (float64) into the launch's output as the kernel stores it."""
    d = lc.desc
    if lc.out_u8 is not None:
        lc.out_u8[0] = quant_u8(v.float(), lc.inv_s)
    if lc.out_f32 is not None:
        lc.out_f32.copy_(v[:, :d["n_valid"]].to(lc.out_f32.dtype))
        return
    out = lc.out
    if out is None:
        return
    out.fill_(float("nan"))
    lo = lc.lo_mask().to(v.device)
    if out.dtype == torch.float64:          # exact mode: the value, a zero lo plane
        out[0] = v
        if out.shape[0] == 2:
            out[1][lo] = 0.0
        return
    v32 = v.float()
    if out.dtype == torch.float16:
        out[0] = v32.clamp(-FP16_MAX, FP16_MAX).half()
        return
    hi = v32.bfloat16()
    out[0] = hi
    if out.shape[0] == 2:
        out[1][lo] = (v32 - hi.float()).bfloat16()[lo]


def fake_gemm(lc):
    """The float64 fake of ``vp3d_conv_gemm``: computes and stores one launch."""
    v, _ = fake_conv(lc)
    store(lc, v)


def gpu_gemm(lc):
    """One launch through ``vp3d_conv_gemm`` with the replay's own buffers."""
    d = lc.desc
    kw = {}
    if lc.res is not None:
        assert lc.res.shape[0] == d["res_planes"]
        kw = dict(res=lc.res, res_rows_per_sample=d["res_rows_per_sample"],
                  res_row_step=d["res_row_step"], res_row_off=d["res_row_off"],
                  res_sample_div=d["res_sample_div"])
    assert lc.a.shape[0] == d["a_planes"]
    if lc.out_u8 is not None:
        kw.update(out_u8=lc.out_u8, out_u8_inv_scale=lc.inv_s)
    conv_gemm(lc.a, d["samples"], d["a_rows"], d["a_ld"], lc.w, d["taps"], d["k_per_tap"],
              d["n_pad"], per_sample_tiles=d["per_sample_tiles"], tap_row_step=d["tap_row_step"],
              tap_col_step=d["tap_col_step"], out_rows=d["out_rows"], precision=d["precision"],
              scale=lc.scale, shift=lc.shift, relu=bool(d["relu"]), out=lc.out,
              out_f32=lc.out_f32, out_f32_cols=d["n_valid"] if lc.out_f32 is not None else None,
              out_plane_stride=d["out_plane_stride"], a_plane_stride=d["a_plane_stride"],
              lo_row_begin=d["lo_row_begin"], lo_row_end=d["lo_row_end"], **kw)


class Replay:
    """Result of ``replay``: y (N, L_out, J_out, 3), the launches in order (``launch_count``
    counts the input pack too, like ``vp3d_last_launch_count``), the plan and the activations
    [(name, level, buffer)] in forward_numpy's collect order: X_0, H_1, X_1, H_2, X_2, ...
    (int8: X_0, Q_0, H_1, X_1, Q_1, ..., H_B, X_B, the Q and H buffers u8 codes)."""

    def __init__(self, plan, y, launches, acts):
        self.plan, self.y, self.launches, self.acts = plan, y, launches, acts
        self.launch_count = 1 + len(launches)

    def activation(self, k):
        """Activation k de-permuted to (N, L, c_real) float64 (hi + lo where lo was written)."""
        _, level, buf = self.acts[k]
        return stored_value(buf)[self.plan.region_rows(level).to(buf.device)][..., :self.plan.c_real]


def stored_value(buf):
    """float64 value of stored planes [planes][rows][ld]: hi + lo where the lo plane was written."""
    v = buf[0].double()
    if buf.shape[0] == 2:
        lo = buf[1].double()
        v = v + torch.where(torch.isnan(lo), torch.zeros_like(lo), lo)
    return v


def replay(sd, cfg, x, precision, gemm, *, exact=False, collect=None, amax=None):
    """Run the eval forward's schedule for input x (N, T, J, F) with `gemm` executing every conv
    GEMM (``gpu_gemm`` or ``fake_gemm``).  exact: float64 operands and activations (use with
    ``fake_gemm``).  collect: a list that receives the de-permuted activations (numpy float64,
    forward_numpy's collect order; int8: int8_oracle.forward_int8's, without the last block's
    absent Q).  amax: the 2B calibration maxima of precision "int8" (``int8_calibration()``)."""
    N, T = int(x.shape[0]), int(x.shape[1])
    p = Plan(cfg, precision, N, T)
    i8 = p.int8
    if i8 and (exact or amax is None):
        raise ValueError("the int8 replay needs amax and runs in the kernels' formats (exact=False)")
    st = Storage(p, exact, x.device)
    pk = pack_weights(sd, p, st)
    if i8:
        pack_int8(sd, p, amax, pk, x.device)
    fw, C, L, R, nb, planes = p.fw, p.C, p.L, p.R, p.nb, p.planes
    xs = x.reshape(N, T, p.c_in_raw).to(torch.float64 if exact else torch.float32)
    launches, acts = [], []

    def prec(layer_x3):
        return K_FP16 if p.f16 else (K_BF16X3 if layer_x3 else K_BF16)

    def run(name, desc, a, w, aff, res=None, out=None, out_f32=None, out_u8=None, inv_s=None):
        lc = Launch(name, desc, a, w, aff[0], aff[1], res=res, out=out, out_f32=out_f32,
                    out_u8=out_u8, inv_s=inv_s)
        gemm(lc)
        launches.append(lc)
        return lc

    def empty_u8(rows):
        # (u8 has no NaN: rows nobody writes keep 0xFF; the GPU test reruns each launch on 0x00)
        return torch.full((1, rows, C), 255, dtype=torch.uint8, device=x.device)

    # ---- input pack + expand
    if p.strided:
        k0 = fw[0] * p.c_in_raw
        vals = torch.zeros(N * L[0], p.k0_pad, dtype=xs.dtype, device=x.device)
        rows = p.region_rows(0).to(x.device).flatten()
        vals[rows, :k0] = xs[:, :L[0] * fw[0]].reshape(N * L[0], k0)
        a0 = st.planes_of(vals, planes)
        desc = new_desc(samples=1, a_rows=N * L[0], a_ld=p.k0_pad, taps=1, k_per_tap=p.k0_pad,
                        per_sample_tiles=0, out_rows=N * L[0])
        w0 = pk["expand_flat"]
    else:
        vals = torch.zeros(N * T, p.c_in_pad, dtype=xs.dtype, device=x.device)
        vals[:, :p.c_in_raw] = xs.reshape(N * T, p.c_in_raw)
        a0 = st.planes_of(vals, planes)
        desc = new_desc(samples=N, a_rows=T, a_ld=p.c_in_pad, taps=fw[0], k_per_tap=p.c_in_pad,
                        per_sample_tiles=1, tap_row_step=1, out_rows=L[0])
        w0 = pk["expand_dil"]
    lo_b, lo_e = p.lo_range(0)
    desc.update(a_planes=planes, precision=prec(p.x3[0]), out_planes=planes, res_planes=planes,
                relu=1, n_pad=C, out_ld=C, out_plane_stride=R[0] * C,
                lo_row_begin=lo_b, lo_row_end=lo_e)
    xcur = st.empty(planes, R[0], C)
    # int8: the fp16 expand also writes Q_0, the u8 input of block 1
    qcur = empty_u8(R[0]) if i8 and nb > 0 else None
    run("expand", desc, a0, w0, pk["expand_aff"], out=xcur, out_u8=qcur,
        inv_s=pk["inv_s"][0] if qcur is not None else None)
    acts.append(("X0", 0, xcur))
    if qcur is not None:
        acts.append(("Q0", 0, qcur))

    # ---- residual blocks
    for i in range(1, nb + 1):
        x3 = p.x3[i]
        Lin, Lout = L[i - 1], L[i]
        h_planes = 2 if x3 else 1      # H only needs a lo plane when its consumer is split-bf16
        h = empty_u8(N * Lout) if i8 else st.empty(h_planes, N * Lout, C)
        desc = new_desc(a_planes=planes, precision=prec(x3), out_planes=h_planes,
                        res_planes=planes, taps=p.taps[i], k_per_tap=C, n_pad=C, relu=1,
                        out_plane_stride=N * Lout * C, out_ld=C, a_ld=C)
        if p.strided:
            desc.update(tap_row_step=R[i], samples=1, a_rows=N * Lin, per_sample_tiles=0,
                        out_rows=N * Lout)
        else:
            desc.update(samples=N, a_rows=Lin, per_sample_tiles=1, tap_row_step=p.dilation[i],
                        out_rows=Lout)
        if i8:   # Q_{i-1} x s8 -> H, u8 alone (the K per tap padded to 128 past the row of C)
            desc.update(precision=K_INT8, k_per_tap=p.k_conv, out_plane_stride=0)
            run(f"block {i} conv 1", desc, qcur, pk[f"conv{2 * (i - 1)}"],
                pk[f"aff{2 * (i - 1)}"], out_u8=h, inv_s=pk["inv_s"][2 * (i - 1) + 1])
        else:
            run(f"block {i} conv 1", desc, xcur, pk[f"conv{2 * (i - 1)}"],
                pk[f"aff{2 * (i - 1)}"], out=h)
        acts.append((f"H{i}", i, h))

        xnext = st.empty(planes, N * Lout, C)
        lo_b, lo_e = p.lo_range(i)
        desc = new_desc(a_planes=h_planes, precision=prec(x3), out_planes=planes,
                        res_planes=planes, samples=1, a_rows=N * Lout, a_ld=C, taps=1,
                        k_per_tap=C, n_pad=C, per_sample_tiles=0, out_rows=N * Lout, relu=1,
                        out_plane_stride=N * Lout * C, out_ld=C, lo_row_begin=lo_b,
                        lo_row_end=lo_e)
        if p.strided:
            desc.update(res_row_step=1, res_row_off=(fw[i] // 2 + p.shift_str[i]) * R[i])
        else:
            desc.update(samples=N, a_rows=Lout, per_sample_tiles=1, out_rows=Lout,
                        res_rows_per_sample=Lin, res_row_step=1,
                        res_row_off=p.pad[i] + p.shift_dil[i])
        qnext = None
        if i8:   # H x s8 + X_{i-1} -> X_i in fp16, and Q_i for the next block
            desc.update(precision=K_INT8, k_per_tap=p.k_conv)
            qnext = empty_u8(N * Lout) if i < nb else None
        run(f"block {i} conv 2", desc, h, pk[f"conv{2 * (i - 1) + 1}"],
            pk[f"aff{2 * (i - 1) + 1}"], res=xcur, out=xnext, out_u8=qnext,
            inv_s=pk["inv_s"][2 * i] if qnext is not None else None)
        acts.append((f"X{i}", i, xnext))
        if qnext is not None:
            acts.append((f"Q{i}", i, qnext))
        xcur, qcur = xnext, qnext

    # ---- shrink into fp32 (N, L_out, J_out, 3)
    y = torch.full((R[nb], p.c_out_raw), float("nan"),
                   dtype=torch.float64 if exact else torch.float32, device=x.device)
    desc = new_desc(a_planes=planes, precision=prec(p.x3[nb + 1]), out_planes=planes,
                    res_planes=planes, samples=1, a_rows=R[nb], a_ld=C, taps=1, k_per_tap=C,
                    n_pad=p.c_out_pad, per_sample_tiles=0, out_rows=R[nb],
                    out_f32_ld=p.c_out_raw, n_valid=p.c_out_raw)
    run("shrink", desc, xcur, pk["shrink"], pk["shrink_aff"], out_f32=y)
    rep = Replay(p, y.reshape(N, L[nb], p.c_out_raw // 3, 3), launches, acts)
    if collect is not None:
        for k in range(len(acts)):
            collect.append(rep.activation(k).cpu().numpy())
    return rep
