"""Python restatement of the training step of ``vp3d_forward_train_ex`` / ``vp3d_backward_ex``
(train_api.cu): ``train_layout`` rows, ``train_convs``, ``wgrad_desc``, ``dgrad_desc`` and the
launch order of the forward and of ``backward_impl``, for both layouts (strided
TemporalModelOptimized1f: flat rows, the expand conv's taps merged into one GEMM over w0 frames
per row, a first conv's taps column blocks of a w*C-wide view; dilated TemporalModel: per-sample
tiles, the data gradient a transposed convolution with ``tap_row_step = -step``) and both training
precisions (bf16: one plane, the BatchNorm-backward sums fused into the data-gradient GEMMs and
folded by ``ordered_col_sums``; bf16x3: hi + lo planes, ``bn_bwd_reduce``).

``replay(sd, cfg, x, gy, precision, ops, ...)`` runs every launch through ``ops``:

* ``GpuOps``  the operator-level C entries (``vp3d_conv_gemm``, ``vp3d_wgrad_gemm``,
  ``vp3d_bn_stats_finalize``, ``vp3d_bn_apply``, ``vp3d_bn_bwd_reduce``, ``vp3d_ordered_col_sums``,
  ``vp3d_bn_bwd_apply``) on NaN-prefilled buffers the replay owns.  Every launch then computes what
  the model's own launch of the same arguments computes, so y, the gradients, the running
  statistics and dx equal the model's bit for bit.
* ``FakeOps``  the same formulas in float64 on float64 operands and activations (nothing is
  rounded), so the schedule can be checked without a GPU against the float64 training step.

Launches without a C entry are restated in torch: the input and dY packs (round-to-nearest bf16
hi + lo split), the shrink bias affine, the weight packs (forward and transposed), the frozen
BatchNorm fold and the tail copy of a strided dx.  The shrink-bias gradient (``launch_col_sum_f32``)
is a float64 sum here; it is not part of the bit tie.

Every launch is kept as a ``Rec`` (kind, name, descriptor, inputs, outputs) in launch order, and
the forward's and the backward's launches are counted as train_api.cu counts them (2 per weight
gradient, 2 per ``bn_bwd_reduce``, finalize + apply per forward BatchNorm, ...).

``mutate`` (a set of names) switches on deliberately wrong schedules that the tests must reject:
``"skip_off"`` (the skip connection's RowMap offset one frame off), ``"tap_sign"`` (the dilated
data gradient with +step), ``"pingpong"`` (the first conv's BatchNorm backward reading G_i from
the other buffer of the g0 / g1 pair).
"""
import ctypes
from dataclasses import dataclass, field

import torch

import eval_replay as er
from oracle import train_emulation as emu
from test_gpu_wgrad_gemm import Geo, _dw, _products
from videopose3d_b200 import _capi

EPS = 1e-5
MOMENTUM = 0.1
REDUCE_SCRATCH = 32 * 3 * 8192   # kReduceScratchFloats
REDUCE_COUNTERS = 8192 // 32


def round_up(v, m):
    return (v + m - 1) // m * m


class TrainPlan:
    """The plan fields the training step reads (vp3d_plan_create, layer_rows)."""

    def __init__(self, cfg, precision, N, T):
        if precision not in ("bf16", "bf16x3"):
            raise ValueError(f"unknown training precision {precision!r}")
        fw = [int(w) for w in cfg["fw"]]
        causal, dense = bool(cfg.get("causal", False)), bool(cfg.get("dense", False))
        self.fw, self.nb, self.N, self.T = fw, len(fw) - 1, N, T
        self.precision = precision
        self.strided = cfg["cls"] != "TemporalModel"
        self.c_real = cfg["C"]
        self.C = round_up(cfg["C"], 64)
        self.c_in_raw = cfg["J"] * cfg["F"]
        self.c_out_raw = cfg["Jout"] * 3
        self.c_in_pad = round_up(self.c_in_raw, 64)
        self.k0_pad = round_up(self.c_in_raw * fw[0], 64)
        self.c_out_pad = round_up(self.c_out_raw, 64)
        self.dy_ld = round_up(self.c_out_raw, 128)     # K of shrink_t: the padded dY's pitch
        self.planes = 2 if precision == "bf16x3" else 1
        self.f16 = self.int8 = False                   # (eval_replay.Storage / pack_weights)
        self.kprec = er.K_BF16X3 if self.planes == 2 else er.K_BF16
        self.pad, self.shift_dil, self.shift_str = [fw[0] // 2], [0], [0]
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
        if self.strided:
            L = [T // fw[0]]
            for w in fw[1:]:
                L.append(L[-1] // w)
            for i in range(1, self.nb + 1):
                if L[i - 1] != fw[i] * L[i]:
                    raise ValueError("strided training needs layer lengths divisible by the width")
        else:
            L = [T - fw[0] + 1]
            for i in range(1, self.nb + 1):
                L.append(L[-1] - 2 * self.pad[i])
        if min(L) < 1:
            raise ValueError(f"sequence of {T} frames is too short")
        self.L = L
        self.R = [N * v for v in L]
        # train_layout: the weight-gradient split partials (their size caps the split count)
        max_taps = max([1] + self.taps[1:])
        if not self.strided:
            max_taps = max(max_taps, fw[0])
        n_max = max(self.C, self.k0_pad, self.c_in_pad)
        self.partial_bytes = 8 * max_taps * round_up(self.C, 128) * round_up(n_max, 64) * 4


# ---------------------------------------------------------------------------------------- packs
def pack_transposed(sd, p, st):
    """The transposed packs of pack_conv_weight_t_kernel: conv_t [taps][ci (n_pad C)][co (k_pad C)],
    shrink_t [1][C][dy_ld] (K padded to 128), expand_t strided: one merged slab
    [tap*c_in + ci (k0_pad)][co (C)], dilated: [w0][c_in_pad][C]; hi + lo bf16, zero padded."""
    dev = st.device
    src = torch.float64 if st.exact else torch.float32

    def w_of(name):
        return sd[name].detach().to(device=dev, dtype=src)

    def pack_t(w, n_pad, k_pad, merged):
        co, ci, k = w.shape
        if merged:
            buf = torch.zeros(1, n_pad, k_pad, dtype=src, device=dev)
            buf[0, :k * ci, :co] = w.permute(2, 1, 0).reshape(k * ci, co)
        else:
            buf = torch.zeros(k, n_pad, k_pad, dtype=src, device=dev)
            buf[:, :ci, :co] = w.permute(2, 1, 0)
        return st.planes_of(buf, p.planes).contiguous()

    pk = {f"conv_t{j}": pack_t(w_of(f"layers_conv.{j}.weight"), p.C, p.C, False)
          for j in range(2 * p.nb)}
    pk["shrink_t"] = pack_t(w_of("shrink.weight"), p.C, p.dy_ld, False)
    ew = w_of("expand_conv.weight")
    pk["expand_t"] = pack_t(ew, p.k0_pad, p.C, True) if p.strided else \
        pack_t(ew, p.c_in_pad, p.C, False)
    return pk


def bn_fold_train(bn, c_pad, exact):
    """launch_bn_fold with the mean / invstd outputs of a frozen-BatchNorm training forward:
    eval_replay.bn_fold's scale / shift, mean = running_mean and invstd = 1 / sqrtf(var + eps) in
    fp32 (each IEEE operation restated in float64 and rounded once; float64 in exact mode)."""
    scale, shift = er.bn_fold(bn, c_pad, exact)
    m, v = bn["running_mean"].detach().cpu(), bn["running_var"].detach().cpu()
    c = m.numel()
    dt = torch.float64 if exact else torch.float32
    mean = torch.zeros(c_pad, dtype=dt)
    inv = torch.zeros(c_pad, dtype=dt)
    mean[:c] = m.to(dt)
    if exact:
        inv[:c] = 1.0 / torch.sqrt(v.double() + EPS)
    else:
        eps = float(torch.tensor(EPS, dtype=torch.float32))
        root = torch.sqrt((v.double() + eps).float().double()).float()
        inv[:c] = (1.0 / root.double()).float()
    return scale, shift, mean, inv


# ------------------------------------------------------------------------------------ launches
@dataclass
class Rec:
    """One launch: kind (conv / stats_finalize / bn_fold / bn_apply / wgrad / bn_bwd_reduce /
    ordered_col_sums / bn_bwd_apply / pack / dx_tail / col_sum), its name, layer and descriptor,
    and the tensors it read and wrote."""
    kind: str
    name: str
    layer: int = -1
    desc: dict = field(default_factory=dict)
    ins: dict = field(default_factory=dict)
    outs: dict = field(default_factory=dict)


class ConvLaunch(er.Launch):
    """A training conv GEMM: eval_replay.Launch (descriptor, A, W, affine) plus the training
    epilogue's options: `skip` (tensor [planes][rows][ld], dict of res_* fields: a column block
    res_col_begin / res_cols, or rows shifted by res_row_off with res_check_rows), `stats` (per-slab
    sum / sumsq of the output [slabs][2][n_pad]) and `bnb` (the fused BatchNorm-backward sums:
    dict(z, scale, shift, mean, invstd, sums, c, p, seed, layer))."""

    def __init__(self, name, desc, a, w, scale, shift, out=None, out_f32=None, skip=None,
                 stats=None, bnb=None):
        super().__init__(name, desc, a, w, scale, shift, out=out, out_f32=out_f32)
        self.skip, self.stats, self.bnb = skip, stats, bnb

    def slabs(self):
        d = self.desc
        return (d["samples"] if d["per_sample_tiles"] else 1) * -(-d["out_rows"] // er.BLOCK_M) * 4

    def per_slab(self, t):
        """[total_rows, n] -> [slabs, n] sums over each 32-row slab of the GEMM's row tiling."""
        d = self.desc
        s = d["samples"] if d["per_sample_tiles"] else 1
        t = t.reshape(s, -1, t.shape[-1])
        tiles = -(-t.shape[1] // er.BLOCK_M)
        pad = torch.zeros(s, tiles * er.BLOCK_M - t.shape[1], t.shape[-1], dtype=t.dtype,
                          device=t.device)
        return torch.cat([t, pad], 1).reshape(s * tiles * 4, 32, t.shape[-1]).sum(1)

    def skip_value(self, v):
        """v + the skip connection's term, as the epilogue adds it (float64)."""
        if self.skip is None:
            return v
        res, kw = self.skip
        rv = er.stored_value(res)
        d = self.desc
        if kw.get("res_cols"):
            cb, nc = kw["res_col_begin"], kw["res_cols"]
            v = v.clone()
            v[:, cb:cb + nc] += rv
            return v
        # per-sample rows: G_in[n, t] += res[n, t + res_row_off] where that row exists
        rps = kw["res_rows_per_sample"]
        t = torch.arange(d["out_rows"], device=v.device) + kw["res_row_off"]
        ok = (t >= 0) & (t < rps)
        add = torch.zeros(d["samples"], d["out_rows"], v.shape[-1], dtype=v.dtype, device=v.device)
        add[:, ok] = rv.reshape(d["samples"], rps, -1)[:, t[ok]]
        return v + add.reshape(v.shape)

    def bnb_dy(self, g):
        """dY of the layer below from the stored gradient g [total_rows, n_pad] (float64):
        g * mask * [Z*scale + shift > 0], channel = column % c, mask element = row * n_pad + column.
        Returns (dy, z - mean) per element."""
        b = self.bnb
        rows, n = g.shape
        ch = torch.arange(n, device=g.device) % b["c"]
        z = b["z"][0].double().reshape(rows, n)
        live = (z * b["scale"].double()[ch] + b["shift"].double()[ch]) > 0
        dy = g * live
        if b["p"] > 0:
            mask = emu.dropout_mask(b["seed"], b["layer"], rows * n // b["c"], b["c"], b["c"], b["p"])
            dy = dy * mask.to(g.device).reshape(rows, n)
        return dy, z - b["mean"].double()[ch]


def _ptr(t):
    return None if t is None else t.data_ptr()


class GpuOps:
    """The launches through the operator-level C entries."""
    exact = False

    def __init__(self, device):
        self.device = device
        self.lib = _capi.load()
        self.scratch = torch.full((REDUCE_SCRATCH,), float("nan"), device=device)
        self.counter = torch.zeros(REDUCE_COUNTERS, dtype=torch.int32, device=device)

    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def _check(self, st, what):
        torch.cuda.synchronize()
        assert st == 0, f"{what}: {self.lib.vp3d_last_error()}"

    def _red(self):
        return (self.scratch.data_ptr(), self.scratch.numel(), self.counter.data_ptr(),
                self.counter.numel())

    def conv(self, lc):
        d = lc.desc
        kw = {}
        if lc.skip is not None:
            res, rk = lc.skip
            kw.update(res=res, **rk)
        if lc.stats is not None:
            lc.stats.fill_(float("nan"))
            kw["stats"] = lc.stats
        if lc.bnb is not None:
            b = lc.bnb
            b["sums"].fill_(float("nan"))
            kw.update(bnb_z=b["z"], bnb_scale=b["scale"], bnb_shift=b["shift"], bnb_mean=b["mean"],
                      bnb_invstd=b["invstd"], bnb_sums=b["sums"], bnb_c=b["c"], bnb_p=b["p"],
                      bnb_seed=b["seed"], bnb_layer=b["layer"])
        er.conv_gemm(lc.a, d["samples"], d["a_rows"], d["a_ld"], lc.w, d["taps"], d["k_per_tap"],
                     d["n_pad"], per_sample_tiles=d["per_sample_tiles"],
                     tap_row_step=d["tap_row_step"], tap_col_step=d["tap_col_step"],
                     out_rows=d["out_rows"], precision=d["precision"], scale=lc.scale,
                     shift=lc.shift, relu=False, out=lc.out, out_f32=lc.out_f32,
                     out_f32_cols=d["n_valid"] if lc.out_f32 is not None else None,
                     out_plane_stride=d["out_plane_stride"], **kw)

    def stats_finalize(self, lc, gamma, beta, rm, rv, c, c_real, out):
        d = lc.desc
        for t in out.values():
            t.fill_(float("nan"))
        tps = -(-d["out_rows"] // er.BLOCK_M) if d["per_sample_tiles"] else 0
        st = self.lib.vp3d_bn_stats_finalize(
            lc.stats.data_ptr(), lc.slabs(), d["per_sample_tiles"], d["out_rows"], tps,
            gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), MOMENTUM, EPS,
            out["scale"].data_ptr(), out["shift"].data_ptr(), out["mean"].data_ptr(),
            out["invstd"].data_ptr(), c, c_real, *self._red(), self._stream())
        self._check(st, "bn_stats_finalize")

    def bn_apply(self, z, x, rows, c, scale, shift, p, seed, layer, res, rmap):
        x.fill_(float("nan"))
        div, rps, step, off = rmap
        st = self.lib.vp3d_bn_apply(z.data_ptr(), z[0].numel(), x.data_ptr(), x[0].numel(),
                                    z.shape[0], rows, c, scale.data_ptr(), shift.data_ptr(), p,
                                    seed, layer, _ptr(res), 0 if res is None else res[0].numel(),
                                    div, rps, step, off, self._stream())
        self._check(st, "bn_apply")

    def wgrad(self, w, dz, x, grad, partial):
        grad.fill_(float("nan"))
        d = _capi.WgradDesc()
        d.dz, d.x, d.grad, d.partial = dz.data_ptr(), x.data_ptr(), grad.data_ptr(), partial.data_ptr()
        d.partial_bytes = partial.numel() * 4
        for k in ("dz_ld", "x_ld", "planes", "rows", "per_sample", "samples", "x_rows", "taps",
                  "tap_row_step", "tap_col_step", "c_out", "c_in_cols", "c_in", "taps_out",
                  "merged"):
            setattr(d, k, w[k])
        st = self.lib.vp3d_wgrad_gemm(ctypes.byref(d), self._stream())
        self._check(st, "wgrad_gemm")

    def bn_bwd_reduce(self, g, z, rows, c, v, p, seed, layer, partials, sums):
        sums.fill_(float("nan"))
        st = self.lib.vp3d_bn_bwd_reduce(
            g.data_ptr(), g[0].numel(), z.data_ptr(), z[0].numel(), z.shape[0], rows, c,
            v["scale"].data_ptr(), v["shift"].data_ptr(), v["mean"].data_ptr(),
            v["invstd"].data_ptr(), p, seed, layer, partials.data_ptr(), partials.numel(),
            sums.data_ptr(), *self._red(), self._stream())
        self._check(st, "bn_bwd_reduce")

    def ordered_col_sums(self, lc, c, invstd, sums):
        sums.fill_(float("nan"))
        n_pad = lc.desc["n_pad"]
        st = self.lib.vp3d_ordered_col_sums(lc.bnb["sums"].data_ptr(), lc.slabs(), 2, n_pad, c,
                                            n_pad // c, None, invstd.data_ptr(), sums.data_ptr(),
                                            sums[c:].data_ptr(), *self._red(), self._stream())
        self._check(st, "ordered_col_sums")

    def bn_bwd_apply(self, g, z, dz, rows, c, v, p, seed, layer, sums, dgamma, dbeta, c_real,
                     frozen):
        for t in (dz, dgamma, dbeta):
            t.fill_(float("nan"))
        st = self.lib.vp3d_bn_bwd_apply(
            g.data_ptr(), g[0].numel(), z.data_ptr(), z[0].numel(), dz.data_ptr(), dz[0].numel(),
            z.shape[0], rows, c, v["scale"].data_ptr(), v["shift"].data_ptr(),
            v["mean"].data_ptr(), v["invstd"].data_ptr(), p, seed, layer, sums.data_ptr(),
            dgamma.data_ptr(), dbeta.data_ptr(), c_real, int(frozen), self._stream())
        self._check(st, "bn_bwd_apply")


class FakeOps:
    """The same launches as float64 formulas on float64 operands: nothing is rounded, so the
    replay is the training step's algorithm in float64."""
    exact = True

    def __init__(self, device):
        self.device = device

    def conv(self, lc):
        base = er.Launch(lc.name, lc.desc, lc.a, lc.w,
                         lc.scale if lc.scale is not None else _ones(lc),
                         lc.shift if lc.shift is not None else _zeros(lc))
        v, _ = er.fake_conv(base)
        v = lc.skip_value(v)
        if lc.stats is not None:
            lc.stats.copy_(torch.stack([lc.per_slab(v), lc.per_slab(v * v)], 1))
        er.store(lc, v)
        if lc.bnb is not None:
            dy, zc = lc.bnb_dy(er.stored_value(lc.out))
            lc.bnb["sums"].copy_(torch.stack([lc.per_slab(dy), lc.per_slab(dy * zc)], 1))

    def stats_finalize(self, lc, gamma, beta, rm, rv, c, c_real, out):
        s = lc.stats.double().sum(0)
        n = lc.desc["out_rows"] * (lc.desc["samples"] if lc.desc["per_sample_tiles"] else 1)
        mean = s[0] / n
        var = (s[1] / n - mean * mean).clamp_min(0.0)
        inv = 1.0 / torch.sqrt(var + EPS)
        cr = slice(0, c_real)
        for t in out.values():
            t.zero_()
        out["mean"][cr] = mean[cr]
        out["invstd"][cr] = inv[cr]
        out["scale"][cr] = gamma.double() * inv[cr]
        out["shift"][cr] = beta.double() - mean[cr] * out["scale"][cr]
        unb = var[cr] * n / (n - 1) if n > 1 else var[cr]
        rm.copy_((1 - MOMENTUM) * rm.double() + MOMENTUM * mean[cr])
        rv.copy_((1 - MOMENTUM) * rv.double() + MOMENTUM * unb)

    def bn_apply(self, z, x, rows, c, scale, shift, p, seed, layer, res, rmap):
        v = torch.relu(er.stored_value(z) * scale.double() + shift.double())
        if p > 0:
            v = v * emu.dropout_mask(seed, layer, rows, c, c, p).to(v.device)
        if res is not None:
            div, rps, step, off = rmap
            r = torch.arange(rows, device=v.device)
            rr = (r // div) * rps + (r % div) * step + off if div else r * step + off
            v = v + er.stored_value(res)[rr]
        x.zero_()
        x[0] = v

    def wgrad(self, w, dz, x, grad, partial):
        g = wgrad_geo(w)
        s = g.s
        dzp = dz.reshape(dz.shape[0], s, g.rows, g.dz_ld)
        xp = x.reshape(x.shape[0], s, g.xr, g.x_ld)
        grad.copy_(sum(_dw(g, a, b) for a, b in _products(dzp, xp)))

    def _sums(self, g, z, v, p, seed, layer):
        rows, c = g.shape[1], g.shape[2]
        z = er.stored_value(z)
        dy = er.stored_value(g) * ((z * v["scale"].double() + v["shift"].double()) > 0)
        if p > 0:
            dy = dy * emu.dropout_mask(seed, layer, rows, c, c, p).to(dy.device)
        return dy, z

    def bn_bwd_reduce(self, g, z, rows, c, v, p, seed, layer, partials, sums):
        dy, zv = self._sums(g, z, v, p, seed, layer)
        sums[:c] = dy.sum(0)
        sums[c:] = (dy * (zv - v["mean"].double())).sum(0) * v["invstd"].double()

    def ordered_col_sums(self, lc, c, invstd, sums):
        n_pad = lc.desc["n_pad"]
        s = lc.bnb["sums"].double().sum(0).reshape(2, n_pad // c, c).sum(1)
        sums[:c] = s[0]
        sums[c:] = s[1] * invstd.double()

    def bn_bwd_apply(self, g, z, dz, rows, c, v, p, seed, layer, sums, dgamma, dbeta, c_real,
                     frozen):
        dy, zv = self._sums(g, z, v, p, seed, layer)
        sc = v["scale"].double()
        if frozen:
            out = sc * dy
        else:
            xh = (zv - v["mean"].double()) * v["invstd"].double()
            out = sc * (dy - sums[:c].double() / rows - xh * sums[c:].double() / rows)
        dz.zero_()
        dz[0] = out
        dbeta[:c_real] = sums[:c_real]
        dgamma[:c_real] = sums[c:c + c_real]


def _ones(lc):
    return torch.ones(lc.desc["n_pad"], dtype=torch.float64, device=lc.a.device)


def _zeros(lc):
    return torch.zeros(lc.desc["n_pad"], dtype=torch.float64, device=lc.a.device)


def wgrad_geo(w):
    """test_gpu_wgrad_gemm.Geo of a vp3d_wgrad_desc (dict)."""
    return Geo(c_out=w["c_out"], dz_ld=w["dz_ld"], c_in=w["c_in"], x_ld=w["x_ld"], rows=w["rows"],
               taps=w["taps_out"], per_sample=w["per_sample"], samples=w["samples"],
               x_rows=w["x_rows"] if w["per_sample"] else 0, tap_row_step=w["tap_row_step"],
               tap_col_step=w["tap_col_step"], merged=w["merged"])


# --------------------------------------------------------------------------------------- replay
class TrainReplay:
    """Result of ``replay``: the plan, y (N, L_out, J_out, 3), dx or None, the parameter gradients
    and new running statistics by state-dict name, the records and the launch counts of the
    forward and of the backward."""

    def __init__(self, plan):
        self.plan = plan
        self.recs, self.grads, self.stats = [], {}, {}
        self.y = self.dx = None
        self.fwd_launches = self.bwd_launches = 0


def bn_prefix(l):
    return "expand_bn" if l == 0 else f"layers_bn.{l - 1}"


def conv_name(l, nb):
    if l == 0:
        return "expand"
    if l == 2 * nb + 1:
        return "shrink"
    return f"block {(l + 1) // 2} conv {2 - l % 2}"


def replay(sd, cfg, x, gy, precision, ops, *, p_drop=0.0, seed=0, frozen=False, want_dx=False,
           mutate=()):
    """One training step of the model with state dict sd on x (N, T, J, F) and upstream gradient
    gy (y's shape): the forward, then the backward with every parameter gradient [+ dx].  p_drop /
    seed: the dropout probability and the step's seed (train_emulation.step_seed).  frozen: the
    eval-mode backward's frozen-BatchNorm forward (no dropout, running statistics untouched)."""
    mutate = set(mutate)
    dev = x.device
    N, T = int(x.shape[0]), int(x.shape[1])
    p = TrainPlan(cfg, precision, N, T)
    exact = ops.exact
    st = er.Storage(p, exact, dev)
    pk = er.pack_weights(sd, p, st)
    pk.update(pack_transposed(sd, p, st))
    fdt = torch.float64 if exact else torch.float32
    C, nb, fw, L, R, pl = p.C, p.nb, p.fw, p.L, p.R, p.planes
    rep = TrainReplay(p)
    recs = rep.recs
    fwd = {}   # layer -> dict(desc, conv launch, input, Z, act, vec, ...)

    def vec(n=C):
        return torch.full((n,), float("nan"), dtype=fdt, device=dev)

    def param(name):
        return sd[name].detach().to(device=dev, dtype=fdt).clone()

    # ---- forward: shrink bias affine, input pack
    launches = 1
    xs = x.reshape(N, T, p.c_in_raw).to(fdt)
    if p.strided:
        vals = torch.zeros(R[0], p.k0_pad, dtype=fdt, device=dev)
        vals[:, :fw[0] * p.c_in_raw] = xs[:, :L[0] * fw[0]].reshape(R[0], fw[0] * p.c_in_raw)
    else:
        vals = torch.zeros(N * T, p.c_in_pad, dtype=fdt, device=dev)
        vals[:, :p.c_in_raw] = xs.reshape(N * T, p.c_in_raw)
    a0 = st.planes_of(vals, pl).contiguous()
    recs.append(Rec("pack", "input pack", outs=dict(out=a0)))
    launches += 1

    def conv_desc(**kw):
        d = er.new_desc(a_planes=pl, out_planes=pl, res_planes=pl, precision=p.kprec, samples=1)
        d.update({k: int(v) for k, v in kw.items()})
        return d

    # train_convs: the forward descriptors, indexed by BatchNorm layer (shrink at 2B + 1)
    def fwd_conv(l, a, w, **kw):
        d = conv_desc(taps=w.shape[1], k_per_tap=w.shape[3], n_pad=w.shape[2], **kw)
        fwd[l] = dict(desc=d, a=a, w=w)
        return d

    for l in range(0, 2 * nb + 1):
        i = (l + 1) // 2
        inp = fwd[l - 1]["act"] if l else a0    # X_{i-1} (odd l) or H_i (even l)
        if l == 0:
            if p.strided:
                fwd_conv(0, a0, pk["expand_flat"], a_rows=R[0], a_ld=p.k0_pad, out_rows=R[0])
            else:
                fwd_conv(0, a0, pk["expand_dil"], samples=N, a_rows=T, a_ld=p.c_in_pad,
                         out_rows=L[0], per_sample_tiles=1, tap_row_step=1)
        elif l % 2:
            if p.strided:
                # (the w*C-wide row view of X_{i-1}: tap k is column block k)
                fwd_conv(l, inp.reshape(pl, R[i], fw[i] * C), pk[f"conv{l - 1}"], a_rows=R[i],
                         a_ld=fw[i] * C, out_rows=R[i], tap_col_step=C)
            else:
                fwd_conv(l, inp, pk[f"conv{l - 1}"], samples=N, a_rows=L[i - 1], a_ld=C,
                         out_rows=L[i], per_sample_tiles=1, tap_row_step=p.dilation[i])
        else:
            fwd_conv(l, inp, pk[f"conv{l - 1}"], a_rows=R[i], a_ld=C, out_rows=R[i])
        f = fwd[l]
        d = f["desc"]
        d.update(out_plane_stride=R[i] * C, out_ld=C)
        z = st.empty(pl, R[i], C)
        lc = ConvLaunch(conv_name(l, nb), d, f["a"], f["w"], None, None, out=z)
        if not frozen:
            lc.stats = torch.full((lc.slabs(), 2, C), float("nan"), dtype=fdt, device=dev)
        ops.conv(lc)
        launches += 1
        recs.append(Rec("conv", lc.name, l, d, dict(a=f["a"]), dict(out=z, lc=lc)))
        f.update(z=z, lc=lc)
        # BatchNorm (+ ReLU, dropout, skip connection)
        prefix = bn_prefix(l)
        bn = {k: sd[f"{prefix}.{k}"] for k in ("weight", "bias", "running_mean", "running_var")}
        if frozen:
            sc, sh, mu, inv = bn_fold_train(bn, C, exact)
            v = {k: t.to(dev) for k, t in zip(("scale", "shift", "mean", "invstd"), (sc, sh, mu, inv))}
            recs.append(Rec("bn_fold", prefix, l, outs=dict(v)))
        else:
            v = dict(scale=vec(), shift=vec(), mean=vec(), invstd=vec())
            rm, rv = param(f"{prefix}.running_mean"), param(f"{prefix}.running_var")
            gamma, beta = param(f"{prefix}.weight"), param(f"{prefix}.bias")
            rm0, rv0 = rm.clone(), rv.clone()
            ops.stats_finalize(lc, gamma, beta, rm, rv, C, p.c_real, v)
            rep.stats[f"{prefix}.running_mean"], rep.stats[f"{prefix}.running_var"] = rm, rv
            recs.append(Rec("stats_finalize", prefix, l, d,
                            dict(lc=lc, gamma=gamma, beta=beta, rm=rm0, rv=rv0),
                            dict(v, rm=rm, rv=rv)))
        f["vec"] = v
        act = st.empty(pl, R[i], C)
        res, rmap = None, (0, 0, 1, 0)
        if l > 0 and l % 2 == 0:
            res = fwd[l - 2]["act"]   # the block's input X_{i-1}
            off = fw[i] // 2 + p.shift_str[i] if p.strided else p.pad[i] + p.shift_dil[i]
            if "skip_off" in mutate:
                off += 1
            rmap = (0, 0, fw[i], off) if p.strided else (L[i], L[i - 1], 1, off)
            f["res_off"] = off
        ops.bn_apply(z, act, R[i], C, v["scale"], v["shift"], p_drop, seed, l, res, rmap)
        launches += 2
        recs.append(Rec("bn_apply", prefix, l, dict(rmap=rmap),
                        dict(z=z, scale=v["scale"], shift=v["shift"], res=res), dict(out=act)))
        f["act"] = act

    # shrink into fp32 y
    inp = fwd[2 * nb]["act"]
    sh_w = pk["shrink"]
    d = conv_desc(a_rows=R[nb], a_ld=C, out_rows=R[nb], taps=1, k_per_tap=C, n_pad=p.c_out_pad,
                  out_f32_ld=p.c_out_raw, n_valid=p.c_out_raw)
    fwd[2 * nb + 1] = dict(desc=d, a=inp, w=sh_w)
    y = torch.full((R[nb], p.c_out_raw), float("nan"), dtype=fdt, device=dev)
    lc = ConvLaunch("shrink", d, inp, sh_w, *pk["shrink_aff"], out_f32=y)
    ops.conv(lc)
    launches += 1
    recs.append(Rec("conv", "shrink", 2 * nb + 1, d, dict(a=inp), dict(out_f32=y, lc=lc)))
    rep.y = y.reshape(N, L[nb], p.c_out_raw // 3, 3)
    rep.fwd_launches = launches

    # ---- backward
    launches = 0
    top = 2 * nb
    fuse = pl == 1
    dyv = gy.reshape(R[nb], p.c_out_raw).to(device=dev, dtype=fdt)
    vals = torch.zeros(R[nb], p.dy_ld, dtype=fdt, device=dev)
    vals[:, :p.c_out_raw] = dyv
    dyp = st.planes_of(vals, pl).contiguous()
    recs.append(Rec("pack", "dY pack", outs=dict(out=dyp)))
    launches += 1
    rep.grads["shrink.bias"] = dyv.double().sum(0)       # launch_col_sum_f32 (not restated)
    recs.append(Rec("col_sum", "shrink bias", ins=dict(dy=dyv), outs=dict(out=rep.grads["shrink.bias"])))
    launches += 2
    partial = torch.full((p.partial_bytes // 4,), float("nan"), dtype=torch.float32, device=dev)

    def pack_of(l):
        """(c_out, c_in, taps, merged) of the forward pack of conv l (its gradient's shape)."""
        if l == 2 * nb + 1:
            return p.c_out_raw, p.c_real, 1, 0
        if l == 0:
            return p.c_real, p.c_in_raw, fw[0], int(p.strided)
        return p.c_real, p.c_real, p.taps[(l + 1) // 2] if l % 2 else 1, 0

    def wgrad(l, dz, dz_ld, name):
        f = fwd[l]
        fd = f["desc"]
        co, ci, taps, merged = pack_of(l)
        w = dict(dz_ld=dz_ld, x_ld=fd["a_ld"], planes=fd["a_planes"], rows=fd["out_rows"],
                 per_sample=fd["per_sample_tiles"], samples=fd["samples"], x_rows=fd["a_rows"],
                 taps=fd["taps"], tap_row_step=fd["tap_row_step"],
                 tap_col_step=fd["tap_col_step"], c_out=co, c_in=ci, taps_out=taps,
                 merged=merged, c_in_cols=taps * ci if merged else ci)
        grad = torch.full((co, ci, taps), float("nan"), dtype=fdt, device=dev)
        ops.wgrad(w, dz, f["a"], grad, partial)
        rep.grads[name] = grad
        recs.append(Rec("wgrad", name, l, w, dict(dz=dz, x=f["a"]), dict(grad=grad)))
        return 2

    def t_pack(l):
        if l == 2 * nb + 1:
            return pk["shrink_t"]
        return pk["expand_t"] if l == 0 else pk[f"conv_t{l - 1}"]

    def dgrad(l, dz, out=None, res=None, res_off=0, out_f32=None):
        """dgrad_desc of conv l, as a ConvLaunch (not run)."""
        f = fwd[l]
        fd = f["desc"]
        wt = t_pack(l)
        d = conv_desc(taps=wt.shape[1], k_per_tap=wt.shape[3], n_pad=wt.shape[2],
                      a_rows=fd["out_rows"], a_ld=wt.shape[3], out_rows=fd["a_rows"],
                      out_plane_stride=fd["samples"] * fd["a_rows"] * fd["a_ld"],
                      out_ld=fd["a_ld"])
        if fd["per_sample_tiles"]:
            step = fd["tap_row_step"] if "tap_sign" in mutate else -fd["tap_row_step"]
            d.update(samples=fd["samples"], per_sample_tiles=1, tap_row_step=step)
        else:
            d.update(n_pad=d["n_pad"] * d["taps"], taps=1)
            wt = wt.reshape(wt.shape[0], 1, -1, wt.shape[3])
        skip = None
        if res is not None:
            if fd["per_sample_tiles"]:
                rk = dict(res_rows_per_sample=fd["out_rows"], res_row_step=1,
                          res_row_off=-res_off, res_check_rows=1)
            else:
                rk = dict(res_row_step=1, res_col_begin=res_off * C, res_cols=C)
            skip = (res, rk)
        if out_f32 is not None:
            d.update(out_f32_ld=out_f32.shape[-1], n_valid=out_f32.shape[-1])
        return ConvLaunch(conv_name(l, nb), d, dz, wt, None, None, out=out,
                          out_f32=out_f32, skip=skip)

    vecs = {l: fwd[l]["vec"] for l in range(top + 1)}

    def fuse_bnb(lc, layer):
        if not fuse:
            return
        v = vecs[layer]
        lc.bnb = dict(z=fwd[layer]["z"], scale=v["scale"], shift=v["shift"], mean=v["mean"],
                      invstd=v["invstd"], c=C, p=p_drop, seed=seed, layer=layer,
                      sums=torch.full((lc.slabs(), 2, lc.desc["n_pad"]), float("nan"),
                                      dtype=fdt, device=dev))

    def run(lc, l):
        ops.conv(lc)
        recs.append(Rec("dgrad", lc.name, l, lc.desc, dict(a=lc.a), dict(out=lc.out, lc=lc,
                                                                       out_f32=lc.out_f32)))
        return 1

    launches += wgrad(2 * nb + 1, dyp, p.dy_ld, "shrink.weight")
    gb = [None, None]
    cur = 0
    gb[cur] = st.empty(pl, R[nb], C)
    lc = dgrad(2 * nb + 1, dyp, out=gb[cur])
    fuse_bnb(lc, top)
    launches += run(lc, 2 * nb + 1)
    last = lc                       # the GEMM whose fused slab sums the next bn_bwd folds

    for l in range(top, -1, -1):
        i = (l + 1) // 2
        f = fwd[l]
        v = vecs[l]
        src = cur ^ 1 if l % 2 else cur
        if "pingpong" in mutate and l % 2:
            src = cur
        gin = gb[src]
        rows = R[i]
        prefix = bn_prefix(l)
        sums = torch.full((2 * C,), float("nan"), dtype=fdt, device=dev)
        if not fuse:
            partials = torch.full(((((rows + 31) // 32 + 1) * 2 * C),), float("nan"),
                                  dtype=torch.float32, device=dev)
            ops.bn_bwd_reduce(gin, f["z"], rows, C, v, p_drop, seed, l, partials, sums)
            launches += 2
            recs.append(Rec("bn_bwd_reduce", prefix, l, {}, dict(g=gin, z=f["z"], v=v),
                            dict(sums=sums)))
        else:
            ops.ordered_col_sums(last, C, v["invstd"], sums)
            launches += 1
            recs.append(Rec("ordered_col_sums", prefix, l, {}, dict(lc=last, invstd=v["invstd"]),
                            dict(sums=sums)))
        dz = st.empty(pl, rows, C)
        dgamma, dbeta = vec(p.c_real), vec(p.c_real)
        ops.bn_bwd_apply(gin, f["z"], dz, rows, C, v, p_drop, seed, l, sums, dgamma, dbeta,
                         p.c_real, frozen)
        launches += 1
        rep.grads[f"{prefix}.weight"], rep.grads[f"{prefix}.bias"] = dgamma, dbeta
        recs.append(Rec("bn_bwd_apply", prefix, l, {}, dict(g=gin, z=f["z"], v=v, sums=sums),
                        dict(dz=dz, dgamma=dgamma, dbeta=dbeta)))
        launches += wgrad(l, dz, C, "expand_conv.weight" if l == 0 else f"layers_conv.{l - 1}.weight")
        if l > 0:
            fd = f["desc"]
            out = st.empty(pl, fd["samples"] * fd["a_rows"], fd["a_ld"])
            gb[cur ^ 1] = out.reshape(pl, -1, C)   # G_{i-1} or G_H, [rows][C]
            if l % 2:
                lc = dgrad(l, dz, out=out, res=gb[cur], res_off=fwd[l + 1]["res_off"])
            else:
                lc = dgrad(l, dz, out=out)
            fuse_bnb(lc, l - 1)
            launches += run(lc, l)
            last = lc
        elif want_dx:
            fd = f["desc"]
            cols = fw[0] * p.c_in_raw if p.strided else p.c_in_raw
            stage = torch.full((fd["samples"] * fd["a_rows"], cols), float("nan"), dtype=fdt,
                               device=dev)
            lc = dgrad(0, dz, out_f32=stage)
            launches += run(lc, 0)
            tail = p.strided and T != fw[0] * L[0]
            if tail:   # cudaMemcpy2DAsync of each sample's rows, cudaMemset2DAsync of its tail
                dx = torch.zeros(N, T, p.c_in_raw, dtype=fdt, device=dev)
                dx[:, :fw[0] * L[0]] = stage.reshape(N, fw[0] * L[0], p.c_in_raw)
                launches += 2
                recs.append(Rec("dx_tail", "dx tail", ins=dict(stage=stage), outs=dict(dx=dx)))
            else:
                dx = stage.reshape(N, T, p.c_in_raw)
            rep.dx = dx.reshape(x.shape)
        if l % 2:
            cur ^= 1
    rep.bwd_launches = launches
    return rep
