"""GPU: the BatchNorm training passes (videopose3d_b200/csrc/train_ops.cu, reached through the C
entries vp3d_bn_stats_finalize / vp3d_ordered_col_sums / vp3d_bn_apply / vp3d_bn_bwd_reduce /
vp3d_bn_bwd_apply, the launches the training step makes) against float64 formulas of
nn.BatchNorm1d in train mode, ReLU, Dropout and their backward.

Inputs are built from a float64 data matrix rounded once to what the kernels read (bf16 planes,
fp32 vectors / slab partials), so the reference and the kernel see identical values.  Dropout
masks come from oracle/train_emulation.dropout_mask, the restatement of the kernels' own generator.

Gates (u = 2^-24, the fp32 unit round-off):
* stats finalize: |mean - ref| <= k u rms, |var - ref| <= k u rms^2 (var read back from invstd),
  k = 8 sqrt(slabs) + 32, rms^2 = var + mean^2 of the channel.  The rms^2 term is the per-slab
  variance: it is formed in fp32 as sq - sum * mean, whose cancellation costs ~u (1 + mean^2 / var)
  of the slab's variance (DESIGN.md, "Batch statistics"): an offset-heavy channel with
  |mean| / std = 100 keeps ~1e-3 relative accuracy in its variance.  scale / shift / running stats
  follow with one or two extra roundings.  Padding channels are exactly 0.
* ordered_col_sums / bn_bwd_reduce sums: |got - ref| <= 32 u sum|terms|.  These are plain fp32
  additions with round-to-nearest on the CUDA cores, whose errors do not share a sign: for
  random-sign terms they add up to about u sum|terms|, a few times that at most.
* bn_apply: one bf16 rounding of the fp64 value, |got - ref| <= 2^-8 |ref| + 8 u (|z scale| +
  |shift| + |res|) (2^-8: half an ulp of bf16's 8-bit significand); two planes: |lo| is at most half
  an ulp of hi (hi is a rounding of hi + lo) and |hi + lo - ref| <= 2^-16 |ref| + the same fp32 term.
* bn_bwd_apply: one bf16 rounding plus the fp32 affine and the sums' own bounds carried through.
Every gate is shown to reject a perturbed reference in the same test (one slab or part dropped, the
mask of another layer, the residual one row off, n - 1 instead of n).

Dispatch cases hit (asserted by the mirrors _splits / _row_tiling): stats finalize with S = 1, 2,
between, 32 and slab counts far beyond 32 * 128; ordered_col_sums on both sides of each 128-part
step; row_tiling widths G = 8 (C = 64, 192, 320) and G = 128 (C = 1024), each over row counts from
1 to 20013 so that blocks end inside and after the 4-row fast loop."""
import functools
import math

import pytest
import torch

from oracle import train_emulation as emu
from videopose3d_b200 import _capi

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = 1e-5
SEED = 0x5EED_0123_4567_89AB
LAYER = 5


def _splits(n_part):
    """Mirror of pick_splits (train_ops.cu)."""
    return max(1, min(32, (n_part + 127) // 128))


def _row_tiling(rows, c):
    """Mirror of row_tiling: (G, lanes, rows per block)."""
    groups, G = c // 8, 8
    while G * 2 <= 256 and groups % (G * 2) == 0:
        G *= 2
    lanes = 256 // G
    rpb = min(256, rows * (groups // G) // (16 * 132))
    rpb = max(rpb, 4 * lanes)
    return G, lanes, -(-rpb // lanes) * lanes


@functools.lru_cache(maxsize=None)
def _mask(layer, rows, c, p):
    """The kernels' dropout mask of element row * c + channel, fp64 [rows][c] (on the CPU)."""
    return emu.dropout_mask(SEED, layer, rows, c, c, p)


def _lib():
    return _capi.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _scratch(c, dev):
    return (torch.full((96 * c,), float("nan"), dtype=torch.float32, device=dev),
            torch.zeros((c + 31) // 32, dtype=torch.int32, device=dev))


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ---------------------------------------------------------------------------------------------
# stats finalize
# ---------------------------------------------------------------------------------------------
def _slab_rows(dilated, out_rows, tps, N):
    """Row lists of every slab (as the GEMM epilogue defines them) over the flat data matrix."""
    slabs = []
    for n in range(N if dilated else 1):
        tiles = tps if dilated else -(-out_rows // 128)
        for s in range(4 * tiles):
            r0 = min((s // 4) * 128 + (s % 4) * 32, out_rows)   # empty slabs: (end, end)
            r1 = min(r0 + 32, out_rows)
            base = n * out_rows
            slabs.append((base + r0, base + r1))
    return slabs


def _stats_inputs(dev, c, c_real, dilated, out_rows, N, seed, offset_heavy=False):
    g = _gen(dev, seed)
    rows = out_rows * (N if dilated else 1)
    std = torch.rand(c_real, generator=g, device=dev, dtype=torch.float64) * 1.5 + 0.5
    mu = (torch.rand(c_real, generator=g, device=dev, dtype=torch.float64) * 2 - 1) * std
    if offset_heavy:
        mu[:8] = std[:8] * torch.tensor([100, -100, 50, -30, 10, 100, -70, 3], device=dev)
    z = torch.randn(rows, c_real, generator=g, device=dev, dtype=torch.float64) * std + mu
    z[:, c_real // 2] = 0.75           # a constant channel: variance 0
    z = z.to(torch.bfloat16).double()  # the stored activations the GEMM epilogue sums
    tps = -(-out_rows // 128)
    slabs = _slab_rows(dilated, out_rows, tps, N)
    part = torch.full((len(slabs), 2, c), float("nan"), dtype=torch.float64, device=dev)
    cs = torch.cat([torch.zeros(1, c_real, dtype=torch.float64, device=dev), z.cumsum(0)])
    cq = torch.cat([torch.zeros(1, c_real, dtype=torch.float64, device=dev), (z * z).cumsum(0)])
    idx0 = torch.tensor([a for a, _ in slabs], device=dev)
    idx1 = torch.tensor([b for _, b in slabs], device=dev)
    part[:, 0, :c_real] = cs[idx1] - cs[idx0]
    part[:, 1, :c_real] = cq[idx1] - cq[idx0]
    vec = lambda lo, hi: (torch.rand(c, generator=g, device=dev) * (hi - lo) + lo)
    return z, slabs, part.float(), tps, vec(0.5, 1.5), vec(-0.2, 0.2), vec(-0.1, 0.1), vec(0.5, 1.5)


def _stats_ref(z, gamma, beta, rm, rv, c_real, momentum):
    mean = z.mean(0)
    return _stats_ref_moments(mean, ((z - mean) ** 2).mean(0), z.shape[0], gamma, beta, rm, rv,
                              c_real, momentum)


def _stats_ref_moments(mean, var, n, gamma, beta, rm, rv, c_real, momentum):
    """The float64 finalize of a batch of n rows with per-channel mean and (biased) var."""
    inv = 1.0 / torch.sqrt(var + float(torch.tensor(EPS, dtype=torch.float32)))
    sc = gamma[:c_real].double() * inv
    unb = var * n / (n - 1) if n > 1 else var
    return dict(mean=mean, var=var, invstd=inv, scale=sc, shift=beta[:c_real].double() - mean * sc,
                rm=(1 - momentum) * rm[:c_real].double() + momentum * mean,
                rv=(1 - momentum) * rv[:c_real].double() + momentum * unb, n=n)


def _stats_ok(out, ref, k, c_real):
    rms2 = ref["var"] + ref["mean"] ** 2
    tol_m = k * U * rms2.sqrt()
    tol_v = k * U * rms2
    inv = out["invstd"][:c_real].double()
    var = 1.0 / inv ** 2 - float(torch.tensor(EPS, dtype=torch.float32))
    # var recovered from the fp32 invstd carries its rounding: 2 * 2^-24 relative of var + eps
    tol_vr = tol_v + 4 * U * (ref["var"] + EPS)
    dm = (out["mean"][:c_real].double() - ref["mean"]).abs()
    dv = (var - ref["var"]).abs()
    rel_inv = 0.5 * tol_vr / (ref["var"] + EPS) + 2 * U
    sc = out["scale"][:c_real].double()
    m = ref["momentum"]
    n = ref["n"]
    unb = n / (n - 1) if n > 1 else 1.0
    checks = [
        bool((dm <= tol_m).all()),
        bool((dv <= tol_vr).all()),
        bool(((sc - ref["scale"]).abs() <= (rel_inv + 2 * U) * ref["scale"].abs()).all()),
        bool(((out["shift"][:c_real].double() - ref["shift"]).abs() <=
              tol_m * ref["scale"].abs() + ref["mean"].abs() * (rel_inv + 2 * U) * ref["scale"].abs()
              + 4 * U * (ref["shift"].abs() + (ref["mean"] * ref["scale"]).abs())).all()),
        bool(((out["rm"][:c_real].double() - ref["rm"]).abs() <= m * tol_m + 4 * U * (ref["rm"].abs() + 1)).all()),
        bool(((out["rv"][:c_real].double() - ref["rv"]).abs() <= m * unb * tol_vr + 4 * U * ref["rv"].abs()).all()),
    ]
    return all(checks), checks


def _finalize(dev, part, slabs_n, dilated, out_rows, tps, gamma, beta, rm, rv, momentum, c, c_real):
    scratch, counter = _scratch(c, dev)
    outs = []
    for _ in range(2):
        o = {k: torch.full((c,), float("nan"), dtype=torch.float32, device=dev)
             for k in ("scale", "shift", "mean", "invstd")}
        o["rm"], o["rv"] = rm.clone(), rv.clone()
        st = _lib().vp3d_bn_stats_finalize(
            part.data_ptr(), slabs_n, int(dilated), out_rows, tps, gamma.data_ptr(), beta.data_ptr(),
            o["rm"].data_ptr(), o["rv"].data_ptr(), momentum, EPS, o["scale"].data_ptr(),
            o["shift"].data_ptr(), o["mean"].data_ptr(), o["invstd"].data_ptr(), c, c_real,
            scratch.data_ptr(), scratch.numel(), counter.data_ptr(), counter.numel(), _stream())
        torch.cuda.synchronize()
        assert st == 0, _lib().vp3d_last_error()
        assert torch.count_nonzero(counter) == 0, "ticket counters must be reset by the kernel"
        outs.append(o)
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), f"second call differs ({k})"
    return outs[0]


# (c, c_real, dilated, out_rows, N) -> slabs and S = pick_splits(slabs)
STATS_CASES = {
    "flat_c64_one_tile": ((64, 64, False, 90, 1), 4, 1),           # ragged tile, one empty slab
    "flat_c128_c100_S2": ((128, 100, False, 128 * 40 + 33, 1), 164, 2),
    "dilated_c1024_S7": ((1024, 1024, True, 300, 70), 840, 7),       # 3 tiles per sample, empty slabs
    "dilated_c64_S32": ((64, 64, True, 64, 2048), 8192, 32),          # 2 of 4 slabs per tile empty
    "flat_c8192_S5": ((8192, 8192, False, 128 * 150 + 7, 1), 604, 5),
    "flat_c64_far_beyond_cap": ((64, 64, False, 128 * 12000 + 50, 1), 48004, 32),
    "dilated_c128_n_rows1": ((128, 128, True, 1, 3000), 12000, 32),   # one row per sample
    "flat_c64_one_row": ((64, 64, False, 1, 1), 4, 1),                 # n = 1
}


@pytest.mark.parametrize("offset_heavy", [False, True], ids=["centred", "offset100"])
@pytest.mark.parametrize("name", list(STATS_CASES))
def test_bn_stats_finalize_matches_fp64(cuda_device, name, offset_heavy):
    (c, c_real, dilated, out_rows, N), n_slabs, S = STATS_CASES[name]
    dev = cuda_device
    z, slabs, part, tps, gamma, beta, rm, rv = _stats_inputs(dev, c, c_real, dilated, out_rows, N,
                                                             seed=len(name), offset_heavy=offset_heavy)
    assert len(slabs) == n_slabs and _splits(n_slabs) == S
    momentum = float(torch.tensor(0.13, dtype=torch.float32))   # the fp32 value the kernel reads
    o = _finalize(dev, part, n_slabs, dilated, out_rows, tps, gamma, beta, rm, rv, momentum, c, c_real)
    ref = _stats_ref(z, gamma, beta, rm, rv, c_real, momentum)
    ref["momentum"] = momentum
    k = 8 * math.sqrt(n_slabs) + 32
    ok, checks = _stats_ok(o, ref, k, c_real)
    rms2 = ref["var"] + ref["mean"] ** 2
    dm = float(((o["mean"][:c_real].double() - ref["mean"]).abs() / (U * rms2.sqrt())).max())
    print(f"{name} S={S}: mean err {dm:.1f} u rms (gate {k:.0f})")
    assert ok, checks
    for key in ("scale", "shift", "mean", "invstd"):
        assert torch.all(o[key][c_real:] == 0), f"padding channels of {key} must be exactly 0"
    assert torch.equal(o["rm"][c_real:], rm[c_real:]) and torch.equal(o["rv"][c_real:], rv[c_real:])
    cc = c_real // 2   # the constant channel: no variance at all
    assert float(o["mean"][cc]) == 0.75
    if ref["n"] > 1:
        # the gate rejects the statistics of a batch that lost its last 1/8 of the slabs (one split,
        # or one warp's range, dropped by the merge)
        full = [sl for sl in slabs if sl[1] > sl[0]]
        keep = full[: len(full) - max(1, len(full) // 8)]
        rows = torch.cat([torch.arange(a, b, device=dev) for a, b in keep])
        bad = _stats_ref(z[rows], gamma, beta, rm, rv, c_real, momentum)
        bad["momentum"] = momentum
        assert not _stats_ok(o, bad, k, c_real)[0], "gate misses a dropped split"
    # ... and a running variance updated with the biased variance (visible while n is small)
    if 1 < ref["n"] <= 10000:
        bad = dict(ref)
        bad["rv"] = (1 - momentum) * rv[:c_real].double() + momentum * ref["var"]
        assert not _stats_ok(o, bad, k, c_real)[0], "gate misses a biased running variance"


def test_bn_stats_finalize_rejects_too_many_channels(cuda_device):
    c = 8256
    buf = torch.zeros(4 * 2 * c, device=cuda_device)
    scratch, counter = _scratch(c, cuda_device)
    p = buf.data_ptr()
    st = _lib().vp3d_bn_stats_finalize(p, 4, 0, 100, 0, p, p, None, None, 0.1, EPS, p, p, p, p, c, c,
                                       scratch.data_ptr(), scratch.numel(), counter.data_ptr(),
                                       counter.numel(), _stream())
    assert st == -2 and b"8192" in _lib().vp3d_last_error()


# ---------------------------------------------------------------------------------------------
# ordered column sums
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nstat,mul", [(1, False), (2, False), (2, True)])
@pytest.mark.parametrize("n_part,folds,c", [(1, 1, 64), (128, 3, 192), (129, 5, 100),
                                            (256, 7, 1024), (257, 1, 256), (4096, 3, 64),
                                            (4097, 1, 64), (20000, 5, 128)])
def test_ordered_col_sums_matches_fp64(cuda_device, n_part, folds, c, nstat, mul):
    dev = cuda_device
    ld = folds * c + 64
    g = _gen(dev, n_part + folds)
    part = (torch.rand(n_part, nstat, ld, generator=g, device=dev) * 2 - 1)
    part[..., folds * c:] = float("nan")      # columns past the folded blocks are never read
    m1 = torch.rand(c, generator=g, device=dev) + 0.5 if mul else None
    scratch, counter = _scratch(c, dev)
    outs = []
    for _ in range(2):
        o0 = torch.full((c,), float("nan"), device=dev)
        o1 = torch.full((c,), float("nan"), device=dev)
        st = _lib().vp3d_ordered_col_sums(part.data_ptr(), n_part, nstat, ld, c, folds, None,
                                          m1.data_ptr() if mul else None, o0.data_ptr(),
                                          o1.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                          counter.data_ptr(), counter.numel(), _stream())
        torch.cuda.synchronize()
        assert st == 0, _lib().vp3d_last_error()
        assert torch.count_nonzero(counter) == 0
        outs.append((o0, o1))
    same = lambda a, b: torch.equal(a.view(torch.int32), b.view(torch.int32))   # bits, NaN included
    assert same(outs[0][0], outs[1][0]) and same(outs[0][1], outs[1][1])
    pd = part[..., :folds * c].double().reshape(n_part, nstat, folds, c)
    ref = pd.sum((0, 2))
    mag = pd.abs().sum((0, 2))
    k = 32
    print(f"n_part {n_part} (S = {_splits(n_part)}) folds {folds} nstat {nstat}")
    for st_ in range(nstat):
        mulv = m1.double() if (mul and st_ == 1) else 1.0
        got = outs[0][st_].double()
        tol = k * U * mag[st_] * (mulv if mul and st_ == 1 else 1.0) + 2 * U * (ref[st_] * mulv).abs()
        assert bool(((got - ref[st_] * mulv).abs() <= tol).all())
        # the gate rejects the sum with one part missing (a split boundary off by one part)
        if n_part > 1:
            drop = n_part // 2
            bad = (ref[st_] - pd[drop, st_].sum(0)) * mulv
            assert not bool(((got - bad).abs() <= tol).all())
    if nstat == 1:
        assert torch.isnan(outs[0][1]).all(), "out1 untouched with nstat = 1"


# ---------------------------------------------------------------------------------------------
# bn_apply
# ---------------------------------------------------------------------------------------------
def _bf(t, planes):
    hi = t.to(torch.bfloat16)
    if planes == 1:
        return hi.unsqueeze(0).contiguous()
    return torch.stack([hi, (t - hi.double()).to(torch.bfloat16)]).contiguous()


def _val(p):
    return p.double().sum(0)


def _split_exact(p):
    """Two planes (hi, lo): hi is a round-to-nearest bf16 of hi + lo, i.e. |lo| <= half an ulp of hi
    (= when the residual rounded onto the tie)."""
    hi, lo = p[0].double(), p[1].double()
    _, e = torch.frexp(p[0].float())
    half_ulp = torch.ldexp(torch.ones_like(hi), (e - 9).to(torch.int64))
    return bool(torch.where(hi == 0, lo == 0, lo.abs() <= half_ulp).all())


ROWS = [1, 7, 33, 100, 1000, 4099, 20013]


@pytest.mark.parametrize("res_kind", [None, "flat", "div"])
@pytest.mark.parametrize("p", [0.0, 0.25])
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("c", [64, 192, 320, 1024])
def test_bn_apply_matches_fp64(cuda_device, c, planes, p, res_kind):
    dev = cuda_device
    G, lanes, _ = _row_tiling(1000, c)
    assert G == (128 if c == 1024 else 8)
    g = _gen(dev, c + planes)
    sc = torch.rand(c, generator=g, device=dev) + 0.5
    sh = (torch.rand(c, generator=g, device=dev) * 2 - 1) * 0.5
    for rows in ROWS:
        zt = torch.randn(rows, c, generator=g, device=dev, dtype=torch.float64)
        zp = _bf(zt, planes)
        if res_kind == "flat":     # strided residual: row r reads r * step + off
            step, off, div, rps = 3, 1, 0, 0
            res_rows = rows * 3 + 1
        elif res_kind == "div":    # dilated residual: (r / L) * L_prev + (r % L) + off
            div = max(1, rows // 5 if rows >= 5 else rows)
            rps, step, off = div + 6, 1, 3
            res_rows = -(-rows // div) * rps
        else:
            step = off = div = rps = res_rows = 0
        rp = _bf(torch.randn(max(res_rows, 1), c, generator=g, device=dev, dtype=torch.float64),
                 planes) if res_kind else None
        x = torch.full((planes, rows, c), float("nan"), dtype=torch.bfloat16, device=dev)
        st = _lib().vp3d_bn_apply(zp.data_ptr(), rows * c, x.data_ptr(), rows * c, planes, rows, c,
                                  sc.data_ptr(), sh.data_ptr(), p, SEED, LAYER,
                                  rp.data_ptr() if rp is not None else None,
                                  rp[0].numel() if rp is not None else 0, div, rps, step, off,
                                  _stream())
        torch.cuda.synchronize()
        assert st == 0, _lib().vp3d_last_error()
        zv = _val(zp)
        mask = _mask(LAYER, rows, c, p).to(dev) if p > 0 else 1.0
        rmap = (div, rps, step, off)

        def ref_of(mask_, shift_rows=0):
            return _apply_ref(zv, sc, sh, mask_, _val(rp) if rp is not None else None, rmap,
                              shift_rows)
        ref = ref_of(mask)
        got = _val(x)
        tol = _apply_tol(ref, zv, sc, sh, _val(rp) if rp is not None else None, p, planes)
        assert not torch.isnan(got).any()
        assert bool(((got - ref).abs() <= tol).all()), (rows, float((got - ref).abs().max()))
        if planes == 2:
            assert _split_exact(x), "hi is not the bf16 rounding of hi + lo"
        # rejects: the mask of the neighbouring layer, the residual one row off
        if p > 0 and rows >= 100:
            other = _mask(LAYER + 1, rows, c, p).to(dev)
            assert not bool(((got - ref_of(other)).abs() <= tol).all())
        if rp is not None and rows >= 33:
            assert not bool(((got - ref_of(mask, 1)).abs() <= tol).all())


def _apply_ref(zv, sc, sh, mask, res=None, rmap=(0, 0, 1, 0), shift_rows=0):
    """float64 bn_apply: relu(z * scale + shift) * mask [+ res at the RowMap rows (div,
    rows_per_sample, step, off): (r / div) * rows_per_sample + (r % div) * step + off, or
    r * step + off without div; shift_rows reads them that many rows off]."""
    v = torch.relu(zv * sc.double() + sh.double()) * mask
    if res is not None:
        div, rps, step, off = rmap
        r = torch.arange(zv.shape[0], device=zv.device)
        rr = (r // div) * rps + (r % div) * step + off if div else r * step + off
        v = v + res[(rr + shift_rows).clamp(0, res.shape[0] - 1)]
    return v


def _apply_tol(ref, zv, sc, sh, res, p, planes):
    """bn_apply's gate: one rounding to the output planes plus 8 u of the fp32 terms."""
    resmag = res.abs().max() if res is not None else 0.0
    fp32 = 8 * U * ((zv * sc.double()).abs() + sh.double().abs() + resmag) * (1 / (1 - p))
    return (2.0 ** -8 if planes == 1 else 2.0 ** -16) * ref.abs() + fp32


# ---------------------------------------------------------------------------------------------
# backward: reduce + apply
# ---------------------------------------------------------------------------------------------
def _bwd_sums_ref(gv, zv, sc, sh, mean, inv, mask):
    """float64 sums of the BatchNorm backward: dY = G * mask * [z * scale + shift > 0],
    s1 = sum dY, s2 = sum dY (z - mean) * invstd, and their gates 32 u sum|terms| (+ 2 u |s2| for
    the product by invstd).  Returns (dY, s1, s2, tol1, tol2)."""
    live = (zv * sc.double() + sh.double()) > 0
    dy = gv * mask * live
    zc = zv - mean.double()
    s2 = (dy * zc).sum(0) * inv.double()
    k = 32
    return (dy, dy.sum(0), s2, k * U * dy.abs().sum(0),
            k * U * (dy * zc).abs().sum(0) * inv.double() + 2 * U * s2.abs())


def _bwd_apply_ref(dy, zv, sc, mean, inv, sums, n, frozen):
    """float64 dZ of bn_bwd_apply from the kernel's sums over n rows (frozen: scale * dY), and the
    fp32 term of its gate (8 u of the terms of scale dY + B z + D)."""
    scd = sc.double()
    c = scd.shape[0]
    s1, s2 = sums[:c].double(), sums[c:].double()
    if frozen:
        return scd * dy, 8 * U * scd * dy.abs()
    xh = (zv - mean.double()) * inv.double()
    B = (scd * inv.double() * s2 / n).abs()
    fp32 = 8 * U * (scd * dy.abs() + scd * s1.abs() / n + B * (zv.abs() + mean.double().abs()))
    return scd * (dy - s1 / n - xh * s2 / n), fp32


@pytest.mark.parametrize("frozen", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.25])
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("c,c_real,rows", [(64, 64, 4099), (192, 150, 1000), (320, 320, 33),
                                           (1024, 1000, 20013)])
def test_bn_backward_matches_fp64(cuda_device, c, c_real, rows, planes, p, frozen):
    dev = cuda_device
    g = _gen(dev, c + rows)
    sc = torch.rand(c, generator=g, device=dev) + 0.5
    sh = (torch.rand(c, generator=g, device=dev) * 2 - 1) * 0.3
    mean = (torch.rand(c, generator=g, device=dev) * 2 - 1) * 0.2
    inv = torch.rand(c, generator=g, device=dev) + 0.5
    zt = torch.randn(rows, c, generator=g, device=dev, dtype=torch.float64)
    # keep every pre-activation clear of the ReLU kink (fp32 fmaf vs fp64 would disagree there)
    pre = zt * sc.double() + sh.double()
    zt = torch.where(pre.abs() < 1e-3, zt + 3e-3 / sc.double(), zt)
    zp, gp = _bf(zt, planes), _bf(torch.randn(rows, c, generator=g, device=dev, dtype=torch.float64), planes)
    scratch, counter = _scratch(c, dev)
    G, lanes, rpb = _row_tiling(rows, c)
    partials = torch.empty(max(-(-rows // rpb), -(-rows // max(rpb, 32))) * 2 * c + 64, device=dev)
    sums = torch.full((2 * c,), float("nan"), device=dev)
    st = _lib().vp3d_bn_bwd_reduce(gp.data_ptr(), rows * c, zp.data_ptr(), rows * c, planes, rows, c,
                                   sc.data_ptr(), sh.data_ptr(), mean.data_ptr(), inv.data_ptr(), p,
                                   SEED, LAYER, partials.data_ptr(), partials.numel(), sums.data_ptr(),
                                   scratch.data_ptr(), scratch.numel(), counter.data_ptr(),
                                   counter.numel(), _stream())
    torch.cuda.synchronize()
    assert st == 0, _lib().vp3d_last_error()
    assert torch.count_nonzero(counter) == 0
    zv, gv = _val(zp), _val(gp)
    mask = _mask(LAYER, rows, c, p).to(dev) if p > 0 else 1.0
    dy, s1, s2, tol1, tol2 = _bwd_sums_ref(gv, zv, sc, sh, mean, inv, mask)
    live = (zv * sc.double() + sh.double()) > 0
    assert bool(((sums[:c].double() - s1).abs() <= tol1).all())
    assert bool(((sums[c:].double() - s2).abs() <= tol2).all())
    if p > 0:   # rejects the sums of another layer's mask
        other = gv * _mask(LAYER + 1, rows, c, p).to(dev) * live
        assert not bool(((sums[:c].double() - other.sum(0)).abs() <= tol1).all())

    dgamma = torch.full((c,), float("nan"), device=dev)
    dbeta = torch.full((c,), float("nan"), device=dev)
    dz = torch.full((planes, rows, c), float("nan"), dtype=torch.bfloat16, device=dev)
    args = (gp.data_ptr(), rows * c, zp.data_ptr(), rows * c, dz.data_ptr(), rows * c, planes, rows, c,
            sc.data_ptr(), sh.data_ptr(), None if frozen else mean.data_ptr(),
            None if frozen else inv.data_ptr(), p, SEED, LAYER, sums.data_ptr(), dgamma.data_ptr(),
            dbeta.data_ptr(), c_real, int(frozen), _stream())
    st = _lib().vp3d_bn_bwd_apply(*args)
    torch.cuda.synchronize()
    assert st == 0, _lib().vp3d_last_error()
    assert torch.equal(dbeta[:c_real], sums[:c_real]) and torch.equal(dgamma[:c_real], sums[c:c + c_real])
    assert torch.isnan(dgamma[c_real:]).all() and torch.isnan(dbeta[c_real:]).all(), \
        "entries past c_real must stay untouched"

    def ref_dz(n):
        return _bwd_apply_ref(dy, zv, sc, mean, inv, sums, n, frozen)[0]
    ref, fp32 = _bwd_apply_ref(dy, zv, sc, mean, inv, sums, rows, frozen)
    tol = (2.0 ** -8 if planes == 1 else 2.0 ** -16) * ref.abs() + fp32
    got = _val(dz)
    if planes == 2:
        assert _split_exact(dz), "hi is not the bf16 rounding of hi + lo"
    assert not torch.isnan(got).any()
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())
    if not frozen:    # rejects n - 1 in place of n
        assert not bool(((got - ref_dz(rows - 1)).abs() <= tol).all())
    # frozen without sums: no dgamma / dbeta written, the same dz
    if frozen:
        dz2 = torch.full_like(dz, float("nan"))
        dgamma.fill_(float("nan"))
        st = _lib().vp3d_bn_bwd_apply(*(args[:4] + (dz2.data_ptr(),) + args[5:16]
                                        + (None, dgamma.data_ptr(), None) + args[19:]))
        torch.cuda.synchronize()
        assert st == 0 and torch.equal(dz2, dz) and torch.isnan(dgamma).all()
