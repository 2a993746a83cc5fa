"""GPU: dropout training against fp64 references that replay the kernels' own masks.

The training kernels' dropout masks are a pure function of (seed, layer, element)
(oracle/train_emulation.dropout_mask), and the seed of a step is the first draw from torch's CPU
generator (train_emulation.step_seed).  So a training step with dropout has an exact reference:

* op level: the fused BatchNorm-backward epilogue of the data-gradient conv GEMM (single-plane bf16)
  against fp64 sums of dY = G * mask * [Z*scale + shift > 0] and dY * (Z - mean), in the geometries
  the backward launches;
* model level, bf16x3 (fp32-faithful): y, every gradient and the running statistics against the fp64
  masked step (train_emulation.train_step(planes=0, masks), equal to float64 autograd through
  forward_torch(masks) -- tests/test_dropout_reference_cpu.py);
* model level, bf16 (the default training precision, fused BatchNorm backward): against the
  quantisation-aware emulation with the same masks (planes=1)."""
import pytest
import torch

from conftest import load_golden
from gpu_utils import conv_gemm, expected_conv, pack_weight, planes_value, split_planes
from oracle import temporal_model_oracle as orc
from oracle import train_emulation as emu
from test_gpu_train import _build, _rel
import videopose3d_b200 as vp

pytestmark = pytest.mark.gpu

P = 0.25
SEED = 0x2F3A_1B7C_9D40_5E61    # high word nonzero
LAYER = 3


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _block_n(m_tiles, n_pad):
    """The tile width run_conv picks (api.cu)."""
    return 128 if n_pad % 128 == 0 and m_tiles * (n_pad // 128) * 2 >= _num_sms() else 64


def _rand(shape, seed, dev, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) * (hi - lo) + lo).to(dev)


def _check_fused_bnb(dev, *, samples, a_rows, k_per_tap, taps, n_pad, per_sample_tiles,
                     tap_row_step, out_rows, bnb_c, p, res=None, res_kw=None, res_expect=None,
                     block_n=None):
    """Launch the data-gradient GEMM with the fused BatchNorm-backward epilogue twice and check G,
    the slab sums and run-to-run identity.  res_expect(acc) adds the residual to the fp64 G."""
    total = samples * out_rows if per_sample_tiles else out_rows
    tps = (out_rows + 127) // 128
    m_tiles = samples * tps if per_sample_tiles else tps
    assert m_tiles * n_pad // _block_n(m_tiles, n_pad) > _num_sms()     # persistent CTAs
    assert _block_n(m_tiles, n_pad) == block_n
    a = split_planes(_rand((samples * a_rows, k_per_tap), 41, dev), 1)
    w = _rand((n_pad, k_per_tap, taps), 42, dev) / (taps * k_per_tap) ** 0.5
    wp = pack_weight(w, n_pad, k_per_tap, 1)
    z = _rand((total, n_pad), 43, dev).to(torch.bfloat16)
    scale = _rand((bnb_c,), 44, dev, 0.5, 1.5)
    shift = _rand((bnb_c,), 45, dev, -0.2, 0.2)
    mean = _rand((bnb_c,), 46, dev, -0.1, 0.1)
    invstd = _rand((bnb_c,), 47, dev, 0.5, 2.0)
    slabs = 4 * m_tiles
    kw = dict(per_sample_tiles=per_sample_tiles, tap_row_step=tap_row_step, tap_col_step=0,
              out_rows=out_rows, bnb_z=z, bnb_scale=scale, bnb_shift=shift, bnb_mean=mean,
              bnb_invstd=invstd, bnb_c=bnb_c, bnb_p=p, bnb_seed=SEED, bnb_layer=LAYER,
              **(dict(res=res, **res_kw) if res is not None else {}))
    runs = []
    for _ in range(2):
        sums = torch.full((slabs, 2, n_pad), float("nan"), dtype=torch.float32, device=dev)
        out, _ = conv_gemm(a, samples, a_rows, k_per_tap, wp, taps, k_per_tap, n_pad, bnb_sums=sums,
                           **kw)
        runs.append((out[0], sums))
    (g, sums), (g2, sums2) = runs
    # G: one bf16 rounding of the fp64 product (+ residual); where the residual cancels the product,
    # the fp32 accumulation error (bounded by 2^-20 of sum |a w| over the taps) shows
    geo = dict(samples=samples, a_rows=a_rows, taps=taps, k_per_tap=k_per_tap,
               per_sample_tiles=per_sample_tiles, tap_row_step=tap_row_step, tap_col_step=0,
               out_rows=out_rows)
    av = planes_value(a).reshape(samples * a_rows, k_per_tap)
    exp = expected_conv(av, planes_value(wp), **geo)
    acc_err = expected_conv(av.abs(), planes_value(wp).abs(), **geo) * 2 ** -20
    if res_expect is not None:
        exp = res_expect(exp)
    gd = g.double()
    assert not torch.isnan(gd).any()
    assert torch.all((gd - exp).abs() <= exp.abs() * 2 ** -8 + acc_err)
    # sums: fp64 over the kernel's own stored G (the bf16 value the epilogue reduces)
    assert not torch.isnan(sums).any(), "every slab entry is written"
    ch = torch.arange(n_pad, device=dev) % bnb_c
    zd = z.double()
    # element out_row * n_pad + column == (out_row * n_pad / bnb_c + column / bnb_c) * bnb_c + channel
    mask = emu.dropout_mask(SEED, LAYER, total * n_pad // bnb_c, bnb_c, bnb_c, p).to(dev)
    mask = mask.reshape(total, n_pad)
    live = (zd * scale.double()[ch] + shift.double()[ch]) > 0
    dy = gd * mask * live
    t1, t2 = dy, dy * (zd - mean.double()[ch])

    def per_slab(t):
        # slab s = rows [32 s, 32 s + 32) of row tile s // 4 (per sample for per-sample tiles)
        t = t.reshape(samples if per_sample_tiles else 1, -1, n_pad)
        pad = torch.zeros(t.shape[0], tps * 128 - t.shape[1], n_pad, dtype=t.dtype, device=dev)
        return torch.cat([t, pad], 1).reshape(slabs, 32, n_pad)
    for k, t in enumerate((t1, t2)):
        got, want, mag = sums[:, k].double(), per_slab(t).sum(1), per_slab(t.abs()).sum(1)
        bad = (got - want).abs() > 1e-5 * mag
        assert not bad.any(), (k, int(bad.sum()), float((got - want).abs().max()))
    # slabs that start past the last row of their tile's sample hold exact zeros
    first_row = (torch.arange(slabs, device=dev) % (4 * tps)) * 32
    empty = first_row >= out_rows
    assert empty.any() == (out_rows % 128 <= 96 and out_rows % 128 != 0)
    assert torch.all(sums[empty] == 0)
    assert torch.equal(g, g2) and torch.equal(sums, sums2), "second launch differs"


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("C,rows,block_n", [(192, 128 * 150 + 37, 64), (256, 128 * 80 + 45, 128)])
@pytest.mark.parametrize("k_per_tap", [128, None], ids=["shrink", "conv1x1"])
def test_fused_bnb_flat(cuda_device, k_per_tap, C, rows, block_n, p):
    """Shrink data gradient (K = 128: the padded 3 * joints outputs) and a block's 1x1 conv data
    gradient: flat tiles, no residual, channel = column."""
    _check_fused_bnb(cuda_device, samples=1, a_rows=rows, k_per_tap=k_per_tap or C, taps=1, n_pad=C,
                     per_sample_tiles=False, tap_row_step=0, out_rows=rows, bnb_c=C, p=p,
                     block_n=block_n)


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("C,w,causal,rows,block_n", [(64, 3, False, 128 * 50 + 11, 64),
                                                     (128, 3, True, 128 * 50 + 11, 128),
                                                     (128, 5, False, 128 * 30 + 7, 128),
                                                     (192, 5, True, 128 * 10 + 100, 64)])
def test_fused_bnb_strided_first_conv(cuda_device, C, w, causal, rows, block_n, p):
    """Strided block's first conv, data gradient: G_prev[rows, w*C] = dZ1 W1^T with the skip
    gradient G_i added in the column block of the residual tap, (w/2 + shift) * C; the epilogue folds
    the w column blocks onto the C channels of the layer below (column % C) and hashes element
    row * w*C + column, which is element (row*w + tap) * C + channel of that layer."""
    dev = cuda_device
    col0 = (w // 2 + (w // 2 if causal else 0)) * C
    res = split_planes(_rand((rows, C), 48, dev, -2.0, 2.0), 1)

    def res_expect(acc):
        acc[:, col0:col0 + C] += planes_value(res)
        return acc
    _check_fused_bnb(dev, samples=1, a_rows=rows, k_per_tap=C, taps=1, n_pad=w * C,
                     per_sample_tiles=False, tap_row_step=0, out_rows=rows, bnb_c=C, p=p, res=res,
                     res_kw=dict(res_rows_per_sample=0, res_row_step=1, res_row_off=0,
                                 res_col_begin=col0, res_cols=C),
                     res_expect=res_expect, block_n=block_n)


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("C,N,L,w,d,causal,block_n", [(192, 40, 300, 3, 9, False, 64),
                                                      (256, 40, 200, 5, 3, True, 128)])
def test_fused_bnb_dilated_transposed_conv(cuda_device, C, N, L, w, d, causal, block_n, p):
    """Dilated block's first conv, data gradient: per-sample tiles over the L + 2 pad input frames
    (ragged last tile), tap k reads dZ row t - k*d (zero outside the sample), skip gradient from row
    t - (pad + shift) where that row exists."""
    dev = cuda_device
    pad = (w - 1) * d // 2
    off = pad + ((w // 2) * d if causal else 0)
    L_in = L + 2 * pad
    res = split_planes(_rand((N * L, C), 48, dev, -2.0, 2.0), 1)

    def res_expect(acc):
        r = planes_value(res).reshape(N, L, C)
        acc = acc.reshape(N, L_in, C)
        acc[:, off:off + L] += r
        return acc.reshape(N * L_in, C)
    _check_fused_bnb(dev, samples=N, a_rows=L, k_per_tap=C, taps=w, n_pad=C, per_sample_tiles=True,
                     tap_row_step=-d, out_rows=L_in, bnb_c=C, p=p, res=res,
                     res_kw=dict(res_rows_per_sample=L, res_row_step=1, res_row_off=-off,
                                 res_check_rows=1),
                     res_expect=res_expect, block_n=block_n)


# ---------------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------------
# torch seed per fixture, chosen on a CPU so that the masked fp64 step keeps every pre-activation
# clear of the ReLU kink (min |pre-activation| in brackets; the split-bf16 round-off is ~1e-5)
MODEL_SEEDS = {"opt_333_c128_train": 62,          # 1.14e-4
               "opt_33_c40_train": 198,           # 2.76e-4
               "opt_35_c128_train_causal": 195,   # 2.13e-4
               "tm_333_c128_train": 175}          # 1.32e-4
MIN_MARGIN = 1e-4


def _masked_case(name):
    meta, sd, x, _, new = load_golden(name)
    dilated = meta["cls"] == "TemporalModel"
    seed = MODEL_SEEDS[name]
    masks = emu.model_masks(emu.step_seed(seed), meta["fw"], x.shape[0], x.shape[1], meta["C"], P,
                            dilated=dilated)
    return meta, sd, x, torch.from_numpy(new["gy"]), dilated, seed, masks


def _step(m, x, gy, seed):
    torch.manual_seed(seed)            # the step draws its dropout seed right after this
    y = m(x.to(gy.device))
    (y * gy).sum().backward()
    return y.detach()


@pytest.mark.parametrize("name", list(MODEL_SEEDS))
def test_bf16x3_dropout_step_matches_masked_fp64_reference(cuda_device, name):
    meta, sd, x, gy, dilated, seed, masks = _masked_case(name)
    ref = emu.train_step(sd, x, gy, meta["fw"], causal=meta["causal"], planes=0,
                         momentum=meta["momentum"], dilated=dilated, masks=masks)
    assert ref["min_abs_preact"] >= MIN_MARGIN, "the chosen seed puts a unit on the ReLU kink"
    m = _build(meta, sd, cuda_device, "bf16x3", dropout=P)
    y = _step(m, x, gy.to(cuda_device), seed)
    dist = {"y": _rel(y, ref["y"].numpy())}
    for k, prm in m.named_parameters():
        dist[k] = _rel(prm.grad, ref["grads"][k].numpy())
    sd_new = m.state_dict()
    for k, v in ref["new_stats"].items():
        dist[k] = _rel(sd_new[k], v.numpy())
    worst = max(dist, key=dist.get)
    print(f"{name} bf16x3 p={P}: margin {ref['min_abs_preact']:.2e}, worst {worst} {dist[worst]:.2e}")
    bad = {k: v for k, v in dist.items() if not v <= 1e-3}
    assert not bad, bad


def _big_strided_case():
    arc, C, N, T = [3, 3, 3], 256, 512, 27
    sd = orc.make_state_dict(17, 2, 17, arc, C, seed=61)
    x = orc.make_input(N, T, seed=62)
    gy = torch.randn(N, 1, 17, 3, generator=torch.Generator().manual_seed(63))
    meta = dict(cls="TemporalModelOptimized1f", J=17, F=2, Jout=17, fw=arc, C=C, causal=False,
                dense=False, momentum=0.1)
    return meta, sd, x, gy


@pytest.mark.parametrize("name", list(MODEL_SEEDS) + ["opt_333_c256_n512"])
def test_bf16_dropout_step_matches_masked_emulation(cuda_device, name):
    """Default precision (single-plane bf16: BatchNorm-backward sums fused into the data-gradient
    GEMMs) with the gates of test_bf16_train_step_matches_quantisation_aware_emulation, the dilated
    model included.  opt_333_c256_n512 runs 128-wide tiles and persistent CTAs in the backward."""
    if name in MODEL_SEEDS:
        meta, sd, x, gy, dilated, seed, masks = _masked_case(name)
    else:
        meta, sd, x, gy = _big_strided_case()
        dilated, seed = False, 64
        masks = emu.model_masks(emu.step_seed(seed), meta["fw"], x.shape[0], x.shape[1], meta["C"],
                                P)
    ref = emu.train_step(sd, x, gy, meta["fw"], causal=meta["causal"], planes=1,
                         momentum=meta["momentum"], dilated=dilated, masks=masks)
    m = _build(meta, sd, cuda_device, "bf16", dropout=P)
    y = _step(m, x, gy.to(cuda_device), seed)
    y_dist = emu.rel_max(y, ref["y"])
    l2 = {k: emu.rel_l2(prm.grad, ref["grads"][k]) for k, prm in m.named_parameters()}
    sd_new = m.state_dict()
    st = {k: emu.rel_max(sd_new[k], v) for k, v in ref["new_stats"].items()}
    print(f"{name} bf16 p={P} vs masked emulation: y {y_dist:.2e}, grad rel-L2 worst "
          f"{max(l2.values()):.2e}, running stats worst {max(st.values()):.2e}")
    assert y_dist <= 3e-2
    bad = {k: v for k, v in l2.items() if not v <= 5e-2}
    assert not bad, f"gradient mismatch vs emulation (relative L2): {bad}"
    bad = {k: v for k, v in st.items() if not v <= 1e-2}
    assert not bad, bad
