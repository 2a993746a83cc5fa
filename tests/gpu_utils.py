"""Helpers for the GPU tests: build operands for the op-level C-ABI entry (vp3d_conv_gemm) from
plain torch tensors and compute the fp64 expectation of the same fused op."""
import ctypes

import torch

from videopose3d_b200 import _capi


def split_planes(t, planes):
    """fp32 tensor -> bf16 [planes, ...] (hi, lo) exactly as the kernels split values."""
    hi = t.to(torch.bfloat16)
    if planes == 1:
        return hi.unsqueeze(0).contiguous()
    lo = (t - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo]).contiguous()


def planes_value(p):
    """bf16 [planes, ...] -> the fp64 value the kernel operand represents."""
    return p.double().sum(dim=0)


def pack_weight(w, n_pad, k_pad, planes):
    """torch Conv1d weight (Cout, Cin, K) fp32 -> bf16 [planes][K][n_pad][k_pad]."""
    co, ci, k = w.shape
    buf = torch.zeros(k, n_pad, k_pad, dtype=torch.float32, device=w.device)
    buf[:, :co, :ci] = w.permute(2, 0, 1)
    return split_planes(buf, planes)


def conv_gemm(a_planes_t, samples, a_rows, a_ld, w_planes_t, taps, k_per_tap, n_pad, *,
              per_sample_tiles, tap_row_step, tap_col_step, out_rows, precision=0, scale=None,
              shift=None, relu=False, res=None, res_rows_per_sample=0, res_row_step=1, res_row_off=0,
              res_sample_div=0, res_col_begin=0, res_cols=0, res_check_rows=0, out_planes=1,
              out_f32_cols=None, stats=None, bnb_z=None, bnb_scale=None, bnb_shift=None,
              bnb_mean=None, bnb_invstd=None, bnb_sums=None, bnb_c=0, bnb_p=0.0, bnb_seed=0,
              bnb_layer=0, out=None, out_f32=None, out_plane_stride=0, a_plane_stride=0,
              lo_row_begin=0, lo_row_end=0, out_u8=None, out_u8_ld=None, out_u8_inv_scale=None):
    """Launch vp3d_conv_gemm; returns (out_bf16_planes or None, out_f32 or None).
    bnb_*: the fused BatchNorm-backward reductions (see vp3d_conv_desc); bnb_z is a bf16 tensor
    with the output's [rows][n_pad] view, the vectors fp32 [bnb_c], bnb_sums fp32 [slabs][2][n_pad].
    out / out_f32: caller-owned outputs ([planes][rows][ld] 16-bit, or [rows][ld] fp32, ld = the
    row pitch); they are filled with NaN before the launch, like the ones allocated here, so that
    whatever the kernel leaves unwritten (a lo plane outside [lo_row_begin, lo_row_end)) reads NaN.
    out_plane_stride / a_plane_stride: 0 = the planes are contiguous.
    precision VP3D_PRECISION_INT8 (4): A is u8 [1][rows][a_ld] and W s8 [taps][n_pad][k_per_tap].
    out_u8: a caller-owned u8 output [.., rows, out_u8_ld] (default ld: its last dimension) of the
    codes of every stored value times out_u8_inv_scale; u8 has no NaN, so it is left as the caller
    filled it.  With out_u8 and no `out`, the launch writes u8 alone (int8 without a residual)."""
    lib = _capi.load()
    dev = a_planes_t.device
    total_rows = samples * out_rows if per_sample_tiles else out_rows
    d = _capi.ConvDesc()
    d.a = a_planes_t.data_ptr(); d.a_planes = a_planes_t.shape[0]
    d.a_plane_stride = a_plane_stride
    d.lo_row_begin = lo_row_begin; d.lo_row_end = lo_row_end
    d.samples = samples; d.a_rows = a_rows; d.a_ld = a_ld
    d.w = w_planes_t.data_ptr(); d.taps = taps; d.k_per_tap = k_per_tap; d.n_pad = n_pad
    d.per_sample_tiles = int(per_sample_tiles); d.tap_row_step = tap_row_step
    d.tap_col_step = tap_col_step; d.out_rows = out_rows; d.precision = precision
    keep = []
    if scale is not None:
        d.scale = scale.data_ptr(); d.shift = shift.data_ptr()
    d.relu = int(relu)
    if res is not None:
        d.res = res.data_ptr(); d.res_planes = res.shape[0]
        d.res_plane_stride = res[0].numel(); d.res_ld = res.shape[-1]
        d.res_rows_per_sample = res_rows_per_sample; d.res_row_step = res_row_step
        d.res_row_off = res_row_off; d.res_sample_div = res_sample_div
        d.res_col_begin = res_col_begin; d.res_cols = res_cols; d.res_check_rows = res_check_rows
    if bnb_z is not None:
        d.bnb_z = bnb_z.data_ptr()
        d.bnb_scale = bnb_scale.data_ptr(); d.bnb_shift = bnb_shift.data_ptr()
        d.bnb_mean = bnb_mean.data_ptr(); d.bnb_invstd = bnb_invstd.data_ptr()
        d.bnb_sums = bnb_sums.data_ptr(); d.bnb_c = bnb_c; d.bnb_p = bnb_p
        d.bnb_seed = bnb_seed; d.bnb_layer = bnb_layer
    out32 = out_f32
    if out is not None:
        out.fill_(float("nan"))
        d.out = out.data_ptr(); d.out_planes = out.shape[0]
        d.out_plane_stride = out_plane_stride or out[0].numel(); d.out_ld = out.shape[-1]
    elif out32 is not None:
        out32.fill_(float("nan"))
        d.out_f32 = out32.data_ptr(); d.out_f32_ld = out32.shape[-1]
        d.n_valid = out_f32_cols or out32.shape[-1]
    elif out_f32_cols is None and out_u8 is None:
        out = torch.full((out_planes, total_rows, n_pad), float("nan"),
                         dtype=torch.float16 if precision in (3, 4) else torch.bfloat16, device=dev)
        d.out = out.data_ptr(); d.out_planes = out_planes; d.out_plane_stride = out[0].numel()
        d.out_ld = n_pad
    elif out_f32_cols is not None:
        out32 = torch.full((total_rows, out_f32_cols), float("nan"), dtype=torch.float32, device=dev)
        d.out_f32 = out32.data_ptr(); d.out_f32_ld = out_f32_cols; d.n_valid = out_f32_cols
    if out_u8 is not None:
        assert out_u8.dtype == torch.uint8 and out_u8_inv_scale is not None
        d.out_u8 = out_u8.data_ptr(); d.out_u8_ld = out_u8_ld or out_u8.shape[-1]
        d.out_u8_inv_scale = float(out_u8_inv_scale)
    if stats is not None:
        d.stats = stats.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream
    _capi.check(lib.vp3d_conv_gemm(ctypes.byref(d), stream), "vp3d_conv_gemm")
    torch.cuda.synchronize()
    return out, out32


def expected_conv(a_val, w_val, *, samples, a_rows, taps, k_per_tap, per_sample_tiles, tap_row_step,
                  tap_col_step, out_rows):
    """fp64 expectation of the raw accumulator.  a_val: [samples*a_rows, a_ld] fp64,
    w_val: [taps, n_pad, k_per_tap] fp64.  Returns [total_rows, n_pad]."""
    a_ld = a_val.shape[-1]
    a3 = a_val.reshape(samples, a_rows, a_ld)
    n_pad = w_val.shape[1]
    if per_sample_tiles:
        acc = torch.zeros(samples, out_rows, n_pad, dtype=torch.float64, device=a_val.device)
        for tap in range(taps):
            c0 = tap * tap_col_step
            # output row t reads input row t + tap*tap_row_step (either sign); TMA zero-fills the
            # rows outside the sample
            src = torch.arange(out_rows, device=a_val.device) + tap * tap_row_step
            ok = (src >= 0) & (src < a_rows)
            rows = torch.zeros(samples, out_rows, k_per_tap, dtype=torch.float64, device=a_val.device)
            rows[:, ok] = a3[:, src[ok], c0:c0 + k_per_tap]
            acc += rows @ w_val[tap].T
        return acc.reshape(samples * out_rows, n_pad)
    acc = torch.zeros(out_rows, n_pad, dtype=torch.float64, device=a_val.device)
    flat = a3.reshape(samples * a_rows, a_ld)
    for tap in range(taps):
        r0 = tap * tap_row_step
        c0 = tap * tap_col_step
        acc += flat[r0:r0 + out_rows, c0:c0 + k_per_tap] @ w_val[tap].T
    return acc


def expected_residual(res_val, n_pad, *, samples, out_rows, per_sample_tiles, res_rows_per_sample=0,
                      res_row_step=1, res_row_off=0, res_sample_div=0, res_check_rows=0,
                      res_col_begin=0, res_cols=0):
    """fp64 value the epilogue adds to every output element, [total_rows, n_pad] (zero where
    nothing is added).  res_val: [planes, rows, res_ld] fp64, the planes summed.
    Output row t of sample s (flat tiles: s = 0, t = the row; with res_sample_div, s = t // div and
    t = t % div) reads residual row s * res_rows_per_sample + t * res_row_step + res_row_off; with
    res_check_rows a row whose in-sample index t * step + off falls outside [0, res_rows_per_sample)
    adds nothing (a per-sample TMA map zero-fills those rows the same way).  Output column c reads
    residual column c - res_col_begin when its 64-column store block [c0, c0 + 64) starts inside
    [res_col_begin, res_col_begin + res_cols) (res_cols 0: n_pad)."""
    dev = res_val.device
    total = samples * out_rows if per_sample_tiles else out_rows
    r = torch.arange(total, device=dev)
    if per_sample_tiles:
        smp, t = r // out_rows, r % out_rows
    elif res_sample_div > 0:
        smp, t = r // res_sample_div, r % res_sample_div
    else:
        smp, t = torch.zeros_like(r), r
    in_sample = t * res_row_step + res_row_off
    ok = torch.ones_like(r, dtype=torch.bool)
    if res_check_rows:
        ok = (in_sample >= 0) & (in_sample < res_rows_per_sample)
    src = smp * res_rows_per_sample + in_sample
    cols = res_cols if res_cols > 0 else n_pad
    c = torch.arange(n_pad, device=dev)
    cb = c // 64 * 64
    col_ok = (cb >= res_col_begin) & (cb < res_col_begin + cols)
    val = res_val.sum(0)
    out = torch.zeros(total, n_pad, dtype=torch.float64, device=dev)
    rows_ok, cols_ok = torch.nonzero(ok).flatten(), torch.nonzero(col_ok).flatten()
    out[rows_ok[:, None], cols_ok[None, :]] = \
        val[src[rows_ok][:, None], (cols_ok - res_col_begin)[None, :]].double()
    return out
