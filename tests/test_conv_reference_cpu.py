"""CPU: the float64 conv GEMM references of gpu_utils (expected_conv, expected_residual) against
plain Python loops over (sample, row, tap, channel), on tiny shapes: a wrong reference fails here,
not only next to the kernel it is meant to judge."""
import pytest
import torch

from gpu_utils import expected_conv, expected_residual


def _naive_conv(a, w, *, samples, a_rows, taps, k_per_tap, per_sample_tiles, tap_row_step,
                tap_col_step, out_rows):
    n_pad = w.shape[1]
    total = samples * out_rows if per_sample_tiles else out_rows
    out = [[0.0] * n_pad for _ in range(total)]
    for r in range(total):
        s, t = (r // out_rows, r % out_rows) if per_sample_tiles else (0, r)
        for tap in range(taps):
            src = t + tap * tap_row_step
            if per_sample_tiles and not 0 <= src < a_rows:
                continue            # TMA zero-fills the rows outside the sample
            row = s * a_rows + src
            for co in range(n_pad):
                for ci in range(k_per_tap):
                    out[r][co] += float(a[row, tap * tap_col_step + ci]) * float(w[tap, co, ci])
    return torch.tensor(out, dtype=torch.float64)


def _naive_residual(res, n_pad, *, samples, out_rows, per_sample_tiles, res_rows_per_sample=0,
                    res_row_step=1, res_row_off=0, res_sample_div=0, res_check_rows=0,
                    res_col_begin=0, res_cols=0):
    total = samples * out_rows if per_sample_tiles else out_rows
    cols = res_cols or n_pad
    out = [[0.0] * n_pad for _ in range(total)]
    for r in range(total):
        if per_sample_tiles:
            s, t = r // out_rows, r % out_rows
        elif res_sample_div:
            s, t = r // res_sample_div, r % res_sample_div
        else:
            s, t = 0, r
        i = t * res_row_step + res_row_off
        if res_check_rows and not 0 <= i < res_rows_per_sample:
            continue
        for c in range(n_pad):
            if res_col_begin <= c // 64 * 64 < res_col_begin + cols:
                for pl in range(res.shape[0]):
                    out[r][c] += float(res[pl, s * res_rows_per_sample + i, c - res_col_begin])
    return torch.tensor(out, dtype=torch.float64)


CONVS = [  # samples, a_rows, a_ld, taps, k_per_tap, per_sample, tap_row_step, tap_col_step, out_rows
    (1, 5, 6, 3, 2, False, 0, 2, 5),          # flat: taps as column blocks of one row
    (1, 9, 2, 3, 2, False, 3, 0, 3),          # flat: taps as tap-major row regions
    (2, 7, 3, 3, 3, True, 2, 0, 5),           # dilated: the last tap reads past the sample
    (3, 6, 2, 3, 2, True, -2, 0, 6),          # dilated, negative step: reads before the sample
    (2, 4, 2, 2, 2, True, 3, 0, 4),           # a tap that leaves the sample after one row
]


@pytest.mark.parametrize("g", CONVS)
def test_expected_conv_matches_loops(g):
    samples, a_rows, a_ld, taps, k, per_sample, rstep, cstep, out_rows = g
    gen = torch.Generator().manual_seed(sum(g[:5]))
    a = torch.randint(-4, 5, (samples * a_rows, a_ld), generator=gen).double()
    w = torch.randint(-3, 4, (taps, 3, k), generator=gen).double()
    geo = dict(samples=samples, a_rows=a_rows, taps=taps, k_per_tap=k, per_sample_tiles=per_sample,
               tap_row_step=rstep, tap_col_step=cstep, out_rows=out_rows)
    assert torch.equal(expected_conv(a, w, **geo), _naive_conv(a, w, **geo))


RESIDUALS = [  # (samples, out_rows, per_sample, res rows, res_ld, planes, n_pad, map)
    (1, 6, False, 9, 64, 1, 64, dict(res_row_off=3)),
    (1, 4, False, 12, 64, 2, 64, dict(res_row_step=3, res_row_off=2)),
    (1, 8, False, 15, 128, 1, 128, dict(res_rows_per_sample=5, res_row_off=1, res_sample_div=4)),
    (1, 9, False, 12, 64, 1, 64,
     dict(res_rows_per_sample=4, res_row_off=-1, res_sample_div=3, res_check_rows=1)),
    (2, 5, True, 12, 64, 2, 64, dict(res_rows_per_sample=6, res_row_off=2, res_check_rows=1)),
    (2, 3, True, 16, 64, 1, 64, dict(res_rows_per_sample=8, res_row_step=2, res_row_off=1)),
    (1, 3, False, 3, 128, 1, 192, dict(res_col_begin=64, res_cols=128)),
    (1, 3, False, 3, 64, 1, 192, dict(res_col_begin=128, res_cols=64)),
]


@pytest.mark.parametrize("g", RESIDUALS)
def test_expected_residual_matches_loops(g):
    samples, out_rows, per_sample, rows, ld, planes, n_pad, rmap = g
    gen = torch.Generator().manual_seed(rows * ld + n_pad)
    res = torch.randint(-9, 10, (planes, rows, ld), generator=gen).double()
    kw = dict(samples=samples, out_rows=out_rows, per_sample_tiles=per_sample, **rmap)
    got = expected_residual(res, n_pad, **kw)
    exp = _naive_residual(res, n_pad, **kw)
    assert torch.equal(got, exp)
    assert got.abs().sum() > 0
