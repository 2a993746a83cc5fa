"""CPU: the host side of TemporalModel.predict -- the grouping of clips into GEMM chains, the row
tables every chain reads, the argument checks of the C entry points, and the Python validation,
all of which run before any device work."""
import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi
from videopose3d_b200.clips import (DEFAULT_MAX_ROWS, clip_chains, clip_rows, clip_tables)

LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


def _lengths(seed, n, lo=1, hi=400):
    return [int(v) for v in np.random.RandomState(seed).randint(lo, hi, n)]


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("rf,max_rows", [(27, 1), (27, 600), (243, 5000), (243, DEFAULT_MAX_ROWS)])
def test_clip_chains_cover_every_clip_in_order(rf, max_rows, augment):
    lengths = _lengths(rf + max_rows, 300)
    chains = clip_chains(lengths, rf, augment, max_rows)
    # every clip in exactly one chain, chains contiguous and in input order
    assert [i for a, b in chains for i in range(a, b)] == list(range(len(lengths)))
    assert all(b > a for a, b in chains)
    for a, b in chains:
        rows = sum(clip_rows(n, rf, augment) for n in lengths[a:b])
        # a chain exceeds max_rows only when it holds a single clip
        assert rows <= max_rows or b - a == 1
        # a clip's rows include its mirrored copy: both copies always share the chain
        assert rows == sum((2 if augment else 1) * (n + rf - 1) for n in lengths[a:b])
    # greedy: the next clip would not have fitted into the chain before it
    for (a, b), (c, _) in zip(chains, chains[1:]):
        assert sum(clip_rows(n, rf, augment) for n in lengths[a:c + 1]) > max_rows
    assert clip_chains(lengths, rf, augment, max_rows) == chains   # deterministic


def test_clip_chains_small_cases():
    assert clip_chains([1], 3, False, 1) == [(0, 1)]
    assert clip_chains([5, 5, 5], 3, False, 21) == [(0, 3)]         # 3 x 7 rows
    assert clip_chains([5, 5, 5], 3, False, 20) == [(0, 2), (2, 3)]
    assert clip_chains([5, 5, 5], 3, True, 28) == [(0, 2), (2, 3)]  # 14 rows each
    assert clip_chains([100, 1, 1], 3, False, 10) == [(0, 1), (1, 3)]
    assert clip_chains([], 3, False) == []
    with pytest.raises(ValueError):
        clip_chains([3], 3, False, 0)


@pytest.mark.parametrize("augment", [False, True])
def test_row_tables_match_a_brute_force_restatement(augment):
    rf, copies = 27, 2 if augment else 1
    lengths = _lengths(7, 60, hi=90)
    chains, first, rows = clip_tables(lengths, rf, augment, max_rows=700)
    # input / output rows: the clips one after the other
    x_rows, y_rows = [], []
    for i, n in enumerate(lengths):
        x_rows += [(i, f) for f in range(n)]
        y_rows += [(i, t) for t in range(n)]
    for i, n in enumerate(lengths):
        assert x_rows[first[i]] == (i, 0) and x_rows[first[i] + n - 1] == (i, n - 1)
        assert y_rows[first[i]] == (i, 0)
    # packed rows of each chain: every copy edge-padded, (pad + shift) | T | (pad - shift)
    pad = (rf - 1) // 2
    for causal in (False, True):
        shift = pad if causal else 0
        for (a, b), r in zip(chains, rows):
            packed = []
            for i in range(a, b):
                frames = [0] * (pad + shift) + list(range(lengths[i])) + \
                    [lengths[i] - 1] * (pad - shift)
                for copy in range(copies):
                    packed += [(i, copy, f) for f in frames]
            assert len(packed) == r
            # the chain's output row t reads packed rows [t, t + rf): the first T rows of a copy
            # are exactly that clip's padded frames, as the per-clip forward sees them
            row = 0
            for i in range(a, b):
                for copy in range(copies):
                    for t in range(lengths[i]):
                        window = packed[row + t: row + t + rf]
                        assert all(w[:2] == (i, copy) for w in window)
                        assert [w[2] for w in window] == \
                            [min(max(t + k - pad - shift, 0), lengths[i] - 1) for k in range(rf)]
                    row += lengths[i] + rf - 1


def test_clip_entry_points_report_errors_without_gpu():
    """Argument checks of vp3d_forward_clips run before any device work: status codes and
    messages, not crashes."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    kps = (_capi.ctypes.c_int32 * 17)(*range(17))
    ptr = _capi.ctypes.cast(kps, _capi.ctypes.c_void_p)

    def call(plan=None, x=fake, first=fake, length=fake, clips=1, rows=243, flags=0, kps=None,
             joints=None, y=fake, y_first=fake):
        return lib.vp3d_forward_clips(plan, x, first, length, clips, rows, flags, kps, joints, y,
                                      y_first, fake, 1 << 30, None)

    assert lib.vp3d_clips_workspace_bytes(None, 243, 0) == 0
    for kw in (dict(x=None), dict(first=None), dict(length=None), dict(y=None), dict(y_first=None)):
        assert call(**kw) == -1
        assert b"null x, clip table or y" in lib.vp3d_last_error()
    for clips in (0, -3):
        assert call(clips=clips) == -1
        assert b"clips must be >= 1" in lib.vp3d_last_error()
    assert call(kps=ptr) == -1
    assert b"without VP3D_CLIPS_AUGMENT" in lib.vp3d_last_error()
    assert call(flags=_capi.VP3D_CLIPS_AUGMENT) == -1
    assert b"needs kps_src" in lib.vp3d_last_error()
    assert call(flags=4) == -1
    assert b"unknown flags" in lib.vp3d_last_error()
    for rows in (0, -1):
        assert call(rows=rows) == -1
        assert b"positive multiple" in lib.vp3d_last_error()
    assert call(rows=243, flags=_capi.VP3D_CLIPS_AUGMENT, kps=ptr) == -1   # odd with two copies
    assert b"positive multiple of 2" in lib.vp3d_last_error()
    assert call(rows=1 << 31) == -2
    assert b"overflow" in lib.vp3d_last_error()
    assert call() == -1
    assert b"forward_clips: null plan" in lib.vp3d_last_error()


def _model(cls=vp.TemporalModel, **kw):
    m = cls(17, 2, 17, filter_widths=[3, 3, 3], channels=64, **kw)
    return m.eval().set_precision("fp16")


def test_predict_validates_before_any_device_work():
    m = _model()
    x = torch.zeros(30, 17, 2)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            m.predict([x])
        with pytest.raises(ValueError, match=r"\(T >= 1, 17, 2\)"):
            m.predict([torch.zeros(30, 16, 2)])
        with pytest.raises(ValueError, match=r"\(T >= 1, 17, 2\)"):
            m.predict([torch.zeros(30, 17, 3)])
        with pytest.raises(ValueError, match=r"\(T >= 1, 17, 2\)"):
            m.predict([torch.zeros(0, 17, 2)])
        with pytest.raises(TypeError, match="float32"):
            m.predict([torch.zeros(30, 17, 2, dtype=torch.float64)])
        with pytest.raises(ValueError, match="at least one sequence"):
            m.predict([])
        with pytest.raises(ValueError, match="augment=True"):
            m.predict([x], kps_left=LEFT, kps_right=RIGHT)
        with pytest.raises(ValueError, match="joints_left"):
            m.predict([x], augment=True, kps_left=LEFT, kps_right=RIGHT)
        with pytest.raises(RuntimeError, match="eval"):
            _model().train().predict([x])
        with pytest.raises(NotImplementedError, match="mixed"):
            _model().set_precision("mixed").predict([x])
        with pytest.raises(NotImplementedError, match="loads into"):
            _model(vp.TemporalModelOptimized1f).predict([x])


def test_predict_is_inference_only():
    m = _model()
    x = torch.zeros(30, 17, 2)
    # parameters require grad by default: outside no_grad predict refuses instead of detaching
    with pytest.raises(RuntimeError, match="inference-only"):
        m.predict([x.clone()], max_rows=64)
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.predict([x.clone().requires_grad_()])
    # without any tensor that requires grad the checks pass on to the device check
    with pytest.raises(RuntimeError, match="CUDA"):
        m.predict([x])
