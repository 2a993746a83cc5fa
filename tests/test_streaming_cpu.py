"""CPU: the host side of streaming sessions -- frame bookkeeping against brute force, ring sizes,
argument validation, the C-ABI error paths, and the reference-produced fixtures."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from videopose3d_b200 import _capi, streaming
from videopose3d_b200.streaming import FrameBook

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "stream")


def _brute_force(T, lookahead, chunks):
    """Which frame each pushed row carries: output frame t needs input frames up to t + lookahead
    (clipped at T - 1 by the end padding), so it is returned with the row of input frame
    t + lookahead -- the pushes, then the `lookahead` rows of finish()."""
    rows = [-1] * (T + lookahead)
    for t in range(T):
        rows[t + lookahead] = t
    out, i = [], 0
    for k in list(chunks) + [lookahead]:
        out.append(rows[i:i + k])
        i += k
    return out


@pytest.mark.parametrize("lookahead", [0, 1, 4, 13, 121])
@pytest.mark.parametrize("seed", range(4))
def test_frame_book_matches_brute_force(lookahead, seed):
    rng = np.random.RandomState(seed)
    T = int(rng.randint(1, 60))
    chunks, t = [], 0
    while t < T:
        k = int(min(T - t, rng.randint(1, 9)))
        chunks.append(k)
        t += k
    book = FrameBook(2, lookahead)
    got = [book.push(chunks[0], [True, False])] + [book.push(k) for k in chunks[1:]] + [book.finish()]
    want = _brute_force(T, lookahead, chunks)
    for g, w in zip(got, want):
        assert g[0].tolist() == w
        assert (g[1] == -1).all()                 # never started
    seen = np.concatenate([g[0] for g in got])
    assert sorted(seen[seen >= 0].tolist()) == list(range(T))
    assert not book.active.any()                  # finish leaves every slot idle
    assert (book.push(3) == -1).all()


def test_frame_book_mid_stream_start():
    """A slot that starts while others run counts from its own first frame; a restart drops the
    old sequence (its last `lookahead` frames are never returned)."""
    book = FrameBook(3, 2)
    book.push(4, [True, False, False])
    f = book.push(3, [False, True, False])
    assert f[0].tolist() == [2, 3, 4] and f[1].tolist() == [-1, -1, 0] and f[2].tolist() == [-1] * 3
    f = book.push(2, [True, False, True])
    assert f[0].tolist() == [-1, -1] and f[1].tolist() == [1, 2] and f[2].tolist() == [-1, -1]
    f = book.finish()
    assert f[0].tolist() == [0, 1] and f[1].tolist() == [3, 4] and f[2].tolist() == [0, 1]


@pytest.mark.parametrize("fw,dense", [([3, 3, 3], False), ([3, 3, 3, 3, 3], False),
                                      ([3, 5, 3], False), ([3, 3], True), ([1], False)])
def test_ring_sizes(fw, dense):
    m = vp.TemporalModel(17, 2, 17, fw, channels=64, dense=dense)
    hist = streaming.ring_history(fw, dense)
    assert hist == [2 * p for p in m.pad]
    assert sum(hist) == m.receptive_field() - 1
    if fw == [3, 3, 3, 3, 3]:
        assert hist == [2, 6, 18, 54, 162]
        big = vp.TemporalModel(17, 2, 17, fw, channels=1024)
        # C = 1024 fp16: about 240 frames x 1024 x 2 B per stream and copy, mirrored, plus K + 1
        per = streaming.ring_bytes_per_stream(big, max_frames=1)
        assert per == 2 * ((2 + 2) * 64 + sum(h + 2 for h in hist[1:]) * 1024) * 2


def test_lookahead():
    assert streaming.lookahead(vp.TemporalModel(17, 2, 17, [3, 3, 3], causal=True)) == 0
    assert streaming.lookahead(vp.TemporalModel(17, 2, 17, [3, 3, 3])) == 13
    assert streaming.lookahead(vp.TemporalModel(17, 2, 17, [3, 3, 3, 3, 3])) == 121


def test_push_input_validation():
    x = torch.zeros(2, 3, 17, 2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        streaming.check_push_input(x, 2, 4, 17, 2)


def test_sessions_refuse_cpu_models_and_unsupported_configs():
    m = vp.TemporalModel(17, 2, 17, [3, 3], channels=64).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.streaming(streams=2)
    with pytest.raises(RuntimeError, match="eval"):
        m.train().streaming(streams=2)
    m.eval().set_precision("mixed")
    with pytest.raises(NotImplementedError, match="mixed"):
        m.streaming(streams=2)
    opt = vp.TemporalModelOptimized1f(17, 2, 17, [3, 3], channels=64).eval()
    with pytest.raises(NotImplementedError, match="loads into"):
        opt.streaming(streams=2)


def test_stream_entry_points_report_errors_without_gpu():
    """Argument checks run before any device work: status codes, not crashes."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    assert lib.vp3d_stream_state_bytes(None, 4, 1) == 0
    assert lib.vp3d_stream_init(None, fake, 1 << 20, 0, 1, None) == -1          # S < 1
    assert b"streams" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init(None, fake, 1 << 20, 4, 0, None) == -1          # K < 1
    assert lib.vp3d_stream_init(None, None, 1 << 20, 4, 1, None) == -1
    assert lib.vp3d_stream_push(None, None, fake, 1, None, fake, fake, None) == -1
    assert b"null state" in lib.vp3d_last_error()
    assert lib.vp3d_stream_push(None, fake, fake, 0, None, fake, fake, None) == -1
    assert b"k must be" in lib.vp3d_last_error()
    assert lib.vp3d_stream_push(None, fake, fake, 1, None, fake, fake, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert lib.vp3d_stream_finish(None, None, None, None, None) == -1
    assert lib.vp3d_stream_release(None, None) == -1
    assert lib.vp3d_stream_lookahead(None) == -1


def test_fixture_set_covers_the_cases():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_stream_golden as mk
    finally:
        sys.path.pop(0)
    names = sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))
    assert names == sorted(mk.CASES)
    for n in names:
        assert os.path.getsize(os.path.join(GOLDEN, n + ".npz")) < 1 << 20
        z = np.load(os.path.join(GOLDEN, n + ".npz"))
        meta = json.loads(str(z["meta"]))
        assert z["y"].shape == (meta["T"], meta["Jout"], 3)


@pytest.mark.parametrize("name", ["tm_333_c64", "tm_333_c64_causal", "tm_33_c64_dense",
                                  "tm_353_c128_traj"])
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_stream_golden as mk
    finally:
        sys.path.pop(0)
    fresh = mk.make_case(name, ref)
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    assert np.array_equal(fresh["x"], z["x"])
    assert np.array_equal(fresh["y"], z["y"])
    assert str(fresh["meta"]) == str(z["meta"])
