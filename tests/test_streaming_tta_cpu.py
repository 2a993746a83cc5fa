"""CPU: the host side of augmented (test-time flip) streaming sessions -- argument validation before
any device work, the mirror maps, ring sizes, the C-ABI error paths of the _ex entries, and the
reference-produced fixtures."""
import json
import os
import sys

import numpy as np
import pytest

import videopose3d_b200 as vp
from videopose3d_b200 import _capi, streaming
from videopose3d_b200.generators import mirror_source

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "stream_tta")
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


def _maker():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_stream_tta_golden as mk
    finally:
        sys.path.pop(0)
    return mk


def _cpu_model(jout=17):
    return vp.TemporalModel(17, 2, jout, [3, 3], channels=64).eval()


@pytest.mark.parametrize("kw,match", [
    (dict(), "needs kps_left/kps_right"),
    (dict(kps_left=LEFT), "go together"),
    (dict(kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT), "go together"),
    (dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT), "go together"),
    (dict(kps_left=LEFT, kps_right=[1, 2, 3, 14, 15, 17], joints_left=LEFT, joints_right=RIGHT),
     "out of range"),
    (dict(kps_left=[-1] + LEFT[1:], kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT),
     "out of range"),
    (dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=[1, 2, 3, 14, 15, 99]),
     "out of range"),
    (dict(kps_left=LEFT, kps_right=RIGHT), "num_joints_out"),
])
def test_augment_validation_before_device_work(kw, match):
    """A CPU model would fail the CUDA check; these errors come first."""
    with pytest.raises(ValueError, match=match):
        _cpu_model().streaming(streams=2, augment=True, **kw)


@pytest.mark.parametrize("kw", [dict(kps_left=LEFT, kps_right=RIGHT), dict(joints_left=LEFT),
                                dict(joints_right=RIGHT)])
def test_lists_without_augment_are_an_error(kw):
    with pytest.raises(ValueError, match="only used with augment=True"):
        _cpu_model().streaming(streams=2, **kw)


def test_trajectory_model_needs_no_joint_lists():
    """J_out = 1: the lists validate, then the CPU model fails the device check as without augment."""
    m = _cpu_model(jout=1)
    kps, joints = streaming.augment_maps(m, True, LEFT, RIGHT)
    assert joints is None and np.array_equal(kps, mirror_source(17, LEFT, RIGHT))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.streaming(streams=2, augment=True, kps_left=LEFT, kps_right=RIGHT)
    with pytest.raises(ValueError, match="out of range"):   # a pose model's lists on J_out = 1
        m.streaming(streams=2, augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT,
                    joints_right=RIGHT)


def test_maps_are_the_generators():
    m = vp.TemporalModel(15, 2, 17, [3, 3], channels=64).eval()
    kl, kr = [3, 4, 5], [6, 7, 8]
    kps, joints = streaming.augment_maps(m, True, kl, kr, LEFT, RIGHT)
    assert kps.dtype == np.int32 and joints.dtype == np.int32
    assert np.array_equal(kps, mirror_source(15, kl, kr))
    assert np.array_equal(joints, mirror_source(17, LEFT, RIGHT))
    assert streaming.augment_maps(m, False) == (None, None)


@pytest.mark.parametrize("fw", [[3, 3, 3], [3, 3, 3, 3, 3], [3, 5, 3]])
@pytest.mark.parametrize("max_frames", [1, 7])
def test_augmented_rings_are_twice_the_plain_ones(fw, max_frames):
    m = vp.TemporalModel(17, 2, 17, fw, channels=1024)
    plain = streaming.ring_bytes_per_stream(m, max_frames)
    assert streaming.ring_bytes_per_stream(m, max_frames, augment=True) == 2 * plain
    assert streaming.ring_bytes_per_stream(m, max_frames, planes=2, augment=True) == 4 * plain


def test_stream_ex_entry_points_report_errors_without_gpu():
    """Argument checks of the _ex entries run before any device work: status codes, not crashes."""
    lib = _capi.load()
    fake = 1 << 20   # never dereferenced: the checks fail first
    aug = _capi.VP3D_STREAM_AUGMENT
    kps = mirror_source(17, LEFT, RIGHT)
    kp = kps.ctypes.data
    assert lib.vp3d_stream_state_bytes_ex(None, 4, 1, 0) == 0
    assert lib.vp3d_stream_state_bytes_ex(None, 4, 1, aug) == 0
    assert lib.vp3d_stream_init_ex(None, fake, 1 << 20, 4, 1, 0, None, None, None) == -1
    assert b"null plan" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(fake, None, 1 << 20, 4, 1, 0, None, None, None) == -1
    assert b"null state" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 0, 1, aug, kp, None, None) == -1
    assert b"streams" in lib.vp3d_last_error()
    for flags in (2, 1 << 30, -1):
        assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, flags, kp, None, None) == -1
        assert b"unknown flags" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, aug, None, None, None) == -1
    assert b"needs kps_src" in lib.vp3d_last_error()
    assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, aug, None, kp, None) == -1
    assert b"needs kps_src" in lib.vp3d_last_error()
    for maps in ((kp, None), (None, kp), (kp, kp)):
        assert lib.vp3d_stream_init_ex(fake, fake, 1 << 20, 4, 1, 0, *maps, None) == -1
        assert b"without VP3D_STREAM_AUGMENT" in lib.vp3d_last_error()


def test_fixture_set_covers_the_cases():
    mk = _maker()
    names = sorted(n[:-4] for n in os.listdir(GOLDEN) if n.endswith(".npz"))
    assert names == sorted(mk.CASES)
    assert mk.LEFT == LEFT and mk.RIGHT == RIGHT
    for n in names:
        assert os.path.getsize(os.path.join(GOLDEN, n + ".npz")) < 1 << 20
        z = np.load(os.path.join(GOLDEN, n + ".npz"))
        meta = json.loads(str(z["meta"]))
        assert z["x"].shape == (meta["T"], meta["J"], meta["F"])
        assert z["y"].shape == (meta["T"], meta["Jout"], 3)


@pytest.mark.parametrize("name", ["tta_333_c64", "tta_333_c64_causal", "tta_33_c64_dense",
                                  "tta_353_c128_traj"])
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    fresh = _maker().make_case(name, ref)
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    assert np.array_equal(fresh["x"], z["x"])
    assert np.array_equal(fresh["y"], z["y"])
    assert str(fresh["meta"]) == str(z["meta"])
