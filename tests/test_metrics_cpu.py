"""CPU: the evaluation-metric oracle against the reference's values, the fixtures against a fresh
run of the reference, and the CPU-side contract of `vp3d_pose_errors` / `videopose3d_b200.metrics`
(argument checks before any launch, CUDA tensors only)."""
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as mo
from videopose3d_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS_DIR = os.path.join(ROOT, "tests", "golden", "metrics")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(METRICS_DIR, "*.npz")))


def load_case(name):
    z = np.load(os.path.join(METRICS_DIR, name + ".npz"))
    return json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}


def oracle_values(meta, case):
    if meta["kind"] == "n_mpjpe":
        return np.array([mo.mpjpe(case["pred"], case["batch_3d"]),
                         mo.n_mpjpe(case["pred"], case["batch_3d"])])
    e, _ = mo.sequence_errors(case["pred"], case["batch_3d"], meta["joints_left"], meta["joints_right"])
    return e


def test_fixture_set_covers_the_cases():
    assert len(NAMES) >= 6
    metas = {n: load_case(n)[0] for n in NAMES}
    assert {m["J"] for m in metas.values()} >= {15, 17}
    assert any(m["copies"] == 2 and m["joints_left"] for m in metas.values())
    assert any(m["kind"] == "n_mpjpe" for m in metas.values())
    mirrored = [n for n in NAMES if load_case(n)[1]["det_h_negative"] > 0]
    assert mirrored, "no fixture exercises the reflection branch of Procrustes"
    for n in NAMES:
        assert os.path.getsize(os.path.join(METRICS_DIR, n + ".npz")) < 1 << 20


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_values(name):
    meta, case = load_case(name)
    got = oracle_values(meta, case)
    np.testing.assert_allclose(got, case["ref64"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(got, case["ref32"], rtol=1e-5, atol=0)


@pytest.mark.parametrize("name", NAMES)
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_metrics_golden as mk
    finally:
        sys.path.pop(0)
    fresh = mk.make_case(name, ref)
    _, stored = load_case(name)
    assert np.array_equal(fresh["pred"], stored["pred"])
    assert np.array_equal(fresh["batch_3d"], stored["batch_3d"])
    assert int(fresh["det_h_negative"]) == int(stored["det_h_negative"])
    np.testing.assert_allclose(fresh["ref64"], stored["ref64"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(fresh["ref32"], stored["ref32"], rtol=1e-6, atol=0)


def test_pose_errors_reports_errors_without_gpu():
    """Argument checks run before any device work: status codes, not crashes."""
    lib = _capi.load()
    ALL = 15
    assert lib.vp3d_pose_errors_scratch_bytes(0) == 0
    assert lib.vp3d_pose_errors_scratch_bytes(1) >= 32
    assert lib.vp3d_pose_errors_scratch_bytes(10 ** 7) >= lib.vp3d_pose_errors_scratch_bytes(1000)
    # frames == 0: nothing to do, whatever the pointers
    assert lib.vp3d_pose_errors(None, 1, None, None, 0, 17, ALL, None, None, None, 0, None) == 0
    assert lib.vp3d_pose_errors(None, 1, None, None, 5, 33, ALL, None, None, None, 0, None) == -2
    assert b"joints" in lib.vp3d_last_error()
    assert lib.vp3d_pose_errors(None, 1, None, None, 5, 0, ALL, None, None, None, 0, None) == -1
    assert lib.vp3d_pose_errors(None, 3, None, None, 5, 17, ALL, None, None, None, 0, None) == -1
    assert lib.vp3d_pose_errors(None, 1, None, None, -1, 17, ALL, None, None, None, 0, None) == -1
    assert lib.vp3d_pose_errors(None, 1, None, None, 5, 17, 16, None, None, None, 0, None) == -1
    assert b"4-bit mask" in lib.vp3d_last_error()
    assert lib.vp3d_pose_errors(None, 1, None, None, 5, 17, ALL, None, None, None, 0, None) == -1
    assert b"null" in lib.vp3d_last_error()
    fake = 1 << 20   # never dereferenced: the checks fail first
    assert lib.vp3d_pose_errors(fake, 1, None, None, 5, 17, ALL, None, fake, fake, 64, None) == -1
    assert lib.vp3d_pose_errors(fake, 2, None, None, 5, 17, 0, None, None, None, 0, None) == -1
    assert b"nothing to compute" in lib.vp3d_last_error()


def test_metrics_refuse_cpu_tensors():
    from videopose3d_b200 import metrics
    p = torch.randn(2, 10, 17, 3)
    t = torch.randn(10, 17, 3)
    for call in (lambda: metrics.p_mpjpe(t, t.clone()),
                 lambda: metrics.n_mpjpe(p[:1], p[:1].clone()),
                 lambda: metrics.mean_velocity_error(t, t.clone()),
                 lambda: metrics.flip_average(p, [1], [2]),
                 lambda: metrics.pose_errors(p, t, [1], [2])):
        with pytest.raises(RuntimeError, match="CUDA float32"):
            call()
    with pytest.raises(RuntimeError, match="CUDA float32"):
        metrics.p_mpjpe(t.numpy(), t.numpy())
