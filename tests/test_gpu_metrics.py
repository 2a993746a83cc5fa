"""GPU: the evaluation metrics (csrc/pose_loss.cu, videopose3d_b200.metrics) against the
reference's values stored in tests/golden/metrics, against the float64 oracle on a large random
input, bit for bit against the torch flip-average expression of run.py:677-680, run to run, and
end to end: `metrics.evaluate()` against run.py's evaluate() loop, and run.py itself with the
metrics swapped in."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from oracle import metrics_oracle as mo
from oracle import stage_ref
from oracle import temporal_model_oracle as orc
from videopose3d_b200 import metrics
from videopose3d_b200.generators import UnchunkedGenerator

from test_metrics_cpu import NAMES, load_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


def _target(batch_3d, dev):
    t = torch.from_numpy(batch_3d[:1].copy()).to(dev)
    t[:, :, 0] = 0                                         # run.py:688
    return t


@pytest.mark.parametrize("name", NAMES)
def test_metrics_match_reference_fixtures(name, cuda_device):
    meta, case = load_case(name)
    pred = torch.from_numpy(case["pred"]).to(cuda_device)
    if meta["kind"] == "n_mpjpe":
        got = np.array([float(metrics.n_mpjpe(pred, torch.from_numpy(case["batch_3d"]).to(cuda_device)))])
        ref64, ref32 = case["ref64"][1:], case["ref32"][1:]
    else:
        tgt = _target(case["batch_3d"], cuda_device)
        means, avg = metrics.pose_errors(pred, tgt, meta["joints_left"], meta["joints_right"])
        got = means.cpu().numpy()
        ref64, ref32 = case["ref64"], case["ref32"]
        # the single-metric entries agree with the fused call
        J = meta["J"]
        a3, t3 = avg.reshape(-1, J, 3), tgt.reshape(-1, J, 3)
        assert float(metrics.p_mpjpe(a3, t3)) == got[1]
        assert float(metrics.n_mpjpe(avg, tgt)) == got[2]
        assert float(metrics.mean_velocity_error(a3, t3)) == got[3]
    np.testing.assert_allclose(got, ref64, rtol=1e-6, atol=0)
    np.testing.assert_allclose(got, ref32, rtol=1e-5, atol=0)


def test_half_million_random_frames_against_oracle(cuda_device):
    rng = np.random.RandomState(0)
    F, J = 500_000, 17
    t = rng.normal(0, 0.25, (F, J, 3))
    p = t + rng.normal(0, 0.03, t.shape)
    half = F // 2                                         # rotated, scaled, shifted; some mirrored
    q = rng.normal(size=(half, 3, 3))
    r, _ = np.linalg.qr(q)
    r[::4, :, 0] *= -1                                    # improper: the reflection branch
    p[:half] = np.einsum("fja,fab->fjb", p[:half], r) * rng.uniform(0.7, 1.3, (half, 1, 1)) + 0.3
    p32, t32 = p.astype(np.float32), t.astype(np.float32)
    got = metrics.pose_errors(torch.from_numpy(p32[None]).to(cuda_device),
                              torch.from_numpy(t32).to(cuda_device), return_averaged=False)[0]
    want = np.array([mo.mpjpe(p32, t32), mo.p_mpjpe(p32, t32), mo.n_mpjpe(p32, t32),
                     mo.mean_velocity_error(p32, t32)])
    assert (np.linalg.det(r) < 0).any()
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-8, atol=0)


@pytest.mark.parametrize("lists", [(LEFT, RIGHT), None])
def test_flip_average_is_bit_identical_to_torch(lists, cuda_device):
    g = torch.Generator().manual_seed(3)
    pred = (torch.randn(2, 777, 17, 3, generator=g) * 0.4).to(cuda_device)
    want = pred.clone()                                     # run.py:677-680, literally
    want[1, :, :, 0] *= -1
    if lists is not None:
        jl, jr = lists
        want[1, :, jl + jr] = want[1, :, jr + jl]
    want = torch.mean(want, dim=0, keepdim=True)
    left, right = lists if lists is not None else (None, None)
    got = metrics.flip_average(pred, left, right)
    assert torch.equal(got, want)
    _, avg = metrics.pose_errors(pred, torch.zeros(777, 17, 3, device=cuda_device), left, right)
    assert torch.equal(avg, want)


def test_two_calls_give_identical_bits(cuda_device):
    g = torch.Generator().manual_seed(4)
    pred = (torch.randn(2, 20_000, 17, 3, generator=g) * 0.3).to(cuda_device)
    tgt = (torch.randn(20_000, 17, 3, generator=g) * 0.3).to(cuda_device)
    a, avg_a = metrics.pose_errors(pred, tgt, LEFT, RIGHT)
    b, avg_b = metrics.pose_errors(pred, tgt, LEFT, RIGHT)
    assert torch.equal(a, b) and torch.equal(avg_a, avg_b)


def _runpy_evaluate(model, gen, left, right):
    """run.py:652-721 transcribed, with the float64 oracle for the four metrics."""
    acc, n = np.zeros(4), 0
    with torch.no_grad():
        model.eval()
        for _, batch, batch_2d in gen.next_epoch():
            pred = model(batch_2d)
            e, w = mo.sequence_errors(pred.cpu().numpy(), batch.cpu().numpy(),
                                      left if gen.augment_enabled() else None, right)
            acc += w * e
            n += w
    return acc / n * 1000


@pytest.mark.parametrize("augment", [True, False])
def test_evaluate_matches_run_py_loop(augment, cuda_device):
    arc, C = [3, 3, 3], 64
    m = vp.TemporalModel(17, 2, 17, filter_widths=arc, channels=C)
    m.load_state_dict(orc.make_state_dict(17, 2, 17, arc, C, seed=21))
    m = m.to(cuda_device)
    rng = np.random.RandomState(5)
    lens = [90, 301, 47, 160]
    p2 = [rng.uniform(-1, 1, (n, 17, 2)).astype(np.float32) for n in lens]
    p3 = [(rng.normal(0, 0.3, (n, 17, 3)) + [0, 0, 4]).astype(np.float32) for n in lens]
    kw = dict(pad=m.receptive_field() // 2, causal_shift=0, augment=augment, kps_left=LEFT,
              kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT, device=cuda_device)
    want = _runpy_evaluate(m, UnchunkedGenerator(None, p3, p2, **kw), LEFT, RIGHT)
    got = metrics.evaluate(m, UnchunkedGenerator(None, p3, p2, **kw), LEFT, RIGHT)
    print("evaluate()", got, "run.py loop", want)
    np.testing.assert_allclose(np.array(got), want, rtol=1e-5, atol=0)
    first = metrics.evaluate(m, UnchunkedGenerator(None, p3, p2, **kw), LEFT, RIGHT,
                             return_predictions=True)
    assert tuple(first.shape) == (lens[0], 17, 3)


FINAL_RE = {k: re.compile(p + r" ([0-9.eE+-]+) mm") for k, p in {
    "p1": r"Protocol #1 Error \(MPJPE\):", "p2": r"Protocol #2 Error \(P-MPJPE\):",
    "p3": r"Protocol #3 Error \(N-MPJPE\):", "vel": r"Velocity Error \(MPJVE\):"}.items()}


def test_run_py_evaluate_with_metrics_swapped(tmp_path):
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    work = str(tmp_path)
    py = sys.executable
    env = dict(os.environ, OMP_NUM_THREADS="4", NVIDIA_TF32_OVERRIDE="0")
    subprocess.run([py, os.path.join(ROOT, "tools", "make_synthetic_h36m.py"), "--reference", ref,
                    "--out", os.path.join(work, "data"), "--frames", "300", "--subjects", "S1,S9",
                    "--actions", "Walking,Directions 1"], cwd=work, env=env, check=True,
                   capture_output=True, timeout=600)
    os.makedirs(os.path.join(work, "ck"))
    shutil.copy(os.path.join(ROOT, "tests", "golden", "run_py_epoch_1.pt"), os.path.join(work, "ck"))
    args = ["-k", "gt", "-arc", "3,3", "-ch", "4", "-str", "S1", "-ste", "S9", "--evaluate",
            "run_py_epoch_1.pt", "-c", "ck"]
    outs = {}
    for swap in ("model", "model,metrics"):
        r = subprocess.run([py, os.path.join(ROOT, "tools", "run_reference.py"), "--reference", ref,
                            "--swap", swap, "--"] + args, cwd=work, env=env, capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, (swap, r.stdout[-1500:], r.stderr[-3000:])
        outs[swap] = {k: [float(v) for v in rx.findall(r.stdout)] for k, rx in FINAL_RE.items()}
    print(outs)
    base, fused = outs["model"], outs["model,metrics"]
    for k in FINAL_RE:
        assert base[k] and len(base[k]) == len(fused[k]), (k, base, fused)
        np.testing.assert_allclose(fused[k], base[k], rtol=1e-5, atol=0, err_msg=k)
