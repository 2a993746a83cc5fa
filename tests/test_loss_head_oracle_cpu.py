"""CPU: the float64 oracle of the training loss kernels (oracle/loss_head_oracle.py) against the
reference's own functions (common/loss.py mpjpe / weighted_mpjpe, common/camera.py project_to_2d /
project_to_2d_linear) and a literal transcription of the bone-length term of run.py:383-387,
against gradcheck, and against the committed semi-supervised goldens; plus the host-side checks of
the loss wrappers that need no GPU."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import loss_head_oracle as lo
from videopose3d_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
H36M_PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]


def _reference():
    """(common.loss, common.camera) of the reference, or skip."""
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    import common.camera as camera
    import common.loss as loss
    return loss, camera


def _case(seed, n, f, j, n_lab=None):
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(n, f, j, 3, generator=g, dtype=torch.float64) * 0.3
    traj = torch.randn(n, f, 1, 3, generator=g, dtype=torch.float64) * 0.3
    traj[..., 2] += 4.5
    pos[0, 0, 0, 0] = 9.0                          # beyond the clamp
    n_lab = n // 2 if n_lab is None else n_lab
    in3 = torch.randn(n_lab, f, j, 3, generator=g, dtype=torch.float64) * 0.4
    in3[:, :, 0, 2] = torch.rand(n_lab, f, generator=g, dtype=torch.float64) * 3 + 3
    cam = torch.cat([torch.rand(n - n_lab, 2, generator=g, dtype=torch.float64) + 1.0,
                     torch.randn(n - n_lab, 2, generator=g, dtype=torch.float64) * 0.1,
                     torch.randn(n - n_lab, 3, generator=g, dtype=torch.float64) * 0.1,
                     torch.randn(n - n_lab, 2, generator=g, dtype=torch.float64) * 0.01], dim=1)
    t2 = torch.randn(n - n_lab, f, j, 2, generator=g, dtype=torch.float64) * 0.3
    return pos, traj, in3, cam, t2


def _rel(a, b):
    return float(abs(a - b) / abs(b))


@pytest.mark.parametrize("f,j", [(1, 17), (5, 15), (3, 1)])
def test_oracle_matches_reference_functions(f, j):
    loss, camera = _reference()
    pos, traj, in3, cam, t2 = _case(1 + j, 8, f, j)
    n_lab = in3.shape[0]
    assert _rel(lo.mpjpe(pos[:n_lab], in3), loss.mpjpe(pos[:n_lab], in3)) <= 1e-12
    w = 1 / in3[:, :, :1, 2]
    assert _rel(lo.weighted_mpjpe(traj[:n_lab], in3[:, :, :1], w),
                loss.weighted_mpjpe(traj[:n_lab], in3[:, :, :1], w)) <= 1e-12
    X = pos[n_lab:] + traj[n_lab:]
    for ours, theirs in ((lo.project_to_2d, camera.project_to_2d),
                         (lo.project_to_2d_linear, camera.project_to_2d_linear)):
        a, b = ours(X, cam), theirs(X, cam)
        assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max())
    if j > 1:
        parents = H36M_PARENTS if j == 17 else [-1] + list(range(j - 1))
        # run.py:383-386, literally
        dists = pos[:, :, 1:] - pos[:, :, parents[1:]]
        bone_lengths = torch.mean(torch.norm(dists, dim=3), dim=1)
        penalty = torch.mean(torch.abs(torch.mean(bone_lengths[:n_lab], dim=0)
                                       - torch.mean(bone_lengths[n_lab:], dim=0)))
        assert _rel(lo.bone_length_penalty(pos, n_lab, parents), penalty) <= 1e-12


def test_one_joint_penalty_is_nan_like_the_reference():
    pos = _case(3, 6, 2, 1)[0]
    assert torch.isnan(lo.bone_length_penalty(pos, 3, [-1]))
    dists = pos[:, :, 1:] - pos[:, :, [-1][1:]]                 # run.py:383 with one joint
    assert torch.isnan(torch.mean(torch.abs(torch.mean(torch.mean(torch.norm(dists, dim=3), dim=1)[:3],
                                                       dim=0))))


@pytest.mark.parametrize("linear", [False, True])
def test_oracle_passes_gradcheck(linear):
    pos, traj, in3, cam, t2 = _case(7, 6, 2, 5)
    parents = [-1, 0, 1, 0, 3]
    pos[0, 0, 0, 0] = 0.2                       # keep every point off the clamp's kinks

    def head(p, t):
        total, _ = lo.semi_loss_head(p, t, in3, cam, t2, parents, linear=linear)
        return total
    assert torch.autograd.gradcheck(head, (pos.clone().requires_grad_(), traj.clone().requires_grad_()),
                                    eps=1e-6, atol=1e-7, rtol=1e-5)
    w = torch.rand(6, 2, 1, dtype=torch.float64) + 0.5
    assert torch.autograd.gradcheck(lambda p: lo.weighted_mpjpe(p, pos.detach(), w),
                                    (traj.expand(6, 2, 5, 3).clone().requires_grad_(),))


def _load_semi():
    z = dict(np.load(os.path.join(GOLDEN_DIR, "semi_333_c64.npz")))
    z.update(np.load(os.path.join(GOLDEN_DIR, "semi_333_c64_lin.npz")))
    return json.loads(str(z["meta"])), z


@pytest.mark.parametrize("tag,linear", [("full/", False), ("lin/", True)])
def test_oracle_reproduces_semi_goldens(tag, linear):
    """The goldens were computed in fp32 by the reference: the oracle in float64 on the same fp32
    inputs agrees to fp32 round-off (a few 2^-24 of each value; gradients per tensor's scale)."""
    meta, z = _load_semi()
    pad = meta["pad"]
    d = lambda a: torch.from_numpy(np.asarray(a)).double()  # noqa: E731
    pos = d(z[tag + "pred_pos"]).requires_grad_(True)
    traj = d(z[tag + "pred_traj"]).requires_grad_(True)
    t2 = d(z["inputs_2d_semi"])[:, pad:-pad, :, :2]
    total, terms = lo.semi_loss_head(pos, traj, d(z["inputs_3d"]), d(z["cam_semi"]), t2,
                                     meta["parents"], linear=linear)
    total.backward()
    ref = z[tag + "losses"]
    got = [float(t.detach()) for t in terms] + [float(total.detach())]
    for i in range(5):
        assert abs(got[i] - ref[i]) <= 1e-6 * abs(ref[i]), (i, got, ref)
    for g, name in ((pos.grad, "d_pred_pos"), (traj.grad, "d_pred_traj")):
        r = z[tag + name].astype(np.float64)
        assert np.abs(g.numpy() - r).max() <= 1e-5 * np.abs(r).max(), name


def test_loss_entry_points_report_errors_without_gpu():
    lib = _capi.load()
    for name in ("vp3d_mpjpe_fwd_bwd_ex", "vp3d_mpjpe_scratch_bytes",
                 "vp3d_projected_mpjpe_fwd_bwd_ex", "vp3d_projected_mpjpe_scratch_bytes"):
        assert hasattr(lib, name)
    # one partial per block plus the ticket; a single block needs none; the grid stops at 4096
    assert lib.vp3d_mpjpe_scratch_bytes(0) == 0 and lib.vp3d_mpjpe_scratch_bytes(256) == 0
    assert lib.vp3d_mpjpe_scratch_bytes(257) == 3 * 4
    assert lib.vp3d_mpjpe_scratch_bytes(1024 * 17) == 69 * 4
    assert lib.vp3d_mpjpe_scratch_bytes(10 ** 9) == 4097 * 4
    assert lib.vp3d_projected_mpjpe_scratch_bytes(64, 243) == (61 + 1) * 4
    assert lib.vp3d_projected_mpjpe_scratch_bytes(64, 0) == 0
    assert lib.vp3d_mpjpe_fwd_bwd_ex(None, None, None, 4, 0, None, None, None, 0, None) == -1
    assert lib.vp3d_mpjpe_fwd_bwd_ex(None, None, None, 4, 3, None, None, None, 0, None) == -1
    assert b"null loss" in lib.vp3d_last_error()
    loss = _capi.ctypes.c_float()
    fake = _capi.ctypes.addressof(loss)   # never dereferenced: the call fails before any launch
    assert lib.vp3d_mpjpe_fwd_bwd_ex(fake, fake, None, 1000, 3, fake, None, None, 0, None) == -4
    assert b"scratch too small" in lib.vp3d_last_error()
    assert lib.vp3d_projected_mpjpe_fwd_bwd_ex(fake, fake, fake, fake, 8, 243, 17, 0, fake, None, None,
                                               fake, 4, None) == -4
    assert lib.vp3d_semi_loss_fwd_bwd(None, None, None, None, None, None, 2, 2, 1, 33, 0, 15, fake,
                                      None, None, fake, 1 << 20, None) == -1
    assert b"at most 32 joints" in lib.vp3d_last_error()


def test_semi_loss_refuses_parents_outside_the_pose():
    """Checked on the host before anything reaches the device (before the CUDA-tensor check too)."""
    from videopose3d_b200 import loss as vloss
    p = torch.zeros(4, 1, 5, 3)
    for parents in ([-1, 0, 1, 5, 0], [-1, 0, -1, 2, 0], [-1, 0, 1], [-1, 0, 1, 2, 3, 4]):
        with pytest.raises(ValueError, match="parents"):
            vloss.bone_length_penalty(p, 2, parents)
        with pytest.raises(ValueError, match="parents"):
            vloss.semi_supervised_loss(p, p[:, :, :1], p[:2], torch.zeros(2, 9), p[2:, :, :, :2], parents)
    with pytest.raises(RuntimeError, match="CUDA float32"):          # a valid list gets that far
        vloss.bone_length_penalty(p, 2, [-1, 0, 1, 2, 0])
