"""CPU: the float64 oracles of the differentiable pose losses (oracle/pose_loss_oracle.py) against
the reference's functions and against each other -- the Horn-form reverse-mode derivative of
P-MPJPE against autograd through the SVD and against finite differences -- the golden files, and
the CPU-side contract of `vp3d_pose_loss_fwd_bwd` / `videopose3d_b200.loss` (argument checks before
any launch, CUDA tensors only)."""
import glob
import json
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from oracle import pose_loss_oracle as po
from videopose3d_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden", "pose_loss")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


def load_case(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}


def _maker():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_pose_loss_golden as mk
    finally:
        sys.path.pop(0)
    return mk


def _reference():
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    return _maker()._reference_loss(ref)


def _random_pair(seed, shape, mirrored=False):
    rng = np.random.RandomState(seed)
    t = rng.normal(0, 0.3, shape)
    p = t + rng.normal(0, 0.05, shape)
    if mirrored:
        p[..., 0] *= -1
    return p, t


def _oracle_terms(p, t):
    pt, tt = torch.from_numpy(p), torch.from_numpy(t)
    out = []
    for fn in po.TERMS:
        try:
            out.append(float(fn(pt, tt)))
        except RuntimeError:   # the SVD of a NaN matrix
            out.append(float("nan"))
    return np.array(out)


@pytest.mark.parametrize("seed,shape,mirrored", [(1, (40, 17, 3), False), (2, (25, 15, 3), True),
                                                 (3, (6, 5, 3), False), (4, (30, 32, 3), True)])
def test_oracle_matches_reference_functions(seed, shape, mirrored):
    ref = _reference()
    p, t = _random_pair(seed, shape, mirrored)
    mk = _maker()
    np.testing.assert_allclose(_oracle_terms(p, t), mk.reference_terms(ref, p, t), rtol=1e-12, atol=0)
    # the reference's NumPy functions directly, on the shapes they take
    pt, tt = torch.from_numpy(p), torch.from_numpy(t)
    np.testing.assert_allclose(float(po.p_mpjpe(pt, tt)), ref.p_mpjpe(p.copy(), t.copy()), rtol=1e-12)
    np.testing.assert_allclose(float(po.mean_velocity_error(pt, tt)), ref.mean_velocity_error(p, t),
                               rtol=1e-12)


def test_velocity_runs_along_frames_within_each_sample():
    ref = _reference()
    p, t = _random_pair(5, (3, 20, 17, 3))
    got = float(po.mean_velocity_error(torch.from_numpy(p), torch.from_numpy(t)))
    want = np.mean([ref.mean_velocity_error(a, b) for a, b in zip(p, t)])
    np.testing.assert_allclose(got, want, rtol=1e-12)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        assert np.isnan(ref.mean_velocity_error(p[0, :1], t[0, :1]))
    assert np.isnan(float(po.mean_velocity_error(torch.from_numpy(p[:, :1]), torch.from_numpy(t[:, :1]))))


@pytest.mark.parametrize("seed,shape,mirrored", [(11, (40, 17, 3), False), (12, (25, 15, 3), True),
                                                 (13, (2, 9, 17, 3), False), (14, (7, 3, 3), True)])
def test_horn_reverse_mode_matches_autograd_through_the_svd(seed, shape, mirrored):
    p, t = _random_pair(seed, shape, mirrored)
    pt = torch.tensor(p, requires_grad=True)
    v = po.p_mpjpe(pt, torch.from_numpy(t))
    v.backward()
    value, grad, degenerate = po.p_mpjpe_horn(p, t)
    assert degenerate == 0
    np.testing.assert_allclose(value, float(v.detach()), rtol=1e-12)
    g = pt.grad.numpy()
    assert np.abs(grad - g).max() <= 1e-10 * np.abs(g).max()


class _HornPMpjpe(torch.autograd.Function):
    """The NumPy Horn form as an autograd function: forward value, backward the reverse formula."""
    @staticmethod
    def forward(ctx, p, t):
        v, g, _ = po.p_mpjpe_horn(p.detach().numpy(), t.numpy())
        ctx.g = torch.from_numpy(g)
        return p.new_tensor(v)

    @staticmethod
    def backward(ctx, go):
        return go * ctx.g, None


@pytest.mark.parametrize("mirrored", [False, True])
def test_horn_reverse_mode_passes_gradcheck(mirrored):
    p, t = _random_pair(21 + mirrored, (4, 6, 3), mirrored)
    pt = torch.tensor(p, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x: _HornPMpjpe.apply(x, torch.from_numpy(t)), (pt,),
                                    eps=1e-6, atol=1e-7, rtol=1e-5)
    assert torch.autograd.gradcheck(lambda x: po.p_mpjpe(x, torch.from_numpy(t)), (pt,),
                                    eps=1e-6, atol=1e-7, rtol=1e-5)


def test_n_mpjpe_gradient_keeps_the_scale_derivative():
    """The scale minimises a squared error but the loss is unsquared: freezing s changes the gradient."""
    p, t = _random_pair(31, (5, 17, 3))
    pt = torch.tensor(p, requires_grad=True)
    po.n_mpjpe(pt, torch.from_numpy(t)).backward()
    pf = torch.tensor(p, requires_grad=True)
    tt = torch.from_numpy(t)
    s = ((tt * pf).sum(-1).mean(-1) / (pf * pf).sum(-1).mean(-1)).detach()[..., None, None]
    po.mpjpe(s * pf, tt).backward()
    assert (pt.grad - pf.grad).abs().max() > 1e-3 * pt.grad.abs().max()
    assert torch.autograd.gradcheck(lambda x: po.n_mpjpe(x, tt), (pt.detach().requires_grad_(),))


def test_degenerate_rotation_gets_the_fixed_rotation_gradient():
    """Exactly collinear prediction joints: the top two eigenvalues of N(H) coincide; the pose is
    counted and its gradient (rotation held fixed) is finite."""
    rng = np.random.RandomState(41)
    t = rng.normal(0, 0.3, (3, 17, 3))
    p = t + rng.normal(0, 0.05, t.shape)
    p[1] = np.outer(np.linspace(-0.5, 0.5, 17), [1.0, 0.0, 0.0])
    value, grad, degenerate = po.p_mpjpe_horn(p, t)
    assert degenerate == 1
    assert np.isfinite(value) and np.isfinite(grad).all()
    np.testing.assert_allclose(value, float(po.p_mpjpe(torch.from_numpy(p), torch.from_numpy(t))),
                               rtol=1e-12)


def test_fixture_set_covers_the_cases():
    assert len(NAMES) >= 8
    metas = {n: load_case(n)[0] for n in NAMES}
    shapes = [tuple(m["shape"]) for m in metas.values()]
    assert {s[-2] for s in shapes} >= {1, 15, 17}
    assert any(len(s) == 3 for s in shapes) and any(len(s) == 4 for s in shapes)
    assert (1024, 1, 17, 3) in shapes and (4, 243, 17, 3) in shapes
    kinds = {m["kind"] for m in metas.values()}
    assert {"mirrored", "near_collinear", "zero"} <= kinds
    for n in NAMES:
        meta, case = load_case(n)
        p = case["pred"].astype(np.float64).reshape(-1, meta["shape"][-2], 3)
        t = case["target"].astype(np.float64).reshape(p.shape)
        if meta["kind"] == "mirrored":
            x0, y0 = t - t.mean(1, keepdims=True), p - p.mean(1, keepdims=True)
            assert (np.linalg.det(np.einsum("fja,fjb->fab", x0, y0)) < 0).all()
        if meta["kind"] == "zero":
            assert np.isnan(case["terms"][1]) and np.isnan(case["terms"][2])
        if meta["shape"][-3] == 1:
            assert np.isnan(case["terms"][3])
        assert os.path.getsize(os.path.join(GOLDEN_DIR, n + ".npz")) < 1 << 20


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_golden(name):
    meta, case = load_case(name)
    p, t = case["pred"].astype(np.float64), case["target"].astype(np.float64)
    with np.errstate(all="ignore"):
        np.testing.assert_allclose(_oracle_terms(p, t), case["terms"], rtol=1e-12, atol=0)
        _, _, degenerate = po.p_mpjpe_horn(p, t)
    assert degenerate == int(case["degenerate"])
    g = _maker().oracle_grad(case["pred"], case["target"], tuple(case["weights"]))
    if g is None:
        assert np.isnan(case["grad"]).all()
    else:
        np.testing.assert_allclose(g, case["grad"], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("name", NAMES)
def test_fixtures_regenerate_from_the_reference(name):
    from oracle import stage_ref
    ref = stage_ref.reference_dir()
    if ref is None:
        pytest.skip("no reference checkout and no staged archive (oracle/stage_ref.py)")
    fresh = _maker().make_case(name, ref)
    _, stored = load_case(name)
    assert np.array_equal(fresh["pred"], stored["pred"])
    assert np.array_equal(fresh["target"], stored["target"])
    np.testing.assert_allclose(fresh["terms"], stored["terms"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(fresh["grad"], stored["grad"], rtol=1e-12, atol=1e-14)


def test_pose_loss_entry_points_report_errors_without_gpu():
    ct = _capi.ctypes
    lib = _capi.load()
    for name in ("vp3d_pose_loss_fwd_bwd", "vp3d_pose_loss_scratch_bytes"):
        assert name in _capi.SIGNATURES and hasattr(lib, name)
    assert _capi.SIGNATURES["vp3d_pose_loss_fwd_bwd"][0] is ct.c_int
    assert len(_capi.SIGNATURES["vp3d_pose_loss_fwd_bwd"][1]) == 13
    assert lib.vp3d_pose_loss_scratch_bytes(1, 0) == 0
    assert lib.vp3d_pose_loss_scratch_bytes(1, 1) >= 40
    assert lib.vp3d_pose_loss_scratch_bytes(243, 10 ** 5) >= lib.vp3d_pose_loss_scratch_bytes(1, 1024)
    w = (ct.c_double * 4)(1.0, 0.0, 0.0, 0.0)
    zero = (ct.c_double * 4)()
    call = lambda F, S, J, wt, scratch=None, nbytes=0: lib.vp3d_pose_loss_fwd_bwd(  # noqa: E731
        None, None, F, S, J, wt, None, None, None, None, scratch, nbytes, None)
    assert call(1, 0, 17, w) == 0                     # no poses: nothing to do
    assert call(1, 4, 33, w) == -2
    assert b"joints" in lib.vp3d_last_error()
    assert call(0, 4, 17, w) == -1
    assert call(1, -1, 17, w) == -1
    assert call(1, 4, 0, w) == -1
    assert call(1, 4, 17, None) == -1
    assert call(1, 4, 17, zero) == -1
    assert b"nothing to compute" in lib.vp3d_last_error()
    assert call(1, 4, 17, w) == -1
    assert b"null" in lib.vp3d_last_error()
    assert _capi.VP3D_POSE_LOSS_MPJPE == 1 and _capi.VP3D_POSE_LOSS_VELOCITY == 8


def test_pose_losses_refuse_cpu_tensors():
    from videopose3d_b200 import loss as vloss
    p = torch.randn(2, 10, 17, 3)
    for call in (lambda: vloss.n_mpjpe(p, p.clone()), lambda: vloss.p_mpjpe(p[0], p[0].clone()),
                 lambda: vloss.mean_velocity_error(p[0], p[0].clone()),
                 lambda: vloss.pose_loss(p, p.clone(), velocity=1.0)):
        with pytest.raises(RuntimeError, match="CUDA float32"):
            call()
    with pytest.raises(ValueError, match="every term weight is 0"):
        vloss.pose_loss(p, p.clone(), mpjpe=0.0)
