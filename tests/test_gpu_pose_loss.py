"""GPU: the differentiable pose losses (`vp3d_pose_loss_fwd_bwd`, csrc/pose_loss.cu) against the
reference's values and the float64 oracles: every golden term by term and combined (values within
1e-6 relative, gradients within 1e-5 of max |g|), the forward equal to the float64 evaluation
metrics rounded to fp32, reproducible bits, the degenerate-rotation rule, NaN where the reference
gives NaN, retain_graph, non-contiguous inputs, three training steps of a TemporalModel against a
torch-expression loss, and a velocity prior on the 2-D input of a frozen model."""
import numpy as np
import pytest
import torch

import videopose3d_b200 as vp
from oracle import pose_loss_oracle as po
from test_pose_loss_cpu import NAMES, load_case
from videopose3d_b200 import loss as vloss
from videopose3d_b200 import metrics

pytestmark = pytest.mark.gpu

ONE_TERM = (lambda p, t: vloss.pose_loss(p, t)[0], vloss.n_mpjpe, vloss.p_mpjpe, vloss.mean_velocity_error)


def _grad_close(got, want, tol=1e-5):
    got = got.double().cpu().numpy()
    scale = np.abs(want).max()
    err = np.abs(got - want).max()
    assert err <= tol * scale, (err, scale)


def _value_close(got, want, rtol=1e-6):
    got = np.asarray(got, dtype=np.float64)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=0, equal_nan=True)


def _oracle_term_grad(k, pred, target):
    p = torch.tensor(pred, dtype=torch.float64, requires_grad=True)
    try:
        v = po.TERMS[k](p, torch.tensor(target, dtype=torch.float64))
    except RuntimeError:    # the SVD of a NaN matrix
        return None
    v.backward()
    return p.grad.numpy()


@pytest.mark.parametrize("name", NAMES)
def test_combined_loss_matches_golden(cuda_device, name):
    _, case = load_case(name)
    w = case["weights"]
    p = torch.from_numpy(case["pred"]).to(cuda_device).requires_grad_()
    t = torch.from_numpy(case["target"]).to(cuda_device)
    loss, terms, deg = vloss.pose_loss(p, t, *w, return_degenerate=True)
    loss.backward()
    _value_close(terms.cpu().numpy(), case["terms"])
    _value_close(float(loss.detach()), float(np.dot(w, case["terms"])))
    assert int(deg) == int(case["degenerate"])
    if np.isfinite(case["grad"]).all():
        _grad_close(p.grad, case["grad"])
    else:
        assert not torch.isfinite(p.grad).all()


@pytest.mark.parametrize("k", range(4))
@pytest.mark.parametrize("name", NAMES)
def test_each_term_matches_golden(cuda_device, name, k):
    _, case = load_case(name)
    p = torch.from_numpy(case["pred"]).to(cuda_device).requires_grad_()
    t = torch.from_numpy(case["target"]).to(cuda_device)
    v = ONE_TERM[k](p, t)
    assert v.dim() == 0 and v.dtype == torch.float32 and v.is_cuda and v.requires_grad
    _value_close(float(v), case["terms"][k])
    v.backward()
    want = _oracle_term_grad(k, case["pred"], case["target"])
    if want is None or not np.isfinite(case["terms"][k]) and k != 3:
        assert np.isnan(float(v))
    else:
        assert torch.isfinite(p.grad).all()
        if np.abs(want).max() > 0:
            _grad_close(p.grad, want)
        else:
            assert float(p.grad.abs().max()) == 0.0   # velocity of single frames: no differences


@pytest.mark.parametrize("name", [n for n in NAMES if n.startswith("seq_") or n.startswith("mirrored")
                                  or n.startswith("batch_n4")])
def test_forward_equals_float64_metrics_rounded(cuda_device, name):
    # The loss and the metrics are two instances of one kernel with the same per-pose code, so the
    # fp32 loss term is the fp64 metric rounded once, bit for bit, when both launches use the same
    # grid.  That holds here: every case has at most 972 poses, i.e. at most 122 blocks of 8 poses,
    # below both grid caps on a 132-SM H100 (one loss block or two metric blocks per SM).
    _, case = load_case(name)
    p = torch.from_numpy(case["pred"]).to(cuda_device)
    t = torch.from_numpy(case["target"]).to(cuda_device)
    J = p.shape[-2]
    p3, t3 = p.reshape(-1, J, 3), t.reshape(-1, J, 3)
    pairs = [(vloss.p_mpjpe(p3, t3), metrics.p_mpjpe(p3, t3)),
             (vloss.n_mpjpe(p3[None], t3[None]), metrics.n_mpjpe(p3[None], t3[None]))]
    if p.dim() == 3:
        pairs.append((vloss.mean_velocity_error(p, t), metrics.mean_velocity_error(p, t)))
    for ours, ref in pairs:
        ref32 = np.float32(float(ref))
        if np.isnan(ref32):
            assert np.isnan(float(ours))
            continue
        assert np.float32(float(ours)) == ref32, (float(ours), float(ref))


def test_two_runs_give_identical_bits(cuda_device):
    _, case = load_case("batch_n4_t243_j17")
    t = torch.from_numpy(case["target"]).to(cuda_device)
    out = []
    for _ in range(2):
        p = torch.from_numpy(case["pred"]).to(cuda_device).requires_grad_()
        loss, terms = vloss.pose_loss(p, t, 1.0, 0.5, 0.25, 2.0)
        loss.backward()
        out.append((loss.detach().clone(), terms, p.grad))
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_degenerate_poses_are_counted_and_finite(cuda_device):
    rng = np.random.RandomState(5)
    t = rng.normal(0, 0.3, (6, 17, 3)).astype(np.float32)
    p = (t + rng.normal(0, 0.05, t.shape)).astype(np.float32)
    for f in (1, 4):   # exactly collinear joints along x: H has rank 1, lambda_0 = lambda_1
        p[f] = np.outer(np.linspace(-0.5, 0.5, 17), [1.0, 0.0, 0.0])
    pd = torch.from_numpy(p).to(cuda_device).requires_grad_()
    loss, terms, deg = vloss.pose_loss(pd, torch.from_numpy(t).to(cuda_device), mpjpe=0.0, p_mpjpe=1.0,
                                       return_degenerate=True)
    loss.backward()
    assert int(deg) == 2
    assert torch.isfinite(pd.grad).all() and float(pd.grad.abs().max()) > 0
    _value_close(float(loss), float(po.p_mpjpe(torch.from_numpy(p).double(), torch.from_numpy(t).double())))
    _, _, want_deg = po.p_mpjpe_horn(p, t)
    assert want_deg == 2


def test_nan_where_the_reference_gives_nan(cuda_device):
    z = torch.zeros(2, 5, 17, 3, device=cuda_device)
    t = torch.randn(2, 5, 17, 3, device=cuda_device)
    assert torch.isnan(vloss.n_mpjpe(z, t)) and torch.isnan(vloss.p_mpjpe(z, t))
    assert torch.isnan(vloss.mean_velocity_error(t[:, :1], t[:, :1] * 2))
    assert torch.isnan(vloss.pose_loss(t[:, :1], z[:, :1], velocity=1.0)[0])
    assert torch.isfinite(vloss.pose_loss(t[:, :1], z[:, :1], velocity=0.0)[0])
    assert torch.isnan(vloss.pose_loss(t[:, :0], z[:, :0])[0])   # mean of nothing


def test_retain_graph_gives_the_gradient_again(cuda_device):
    p = torch.randn(3, 9, 17, 3, device=cuda_device, requires_grad=True)
    t = torch.randn(3, 9, 17, 3, device=cuda_device)
    loss, _ = vloss.pose_loss(p, t, 1.0, 1.0, 1.0, 1.0)
    (2.0 * loss).backward(retain_graph=True)
    g1 = p.grad.clone()
    loss.backward()
    torch.testing.assert_close(p.grad, 1.5 * g1, rtol=1e-6, atol=0)
    # no gradient requested: same forward bits
    loss2, _ = vloss.pose_loss(p.detach(), t, 1.0, 1.0, 1.0, 1.0)
    assert torch.equal(loss2, loss.detach())


def test_non_contiguous_input(cuda_device):
    base = torch.randn(17, 40, 3, device=cuda_device)
    tb = torch.randn(17, 40, 3, device=cuda_device)
    p, t = base.transpose(0, 1).requires_grad_(), tb.transpose(0, 1)
    assert not p.is_contiguous()
    loss, terms = vloss.pose_loss(p, t, 1.0, 1.0, 1.0, 1.0)
    loss.backward()
    pc = p.detach().contiguous().requires_grad_()
    loss_c, terms_c = vloss.pose_loss(pc, t.contiguous(), 1.0, 1.0, 1.0, 1.0)
    loss_c.backward()
    assert torch.equal(loss, loss_c) and torch.equal(terms, terms_c) and torch.equal(p.grad, pc.grad)


def _torch_pose_loss(y, t, weights):
    """The torch-expression loss: the oracle's statements in float32 on the device."""
    total = 0.0
    for w, fn in zip(weights, po.TERMS):
        total = total + w * fn(y, t)
    return total


def test_training_steps_match_torch_expression_loss(cuda_device):
    from oracle import temporal_model_oracle as orc
    from videopose3d_b200.optim import FusedAdam
    weights = (1.0, 0.5, 0.5, 1.0)
    arc, C, N, T_out = [3, 3, 3], 128, 8, 9
    sd = orc.make_state_dict(17, 2, 17, arc, C, seed=8)
    x = orc.make_input(N, 27 + T_out - 1, 17, 2, seed=9).to(cuda_device)
    target = torch.from_numpy(np.random.RandomState(10).normal(0, 0.2, (N, T_out, 17, 3))
                              .astype(np.float32)).to(cuda_device)
    runs = []
    for fused in (True, False):
        m = vp.TemporalModel(17, 2, 17, filter_widths=arc, dropout=0.0, channels=C)
        m.load_state_dict(sd)
        m = m.to(cuda_device).set_train_precision("bf16x3").train()
        opt = FusedAdam(m.parameters(), lr=1e-3, amsgrad=True)
        losses, first_grads = [], None
        for _ in range(3):
            opt.zero_grad()
            y = m(x)
            assert y.shape == target.shape
            loss = (vloss.pose_loss(y, target, *weights)[0] if fused
                    else _torch_pose_loss(y, target, weights))
            loss.backward()
            if first_grads is None:
                first_grads = {n: q.grad.detach().cpu().double() for n, q in m.named_parameters()}
            opt.step()
            losses.append(float(loss))
        runs.append((losses, first_grads,
                     {k: v.detach().cpu().double() for k, v in m.state_dict().items()}))
    (l_f, g_f, sd_f), (l_t, g_t, sd_t) = runs
    np.testing.assert_allclose(l_f, l_t, rtol=1e-4)
    # the loss gradient differs by fp32 rounding only: the first step's parameter gradients hold
    # the 1e-3 max-norm gate; after the Adam steps (whose first update is +-lr wherever a gradient
    # is nonzero, so a gradient at round-off level may flip) the parameters hold it in relative L2
    for k, v in g_t.items():
        err = float((g_f[k] - v).abs().max() / v.abs().max().clamp_min(1e-30))
        assert err <= 1e-3, (k, err)
    for k, v in sd_t.items():
        if k.endswith("num_batches_tracked"):
            assert torch.equal(sd_f[k], v)
            continue
        err = float((sd_f[k] - v).norm() / v.norm().clamp_min(1e-30))
        assert err <= 1e-3, (k, err)


def test_velocity_prior_gives_input_gradient_through_frozen_model(cuda_device):
    from oracle import temporal_model_oracle as orc
    m = vp.TemporalModel(17, 2, 17, filter_widths=[3, 3, 3], channels=64)
    m.load_state_dict(orc.make_state_dict(17, 2, 17, [3, 3, 3], 64, seed=12))
    m = m.to(cuda_device).eval()
    for prm in m.parameters():
        prm.requires_grad_(False)
    x = orc.make_input(1, 60, 17, 2, seed=13).to(cuda_device).requires_grad_()
    y = m(x)
    prior = vloss.mean_velocity_error(y, torch.zeros_like(y))
    prior.backward()
    assert torch.isfinite(prior) and float(prior) > 0
    assert x.grad is not None and torch.isfinite(x.grad).all() and float(x.grad.abs().max()) > 0
