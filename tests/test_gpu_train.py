"""GPU: training-mode parity of TemporalModelOptimized1f (forward with BatchNorm batch statistics,
running-stat update, backward for every parameter) against goldens produced by the real reference
(forward output, updated running stats, autograd gradients; dropout = 0).

Gates (SURVEY.md §8d G1): bf16x3 (fp32-faithful) mode: max|new - ref| / max|ref| <= 1e-3 on the
output, every parameter gradient and the post-step running statistics.  bf16 mode: <= 5e-2.
Dropout (p > 0) is statistically equal to torch's, not bitwise: checked here through keep-rate /
determinism properties and a directional finite-difference check of the gradients, and in
tests/test_gpu_train_dropout.py against references that replay the kernels' own masks."""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
import videopose3d_b200 as vp

pytestmark = pytest.mark.gpu

TRAIN_CASES = [n for n in golden_names() if n.startswith("opt") and "train" in n]
TM_TRAIN_CASES = [n for n in golden_names() if n.startswith("tm") and "train" in n]


def _build(meta, sd, dev, precision, dropout=0.0):
    kw = dict(filter_widths=meta["fw"], causal=meta["causal"], dropout=dropout, channels=meta["C"])
    if meta["cls"] == "TemporalModel":
        m = vp.TemporalModel(meta["J"], meta["F"], meta["Jout"], dense=meta["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(meta["J"], meta["F"], meta["Jout"], **kw)
    m.load_state_dict(sd)
    m = m.to(dev).train().set_train_precision(precision)
    m.set_bn_momentum(meta.get("momentum", 0.1))
    return m


def _rel(a, b):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else a
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_bf16_train_step_matches_quantisation_aware_emulation(cuda_device, name):
    """bf16 mode: ReLU mask flips make a small-batch comparison with an fp32 reference ill-posed
    (see oracle/train_emulation.py); compare with the emulation that rounds at the same points
    (<= 3e-2 of each tensor's scale: bf16 ties may still round differently) and report the distance
    to the fp32 reference."""
    from oracle import train_emulation as emu
    meta, sd, x, y_ref, new = load_golden(name)
    ref = emu.train_step(sd, x, torch.from_numpy(new["gy"]), meta["fw"], causal=meta["causal"],
                         planes=1, momentum=meta["momentum"])
    m = _build(meta, sd, cuda_device, "bf16")
    y = m(x.to(cuda_device))
    assert emu.rel_max(y, ref["y"]) <= 3e-2
    assert _rel(y, y_ref) <= 5e-2
    (y * torch.from_numpy(new["gy"]).to(cuda_device)).sum().backward()
    worst = {k: emu.rel_l2(prm.grad, ref["grads"][k]) for k, prm in m.named_parameters()}
    worst_max = {k: emu.rel_max(prm.grad, ref["grads"][k]) for k, prm in m.named_parameters()}
    vs_fp32 = max(emu.rel_l2(prm.grad, new["grad/" + k]) for k, prm in m.named_parameters())
    print(f"{name}: grad deviation vs emulation: L2 {max(worst.values()):.2e} max-norm "
          f"{max(worst_max.values()):.2e}; L2 vs fp32 reference {vs_fp32:.2e}")
    bad = {k: v for k, v in worst.items() if not v <= 5e-2}
    assert not bad, f"gradient mismatch vs emulation (relative L2): {bad}"
    sd_new = m.state_dict()
    for k, v in ref["new_stats"].items():
        assert emu.rel_max(sd_new[k], v) <= 1e-2, k


@pytest.mark.parametrize("precision,tol", [("bf16x3", 1e-3)])
@pytest.mark.parametrize("name", TRAIN_CASES + TM_TRAIN_CASES)
def test_train_step_matches_reference(cuda_device, name, precision, tol):
    meta, sd, x, y_ref, new = load_golden(name)
    m = _build(meta, sd, cuda_device, precision)
    y = m(x.to(cuda_device))
    assert y.requires_grad and tuple(y.shape) == y_ref.shape
    assert _rel(y, y_ref) <= tol
    (y * torch.from_numpy(new["gy"]).to(cuda_device)).sum().backward()
    worst = {}
    for k, prm in m.named_parameters():
        assert prm.grad is not None, k
        worst[k] = _rel(prm.grad, new["grad/" + k])
    bad = {k: v for k, v in worst.items() if not v <= tol}
    assert not bad, f"gradient mismatch: {bad}"
    sd_new = m.state_dict()
    for k, v in new.items():
        if k == "gy" or k.startswith("grad/"):
            continue
        if k.endswith("num_batches_tracked"):
            assert int(sd_new[k]) == int(v)
        else:
            assert _rel(sd_new[k], v) <= tol, k


def test_gradients_accumulate_and_eval_sees_new_stats(cuda_device):
    meta, sd, x, y_ref, new = load_golden("opt_333_c128_train")
    m = _build(meta, sd, cuda_device, "bf16x3")
    xg = x.to(cuda_device)
    gy = torch.from_numpy(new["gy"]).to(cuda_device)
    (m(xg) * gy).sum().backward()
    g1 = m.shrink.weight.grad.clone()
    m.load_state_dict(sd)                       # restore running stats, keep .grad
    (m(xg) * gy).sum().backward()               # autograd accumulates into .grad
    assert _rel(m.shrink.weight.grad, (2 * g1).cpu().numpy()) <= 1e-5
    # eval after training must use the updated running statistics
    from oracle import temporal_model_oracle as orc
    m.eval().set_precision("bf16x3")
    with torch.no_grad():
        y_eval = m(xg)
    sd_now = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    y_o = orc.forward_numpy(sd_now, x.numpy(), meta["fw"], causal=meta["causal"], strided=True)
    assert _rel(y_eval, y_o) <= 1e-3


def test_dropout_statistics_and_determinism(cuda_device):
    _dropout_statistics_and_determinism(cuda_device, "bf16x3")


def test_bf16_dropout_statistics_and_determinism(cuda_device):
    """The default precision: BatchNorm-backward sums fused into the data-gradient GEMMs."""
    _dropout_statistics_and_determinism(cuda_device, "bf16")


def _dropout_statistics_and_determinism(cuda_device, precision):
    meta, sd, x, _, new = load_golden("opt_333_c128_train")
    xg = x.to(cuda_device)
    gy = torch.from_numpy(new["gy"]).to(cuda_device)
    m = _build(meta, sd, cuda_device, precision, dropout=0.25)

    def step(seed):
        m.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        y = m(xg)
        (y * gy).sum().backward()
        return y.detach(), {k: prm.grad.clone() for k, prm in m.named_parameters()}
    (y1, g1), (y2, g2), (y3, _) = step(11), step(11), step(12)
    # same torch seed -> same dropout masks, and every reduction (batch statistics, BatchNorm-backward
    # sums, weight-gradient partials) runs in a fixed order: bit-identical output and gradients
    assert torch.equal(y1, y2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    scale = float(y1.abs().max())
    assert float((y1 - y3).abs().max()) >= 1e-2 * scale, "different seed -> different masks"
    m0 = _build(meta, sd, cuda_device, precision, dropout=0.0)
    y0 = m0(xg).detach()
    assert torch.isfinite(y1).all()
    # dropout perturbs but does not bias the activations grossly
    assert float((y1 - y0).abs().mean()) > 1e-3
    assert float(y1.abs().mean()) < 3 * float(y0.abs().mean()) + 1.0


def test_directional_finite_difference_with_dropout(cuda_device):
    """d/de loss(w + e*d) at e = 0 equals <grad, d> with the dropout masks frozen by the seed."""
    meta, sd, x, _, new = load_golden("opt_333_c128_train")
    xg = x.to(cuda_device)
    gy = torch.from_numpy(new["gy"]).to(cuda_device)
    m = _build(meta, sd, cuda_device, "bf16x3", dropout=0.25)

    def loss():
        torch.manual_seed(21)
        return (m(xg) * gy).sum()

    l0 = loss()
    l0.backward()
    g = torch.Generator().manual_seed(3)
    names = ["layers_conv.1.weight", "layers_bn.0.weight", "expand_conv.weight", "shrink.bias",
             "layers_conv.2.weight", "layers_bn.3.bias"]
    prm = dict(m.named_parameters())
    for k in names:
        d = torch.randn(prm[k].shape, generator=g).to(cuda_device)
        d = d / d.norm() * prm[k].detach().norm() * 2e-3
        analytic = float((prm[k].grad * d).sum())
        with torch.no_grad():
            prm[k].add_(d)
            lp = float(loss())
            prm[k].sub_(2 * d)
            lm = float(loss())
            prm[k].add_(d)
        numeric = (lp - lm) / 2
        assert abs(numeric - analytic) <= 0.08 * max(abs(analytic), abs(numeric)) + 1e-3, \
            (k, numeric, analytic)


def test_cfg3_full_size_train_step(cuda_device):
    """BASELINE configs[2] shape: arc 3^5, N = 1024, T = 243, fwd + bwd + AMSGrad step: finite,
    loss decreases over a few steps on a fixed batch."""
    from oracle import temporal_model_oracle as orc
    arc = [3, 3, 3, 3, 3]
    sd = orc.make_state_dict(17, 2, 17, arc, 1024, seed=0)
    m = vp.TemporalModelOptimized1f(17, 2, 17, filter_widths=arc, dropout=0.25, channels=1024)
    m.load_state_dict(sd)
    m = m.to(cuda_device).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)
    x = orc.make_input(1024, 243, seed=5).to(cuda_device)
    tgt = torch.randn(1024, 1, 17, 3, generator=torch.Generator().manual_seed(6)).to(cuda_device) * 0.3
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = orc.mpjpe(m(x), tgt)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < losses[0], losses


@pytest.mark.parametrize("name", TM_TRAIN_CASES)
def test_dilated_train_bf16_runs_and_is_close(cuda_device, name):
    """TemporalModel (dilated) training in bf16 mode: forward within 5e-2 of the fp32 reference,
    gradients finite and within 35 % (relative L2; ReLU-mask flips on a tiny batch, see
    oracle/train_emulation.py) — the tight check is the bf16x3 case above."""
    from oracle import train_emulation as emu
    meta, sd, x, y_ref, new = load_golden(name)
    m = _build(meta, sd, cuda_device, "bf16")
    y = m(x.to(cuda_device))
    assert _rel(y, y_ref) <= 5e-2
    (y * torch.from_numpy(new["gy"]).to(cuda_device)).sum().backward()
    for k, prm in m.named_parameters():
        assert torch.isfinite(prm.grad).all(), k
        assert emu.rel_l2(prm.grad, new["grad/" + k]) <= 0.35, k


def test_training_loss_curve_tracks_fp32_reference(cuda_device):
    """SURVEY §8d gate G3 (dropout on): the training-loss curve over 300 optimiser steps stays
    within the noise of the reference's.

    Student/teacher regression on synthetic keypoints (arc 3,3,3, C = 128, batch 256, dropout 0.25,
    AMSGrad lr 1e-3, the same batch sequence in every run).  The reference is the oracle's
    torch.nn.functional network trained in fp32 (TF32 off) -- run twice with different dropout
    streams to measure its own run-to-run noise -- against this repo's default bf16 training
    path.  Compared on 50-step window means from step 50 on:
        |ours - mean(ref_a, ref_b)| <= 3 * |ref_a - ref_b| + 8 % of the reference loss.
    """
    from oracle import temporal_model_oracle as orc
    arc, C, N, T, steps, p = [3, 3, 3], 128, 256, 27, 300, 0.25
    dev = cuda_device
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        teacher = {k: v.to(dev) for k, v in orc.make_state_dict(17, 2, 17, arc, C, seed=11).items()}
        x_pool = orc.make_input(4096, T, 17, 2, seed=12).to(dev)
        with torch.no_grad():
            y_pool = orc.forward_torch(teacher, x_pool, arc, strided=True)
        sd0 = orc.make_state_dict(17, 2, 17, arc, C, seed=13)

        def batches():
            g = torch.Generator().manual_seed(99)
            for _ in range(steps):
                idx = torch.randint(0, x_pool.shape[0], (N,), generator=g).to(dev)
                yield x_pool[idx], y_pool[idx]

        def run_reference(seed):
            sd = {k: v.clone().to(dev) for k, v in sd0.items()}
            leaves = [v.requires_grad_(True) for k, v in sd.items()
                      if v.is_floating_point() and "running_" not in k]
            opt = torch.optim.Adam(leaves, lr=1e-3, amsgrad=True)
            torch.manual_seed(seed)
            curve = []
            for xb, yb in batches():
                opt.zero_grad()
                out = orc.forward_torch(sd, xb, arc, strided=True, training=True, momentum=0.1,
                                        update_stats=True, dropout=p)
                loss = torch.mean(torch.norm(out - yb, dim=-1))
                loss.backward()
                opt.step()
                curve.append(loss.item())
            return np.array(curve)

        def run_ours(seed):
            m = vp.TemporalModelOptimized1f(17, 2, 17, filter_widths=arc, dropout=p, channels=C)
            m.load_state_dict(sd0)
            m = m.to(dev).train()
            opt = torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)
            torch.manual_seed(seed)
            curve = []
            for xb, yb in batches():
                opt.zero_grad()
                loss = torch.mean(torch.norm(m(xb) - yb, dim=-1))
                loss.backward()
                opt.step()
                curve.append(loss.item())
            return np.array(curve)

        ref_a, ref_b, ours = run_reference(1), run_reference(2), run_ours(3)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32

    def windows(c):
        return c.reshape(-1, 50).mean(axis=1)
    wa, wb, wo = windows(ref_a), windows(ref_b), windows(ours)
    centre, noise = 0.5 * (wa + wb), np.abs(wa - wb)
    print("ref_a ", np.round(wa, 4), "\nref_b ", np.round(wb, 4), "\nours  ", np.round(wo, 4))
    assert np.isfinite(ours).all()
    assert wo[-1] < 0.6 * wo[0] and centre[-1] < 0.6 * centre[0]      # both learn
    for w in range(1, len(wo)):
        assert abs(wo[w] - centre[w]) <= 3 * noise[w] + 0.08 * centre[w], (w, wo[w], centre[w], noise[w])


# ---------------------------------------------------------------------------------------------
# BASELINE configs[2] shape (arc 3,3,3,3,3, C = 1024) against the real reference: fixture
# tests/golden/big_opt_33333_c1024_train.npz (tests/golden/make_semi_golden.py) -- output, running
# statistics and every parameter gradient (conv-weight gradients as a 4096-entry strided sample
# plus L2 norm and sum) at the full cfg3 batch N = 1024.  SURVEY §8d gate G1: <= 1e-3 in the
# fp32-faithful mode.
# ---------------------------------------------------------------------------------------------
def _load_big():
    import json
    import os
    from conftest import GOLDEN_DIR
    from oracle import temporal_model_oracle as orc
    z = np.load(os.path.join(GOLDEN_DIR, "big_opt_33333_c1024_train.npz"))
    meta = json.loads(str(z["meta"]))
    sd = orc.make_state_dict(meta["J"], meta["F"], meta["Jout"], meta["fw"], meta["C"], seed=meta["seed"])
    check = np.array([float(v.double().sum()) for k, v in sorted(sd.items())])
    assert np.allclose(check, z["sd_check"], rtol=0, atol=1e-9), "seeded parameters differ from the fixture's"
    x = orc.make_input(meta["N"], meta["T"], meta["J"], meta["F"], seed=meta["seed"] + 1)
    return meta, sd, x, z


def test_cfg3_shape_train_step_matches_reference(cuda_device):
    """fp32-faithful kernels against the real reference at the cfg3 shape.

    The forward output and the running statistics hold the 1e-3 gate in the max norm.  For the
    gradients a max-norm gate is ill-posed at this size: of the ~170 M pre-activations a few
    hundred lie within the split-bf16 round-off (~1e-5 of their scale) of the ReLU kink and are
    rounded to the other side than the fp32 reference rounds them; ONE flipped unit in the top
    blocks moves individual gradient entries of that layer by ~1/rows and, through the backward
    pass, every entry below it a little (the small goldens avoid this by choosing seeds without
    near-kink units, impossible here; the fp32 reference against its own float64 run, whose
    round-off is 100x smaller, shows no flip: 1e-6).  The worst tensor is expand_bn, which
    collects every flip above it.  The gates sit well above the spread such flips cause: a wrong kernel (a mis-indexed tap, a missing term, a wrong
    reduction) moves every entry by O(1), not by 1e-3."""
    meta, sd, x, z = _load_big()
    m = _build(meta, sd, cuda_device, "bf16x3")
    y = m(x.to(cuda_device))
    assert _rel(y, z["y"]) <= 1e-3
    (y * torch.from_numpy(z["gy"]).to(cuda_device)).sum().backward()
    med, l2, mx, fn = {}, {}, {}, {}
    for k, prm in m.named_parameters():
        g = prm.grad.reshape(-1)
        idx = torch.from_numpy(z["gidx/" + k]).to(cuda_device)
        ref = z["gval/" + k].astype(np.float64)
        norm, total, gmax = z["gnorm/" + k]
        err = np.abs(g[idx].cpu().numpy().astype(np.float64) - ref)
        med[k] = float(np.median(err) / gmax)
        mx[k] = float(err.max() / gmax)
        l2[k] = float(np.linalg.norm(err) / max(np.linalg.norm(ref), 1e-30))
        n_err = abs(float(g.double().norm()) - norm) / norm
        s_err = abs(float(g.double().sum()) - total) / (norm * np.sqrt(g.numel()))
        fn[k] = max(n_err, s_err)
    print(f"cfg3-shape gradients vs reference: median entry error {max(med.values()):.2e}, rel-L2 "
          f"{max(l2.values()):.2e}, norm/sum functionals {max(fn.values()):.2e}, max entry error "
          f"{max(mx.values()):.2e} (kink flips)")
    assert max(med.values()) <= 3e-3, med
    assert max(l2.values()) <= 2e-2, l2
    assert max(fn.values()) <= 2e-3, fn
    sd_new = m.state_dict()
    for k in z.files:
        if not k.startswith("new/"):
            continue
        if k.endswith("num_batches_tracked"):
            assert int(sd_new[k[4:]]) == int(z[k])
        else:
            assert _rel(sd_new[k[4:]], z[k]) <= 1e-3, k


def test_cfg3_shape_default_bf16_training_is_close_and_reproducible(cuda_device):
    """Default training kernels (bf16 operands) on the cfg3-shape fixture: output within 2e-2 of the
    reference; gradients within bf16's reach (<= 0.2 relative L2 on the stored samples); and two
    identical steps give IDENTICAL gradients: batch
    statistics, BatchNorm-backward sums and weight-gradient partials are all reduced in a fixed
    order (no floating-point atomics)."""
    meta, sd, x, z = _load_big()
    gy = torch.from_numpy(z["gy"]).to(cuda_device)
    grads = []
    for rep in range(2):
        m = _build(meta, sd, cuda_device, "bf16")
        y = m(x.to(cuda_device))
        if rep == 0:
            assert _rel(y, z["y"]) <= 2e-2
        (y * gy).sum().backward()
        grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
    worst = {}
    for k, g in grads[0].items():
        idx = torch.from_numpy(z["gidx/" + k]).to(cuda_device)
        ref = z["gval/" + k].astype(np.float64)
        got = g.reshape(-1)[idx].cpu().numpy().astype(np.float64)
        worst[k] = float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))
    print(f"cfg3-shape bf16 gradients vs fp32 reference (sample rel-L2): worst {max(worst.values()):.2e}")
    assert max(worst.values()) <= 0.2, worst
    noise = max(float((grads[0][k] - grads[1][k]).norm() / grads[0][k].norm().clamp_min(1e-30)) for k in grads[0])
    print(f"run-to-run gradient difference: {noise:.2e}")
    assert noise <= 1e-6      # (was 8e-2 with atomically accumulated batch statistics)


def test_dropout_keep_rate_scale_and_mask_consistency(cuda_device):
    _dropout_keep_rate_scale_and_mask(cuda_device, "bf16x3", "TemporalModel", 64)


@pytest.mark.parametrize("precision,cls,C", [
    (pr, cl, c) for pr in ("bf16x3", "bf16") for cl in ("TemporalModel", "TemporalModelOptimized1f")
    for c in (64, 100) if (pr, cl, c) != ("bf16x3", "TemporalModel", 64)])
def test_dropout_keep_rate_and_mask_across_precisions_models_and_padding(cuda_device, precision, cls, C):
    """The same checks in the default bf16 precision (layer 0's BatchNorm-backward sums come from the
    shrink GEMM's fused epilogue), for the strided model, and with C = 100 on 128 padded channels."""
    _dropout_keep_rate_scale_and_mask(cuda_device, precision, cls, C)


def _dropout_keep_rate_scale_and_mask(cuda_device, precision, cls, C):
    """SURVEY §8d gate G3 on the kernels' own output.  arc [3] (no residual block) with a shrink
    layer that copies the first 51 channels makes the dropout output observable:
    y[..., c] = drop(relu(bn(expand(x))))[..., c].  Against the same step with p = 0: every value is
    either dropped (0) or scaled by exactly 1/(1-p) = 4/3; the units dropped are exactly those the
    mask of oracle/train_emulation.dropout_mask drops (C = 100 runs on 128 padded channels); the kept
    fraction is 0.75 +- 3 sigma; and the backward uses the same mask (d sum(y) / d beta_c = 4/3 x
    #kept positive rows -- in bf16 through the BatchNorm-backward sums fused into the shrink's
    data-gradient GEMM)."""
    J, N, T, p = 17, 64, 50, 0.25
    from oracle import temporal_model_oracle as orc
    from oracle import train_emulation as emu
    sd = orc.make_state_dict(J, 2, J, [3], C, seed=77)
    sd["shrink.weight"] = torch.zeros(51, C, 1)
    sd["shrink.weight"][torch.arange(51), torch.arange(51), 0] = 1.0
    sd["shrink.bias"] = torch.zeros(51)
    x = orc.make_input(N, T, J, 2, seed=78).to(cuda_device)
    outs = {}
    for prob in (0.0, p):
        m = getattr(vp, cls)(J, 2, J, filter_widths=[3], dropout=prob, channels=C)
        m.load_state_dict(sd)
        m = m.to(cuda_device).train().set_train_precision(precision)
        torch.manual_seed(5)
        y = m(x)
        y.sum().backward()
        outs[prob] = (y.detach().reshape(-1, 51), m.expand_bn.bias.grad[:51].clone())
    y0, _ = outs[0.0]
    yp, dbeta = outs[p]
    pos = y0 > 1e-4                                   # rows where ReLU passed a value
    kept = pos & (yp != 0)
    mask = emu.model_masks(emu.step_seed(5), [3], N, T, C, p, dilated=cls == "TemporalModel")[0]
    assert mask.shape[0] == y0.shape[0]
    assert torch.equal(pos & (yp == 0), pos & (mask[:, :51] == 0).to(cuda_device))
    ratio = yp[kept] / y0[kept]
    # scale 1/(1-p), nothing in between (bf16 storage: both values rounded, each by up to half an
    # ulp = 2^-8 relative)
    tol = 1e-3 if precision == "bf16x3" else 4.0 / 3.0 * 2 ** -7
    assert float((ratio - 4.0 / 3.0).abs().max()) <= tol
    assert float(yp[~pos].abs().max()) <= 2e-4                 # dropout never creates values
    n = int(pos.sum())
    rate = float(kept.sum()) / n
    sigma = (p * (1 - p) / n) ** 0.5
    print(f"dropout keep rate {rate:.4f} over {n} activations (3 sigma = {3 * sigma:.4f})")
    assert abs(rate - (1 - p)) <= 3 * sigma
    # per-channel keep rates are unbiased too (no channel / row structure in the mask)
    per_ch = kept.float().sum(0) / pos.float().sum(0).clamp_min(1)
    assert float((per_ch - 0.75).abs().max()) <= 6 * (p * (1 - p) / (n / 51)) ** 0.5
    # backward mask == forward mask: d sum(y)/d beta_c = 4/3 * (# kept activations of channel c
    # with a positive pre-activation); dropped or negative rows contribute nothing
    expect = kept.float().sum(0) * (4.0 / 3.0)
    assert float((dbeta - expect).abs().max()) <= 1e-2 * float(expect.max())


def test_total_causal_shift_and_receptive_field_match_reference(cuda_device):
    """model.py:41-61 for both classes: the Python methods and the C-ABI entry points against values
    produced by the real reference (tests/golden/causal_shift.json)."""
    import json
    import os
    from conftest import GOLDEN_DIR
    from videopose3d_b200 import _capi
    rows = json.load(open(os.path.join(GOLDEN_DIR, "causal_shift.json")))
    assert len(rows) >= 30
    lib = _capi.load()
    for r in rows:
        cls = getattr(vp, r["cls"])
        m = cls(17, 2, 17, filter_widths=r["arc"], causal=r["causal"], channels=64)
        assert m.total_causal_shift() == r["total_causal_shift"], r
        assert m.receptive_field() == r["receptive_field"], r
        assert list(m.pad) == r["pad"] and list(m.causal_shift) == r["causal_shift"], r
        plan = m.to(cuda_device)._get_plan(cuda_device)
        assert lib.vp3d_total_causal_shift(plan) == r["total_causal_shift"], r
        assert lib.vp3d_receptive_field(plan) == r["receptive_field"], r
