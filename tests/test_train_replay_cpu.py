"""CPU: the training schedule restated in Python (train_replay.py) with float64 fakes of every
launch equals the float64 training step, so the row views, tap signs, skip offsets, slab geometry,
fused BatchNorm-backward wiring and the g0 / g1 ping-pong it restates from train_api.cu are the
model's algorithm.  The GPU test (test_gpu_train_layers.py) then ties the same schedule, run through
the C entries, to the model bit for bit.

References: train_emulation.train_step(planes=0, masks=...) (float64, pinned against float64
autograd by test_dropout_reference_cpu.py) for y, every parameter gradient and the new running
statistics; float64 autograd through temporal_model_oracle.forward_torch where the emulation has no
such configuration (the dense model, frozen BatchNorm, the input gradient dx).  Each mutated
schedule (skip offset one frame off, the dilated data gradient's tap sign flipped, the ping-pong
buffers swapped) must be rejected."""
import pytest
import torch

import train_replay as tr
from oracle import temporal_model_oracle as orc
from oracle import train_emulation as emu

TM, OPT = "TemporalModel", "TemporalModelOptimized1f"
P = 0.25
TOL = 1e-9          # float64 against float64, different summation orders


def _cfg(cls, fw, C, J=17, F=2, Jout=17, causal=False, dense=False):
    return dict(cls=cls, fw=list(fw), C=C, J=J, F=F, Jout=Jout, causal=causal, dense=dense)


# (id, cfg, N, T): every architecture of the GPU matrix at small N
ARCHS = [
    ("opt_333_c64", _cfg(OPT, [3, 3, 3], 64), 4, 27),
    ("opt_35_causal", _cfg(OPT, [3, 5], 64, causal=True), 4, 15),
    ("opt_333_c40", _cfg(OPT, [3, 3, 3], 40), 4, 27),
    ("opt_33_c100", _cfg(OPT, [3, 3], 100), 3, 9),
    ("opt_333_j15_f3", _cfg(OPT, [3, 3, 3], 64, J=15, F=3, Jout=15), 3, 27),
    ("opt_333_jout1", _cfg(OPT, [3, 3, 3], 64, Jout=1), 4, 27),
    ("tm_333_dilated", _cfg(TM, [3, 3, 3], 64), 2, 40),
    ("tm_35_causal", _cfg(TM, [3, 5], 64, causal=True), 2, 30),
    ("tm_33_dense", _cfg(TM, [3, 3], 64, dense=True), 2, 20),
    # widths other than 3 and 5, and the 32-joint skeleton (tests/test_gpu_architectures.py)
    ("opt_337", _cfg(OPT, [3, 3, 7], 128), 2, 63),
    ("opt_355_causal", _cfg(OPT, [3, 5, 5], 100, causal=True), 2, 75),
    ("opt_733_t68", _cfg(OPT, [7, 3, 3], 64), 2, 68),
    ("opt_313", _cfg(OPT, [3, 1, 3], 64), 3, 9),
    ("opt_133", _cfg(OPT, [1, 3, 3], 64), 3, 9),
    ("opt_j32_f3", _cfg(OPT, [3, 3, 3], 64, J=32, F=3, Jout=32), 3, 27),
    ("tm_337_dilated", _cfg(TM, [3, 3, 7], 64), 1, 70),
    ("tm_313_dilated", _cfg(TM, [3, 1, 3], 64), 2, 20),
    ("tm_337_dense", _cfg(TM, [3, 3, 7], 64, dense=True), 1, 70),
]


def _case(cfg, N, T, seed=3):
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"],
                             dense=cfg["dense"], seed=seed)
    x = orc.make_input(N, T, cfg["J"], cfg["F"], seed=seed + 1).double()
    rf = orc.arch(cfg["fw"])["receptive_field"]
    L_out = T // rf if cfg["cls"] == OPT else T - rf + 1
    gy = torch.randn(N, L_out, cfg["Jout"], 3, generator=torch.Generator().manual_seed(seed + 2),
                     dtype=torch.float64)
    return sd, x, gy


def _masks(cfg, N, T, p, seed):
    if p == 0:
        return None
    return emu.model_masks(seed, cfg["fw"], N, T, cfg["C"], p, dilated=cfg["cls"] == TM)


def _autograd(sd, cfg, x, gy, masks, frozen=False):
    """float64 autograd through forward_torch: y, parameter gradients, new running stats, dx."""
    sdr = {k: v.double().clone() for k, v in sd.items() if v.dtype.is_floating_point}
    params = {k: v.requires_grad_() for k, v in sdr.items() if "running" not in k}
    xg = x.clone().requires_grad_()
    y = orc.forward_torch(sdr, xg, cfg["fw"], causal=cfg["causal"], dense=cfg["dense"],
                          strided=cfg["cls"] == OPT, training=not frozen, momentum=tr.MOMENTUM,
                          update_stats=True, masks=masks)
    (y * gy).sum().backward()
    grads = {k: v.grad for k, v in params.items()}
    stats = {} if frozen else {k: v for k, v in sdr.items() if "running" in k}
    return dict(y=y.detach(), grads=grads, new_stats=stats, dx=xg.grad)


def _reference(sd, cfg, x, gy, masks):
    if cfg["dense"]:
        return _autograd(sd, cfg, x, gy, masks)
    return emu.train_step(sd, x, gy, cfg["fw"], causal=cfg["causal"], planes=0,
                          momentum=tr.MOMENTUM, dilated=cfg["cls"] == TM, masks=masks)


def _dist(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double().reshape(a.shape)
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def _compare(rep, ref, dx=False):
    """{name: relative max distance} over y, every gradient, the running statistics [and dx]."""
    out = {"y": _dist(rep.y, ref["y"])}
    for k, g in ref["grads"].items():
        out[k] = _dist(rep.grads[k], g)
    for k, s in ref["new_stats"].items():
        out[k] = _dist(rep.stats[k], s)
    if dx:
        out["dx"] = _dist(rep.dx, ref["dx"])
    return out


def _run(cfg, N, T, precision, p=0.0, seed=0x1234_5678_9ABC, **kw):
    sd, x, gy = _case(cfg, N, T)
    rep = tr.replay(sd, cfg, x, gy, precision, tr.FakeOps(x.device), p_drop=p, seed=seed, **kw)
    return sd, x, gy, rep


@pytest.mark.parametrize("p", [0.0, P])
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name,cfg,N,T", ARCHS, ids=[a[0] for a in ARCHS])
def test_float64_replay_is_the_training_step(name, cfg, N, T, precision, p):
    """bf16 runs the fused BatchNorm-backward sums and ordered_col_sums, bf16x3 bn_bwd_reduce."""
    seed = 0x1234_5678_9ABC
    sd, x, gy, rep = _run(cfg, N, T, precision, p, seed)
    ref = _reference(sd, cfg, x, gy, _masks(cfg, N, T, p, seed))
    d = _compare(rep, ref)
    assert len(d) == 1 + len(ref["grads"]) + len(ref["new_stats"])
    bad = {k: v for k, v in d.items() if not v <= TOL}
    assert not bad, bad
    assert not any(torch.isnan(g).any() for g in rep.grads.values())


def _launches(p, dx):
    """The launch counts train_api.cu reports for one step with every parameter gradient."""
    fused = p.planes == 1
    fwd = 2 + 3 * (2 * p.nb + 1) + 1
    bn_bwd = (1 if fused else 2) + 1
    bwd = 1 + 2 + 2 + 1 + (2 * p.nb + 1) * (bn_bwd + 2) + 2 * p.nb
    if dx:
        bwd += 1 + (2 if p.strided and p.T != p.fw[0] * p.L[0] else 0)
    return fwd, bwd


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name,cfg,N,T", [("opt_333_t29", _cfg(OPT, [3, 3, 3], 64), 3, 29),
                                          ("tm_35_causal", _cfg(TM, [3, 5], 64, causal=True), 2, 30),
                                          ("opt_733_t68", _cfg(OPT, [7, 3, 3], 64), 2, 68),
                                          ("opt_133", _cfg(OPT, [1, 3, 3], 64), 2, 9),
                                          ("tm_337_dilated", _cfg(TM, [3, 3, 7], 64), 1, 70)])
def test_float64_replay_input_gradient(name, cfg, N, T, precision):
    """dx: the strided tail (T != w0 * L0: the trailing frames get zero) and the dilated transposed
    expand conv, against float64 autograd; also the launch counts."""
    sd, x, gy, rep = _run(cfg, N, T, precision, want_dx=True)
    ref = _autograd(sd, cfg, x, gy, None)
    d = _compare(rep, ref, dx=True)
    bad = {k: v for k, v in d.items() if not v <= TOL}
    assert not bad, bad
    if cfg["cls"] == OPT:
        assert torch.all(rep.dx[:, rep.plan.fw[0] * rep.plan.L[0]:] == 0)
    assert (rep.fwd_launches, rep.bwd_launches) == _launches(rep.plan, True)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name,cfg,N,T", [("opt_333", _cfg(OPT, [3, 3, 3], 64), 3, 27),
                                          ("tm_333", _cfg(TM, [3, 3, 3], 64), 2, 40)])
def test_float64_replay_frozen_bn(name, cfg, N, T, precision):
    """Frozen BatchNorm (the eval-mode backward): the fixed affine of the running statistics,
    running statistics untouched; gradients and dx against float64 autograd in eval mode."""
    sd, x, gy, rep = _run(cfg, N, T, precision, frozen=True, want_dx=True)
    ref = _autograd(sd, cfg, x, gy, None, frozen=True)
    d = _compare(rep, ref, dx=True)
    bad = {k: v for k, v in d.items() if not v <= TOL}
    assert not bad, bad
    assert rep.stats == {}
    assert (rep.fwd_launches, rep.bwd_launches) == _launches(rep.plan, True)


def test_bn_fold_train_matches_float64():
    """The frozen fold's mean / invstd outputs: mean copied, invstd 1/sqrt(var + eps) in fp32
    (one rounding per operation) within 2 ulp of float64, zero padding."""
    g = torch.Generator().manual_seed(5)
    bn = dict(weight=torch.rand(40, generator=g) + 0.5, bias=torch.randn(40, generator=g),
              running_mean=torch.randn(40, generator=g),
              running_var=torch.rand(40, generator=g) * 4 + 1e-3)
    sc, sh, mu, inv = tr.bn_fold_train(bn, 64, exact=False)
    assert mu.dtype == inv.dtype == torch.float32
    assert torch.equal(mu[:40], bn["running_mean"]) and torch.all(mu[40:] == 0)
    ref = 1.0 / torch.sqrt(bn["running_var"].double() + 1e-5)
    assert torch.all((inv[:40].double() - ref).abs() <= 2 * 2.0 ** -24 * ref)
    assert torch.all(inv[40:] == 0) and torch.all(sc[40:] == 0) and torch.all(sh[40:] == 0)


MUTATIONS = [
    ("skip_off", ("opt_333_c64", _cfg(OPT, [3, 3, 3], 64), 4, 27)),
    ("skip_off", ("tm_333_dilated", _cfg(TM, [3, 3, 3], 64), 2, 40)),
    ("tap_sign", ("tm_333_dilated", _cfg(TM, [3, 3, 3], 64), 2, 40)),
    ("pingpong", ("opt_333_c64", _cfg(OPT, [3, 3, 3], 64), 4, 27)),
    ("pingpong", ("tm_35_causal", _cfg(TM, [3, 5], 64, causal=True), 2, 30)),
    ("tap_sign", ("tm_337_dilated", _cfg(TM, [3, 3, 7], 64), 1, 70)),
]


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("mutation,arch", MUTATIONS, ids=[f"{m}-{a[0]}" for m, a in MUTATIONS])
def test_mutated_schedule_is_rejected(mutation, arch, precision):
    _, cfg, N, T = arch
    seed = 77
    sd, x, gy, rep = _run(cfg, N, T, precision, P, seed, mutate={mutation})
    ref = _reference(sd, cfg, x, gy, _masks(cfg, N, T, P, seed))
    d = _compare(rep, ref)
    worst = max(d.values())
    assert worst > 1e-3, f"{mutation} not rejected: worst distance {worst:.2e}"
