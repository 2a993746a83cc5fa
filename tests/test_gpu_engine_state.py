"""GPU: the per-plan engine state of the models.

* which weight packs each call makes on which plan (vp3d_set_weights recorded through a scripted
  sequence of eval forwards at two precisions, a BatchNorm buffer edit, training steps with the fused
  optimizer, an eval-mode backward, a streaming push and the host pipeline), the launch count the
  model reports and the plan ``model._plan`` is after each call;
* a host-pipeline slot completes on the plan it was submitted on, whatever ran in between;
* the C entry points the model does not call (vp3d_forward_train, vp3d_backward,
  vp3d_backward_staged) give the bits and launches of vp3d_forward_train_ex / vp3d_backward_ex."""
import ctypes

import pytest
import torch

import videopose3d_b200 as vp
from oracle import temporal_model_oracle as orc
from videopose3d_b200 import _capi
from videopose3d_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

ARC, C, N, T = [3, 3, 3], 64, 4, 35
CONV, CONV_T = _capi.VP3D_PACK_CONV, _capi.VP3D_PACK_CONV_T
BN_EVAL, EXPAND_T = _capi.VP3D_PACK_BN_EVAL, _capi.VP3D_PACK_EXPAND_T
_PRECISION_NAMES = {_capi.VP3D_PRECISION_FP16: "fp16", _capi.VP3D_PRECISION_BF16: "bf16",
                    _capi.VP3D_PRECISION_BF16X3: "bf16x3", _capi.VP3D_PRECISION_MIXED: "mixed"}


def _model(dev, dropout=0.0):
    m = vp.TemporalModel(17, 2, 17, filter_widths=ARC, dropout=dropout, channels=C)
    m.load_state_dict(orc.make_state_dict(17, 2, 17, ARC, C, seed=11))
    return m.to(dev).set_precision("fp16").set_train_precision("bf16")


class _Recorder:
    """Wraps vp3d_plan_create (to name each plan by its precision) and vp3d_set_weights (to record
    (precision, what) per call) on the loaded library."""

    def __init__(self, monkeypatch):
        lib = _capi.load()
        self.names, self.packs = {}, []
        create, set_weights = lib.vp3d_plan_create, lib.vp3d_set_weights

        def plan_create(cfg, handle):
            rc = create(cfg, handle)
            self.names[handle._obj.value] = _PRECISION_NAMES[cfg._obj.precision]
            return rc

        def record_set_weights(plan, w, what, stream):
            self.packs.append((self.name(plan), what))
            return set_weights(plan, w, what, stream)

        monkeypatch.setattr(lib, "vp3d_plan_create", plan_create)
        monkeypatch.setattr(lib, "vp3d_set_weights", record_set_weights)

    def name(self, plan):
        """Precision of a plan handle (or of an object ctypes passes as one), None for no plan."""
        if plan is None:
            return None
        return self.names[getattr(plan, "_as_parameter_", plan).value]

    def take(self):
        packs, self.packs = self.packs, []
        return packs


# (step, vp3d_set_weights calls as (plan precision, what), last_launch_count(), precision of
# model._plan) after each step of test_packs_launches_and_last_plan_per_call
EXPECTED = [
    ("eval fp16", [("fp16", CONV | BN_EVAL)], 7, "fp16"),
    ("eval fp16 again", [], 7, "fp16"),
    ("BatchNorm buffer edit, eval fp16", [("fp16", BN_EVAL)], 7, "fp16"),
    ("eval bf16", [("bf16", CONV | BN_EVAL)], 7, "bf16"),
    ("training step 1", [("bf16", CONV | CONV_T)], 4, "bf16"),
    ("training step 2", [], 4, "bf16"),
    ("eval bf16 after training", [("bf16", CONV | BN_EVAL)], 7, "bf16"),
    ("eval-mode backward into x", [("bf16", EXPAND_T)], 31, "bf16"),
    ("streaming push at fp16", [("fp16", CONV | BN_EVAL)], 31, "bf16"),
    ("host submit and wait at fp16", [], 7, "fp16"),
]


def test_packs_launches_and_last_plan_per_call(cuda_device, monkeypatch):
    rec = _Recorder(monkeypatch)
    m = _model(cuda_device).eval()
    x = orc.make_input(N, T, 17, 2, seed=12).to(cuda_device)
    gen = torch.Generator().manual_seed(13)
    target = torch.randn(N, T - 26, 17, 3, generator=gen).to(cuda_device)
    got = []

    def observe(step):
        torch.cuda.synchronize()
        got.append((step, rec.take(), m.last_launch_count(), rec.name(m._plan)))

    with torch.no_grad():
        m(x)
        observe("eval fp16")
        m(x)
        observe("eval fp16 again")
        m.layers_bn[1].running_var.mul_(1.5)
        m(x)
        observe("BatchNorm buffer edit, eval fp16")
        m.set_precision("bf16")(x)
        observe("eval bf16")
    m.train()
    opt = FusedAdam(m.parameters(), lr=1e-3, amsgrad=True)
    for i in range(2):
        opt.zero_grad()
        (m(x) - target).square().mean().backward()
        opt.step()
        observe(f"training step {i + 1}")
    m.eval()
    with torch.no_grad():
        m(x)
    observe("eval bf16 after training")
    xg = x.clone().requires_grad_()
    (m(xg) * target).sum().backward()
    observe("eval-mode backward into x")
    m.set_precision("fp16")
    m.streaming(streams=2, max_frames=1).push(x[:2, :1].contiguous(), start=[True, True])
    observe("streaming push at fp16")
    xh = x.cpu().pin_memory()
    out = torch.empty((N, T - 26, 17, 3), dtype=torch.float32).pin_memory()
    m.forward_host_submit(xh, out, 0)
    m.forward_host_wait(0)
    observe("host submit and wait at fp16")
    report = "\n".join(map(repr, got))
    assert len(got) == len(EXPECTED), report
    for g, e in zip(got, EXPECTED):
        assert g == e, report


def test_host_wait_completes_on_the_plan_of_its_submit(cuda_device):
    """submit at fp16, an eval forward at bf16 in between, then the wait: it completes the fp16
    batch (with the same output as forward_host) and leaves the slot free for the next submit."""
    m = _model(cuda_device).eval()
    x = orc.make_input(N, T, 17, 2, seed=14)
    xh = x.pin_memory()
    want = m.forward_host(xh).clone()
    out = torch.empty_like(want).pin_memory()
    m.forward_host_submit(xh, out, 0)
    with torch.no_grad():
        m.set_precision("bf16")(x.to(cuda_device))
    m.forward_host_wait(0)
    assert torch.equal(out, want)
    m.set_precision("fp16")
    out.zero_()
    m.forward_host_submit(xh, out, 0)
    m.forward_host_wait(0)
    assert torch.equal(out, want)


def test_legacy_training_entries_match_the_ex_entries(cuda_device):
    """vp3d_forward_train + vp3d_backward and vp3d_backward_staged against vp3d_forward_train_ex
    (flags 0) + vp3d_backward_ex on one plan with one dropout seed: the same gradient bits, stage
    callbacks and launch counts."""
    m = _model(cuda_device, dropout=0.25).train()
    x = orc.make_input(N, T, 17, 2, seed=15).to(cuda_device)
    dy = torch.randn(N, T - 26, 17, 3, generator=torch.Generator().manual_seed(16)).to(cuda_device)
    m(x)                                   # creates and packs the bf16 training plan
    torch.cuda.synchronize()
    lib, plan = _capi.load(), m._plan
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    w = m._weights_struct()
    mom = (ctypes.c_float * (1 + len(m.layers_bn)))(*([0.1] * (1 + len(m.layers_bn))))

    def run(ex, staged):
        ws = torch.empty(lib.vp3d_train_workspace_bytes(plan, N, T), dtype=torch.uint8,
                         device=cuda_device)
        y = torch.empty(dy.shape, dtype=torch.float32, device=cuda_device)
        args = (plan, x.data_ptr(), y.data_ptr(), N, T, ctypes.byref(w), mom, 0.25, 1234)
        if ex:
            assert lib.vp3d_forward_train_ex(*args, 0, ws.data_ptr(), ws.numel(), stream) == 0
        else:
            assert lib.vp3d_forward_train(*args, ws.data_ptr(), ws.numel(), stream) == 0
        fwd_launches = lib.vp3d_last_launch_count(plan)
        grads = [torch.empty(p.shape, dtype=torch.float32, device=cuda_device)
                 for p in m._learnable_tensors()]
        g = m._grads_struct(grads)
        stages = []
        cb = _capi.STAGE_FN(lambda stage, _user: stages.append(stage))
        cbp = ctypes.cast(cb, ctypes.c_void_p) if staged else None
        bwd = (plan, dy.data_ptr(), ctypes.byref(g))
        tail = (ws.data_ptr(), ws.numel(), stream)
        if ex:
            assert lib.vp3d_backward_ex(*bwd, None, *tail, cbp, None) == 0
        elif staged:
            assert lib.vp3d_backward_staged(*bwd, *tail, cbp, None) == 0
        else:
            assert lib.vp3d_backward(*bwd, *tail) == 0
        torch.cuda.synchronize()
        return y, grads, stages, fwd_launches, lib.vp3d_last_launch_count(plan)

    for staged in (False, True):
        y0, g0, s0, f0, b0 = run(False, staged)
        y1, g1, s1, f1, b1 = run(True, staged)
        assert torch.equal(y0, y1)
        for a, b in zip(g0, g1):
            assert torch.equal(a, b)
        assert (s0, f0, b0) == (s1, f1, b1)
        assert s0 == (list(range(len(ARC) + 1)) if staged else [])


def test_training_above_the_channel_limit_fails_on_every_forward(cuda_device):
    """Training supports at most 8192 (padded) channels.  A plan above the limit gets no training
    state at all, so every training forward raises the same error instead of the second one running
    on half-built state."""
    m = vp.TemporalModel(17, 2, 17, filter_widths=[3, 3], dropout=0.0, channels=8193)   # 8256 padded
    m = m.to(cuda_device).set_train_precision("bf16").train()
    x = orc.make_input(2, 9, 17, 2, seed=3).to(cuda_device)
    for _ in range(2):
        with pytest.raises(NotImplementedError, match="at most 8192 channels"):
            m(x)
    torch.cuda.synchronize()
