"""GPU: TemporalModel (dilated) training at C = 1024 against float64 autograd, the one model-level
check of the dilated training path above C = 128.

Arc 3^5, C = 1024, N = 256 sequences of T = 243 frames (one output frame each: the last block is
the receptive-field case with one row per sample and dilation 81), fp32-faithful kernels (bf16x3).
Reference: float64 autograd through oracle.temporal_model_oracle.forward_torch on the same GPU.

Gates are those of tests/test_gpu_train.py::test_cfg3_shape_train_step_matches_reference and for
the same reason: the output and the running statistics hold 1e-3 in the max norm, while a few of
the ~10^8 pre-activations sit within the split-bf16 round-off of the ReLU kink, flip, and move single
gradient entries by O(1 / rows) -- so the gradients are gated on the median entry error (3e-3 of
the tensor's largest entry), the relative L2 error (2e-2) and the norm / sum functionals (2e-3).
The test shows the L2 gate rejects a reference whose dilated conv gradient has two taps swapped."""
import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc
from test_gpu_train import _build, _rel

pytestmark = pytest.mark.gpu


def _grad_dist(g, ref):
    g, ref = g.double().reshape(-1), ref.double().reshape(-1)
    err = (g - ref).abs()
    gmax = float(ref.abs().max())
    med = float(err.median()) / gmax
    l2 = float(err.norm() / ref.norm().clamp_min(1e-300))
    n_err = abs(float(g.norm() - ref.norm())) / float(ref.norm())
    s_err = abs(float(g.sum() - ref.sum())) / (float(ref.norm()) * np.sqrt(g.numel()))
    return med, l2, max(n_err, s_err)


def test_dilated_c1024_bf16x3_train_step_matches_fp64_autograd(cuda_device):
    dev = cuda_device
    arc, C, N, T = [3, 3, 3, 3, 3], 1024, 256, 243
    momentum = 0.1
    sd = orc.make_state_dict(17, 2, 17, arc, C, seed=71)
    x = orc.make_input(N, T, seed=72)
    gy = torch.randn(N, 1, 17, 3, generator=torch.Generator().manual_seed(73))
    meta = dict(cls="TemporalModel", J=17, F=2, Jout=17, fw=arc, C=C, causal=False, dense=False,
                momentum=momentum)
    m = _build(meta, sd, dev, "bf16x3")
    y = m(x.to(dev))
    (y * gy.to(dev)).sum().backward()
    torch.cuda.synchronize()

    params = dict(m.named_parameters())
    sd64 = {k: v.to(dev, torch.float64).clone().requires_grad_(k in params) for k, v in sd.items()}
    y64 = orc.forward_torch(sd64, x.to(dev, torch.float64), arc, training=True, momentum=momentum,
                            update_stats=True)
    y64.backward(gy.to(dev, torch.float64))

    y_err = _rel(y, y64.detach().cpu().numpy())
    new = m.state_dict()
    st_err = {k: _rel(new[k], sd64[k].detach().cpu().numpy())
              for k in sd if k.endswith("running_mean") or k.endswith("running_var")}
    dist = {k: _grad_dist(p.grad, sd64[k].grad) for k, p in params.items()}
    med = max(d[0] for d in dist.values())
    l2 = max(d[1] for d in dist.values())
    fn = max(d[2] for d in dist.values())
    print(f"TemporalModel 3^5 C=1024 N={N} bf16x3 vs fp64 autograd: y {y_err:.2e}, running stats "
          f"{max(st_err.values()):.2e}, gradients: median entry {med:.2e}, rel-L2 {l2:.2e}, "
          f"norm/sum {fn:.2e}")
    assert y_err <= 1e-3
    assert max(st_err.values()) <= 1e-3, st_err
    assert med <= 3e-3, {k: d[0] for k, d in dist.items()}
    assert l2 <= 2e-2, {k: d[1] for k, d in dist.items()}
    assert fn <= 2e-3, {k: d[2] for k, d in dist.items()}
    # the L2 gate rejects a per-sample weight gradient with two taps exchanged
    k = "layers_conv.2.weight"
    swapped = sd64[k].grad[:, :, [1, 0, 2]]
    assert _grad_dist(params[k].grad, swapped)[1] > 2e-2
