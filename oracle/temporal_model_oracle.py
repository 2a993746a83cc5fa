"""CPU oracle for the VideoPose3D temporal-convolution hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product path (videopose3d_b200/) imports this file; it is
used by tests/, by ``__graft_entry__.smoke()`` and by ``bench.py``'s cpu_baseline / ``--impl
reference`` legs as the checker and as the timed CPU baseline, never as a fallback.

It restates the algorithm of the reference's ``common/model.py`` twice:

* ``forward_numpy``  — explicit arithmetic in NumPy (channel-last, one matmul per filter tap,
  BatchNorm / ReLU / residual slices written out), float64 or float32.  Independent of torch.nn.
* ``forward_torch``  — the same network through ``torch.nn.functional`` conv1d / batch_norm on CPU,
  i.e. what the reference executes on a host (torch >= 0.4 per README.md:31; MKL-DNN here).  This is
  the CPU baseline that bench.py times ("kind": "port").

Parity pinning: the reference ships no tests or golden vectors (SURVEY.md §4).  Both restatements are
pinned against outputs of the *real* reference classes imported from /root/reference in the build
container (tests/golden/make_golden.py, fixtures committed under tests/golden/*.npz; checked by
tests/test_oracle_golden.py).

Reference lines followed:
  TemporalModelBase.forward            common/model.py:63-77   (view/permute in, permute/view out)
  TemporalModel._forward_blocks        common/model.py:126-138 (dilated, residual slice :130-132)
  TemporalModelOptimized1f._forward_blocks  common/model.py:187-197 (strided, residual :191)
  pad / causal_shift / dilation        common/model.py:107-121, 172-184
  BatchNorm1d semantics                torch.nn.BatchNorm1d (eps 1e-5, biased var for normalisation,
                                       unbiased for running_var), momentum read per call (:36-39)
"""
import numpy as np

EPS = 1e-5


# ---------------------------------------------------------------------------------------------
# architecture bookkeeping (model.py:31, 107-121, 172-184)
# ---------------------------------------------------------------------------------------------
def arch(filter_widths, causal=False, dense=False, strided=False):
    fw = list(filter_widths)
    for w in fw:
        assert w % 2 != 0, 'Only odd filter widths are supported'
    pad = [fw[0] // 2]
    shift = [fw[0] // 2 if causal else 0]
    dil = [1]
    taps = [fw[0]]
    nd = fw[0]
    for w in fw[1:]:
        p = (w - 1) * nd // 2
        pad.append(p)
        if strided:
            shift.append(w // 2 if causal else 0)
        else:
            shift.append((w // 2) * nd if causal else 0)
        dil.append(1 if dense else nd)
        taps.append(2 * p + 1 if dense else w)
        nd *= w
    return dict(widths=fw, pad=pad, shift=shift, dilation=dil, taps=taps,
                receptive_field=1 + 2 * sum(pad))


def receptive_field(filter_widths):
    return arch(filter_widths)["receptive_field"]


def state_dict_to_numpy(sd, dtype=np.float64):
    out = {}
    for k, v in sd.items():
        a = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
        out[k] = a.astype(dtype) if a.dtype.kind == "f" else a
    return out


# ---------------------------------------------------------------------------------------------
# NumPy restatement
# ---------------------------------------------------------------------------------------------
def _conv_cl(x, w, stride=1, dilation=1):
    """Valid 1-D convolution on channel-last data.  x: (N, L, Cin), w: (Cout, Cin, K) (torch
    Conv1d layout).  y[n, t, co] = sum_k sum_ci x[n, t*stride + k*dilation, ci] * w[co, ci, k]."""
    N, L, _ = x.shape
    K = w.shape[2]
    Lout = (L - dilation * (K - 1) - 1) // stride + 1
    assert Lout >= 1, "sequence shorter than the kernel extent"
    y = None
    for k in range(K):
        xs = x[:, k * dilation: k * dilation + (Lout - 1) * stride + 1: stride, :]
        term = xs @ w[:, :, k].T
        y = term if y is None else y + term
    return y


def _bn_cl(x, prefix, sd, training, momentum, new_stats, probe=None):
    g, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
    if training:
        flat = x.reshape(-1, x.shape[-1])
        n = flat.shape[0]
        mean = flat.mean(axis=0)
        var = flat.var(axis=0)  # biased, used for normalisation
        if new_stats is not None:
            unbiased = var * n / max(n - 1, 1)
            new_stats[prefix + ".running_mean"] = (1 - momentum) * sd[prefix + ".running_mean"] + momentum * mean
            new_stats[prefix + ".running_var"] = (1 - momentum) * sd[prefix + ".running_var"] + momentum * unbiased
            new_stats[prefix + ".num_batches_tracked"] = sd[prefix + ".num_batches_tracked"] + 1
    else:
        mean, var = sd[prefix + ".running_mean"], sd[prefix + ".running_var"]
    y = (x - mean) / np.sqrt(var + EPS) * g + b
    if probe is not None:  # distance of the closest pre-activation to the ReLU kink
        probe["min_abs_preact"] = min(probe.get("min_abs_preact", np.inf), float(np.abs(y).min()))
    return y


def forward_numpy(sd, x, filter_widths, causal=False, dense=False, strided=False, training=False,
                  momentum=0.1, dtype=np.float64, return_new_stats=False, collect=None, probe=None):
    """sd: state_dict (numpy or torch values); x: (N, T, J, F).  Dropout is the identity here
    (eval, or training with p = 0).  Returns (N, T_out, J_out, 3) [and the updated BN buffers]."""
    sd = state_dict_to_numpy(sd, dtype)
    a = arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    x = np.asarray(x, dtype=dtype)
    assert x.ndim == 4
    N, T = x.shape[0], x.shape[1]
    h = x.reshape(N, T, -1)                                   # model.py:68-70 (kept channel-last)
    new_stats = {} if return_new_stats else None

    h = _conv_cl(h, sd["expand_conv.weight"], stride=fw[0] if strided else 1)
    h = np.maximum(_bn_cl(h, "expand_bn", sd, training, momentum, new_stats, probe), 0)   # :127 / :188
    if collect is not None:
        collect.append(h)
    for i in range(len(fw) - 1):
        w = fw[i + 1]
        if strided:
            res = h[:, a["shift"][i + 1] + w // 2:: w, :]                           # :191
            z = _conv_cl(h, sd[f"layers_conv.{2 * i}.weight"], stride=w)
            res = res[:, :z.shape[1], :]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = h[:, pad + sh: h.shape[1] - pad + sh, :]                         # :130-132
            z = _conv_cl(h, sd[f"layers_conv.{2 * i}.weight"], dilation=a["dilation"][i + 1])
        z = np.maximum(_bn_cl(z, f"layers_bn.{2 * i}", sd, training, momentum, new_stats, probe), 0)
        if collect is not None:
            collect.append(z)
        z = _conv_cl(z, sd[f"layers_conv.{2 * i + 1}.weight"])
        z = np.maximum(_bn_cl(z, f"layers_bn.{2 * i + 1}", sd, training, momentum, new_stats, probe), 0)
        h = res + z                                                                  # :135 / :194
        if collect is not None:
            collect.append(h)
    y = _conv_cl(h, sd["shrink.weight"]) + sd["shrink.bias"]                          # :137 / :196
    y = y.reshape(N, -1, sd["shrink.weight"].shape[0] // 3, 3)                       # :74-75
    if return_new_stats:
        return y, new_stats
    return y


# ---------------------------------------------------------------------------------------------
# torch.nn.functional restatement (what the reference runs on a CPU) — also the timed CPU baseline
# ---------------------------------------------------------------------------------------------
def forward_torch(sd, x, filter_widths, causal=False, dense=False, strided=False, training=False,
                  momentum=0.1, update_stats=False, dropout=0.0, masks=None):
    """sd: dict of torch tensors (state_dict layout); x: torch (N, T, J, F).  Same math through
    F.conv1d / F.batch_norm in x's dtype on x's device.  `dropout` > 0 applies torch's dropout
    after every ReLU in training mode (model.py:127, 134-135); the default is the identity.
    `masks` ({layer: (N * frames, channels)}, layers numbered as in train_emulation.model_masks)
    instead multiplies given dropout masks in at the same places.
    Differentiable: tensors in `sd` that require grad receive gradients."""
    import torch
    import torch.nn.functional as F

    a = arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    N, T = x.shape[0], x.shape[1]
    h = x.reshape(N, T, -1).permute(0, 2, 1)

    def bn(t, prefix):
        rm, rv = sd[prefix + ".running_mean"], sd[prefix + ".running_var"]
        if training and not update_stats:
            rm, rv = rm.clone(), rv.clone()
        return F.batch_norm(t, rm, rv, sd[prefix + ".weight"], sd[prefix + ".bias"], training,
                            momentum, EPS)

    def act(t, layer):
        t = F.relu(t)
        if masks is not None:
            return t * masks[layer].to(t).reshape(N, t.shape[2], t.shape[1]).permute(0, 2, 1)
        return F.dropout(t, dropout, True) if (training and dropout > 0.0) else t

    h = act(bn(F.conv1d(h, sd["expand_conv.weight"], stride=fw[0] if strided else 1), "expand_bn"), 0)
    for i in range(len(fw) - 1):
        w = fw[i + 1]
        if strided:
            res = h[:, :, a["shift"][i + 1] + w // 2:: w]
            z = F.conv1d(h, sd[f"layers_conv.{2 * i}.weight"], stride=w)
            res = res[:, :, :z.shape[2]]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = h[:, :, pad + sh: h.shape[2] - pad + sh]
            z = F.conv1d(h, sd[f"layers_conv.{2 * i}.weight"], dilation=a["dilation"][i + 1])
        z = act(bn(z, f"layers_bn.{2 * i}"), 2 * i + 1)
        z = act(bn(F.conv1d(z, sd[f"layers_conv.{2 * i + 1}.weight"]), f"layers_bn.{2 * i + 1}"), 2 * i + 2)
        h = res + z
    y = F.conv1d(h, sd["shrink.weight"], sd["shrink.bias"])
    return y.permute(0, 2, 1).reshape(N, -1, sd["shrink.weight"].shape[0] // 3, 3)


# ---------------------------------------------------------------------------------------------
# synthetic parameters / inputs shared by tests, smoke() and bench.py (SURVEY.md §8d)
# ---------------------------------------------------------------------------------------------
def randomize_bn_(sd_or_module, seed=1):
    """BN affine + running stats away from the identity defaults (gamma~U(.5,1.5), beta~N(0,.1),
    running_mean~N(0,.1), running_var~U(.5,1.5)) so that BN bugs cannot hide."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sd = sd_or_module.state_dict() if hasattr(sd_or_module, "state_dict") else sd_or_module
    with torch.no_grad():
        for k, v in sd.items():
            if k.endswith("num_batches_tracked") or "bn" not in k:
                continue
            if k.endswith(".weight") or k.endswith("running_var"):
                v.copy_(torch.rand(v.shape, generator=g) + 0.5)
            else:
                v.copy_(torch.randn(v.shape, generator=g) * 0.1)
    return sd_or_module


def make_state_dict(num_joints_in, in_features, num_joints_out, filter_widths, channels,
                    dense=False, seed=0):
    """Parameters with torch's default Conv1d init ranges (kaiming-uniform a=sqrt(5) == U(-b, b),
    b = 1/sqrt(fan_in)) drawn from a seeded generator, plus randomised BN.  Construction order is
    fixed here (not torch.nn's), so the values depend only on this file and the seed."""
    import torch
    g = torch.Generator().manual_seed(seed)
    a = arch(filter_widths, dense=dense)
    c_in = num_joints_in * in_features

    def conv(co, ci, k):
        bound = 1.0 / (ci * k) ** 0.5
        return (torch.rand(co, ci, k, generator=g) * 2 - 1) * bound

    sd = {}

    def bn(prefix):
        sd[prefix + ".weight"] = torch.rand(channels, generator=g) + 0.5
        sd[prefix + ".bias"] = torch.randn(channels, generator=g) * 0.1
        sd[prefix + ".running_mean"] = torch.randn(channels, generator=g) * 0.1
        sd[prefix + ".running_var"] = torch.rand(channels, generator=g) + 0.5
        sd[prefix + ".num_batches_tracked"] = torch.zeros((), dtype=torch.long)

    bn("expand_bn")
    sd["shrink.weight"] = conv(num_joints_out * 3, channels, 1)
    sd["shrink.bias"] = (torch.rand(num_joints_out * 3, generator=g) * 2 - 1) / channels ** 0.5
    sd["expand_conv.weight"] = conv(channels, c_in, filter_widths[0])
    nb = len(filter_widths) - 1
    for i in range(nb):
        sd[f"layers_conv.{2 * i}.weight"] = conv(channels, channels, a["taps"][i + 1])
        sd[f"layers_conv.{2 * i + 1}.weight"] = conv(channels, channels, 1)
    for j in range(2 * nb):
        bn(f"layers_bn.{j}")
    return sd


def make_input(N, T, J=17, F=2, seed=0):
    """2-D keypoints in normalised screen coordinates, ~U(-1, 1) (camera.py:14-18)."""
    import torch
    g = torch.Generator().manual_seed(seed)
    return torch.rand(N, T, J, F, generator=g) * 2 - 1


def mpjpe(predicted, target):
    """Mean per-joint position error (loss.py:11-17), NumPy or torch inputs."""
    import torch
    p, t = torch.as_tensor(predicted), torch.as_tensor(target)
    assert p.shape == t.shape
    return torch.mean(torch.norm(p - t, dim=len(t.shape) - 1))
