"""Quantisation-aware CPU restatement of one TemporalModelOptimized1f training step.

TEST INFRASTRUCTURE ONLY (see oracle/temporal_model_oracle.py for the rules: only tests/, smoke()
and bench.py's CPU legs may import oracle/).

`train_step(..., planes=0)` is the reference algorithm in float64: forward of common/model.py:187-197
(strided) or :126-138 (`dilated=True`, TemporalModel) in train() mode (BatchNorm batch statistics,
dropout = 0 unless `masks` are given) followed by the analytic backward that autograd performs (conv
weight / data gradients, BatchNorm backward with the sum(dY) and sum(dY * xhat) reductions, ReLU
and dropout masks, residual fan-in).  It is pinned against gradients produced by the real reference
(tests/test_oracle_golden.py::test_train_emulation_matches_reference).

`dropout_mask` restates the kernels' counter-based dropout mask, so that `masks` can replay exactly
the masks a training step of the CUDA path drew.

`planes = 1 / 2` additionally rounds every tensor the CUDA path stores in bf16 (1 plane) or split
bf16 (hi + lo, 2 planes) at exactly the points where the kernels round: packed input and weights,
pre-BN conv outputs Z, activations X / H, incoming gradients G and dZ.  ReLU networks are not
smooth: a pre-activation that sits within the rounding error of zero flips its mask and moves a
gradient by O(1/rows), so a bf16 path cannot be compared with an fp32 reference at tight tolerance
on small batches — but it can be compared tightly with this emulation, which shares its rounding
points.  The fp32-faithful mode (planes = 2) is compared with the reference directly, on fixtures
chosen away from ReLU kinks (tests/golden/make_golden.py).
"""
import numpy as np
import torch

from oracle import temporal_model_oracle as orc

EPS = 1e-5
_U32 = 0xFFFFFFFF


def _mix32(h):
    h = h ^ (h >> 16)
    h = (h * 0x85EBCA6B) & _U32
    h = h ^ (h >> 13)
    h = (h * 0xC2B2AE35) & _U32
    return h ^ (h >> 16)


def dropout_mask(seed, layer, rows, c_real, c_pad, p):
    """The dropout mask the training kernels apply to `layer` (train_ops.cu dropout_keep8): a
    (rows, c_real) float64 tensor of 0 (dropped) and the kernels' fp32 1/(1-p) (kept).

    Element e = row * c_pad + channel (c_pad = the plan's padded channel count), pair P = e >> 1,
    h = mix32(uint32(P) * 0x9E3779B1 + key) with key = seed_lo ^ seed_hi * 0x7F4A7C15 ^
    layer * 0x632BE5AB ^ (P >> 32) * 0x85EBCA77 (wrapping uint32); the even element of the pair reads
    h & 0xFFFF, the odd one h >> 16, and it is kept iff that value >= uint32(fp32(p) * 65536)."""
    e = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(c_pad) +
         np.arange(c_real, dtype=np.uint64)[None, :])
    pair = e >> np.uint64(1)
    key = ((seed & _U32) ^ (((seed >> 32) & _U32) * 0x7F4A7C15 & _U32) ^
           ((layer * 0x632BE5AB) & _U32))
    key = np.uint64(key) ^ (((pair >> np.uint64(32)) * np.uint64(0x85EBCA77)) & np.uint64(_U32))
    h = _mix32(((pair & np.uint64(_U32)) * np.uint64(0x9E3779B1) + key) & np.uint64(_U32))
    u16 = np.where((e & np.uint64(1)) == 1, h >> np.uint64(16), h & np.uint64(0xFFFF))
    p32 = np.float32(p)
    thresh = int(p32 * np.float32(65536.0))                 # truncated, as the kernels convert
    inv_keep = float(np.float32(1.0) / (np.float32(1.0) - p32))
    return torch.from_numpy(np.where(u16 >= thresh, inv_keep, 0.0))


def step_seed(torch_seed):
    """The dropout seed of the training step that runs right after torch.manual_seed(torch_seed):
    _TrainFunction.forward (videopose3d_b200/temporal_model.py) draws it as
    torch.randint(0, 2**62, (1,)) from the CPU generator, and this repeats that draw -- keep the two
    in step."""
    torch.manual_seed(torch_seed)
    return int(torch.randint(0, 2 ** 62, (1,)).item())


def layer_lengths(filter_widths, T, dilated=False):
    """Frames per sample of every layer's output: [expand, block 1, ..., block nb]."""
    a = orc.arch(filter_widths, strided=not dilated)
    fw = a["widths"]
    L = [T - fw[0] + 1 if dilated else T // fw[0]]
    for i in range(1, len(fw)):
        L.append(L[-1] - 2 * a["pad"][i] if dilated else L[-1] // fw[i])
    return L


def model_masks(seed, filter_widths, N, T, channels, p, dilated=False):
    """{layer: mask} for every BatchNorm layer of one training step, numbered as forward_train
    numbers them: 0 = expand_bn, 2i-1 / 2i = layers_bn.2(i-1) / layers_bn.2(i-1)+1 of block i.
    Rows are (sample, frame), sample-major, over the layer's output length."""
    c_pad = -(-channels // 64) * 64
    L = layer_lengths(filter_widths, T, dilated)
    out = {0: dropout_mask(seed, 0, N * L[0], channels, c_pad, p)}
    for i in range(1, len(L)):
        for layer in (2 * i - 1, 2 * i):
            out[layer] = dropout_mask(seed, layer, N * L[i], channels, c_pad, p)
    return out


def _q(t, planes):
    if planes == 0:
        return t
    hi = t.float().to(torch.bfloat16).double()
    if planes == 1:
        return hi
    return hi + (t - hi).float().to(torch.bfloat16).double()


def train_step(sd, x, gy, filter_widths, causal=False, planes=0, momentum=0.1, dilated=False,
               masks=None):
    """sd: state_dict (torch tensors), x: (N, T, J, F), gy: upstream gradient of the output.
    dilated: TemporalModel instead of TemporalModelOptimized1f.  masks: {layer: (rows, channels)}
    dropout masks (model_masks), multiplied in after each ReLU as the kernels do; None = no dropout.
    Returns dict(y=..., grads={name: tensor}, new_stats={name: tensor}, min_abs_preact=float)."""
    q = lambda t: _q(t, planes)
    sd = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    fw = list(filter_widths)
    a = orc.arch(fw, causal, strided=not dilated)
    C = sd["expand_conv.weight"].shape[0]
    x = x.double()
    N, T = x.shape[0], x.shape[1]
    c_in = x.shape[2] * x.shape[3]
    saved, new_stats = {}, {}
    min_pre = float("inf")

    def taps(X, w, d):
        # [rows_out, w, C] view of the conv's input rows: strided (stride = width) rows are w
        # consecutive input rows; dilated rows (n, t) read X[n, t + k*d]
        if not dilated:
            return X.reshape(X.shape[0] // w, w, X.shape[-1])
        Xn = X.reshape(N, -1, X.shape[-1])
        L_out = Xn.shape[1] - (w - 1) * d
        return torch.stack([Xn[:, k * d:k * d + L_out] for k in range(w)], 2).reshape(N * L_out, w, -1)

    def bn(z_exact, prefix, layer):
        # the kernels take the batch statistics from the fp32 accumulators (before rounding) and
        # normalise the stored (rounded) Z with them
        nonlocal min_pre
        n = z_exact.shape[0]
        mu = z_exact.mean(0)
        var = z_exact.var(0, unbiased=False)
        z = q(z_exact)
        inv = 1.0 / torch.sqrt(var + EPS)
        sc = sd[prefix + ".weight"] * inv
        sh = sd[prefix + ".bias"] - mu * sc
        new_stats[prefix + ".running_mean"] = (1 - momentum) * sd[prefix + ".running_mean"] + momentum * mu
        new_stats[prefix + ".running_var"] = ((1 - momentum) * sd[prefix + ".running_var"] +
                                              momentum * var * n / max(n - 1, 1))
        m = masks[layer] if masks is not None else None
        saved[layer] = (z, mu, inv, sc, sh, m)
        y = z * sc + sh
        min_pre = min(min_pre, float(y.abs().min()))
        return torch.relu(y) if m is None else torch.relu(y) * m

    # ---- forward: every conv is a GEMM on [rows, w*C] views of its input (taps)
    if dilated:
        a0 = taps(q(x.reshape(N * T, c_in)), fw[0], 1)
        a0 = a0.reshape(a0.shape[0], fw[0] * c_in)
    else:
        L0 = T // fw[0]
        a0 = q(x.reshape(N, T, c_in)[:, :L0 * fw[0]].reshape(N * L0, fw[0] * c_in))
    w0 = sd["expand_conv.weight"].permute(0, 2, 1).reshape(C, -1)       # [co][tap*c_in + ci]
    X = q(bn(a0 @ q(w0).T, "expand_bn", 0))
    Xs, Hs = [X], [None]
    nb = len(fw) - 1
    offs = [None]
    for i in range(1, nb + 1):
        w, d = fw[i], a["dilation"][i]
        A = taps(X, w, d)
        rows = A.shape[0]
        w1 = sd[f"layers_conv.{2 * (i - 1)}.weight"].permute(0, 2, 1).reshape(C, w * C)
        H = q(bn(A.reshape(rows, w * C) @ q(w1).T, f"layers_bn.{2 * (i - 1)}", 2 * i - 1))
        w2 = sd[f"layers_conv.{2 * (i - 1) + 1}.weight"][:, :, 0]
        Y2 = bn(H @ q(w2).T, f"layers_bn.{2 * (i - 1) + 1}", 2 * i)
        if dilated:                                                        # model.py:130-132
            off = a["pad"][i] + a["shift"][i]
            res = X.reshape(N, -1, C)[:, off:off + rows // N].reshape(rows, C)
        else:                                                              # model.py:191
            off = w // 2 + (w // 2 if causal else 0)
            res = X.reshape(rows, w, C)[:, off]
        X = q(res + Y2)
        Xs.append(X)
        Hs.append(H)
        offs.append(off)
    wsh = sd["shrink.weight"][:, :, 0]
    y = X @ q(wsh).T + sd["shrink.bias"]

    # ---- backward
    gy = gy.double().reshape(-1, y.shape[1])
    grads = {"shrink.bias": gy.sum(0)}
    gyq = q(gy)
    grads["shrink.weight"] = (gyq.T @ Xs[nb])[:, :, None]
    G = q(gyq @ q(wsh))

    def bn_bwd(G, layer):
        z, mu, inv, sc, sh, m = saved[layer]
        dy = G * ((z * sc + sh) > 0)
        if m is not None:
            dy = dy * m
        xh = (z - mu) * inv
        s1, s2, n = dy.sum(0), (dy * xh).sum(0), z.shape[0]
        return q(sc * (dy - s1 / n - xh * s2 / n)), s2, s1

    for i in range(nb, 0, -1):
        w = fw[i]
        c1, c2 = 2 * (i - 1), 2 * (i - 1) + 1
        dz2, dg, db = bn_bwd(G, 2 * i)
        grads[f"layers_bn.{c2}.weight"], grads[f"layers_bn.{c2}.bias"] = dg, db
        grads[f"layers_conv.{c2}.weight"] = (dz2.T @ Hs[i])[:, :, None]
        GH = q(dz2 @ q(sd[f"layers_conv.{c2}.weight"][:, :, 0]))
        dz1, dg, db = bn_bwd(GH, 2 * i - 1)
        grads[f"layers_bn.{c1}.weight"], grads[f"layers_bn.{c1}.bias"] = dg, db
        rows = dz1.shape[0]
        A = taps(Xs[i - 1], w, a["dilation"][i])
        grads[f"layers_conv.{c1}.weight"] = torch.einsum("ro,rkc->ock", dz1, A)
        Gn = torch.einsum("ro,ock->rkc", dz1, q(sd[f"layers_conv.{c1}.weight"]))
        if dilated:
            # transposed convolution: tap k of output row (n, t) came from input row (n, t + k*d)
            d, L_out = a["dilation"][i], rows // N
            Gd = torch.zeros_like(Xs[i - 1]).reshape(N, -1, C)
            for k in range(w):
                Gd[:, k * d:k * d + L_out] += Gn[:, k].reshape(N, L_out, C)
            Gd[:, offs[i]:offs[i] + L_out] += G.reshape(N, L_out, C)       # skip-connection gradient
            G = q(Gd.reshape(-1, C))
        else:
            Gn[:, offs[i]] += G                                            # skip-connection gradient
            G = q(Gn.reshape(rows * w, C))
    dz0, dg, db = bn_bwd(G, 0)
    grads["expand_bn.weight"], grads["expand_bn.bias"] = dg, db
    grads["expand_conv.weight"] = (dz0.T @ a0).reshape(C, fw[0], c_in).permute(0, 2, 1)
    return dict(y=y.reshape(N, -1, y.shape[1] // 3, 3), grads=grads, new_stats=new_stats,
                min_abs_preact=min_pre)


def rel_l2(a, b):
    a = a.detach().cpu().double().numpy() if hasattr(a, "detach") else np.asarray(a, dtype=np.float64)
    b = b.detach().cpu().double().numpy() if hasattr(b, "detach") else np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def rel_max(a, b):
    a = a.detach().cpu().double().numpy() if hasattr(a, "detach") else np.asarray(a, dtype=np.float64)
    b = b.detach().cpu().double().numpy() if hasattr(b, "detach") else np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
