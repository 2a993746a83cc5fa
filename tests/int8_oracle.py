"""Float64 restatement of the 'int8' eval forward (precision VP3D_PRECISION_INT8).

The quantisation and fold formulas are the kernels' own, in fp32 and in this order:
    activation scale      s = fp32(amax / 255) (1 when amax == 0),  inv_s = fp32(1 / s)
    activation code       q = clamp(rint(fp32(fp32(v) * inv_s)), 0, 255)   (cvt.rni.sat.u8.f32)
    weight scale          s_w[co] = fp32(max_{ci,tap} |W| / 127) (1 for an all-zero channel)
    weight code           q_w = clamp(rint(fp32(W / s_w[co])), -127, 127)
    BatchNorm fold        bn_s = fp32(gamma / sqrt(fp32(var + 1e-5))),  bn_t = beta - mean * bn_s
    int8 affine           scale'[co] = fp32(bn_s * fp32(s_w * s_in))
    block epilogue        v = max(fp32(acc) * scale' + bn_t, 0) [+ X_prev];  X = fp16(v), Q = q(v)
The integer sums are exact here as in the kernels; what this restatement computes in float64 and
the kernels in fp32 is the fp16 expand / shrink and the fma of each epilogue.  Expand writes X_0
and Q_0, each block reads Q_{i-1} and H as u8 and writes X_i (fp16) and Q_i; shrink reads X_B.
"""
import numpy as np

from oracle import temporal_model_oracle as orc

F32 = np.float32


def f16(a):
    return np.clip(np.asarray(a, np.float64), -65504.0, 65504.0).astype(np.float16).astype(np.float64)


def act_scales(amax):
    """(s, inv_s) fp32 arrays of the 2B activation maxima."""
    a = np.asarray(amax, F32)
    s = np.where(a > 0, a / F32(255), F32(1)).astype(F32)
    return s, (F32(1) / s).astype(F32)


def quant_act(v, inv_s):
    return np.clip(np.rint(np.asarray(v, F32) * F32(inv_s)), 0, 255).astype(np.float64)


def quant_weight(w):
    """Conv1d weight (Co, Ci, K) -> (s8 codes as float64 (Co, Ci, K), fp32 scales [Co])."""
    w = np.asarray(w, F32)
    amax = np.abs(w).reshape(w.shape[0], -1).max(axis=1)
    s = np.where(amax > 0, amax / F32(127), F32(1)).astype(F32)
    q = np.clip(np.rint(w / s[:, None, None]), -127, 127)
    return q.astype(np.float64), s


def bn_fold(sd, prefix):
    g, b, m, v = (np.asarray(sd[f"{prefix}.{k}"], F32)
                  for k in ("weight", "bias", "running_mean", "running_var"))
    s = (g / np.sqrt(v + F32(1e-5))).astype(F32)
    return s, b.astype(np.float64) - m.astype(np.float64) * s.astype(np.float64)


def int8_affine(sd, layer, s_in):
    """(scale', shift, s8 codes) of layers_conv.{layer} for an input scale s_in."""
    wq, ws = quant_weight(sd[f"layers_conv.{layer}.weight"])
    bs, bt = bn_fold(sd, f"layers_bn.{layer}")
    return (bs * (ws * F32(s_in)).astype(F32)).astype(F32), bt, wq


def forward_int8(sd, x, filter_widths, amax, causal=False, dense=False, strided=False,
                 collect=None):
    """x (N, T, J, F) -> (N, T_out, J_out, 3) float64.  amax: the 2B calibration maxima.
    collect: receives X_0, Q_0, then per block H (u8 codes), X_i, Q_i (numpy, channel-last)."""
    sd = orc.state_dict_to_numpy(sd, np.float32)
    a = orc.arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    s_act, inv = act_scales(amax)
    x = np.asarray(x, np.float64)
    N, T = x.shape[:2]
    h = x.reshape(N, T, -1)
    bs, bt = bn_fold(sd, "expand_bn")
    z = orc._conv_cl(f16(h), f16(sd["expand_conv.weight"]), stride=fw[0] if strided else 1)
    v = np.maximum(z * bs + bt, 0)
    X, Q = f16(v), quant_act(v, inv[0])
    if collect is not None:
        collect += [X, Q]
    nb = len(fw) - 1
    for i in range(nb):
        w = fw[i + 1]
        sc1, sh1, w1 = int8_affine(sd, 2 * i, s_act[2 * i])
        if strided:
            res = X[:, a["shift"][i + 1] + w // 2:: w, :]
            z = orc._conv_cl(Q, w1, stride=w)
            res = res[:, :z.shape[1], :]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = X[:, pad + sh: X.shape[1] - pad + sh, :]
            z = orc._conv_cl(Q, w1, dilation=a["dilation"][i + 1])
        v = np.maximum(z.astype(F32) * sc1 + sh1, 0)
        H = quant_act(v, inv[2 * i + 1])
        sc2, sh2, w2 = int8_affine(sd, 2 * i + 1, s_act[2 * i + 1])
        z = orc._conv_cl(H, w2)
        v = np.maximum(z.astype(F32) * sc2 + sh2, 0) + res
        X = f16(v)
        Q = quant_act(v, inv[2 * i + 2]) if i + 1 < nb else None
        if collect is not None:
            collect += [H, X, Q]
    y = orc._conv_cl(X, f16(sd["shrink.weight"])) + sd["shrink.bias"].astype(np.float64)
    return y.reshape(N, -1, sd["shrink.weight"].shape[0] // 3, 3)


def calibrate(sd, x, filter_widths, causal=False, dense=False, strided=False):
    """The 2B maxima of the fp16 forward's stored activations (X_{i-1}, H_i per block), float64
    restated: what vp3d_calibrate_int8 measures up to the fp32 accumulation of the fp16 GEMMs."""
    sd = orc.state_dict_to_numpy(sd, np.float32)
    a = orc.arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    x = np.asarray(x, np.float64)
    N, T = x.shape[:2]
    bs, bt = bn_fold(sd, "expand_bn")
    X = f16(np.maximum(orc._conv_cl(f16(x.reshape(N, T, -1)), f16(sd["expand_conv.weight"]),
                                    stride=fw[0] if strided else 1) * bs + bt, 0))
    amax = []
    for i in range(len(fw) - 1):
        w = fw[i + 1]
        amax.append(X.max())
        s1, t1 = bn_fold(sd, f"layers_bn.{2 * i}")
        s2, t2 = bn_fold(sd, f"layers_bn.{2 * i + 1}")
        if strided:
            res = X[:, a["shift"][i + 1] + w // 2:: w, :]
            z = orc._conv_cl(X, f16(sd[f"layers_conv.{2 * i}.weight"]), stride=w)
            res = res[:, :z.shape[1], :]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = X[:, pad + sh: X.shape[1] - pad + sh, :]
            z = orc._conv_cl(X, f16(sd[f"layers_conv.{2 * i}.weight"]), dilation=a["dilation"][i + 1])
        H = f16(np.maximum(z * s1 + t1, 0))
        amax.append(H.max())
        X = f16(np.maximum(orc._conv_cl(H, f16(sd[f"layers_conv.{2 * i + 1}.weight"])) * s2 + t2, 0)
                + res)
    return np.asarray(amax, F32)
