"""Float64 restatement of the 'int8' eval forward on a chosen set of residual blocks
(``set_int8_blocks``), the others in fp16.

The int8 blocks are int8_oracle's, formula for formula.  A block outside the set runs as the fp16
forward does: fp16 operands, H and X_i stored in fp16.  The Q_{i-1} an int8 block reads comes
    after the expand or an int8 block: from the epilogue's value v (int8_oracle),
    after an fp16 block: from the STORED fp16 X_{i-1} (the quantise pass, cvt.rni.sat.u8.f32):
        Q = clamp(rint(fp32(fp32(X) * inv_s)), 0, 255)
and is made only where an int8 block reads it.
"""
import numpy as np

import int8_oracle as io
from oracle import temporal_model_oracle as orc

F32 = np.float32


def forward_int8_blocks(sd, x, filter_widths, amax, int8_blocks=None, causal=False, dense=False,
                        strided=False, collect=None):
    """x (N, T, J, F) -> (N, T_out, J_out, 3) float64.  amax: the 2B calibration maxima;
    int8_blocks: the blocks (1..B) that run u8 x s8, None = all (int8_oracle.forward_int8).
    collect: receives X_0, Q_0, then per block H (u8 codes, or fp16 values in an fp16 block), X_i,
    Q_i (numpy, channel-last; None for a Q no int8 block reads)."""
    sd = orc.state_dict_to_numpy(sd, F32)
    a = orc.arch(filter_widths, causal, dense, strided)
    fw = a["widths"]
    nb = len(fw) - 1
    chosen = set(range(1, nb + 1) if int8_blocks is None else int8_blocks)
    int8 = [b in chosen for b in range(1, nb + 2)]   # int8[i]: block i + 1 (False past the last)
    s_act, inv = io.act_scales(amax)
    x = np.asarray(x, np.float64)
    N, T = x.shape[:2]
    bs, bt = io.bn_fold(sd, "expand_bn")
    z = orc._conv_cl(io.f16(x.reshape(N, T, -1)), io.f16(sd["expand_conv.weight"]),
                     stride=fw[0] if strided else 1)
    v = np.maximum(z * bs + bt, 0)
    X, Q = io.f16(v), (io.quant_act(v, inv[0]) if int8[0] else None)
    if collect is not None:
        collect += [X, Q]
    for i in range(nb):
        w = fw[i + 1]

        def conv(t, k):
            if strided:
                return orc._conv_cl(t, k, stride=w)
            return orc._conv_cl(t, k, dilation=a["dilation"][i + 1])

        if strided:
            res = X[:, a["shift"][i + 1] + w // 2:: w, :]
        else:
            pad, sh = a["pad"][i + 1], a["shift"][i + 1]
            res = X[:, pad + sh: X.shape[1] - pad + sh, :]
        if int8[i]:
            sc1, sh1, w1 = io.int8_affine(sd, 2 * i, s_act[2 * i])
            z = conv(Q, w1)
            res = res[:, :z.shape[1], :]
            v = np.maximum(z.astype(F32) * sc1 + sh1, 0)
            H = io.quant_act(v, inv[2 * i + 1])
            sc2, sh2, w2 = io.int8_affine(sd, 2 * i + 1, s_act[2 * i + 1])
            v = np.maximum(orc._conv_cl(H, w2).astype(F32) * sc2 + sh2, 0) + res
            X = io.f16(v)
            Q = io.quant_act(v, inv[2 * i + 2]) if int8[i + 1] else None
        else:
            s1, t1 = io.bn_fold(sd, f"layers_bn.{2 * i}")
            s2, t2 = io.bn_fold(sd, f"layers_bn.{2 * i + 1}")
            z = conv(X, io.f16(sd[f"layers_conv.{2 * i}.weight"]))
            res = res[:, :z.shape[1], :]
            H = io.f16(np.maximum(z * s1 + t1, 0))
            X = io.f16(np.maximum(orc._conv_cl(H, io.f16(sd[f"layers_conv.{2 * i + 1}.weight"]))
                                  * s2 + t2, 0) + res)
            Q = io.quant_act(X, inv[2 * i + 2]) if int8[i + 1] else None
        if collect is not None:
            collect += [H, X, Q]
    y = orc._conv_cl(X, io.f16(sd["shrink.weight"])) + sd["shrink.bias"].astype(np.float64)
    return y.reshape(N, -1, sd["shrink.weight"].shape[0] // 3, 3)
