"""The launch schedule of an 'int8' plan whose block mask (``set_int8_blocks``) leaves some residual
blocks in fp16, restated in torch on eval_replay's pieces (Plan, packs, Launch, descriptors).

``replay_blocks(sd, cfg, x, gemm, amax, int8_blocks)`` runs what ``run_infer_chain`` runs:
the input pack and the fp16 expand (writing Q_0 only when block 1 is int8); per int8 block the two
u8 x s8 GEMMs of eval_replay's "int8" schedule; per fp16 block the two GEMMs of its "fp16" schedule
(fp16 packs, K per tap C, the plain BatchNorm affine), and, where the next block is int8, the
quantise pass that makes Q_i from the stored fp16 X_i (``Replay.quants``, computed with
``eval_replay.quant_u8``); the fp16 shrink.  Every GEMM goes to `gemm` (``eval_replay.gpu_gemm`` or
``fake_gemm``), so with ``gpu_gemm`` the output is the model's bit for bit.  With every block in
the set it is eval_replay.replay(..., "int8"); with none, its "fp16" schedule.
"""
import torch

import eval_replay as er


def replay_blocks(sd, cfg, x, gemm, amax, int8_blocks=None):
    """Returns an ``eval_replay.Replay`` with ``quants`` [(block i, stored X_i, Q_i, inv_s)] of the
    quantise passes, counted in ``launch_count``; acts X_0 [, Q_0], then per block H_i, X_i
    [, Q_i], the Q's present where an int8 block reads them."""
    N, T = int(x.shape[0]), int(x.shape[1])
    p = er.Plan(cfg, er.INT8, N, T)
    int8 = [False] + [int8_blocks is None or i in set(int8_blocks) for i in range(1, p.nb + 2)]
    int8[p.nb + 1] = False   # (no block past the last)
    st = er.Storage(p, False, x.device)
    pk = er.pack_weights(sd, p, st)
    er.pack_int8(sd, p, amax, pk, x.device)
    # an fp16 block's convs: the fp16 plan's packs and affine (same C, same single fp16 plane)
    pk16 = er.pack_weights(sd, er.Plan(cfg, "fp16", N, T), st)
    for j in range(2 * p.nb):
        if not int8[j // 2 + 1]:
            pk[f"conv{j}"], pk[f"aff{j}"] = pk16[f"conv{j}"], pk16[f"aff{j}"]
    fw, C, L, R, nb = p.fw, p.C, p.L, p.R, p.nb
    xs = x.reshape(N, T, p.c_in_raw).float()
    launches, acts, quants = [], [], []

    def run(name, desc, a, w, aff, res=None, out=None, out_f32=None, out_u8=None, inv_s=None):
        lc = er.Launch(name, desc, a, w, aff[0], aff[1], res=res, out=out, out_f32=out_f32,
                       out_u8=out_u8, inv_s=inv_s)
        gemm(lc)
        launches.append(lc)

    def empty_u8(rows):
        return torch.full((1, rows, C), 255, dtype=torch.uint8, device=x.device)

    # ---- input pack + expand (as eval_replay.replay)
    if p.strided:
        k0 = fw[0] * p.c_in_raw
        vals = torch.zeros(N * L[0], p.k0_pad, dtype=xs.dtype, device=x.device)
        vals[p.region_rows(0).to(x.device).flatten(), :k0] = \
            xs[:, :L[0] * fw[0]].reshape(N * L[0], k0)
        desc = er.new_desc(samples=1, a_rows=N * L[0], a_ld=p.k0_pad, taps=1, k_per_tap=p.k0_pad,
                           per_sample_tiles=0, out_rows=N * L[0])
        w0 = pk["expand_flat"]
    else:
        vals = torch.zeros(N * T, p.c_in_pad, dtype=xs.dtype, device=x.device)
        vals[:, :p.c_in_raw] = xs.reshape(N * T, p.c_in_raw)
        desc = er.new_desc(samples=N, a_rows=T, a_ld=p.c_in_pad, taps=fw[0], k_per_tap=p.c_in_pad,
                           per_sample_tiles=1, tap_row_step=1, out_rows=L[0])
        w0 = pk["expand_dil"]
    a0 = st.planes_of(vals, 1)
    desc.update(a_planes=1, precision=er.K_FP16, out_planes=1, res_planes=1, relu=1, n_pad=C,
                out_ld=C, out_plane_stride=R[0] * C)
    xcur = st.empty(1, R[0], C)
    qcur = empty_u8(R[0]) if int8[1] else None
    run("expand", desc, a0, w0, pk["expand_aff"], out=xcur, out_u8=qcur,
        inv_s=pk["inv_s"][0] if qcur is not None else None)
    acts.append(("X0", 0, xcur))
    if qcur is not None:
        acts.append(("Q0", 0, qcur))

    # ---- residual blocks
    for i in range(1, nb + 1):
        Lin, Lout = L[i - 1], L[i]
        h = empty_u8(N * Lout) if int8[i] else st.empty(1, N * Lout, C)
        desc = er.new_desc(a_planes=1, precision=er.K_FP16, out_planes=1, res_planes=1,
                           taps=p.taps[i], k_per_tap=C, n_pad=C, relu=1,
                           out_plane_stride=N * Lout * C, out_ld=C, a_ld=C)
        if p.strided:
            desc.update(tap_row_step=R[i], samples=1, a_rows=N * Lin, per_sample_tiles=0,
                        out_rows=N * Lout)
        else:
            desc.update(samples=N, a_rows=Lin, per_sample_tiles=1, tap_row_step=p.dilation[i],
                        out_rows=Lout)
        if int8[i]:   # Q_{i-1} x s8 -> H, u8 alone (the K per tap padded to 128)
            desc.update(precision=er.K_INT8, k_per_tap=p.k_conv, out_plane_stride=0)
            run(f"block {i} conv 1", desc, qcur, pk[f"conv{2 * (i - 1)}"],
                pk[f"aff{2 * (i - 1)}"], out_u8=h, inv_s=pk["inv_s"][2 * (i - 1) + 1])
        else:
            run(f"block {i} conv 1", desc, xcur, pk[f"conv{2 * (i - 1)}"],
                pk[f"aff{2 * (i - 1)}"], out=h)
        acts.append((f"H{i}", i, h))

        xnext = st.empty(1, N * Lout, C)
        desc = er.new_desc(a_planes=1, precision=er.K_FP16, out_planes=1, res_planes=1, samples=1,
                           a_rows=N * Lout, a_ld=C, taps=1, k_per_tap=C, n_pad=C,
                           per_sample_tiles=0, out_rows=N * Lout, relu=1,
                           out_plane_stride=N * Lout * C, out_ld=C)
        if p.strided:
            desc.update(res_row_step=1, res_row_off=(fw[i] // 2 + p.shift_str[i]) * R[i])
        else:
            desc.update(samples=N, a_rows=Lout, per_sample_tiles=1, out_rows=Lout,
                        res_rows_per_sample=Lin, res_row_step=1,
                        res_row_off=p.pad[i] + p.shift_dil[i])
        qnext = None
        if int8[i]:   # H x s8 + X_{i-1} -> X_i in fp16 [+ Q_i from the epilogue]
            desc.update(precision=er.K_INT8, k_per_tap=p.k_conv)
            qnext = empty_u8(N * Lout) if int8[i + 1] else None
        run(f"block {i} conv 2", desc, h, pk[f"conv{2 * (i - 1) + 1}"],
            pk[f"aff{2 * (i - 1) + 1}"], res=xcur, out=xnext, out_u8=qnext,
            inv_s=pk["inv_s"][2 * i] if qnext is not None else None)
        if int8[i + 1] and not int8[i]:   # the quantise pass: Q_i from the stored fp16 X_i
            qnext = er.quant_u8(xnext[0].float(), pk["inv_s"][2 * i]).unsqueeze(0)
            quants.append((i, xnext, qnext, pk["inv_s"][2 * i]))
        acts.append((f"X{i}", i, xnext))
        if qnext is not None:
            acts.append((f"Q{i}", i, qnext))
        xcur, qcur = xnext, qnext

    # ---- fp16 shrink into fp32 (N, L_out, J_out, 3)
    y = torch.full((R[nb], p.c_out_raw), float("nan"), dtype=torch.float32, device=x.device)
    desc = er.new_desc(a_planes=1, precision=er.K_FP16, out_planes=1, res_planes=1, samples=1,
                       a_rows=R[nb], a_ld=C, taps=1, k_per_tap=C, n_pad=p.c_out_pad,
                       per_sample_tiles=0, out_rows=R[nb], out_f32_ld=p.c_out_raw,
                       n_valid=p.c_out_raw)
    run("shrink", desc, xcur, pk["shrink"], pk["shrink_aff"], out_f32=y)
    rep = er.Replay(p, y.reshape(N, L[nb], p.c_out_raw // 3, 3), launches, acts)
    rep.quants = quants
    rep.launch_count += len(quants)
    return rep
