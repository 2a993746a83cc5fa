#!/usr/bin/env python
"""The int8 eval precision against fp16 on the bench model.

    python tools/bench_int8.py [--steps 20] [--warmup 5] [--runs 3] [--json OUT]

TemporalModel arc 3,3,3,3,3, C = 1024, N = 1024, T = 243 (bench.py's model, seeds and input) on
device tensors: calibration time (one calibrate_int8 call on the batch), then fp16 and int8
forwards alternated, `runs` timed windows each (CUDA events around `steps` forwards), then the
per-launch device times of both precisions (vp3d_profile_launch, programmatic dependent launch off
so that every launch is timed alone) with each GEMM's rate: TFLOP/s for fp16 against 989, TOPS for
the int8 block GEMMs against 1,979 (dense data-sheet peaks).  The card's name and power limit are
read in the same run.

Last, the final evaluation of run.py (metrics.evaluate) on 240 synthetic sequences of 1000-4000
frames with test-time augmentation (the workload of `tools/bench_extra.py --what metrics`): host wall
time of the whole evaluate() in each precision, and the protocol #1 error (MPJPE, mm) of both, int8
calibrated on the first 8 sequences.
"""
import argparse
import json
import os
import sys
import time

os.environ["VP3D_PDL"] = "0"   # (read by the library at its first launch)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import ctypes

    import torch

    import bench
    import videopose3d_b200 as vp
    from eval_launch_times import card_info, strided_launches
    from oracle import temporal_model_oracle as orc
    from videopose3d_b200 import _capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_int8.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    J, F, C, N, T, ARC = bench.J, bench.F, bench.C, bench.N_PER_GPU, bench.T, bench.ARC
    name, power = card_info()
    sd = orc.make_state_dict(J, F, J, ARC, C, seed=0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, causal=False, dropout=0.25, channels=C)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = orc.make_input(N, T, J, F, seed=1).to(dev)
    out = {"card": name, "power_limit_w": power, "N": N, "T": T, "C": C, "arc": ARC}

    # calibration (the fp16 plan packs its weights on the first call: time the second)
    m.calibrate_int8(x)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.calibrate_int8(x)
    torch.cuda.synchronize()
    out["calibrate_ms"] = (time.perf_counter() - t0) * 1e3

    def window(precision):
        m.set_precision(precision)
        with torch.no_grad():
            for _ in range(args.warmup):
                m(x)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                m(x)
            b.record()
            b.synchronize()
        return a.elapsed_time(b) / args.steps

    times = {"fp16": [], "int8": []}
    for _ in range(args.runs):
        for p in ("fp16", "int8"):
            times[p].append(window(p))
    out["forward_ms"] = times
    with torch.no_grad():
        m.set_precision("fp16"); y16 = m(x)
        m.set_precision("int8"); y8 = m(x)
    ref = torch.from_numpy(orc.forward_numpy(sd, x[:64].cpu().numpy(), ARC, strided=True)).float()
    scale = float(ref.abs().max())
    out["rel_err_vs_fp64_first64"] = {
        "fp16": float((y16[:64].cpu() - ref).abs().max()) / scale,
        "int8": float((y8[:64].cpu() - ref).abs().max()) / scale}

    lib = _capi.load()
    launches = strided_launches(ARC, C, N, T, J, F, J)
    per = {}
    for p in ("fp16", "int8"):
        m.set_precision(p)
        rows = []
        with torch.no_grad():
            m(x)
            for k, (label, M, Nn, K) in enumerate(launches):
                lib.vp3d_profile_launch(m._plan, k)
                for _ in range(args.steps):
                    m(x)
                ms, cnt = ctypes.c_float(), ctypes.c_int()
                _capi.check(lib.vp3d_profile_read(m._plan, ctypes.byref(ms), ctypes.byref(cnt)),
                            "vp3d_profile_read")
                t = ms.value / max(cnt.value, 1)
                block = label.startswith("block")   # (C = 1024: the same K in int8)
                rate = 2.0 * M * Nn * K / (t * 1e-3) / 1e12 if M else 0.0
                peak = 1979.0 if (p == "int8" and block) else 989.0
                rows.append({"launch": label, "ms": t, "rate_T": rate,
                             "share_of_peak": rate / peak if M else 0.0})
            lib.vp3d_profile_launch(m._plan, -1)
        per[p] = rows
    out["launches"] = per

    # run.py's final evaluation, fp16 against int8
    import numpy as np
    from videopose3d_b200 import metrics
    from videopose3d_b200.generators import UnchunkedGenerator
    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    lens = np.random.RandomState(0).randint(1000, 4001, 240)
    rng = np.random.RandomState(1)
    p2 = [rng.uniform(-1, 1, (n, J, F)).astype(np.float32) for n in lens]
    p3 = [rng.normal(0, 0.25, (n, J, 3)).astype(np.float32) for n in lens]
    pad = m.receptive_field() // 2
    gen = UnchunkedGenerator(None, p3, p2, pad=pad, causal_shift=0, augment=True, kps_left=left,
                             kps_right=right, joints_left=left, joints_right=right, device=dev)
    calib = []
    for _, _, b2 in gen.next_epoch():
        calib.append(b2.clone())
        if len(calib) == 8:
            break
    m.calibrate_int8(calib)
    ev = {"sequences": int(len(lens)), "frames": int(lens.sum())}
    for p in ("fp16", "int8", "fp16", "int8"):
        m.set_precision(p)
        metrics.evaluate(m, gen, left, right)   # warm (plans, workspace)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e = metrics.evaluate(m, gen, left, right)
        torch.cuda.synchronize()
        ev.setdefault(p, {"wall_s": [], "mpjpe_mm": e[0]})["wall_s"].append(time.perf_counter() - t0)
    ev["p1_difference_mm"] = abs(ev["int8"]["mpjpe_mm"] - ev["fp16"]["mpjpe_mm"])
    out["evaluate"] = ev
    print(json.dumps(out, indent=1))
    for p in ("fp16", "int8"):
        print(f"{p}: forward {min(times[p]):.3f} ms (runs {', '.join(f'{v:.3f}' for v in times[p])})")
        for r in per[p]:
            print(f"  {r['launch']:<22} {r['ms'] * 1e3:8.1f} us  {r['rate_T']:7.1f} T/s  "
                  f"{100 * r['share_of_peak']:5.1f}% of peak")
    print(f"evaluate(): fp16 {ev['fp16']['wall_s']} s, P1 {ev['fp16']['mpjpe_mm']:.4f} mm; "
          f"int8 {ev['int8']['wall_s']} s, P1 {ev['int8']['mpjpe_mm']:.4f} mm; "
          f"difference {ev['p1_difference_mm']:.4f} mm")
    print(f"calibration {out['calibrate_ms']:.2f} ms; card {name}, power limit {power} W")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
