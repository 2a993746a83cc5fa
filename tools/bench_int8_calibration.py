#!/usr/bin/env python
"""Int8 calibration methods (TemporalModel.calibrate_int8(method=...)) on the bench model.

    python tools/bench_int8_calibration.py [--repeats 5] [--eval 64] [--json OUT]

TemporalModel arc 3,3,3,3,3, C = 1024 (bench.py's model and seeds), on device tensors:

1. Calibration time per method (host clock around calibrate_int8, which ends in a device-to-host
   copy): on the bench batch (N = 1024, T = 243), and on the 240 synthetic sequences of 1000-4000
   frames with flip augmentation of tools/bench_int8.py's evaluate() workload, through the device
   UnchunkedGenerator.  Each first call (weight packing, workspace) is untimed.
2. The histogram kernel's per-launch device time (torch.profiler, CUDA activity, its own run).
3. Accuracy per method: the int8 forward against the float64 one on `--eval` held-out bench-batch
   sequences (max |d| / max |ref| and the mean joint distance, x1000 as mm), calibrated on 128
   clean sequences and on the same 128 with about 1 % of the frames scaled by 20 to 50
   (int8_calib_ref.inject_glitches); and the protocol #1 error (MPJPE, mm) of evaluate() on the
   240-sequence workload in int8 (calibrated on its first 8 batches) minus the fp16 one.
4. The int8 forward time on the bench batch (CUDA events), one calibration per method: a sanity
   check that the calibration changes no kernel.

The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

METHODS = ("amax", "percentile", "mse")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--eval", type=int, default=64)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import int8_calib_ref as cr
    import videopose3d_b200 as vp
    from eval_launch_times import card_info
    from oracle import temporal_model_oracle as orc
    from videopose3d_b200 import metrics
    from videopose3d_b200.generators import UnchunkedGenerator

    if not torch.cuda.is_available():
        raise SystemExit("bench_int8_calibration.py needs a CUDA device")
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

    def timed(inputs, method, repeats):
        m.calibrate_int8(inputs, method=method)
        ts = []
        for _ in range(repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.calibrate_int8(inputs, method=method)
            ts.append((time.perf_counter() - t0) * 1e3)
        return ts

    out["calibrate_ms_bench_batch"] = {k: timed(x, k, args.repeats) for k in METHODS}

    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    lens = np.random.RandomState(0).randint(1000, 4001, 240)
    rng = np.random.RandomState(1)
    p2 = [rng.uniform(-1, 1, (n, J, F)).astype(np.float32) for n in lens]
    p3 = [rng.normal(0, 0.25, (n, J, 3)).astype(np.float32) for n in lens]
    gen = UnchunkedGenerator(None, p3, p2, pad=m.receptive_field() // 2, causal_shift=0,
                             augment=True, kps_left=left, kps_right=right, joints_left=left,
                             joints_right=right, device=dev)
    out["calibrate_ms_240_sequences"] = {k: timed(gen, k, 2) for k in METHODS}

    # the histogram kernel alone
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.calibrate_int8(x, method="percentile")
        torch.cuda.synchronize()
    hist_us = [e.device_time for e in prof.events() if "hist_f16_kernel" in e.name]
    amax_us = [e.device_time for e in prof.events() if "amax_f16_kernel" in e.name]
    out["hist_kernel_us"] = hist_us
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.calibrate_int8(x, method="amax")
        torch.cuda.synchronize()
    out["amax_kernel_us"] = [e.device_time for e in prof.events() if "amax_f16_kernel" in e.name]
    assert not amax_us

    # accuracy against float64 on held-out sequences, clean and glitched calibration sets
    xe = x[N - args.eval:]
    ref = orc.forward_numpy(sd, xe.cpu().numpy(), ARC, strided=True)
    xc = x[:128].cpu().numpy()
    xg = torch.from_numpy(cr.inject_glitches(xc, seed=6)).to(dev)
    acc = {}
    m.set_precision("int8")
    for cal_name, cal in (("clean", x[:128]), ("glitch", xg)):
        for k in METHODS:
            m.calibrate_int8(cal, method=k)
            with torch.no_grad():
                y = m(xe).cpu().numpy()
            e_max, e_joint = cr.int8_errors(y, ref)
            acc[f"{cal_name}_{k}"] = {"rel_max": e_max, "joint_mm": 1e3 * e_joint,
                                      "thresholds": m.int8_calibration().tolist()}
    out["accuracy_vs_fp64"] = acc

    # protocol #1 on the 240-sequence workload, int8 per method minus fp16
    calib = []
    for _, _, b2 in gen.next_epoch():
        calib.append(b2.clone())
        if len(calib) == 8:
            break
    m.set_precision("fp16")
    p1 = {"fp16": metrics.evaluate(m, gen, left, right)[0]}
    m.set_precision("int8")
    fwd = {}
    for k in METHODS:
        m.calibrate_int8(calib, method=k)
        p1[k] = metrics.evaluate(m, gen, left, right)[0]
        with torch.no_grad():
            for _ in range(3):
                m(x)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20):
                m(x)
            b.record()
            b.synchronize()
        fwd[k] = a.elapsed_time(b) / 20
    out["p1_mm"] = p1
    out["p1_difference_from_fp16_mm"] = {k: p1[k] - p1["fp16"] for k in METHODS}
    out["int8_forward_ms"] = fwd

    print(json.dumps(out, indent=1))
    for k in METHODS:
        b, s = out["calibrate_ms_bench_batch"][k], out["calibrate_ms_240_sequences"][k]
        print(f"{k:<10} calibrate: bench batch {min(b):8.2f} ms, 240 sequences {min(s):9.1f} ms; "
              f"int8 forward {fwd[k]:.3f} ms; P1 - fp16 {out['p1_difference_from_fp16_mm'][k]:+.4f} mm")
        for c in ("clean", "glitch"):
            r = acc[f"{c}_{k}"]
            print(f"           {c:<6} calibration: max|d|/max|ref| {r['rel_max']:.3e}, mean joint "
                  f"distance {r['joint_mm']:.3f} mm")
    print(f"hist kernel per launch (us): {[round(v, 1) for v in hist_us]}; amax kernel: "
          f"{[round(v, 1) for v in out['amax_kernel_us']]}")
    print(f"card {name}, power limit {power} W")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
