#!/usr/bin/env python
"""Per-launch device times of the eval forward that bench.py measures.

    python tools/eval_launch_times.py [--precision fp16] [--steps 30] [--warmup 10] [--json OUT]

Same model, seeds and inputs as bench.py (TemporalModel arc 3,3,3,3,3, C = 1024, N = 1024,
T = 243, L2 flushed between steps).  The timed steps run under torch.profiler with CUDA
activities; each launch's mean device time over the steps is printed with the FLOPs of the GEMM
it runs (computed from the shapes, K and N as launched, i.e. padded to the tile) and the rate,
together with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def strided_launches(arc, c, n, t, j_in, f_in, j_out):
    """(label, M, N, K) of every launch of the strided eval forward, in launch order; the input
    pack has no GEMM (M = N = K = 0)."""
    pad64 = lambda v: (v + 63) // 64 * 64   # noqa: E731
    out = [("input pack", 0, 0, 0)]
    frames = t // arc[0]
    out.append(("expand", n * frames, pad64(c), pad64(arc[0] * j_in * f_in)))
    for i, w in enumerate(arc[1:], start=1):
        frames //= w
        out.append((f"block {i} {w}-tap conv", n * frames, pad64(c), w * pad64(c)))
        out.append((f"block {i} 1x1 conv", n * frames, pad64(c), pad64(c)))
    out.append(("shrink", n * frames, pad64(j_out * 3), pad64(c)))
    return out


def card_info():
    """(name, power limit in W) of cuda:0, read through NVML or nvidia-smi's query."""
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return name, pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    try:
        import subprocess
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        return name, float(r.stdout.strip().splitlines()[0])
    except Exception:
        return name, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="fp16", choices=["fp16", "bf16", "mixed", "bf16x3"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import videopose3d_b200 as vp
    from oracle import temporal_model_oracle as orc

    if not torch.cuda.is_available():
        raise SystemExit("eval_launch_times.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    J, F, C, N, T, ARC = bench.J, bench.F, bench.C, bench.N_PER_GPU, bench.T, bench.ARC
    sd = orc.make_state_dict(J, F, J, ARC, C, seed=0)
    model = vp.TemporalModel(J, F, J, filter_widths=ARC, causal=False, dropout=0.25, channels=C)
    model.load_state_dict(sd)
    model = model.to(dev).eval().set_precision(args.precision)
    n_buf = 8
    xs = [orc.make_input(N, T, J, F, seed=100 + i).to(dev) for i in range(n_buf)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    shapes = strided_launches(ARC, C, N, T, J, F, J)
    with torch.no_grad():
        model(xs[0])
        torch.cuda.synchronize()
        per_step = model.last_launch_count()
        if per_step != len(shapes):
            raise SystemExit(f"the forward made {per_step} launches, expected {len(shapes)}")
        for i in range(args.warmup):
            flush.zero_()
            model(xs[i % n_buf])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.steps):
                flush.zero_()
                model(xs[i % n_buf])
            torch.cuda.synchronize()
    name, power_w = card_info()

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kernels = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"),
                     key=lambda e: e["ts"])
    # the L2 flush is a PyTorch kernel; everything else belongs to the forward
    ours = [e for e in kernels if "at::" not in e["name"]]
    if len(ours) != per_step * args.steps:
        raise SystemExit(f"{len(ours)} forward kernels in the trace, expected {per_step * args.steps}")
    rows = []
    total_ms = 0.0
    for k, (label, m, n, kk) in enumerate(shapes):
        evs = ours[k::per_step]
        kname = evs[0]["name"]
        if any(e["name"] != kname for e in evs):
            raise SystemExit(f"launch {k} ran different kernels in different steps")
        ms = sum(e["dur"] for e in evs) / len(evs) / 1e3
        flops = 2.0 * m * n * kk
        total_ms += ms
        short = kname.replace("void ", "").replace("vp3d::", "").split("(")[0]
        rows.append({"launch": k, "what": label, "kernel": short, "M": m, "N": n, "K": kk,
                     "ms": ms, "gflop": flops / 1e9, "tflops": flops / (ms * 1e-3) / 1e12 if flops else None})
    gflop = sum(r["gflop"] for r in rows)

    print(f"card: {name}, power limit: {power_w if power_w is not None else 'unknown'} W; "
          f"precision {args.precision}; mean of {args.steps} profiled steps (L2 flushed between steps)")
    print(f"{'#':>2}  {'launch':<20} {'kernel':<56} {'M x N x K':<22} {'ms':>7} {'GFLOP':>7} {'TFLOP/s':>8}")
    for r in rows:
        shape = f"{r['M']} x {r['N']} x {r['K']}" if r["M"] else "-"
        tf = f"{r['tflops']:8.1f}" if r["tflops"] else f"{'-':>8}"
        print(f"{r['launch']:>2}  {r['what']:<20} {r['kernel']:<56} {shape:<22} {r['ms']:7.4f} "
              f"{r['gflop']:7.1f} {tf}")
    print(f"    {'sum of launches':<20} {'':<56} {'':<22} {total_ms:7.4f} {gflop:7.1f} "
          f"{gflop / total_ms:8.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit_w": power_w, "precision": args.precision,
                       "steps": args.steps, "launches": rows, "sum_ms": total_ms}, f, indent=1)


if __name__ == "__main__":
    main()
