#!/usr/bin/env python
"""Fused pose loss vs its torch formulation, forward + backward, on the device.

    python tools/bench_pose_loss.py [--iters 200] [--warmup 20] [--out FILE.json]

Both arms compute mpjpe + n_mpjpe + p_mpjpe + velocity (weights 1, 0.5, 0.5, 1) of a prediction
that requires grad and its gradient:
  fused  videopose3d_b200.loss.pose_loss: one cooperative launch (the backward only scales the
         stored gradient);
  torch  the reference's n_mpjpe (common/loss.py:68-78 restated on torch ops), the torch.linalg.svd
         restatement of p_mpjpe (oracle/pose_loss_oracle.py), a torch.diff velocity, and their
         autograd backward.
Shapes: N = 1024 with T_out = 1 (the training batch of the flagship model) and N = 8 with
T_out = 243, J = 17.  Reports the median over CUDA-event-timed iterations, the kernel launches of
one iteration (torch.profiler), and the GPU's name and power limit read by this process.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pose_loss_oracle as po  # noqa: E402
from videopose3d_b200 import loss as vloss  # noqa: E402

WEIGHTS = (1.0, 0.5, 0.5, 1.0)


def gpu_info():
    """Name and power limit of the GPU, read by this process."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                              "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in out.split(",")[:2]]
    except Exception:
        name, limit = torch.cuda.get_device_name(0), "not read"
    return {"gpu": name, "power_limit": limit}


def torch_loss(y, t):
    return sum(w * fn(y, t) for w, fn in zip(WEIGHTS, po.TERMS))


def fused_loss(y, t):
    return vloss.pose_loss(y, t, *WEIGHTS)[0]


def step(fn, y, t):
    y.grad = None
    fn(y, t).backward()


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    result = dict(gpu_info(), rows=[])
    for N, T in ((1024, 1), (8, 243)):
        g = torch.Generator(device=dev).manual_seed(0)
        t = torch.randn(N, T, 17, 3, device=dev, generator=g) * 0.3
        y = (t + 0.05 * torch.randn(N, T, 17, 3, device=dev, generator=g)).requires_grad_()
        row = {"N": N, "T_out": T, "J": 17}
        for arm, fn in (("fused", fused_loss), ("torch", torch_loss)):
            call = lambda fn=fn: step(fn, y, t)  # noqa: E731
            row[f"{arm}_ms"] = round(median_ms(call, args.iters, args.warmup), 4)
            row[f"{arm}_launches"] = launches(call)
        row["speedup"] = round(row["torch_ms"] / row["fused_ms"], 2)
        result["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
