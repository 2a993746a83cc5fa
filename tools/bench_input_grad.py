#!/usr/bin/env python
"""Cost of the input gradient and of eval-mode autograd (H100; prints one JSON line per arm).

    python tools/bench_input_grad.py [--reps 20] [--warmup 5]

(a) TemporalModelOptimized1f training step, arc 3^5, C 1024, N 1024, T 243, bf16: forward +
    backward with x.requires_grad off vs on (the expand conv's data gradient).
(b) Test-time refinement step: TemporalModel in eval(), arc 3^5, C 1024, x (2, 2242, 17, 2)
    requiring grad, parameters frozen: forward + backward, against the reference's class in eval()
    on the same GPU (cuDNN fp32, TF32 at torch's defaults).
(c) (b) with every parameter requiring grad: a frozen-BatchNorm fine-tune step.

Arms alternate within every repetition; times are CUDA-event medians of forward + backward.  The
reference is read only through oracle.stage_ref.reference_dir()."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import videopose3d_b200 as vp  # noqa: E402
from oracle import stage_ref  # noqa: E402
from oracle import temporal_model_oracle as orc  # noqa: E402

ARC = [3, 3, 3, 3, 3]


def card():
    """Name and power limit of the GPU, read by this process."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                              "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in out.split(",")[:2]]
    except Exception:
        name, limit = torch.cuda.get_device_name(0), "not read"
    return {"gpu": name, "power_limit": limit}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def run(arms, reps, warmup):
    """{arm: (median ms, launches)}; arms alternate inside every repetition."""
    for _ in range(warmup):
        for fn, _ in arms.values():
            fn()
    ev = {k: [] for k in arms}
    launches = {}
    for _ in range(reps):
        for k, (fn, count) in arms.items():
            ev[k].append(timed(fn))
            launches[k] = count()   # the backward just run (the arms share nothing else)
    torch.cuda.synchronize()
    out = {}
    for k in arms:
        ms = sorted(a.elapsed_time(b) for a, b in ev[k])
        out[k] = (ms[len(ms) // 2], launches[k])
    return out


def step(m, x, gy, x_grad, p_grad):
    for p in m.parameters():
        p.requires_grad_(p_grad)
        p.grad = None
    xd = x.detach().requires_grad_(x_grad)
    (m(xd) * gy).sum().backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    info = card()
    print(json.dumps(info), flush=True)
    sd = orc.make_state_dict(17, 2, 17, ARC, 1024, seed=3)

    # (a) training step, input gradient off / on
    m = vp.TemporalModelOptimized1f(17, 2, 17, ARC, dropout=0.25, channels=1024)
    m.load_state_dict(sd)
    m = m.to(dev).train().set_train_precision("bf16")
    x = orc.make_input(1024, 243, seed=4).to(dev)
    gy = torch.randn(1024, 1, 17, 3, device=dev)
    res = run({"train_x_off": (lambda: step(m, x, gy, False, True), m.last_launch_count),
               "train_x_on": (lambda: step(m, x, gy, True, True), m.last_launch_count)},
              args.reps, args.warmup)
    for k, (ms, n) in res.items():
        print(json.dumps(dict(info, arm=k, ms=round(ms, 3), backward_launches=n)), flush=True)

    # (b), (c) eval-mode refinement / frozen-BatchNorm fine-tune against the reference class
    ref = stage_ref.import_reference()
    tm = vp.TemporalModel(17, 2, 17, ARC, channels=1024)
    tm.load_state_dict(sd)
    tm = tm.to(dev).eval()
    x = orc.make_input(2, 2000 + 242, seed=5).to(dev)
    gy = torch.randn(2, 2000, 17, 3, device=dev)
    arms = {"refine_ours": (lambda: step(tm, x, gy, True, False), tm.last_launch_count),
            "finetune_ours": (lambda: step(tm, x, gy, True, True), tm.last_launch_count)}
    if ref is not None:
        rm = ref.TemporalModel(17, 2, 17, ARC, channels=1024)
        rm.load_state_dict(sd)
        rm = rm.to(dev).eval()
        arms["refine_reference"] = (lambda: step(rm, x, gy, True, False), lambda: None)
        arms["finetune_reference"] = (lambda: step(rm, x, gy, True, True), lambda: None)
    res = run(arms, args.reps, args.warmup)
    for k, (ms, n) in res.items():
        print(json.dumps(dict(info, arm=k, ms=round(ms, 3), backward_launches=n)), flush=True)


if __name__ == "__main__":
    main()
