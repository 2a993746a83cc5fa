#!/usr/bin/env python
"""Launch time of the mpjpe and projected-mpjpe loss kernels (forward + gradient), CUDA events.

    python tools/bench_loss_kernels.py [--entry ex|plain] [--reps 7] [--iters 200]

Times the C entry points of the library `_capi` loads (VP3D_LIB_PATH selects another build, e.g.
the parent commit's, to compare; `--entry plain` is then the only entry point it has) at
N x T x J = 1024 x 1 x 17 and 64 x 243 x 17.  Each repetition is `iters` back-to-back calls between
two events; prints one JSON line per case with the median and the range over the repetitions, in
microseconds per call, and the device name and power limit they were measured on.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from videopose3d_b200 import _capi  # noqa: E402


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entry", choices=["ex", "plain"], default="ex")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    # the library alone, with only the signatures used here: an older build lacks the `_ex` entries
    lib = _capi.ctypes.CDLL(_capi.lib_path())
    for name in ("vp3d_mpjpe_fwd_bwd", "vp3d_projected_mpjpe_fwd_bwd") + (
            ("vp3d_mpjpe_scratch_bytes", "vp3d_mpjpe_fwd_bwd_ex", "vp3d_projected_mpjpe_scratch_bytes",
             "vp3d_projected_mpjpe_fwd_bwd_ex") if args.entry == "ex" else ()):
        getattr(lib, name).restype, getattr(lib, name).argtypes = _capi.SIGNATURES[name]
    stream = torch.cuda.current_stream(dev).cuda_stream
    g = torch.Generator().manual_seed(0)
    info = _device_info()
    for n, t, j in ((1024, 1, 17), (64, 243, 17)):
        pred = torch.randn(n, t, j, 3, generator=g).to(dev)
        tgt = torch.randn(n, t, j, 3, generator=g).to(dev)
        traj = (torch.randn(n, t, 1, 3, generator=g) + torch.tensor([0.0, 0.0, 4.5])).to(dev)
        cam = torch.cat([torch.rand(n, 2, generator=g) + 1, torch.randn(n, 7, generator=g) * 0.05], 1).to(dev)
        t2 = torch.randn(n, t, j, 2, generator=g).to(dev)
        loss = torch.empty((), device=dev)
        dpred, dtraj = torch.empty_like(pred), torch.empty_like(traj)
        joints = n * t * j
        if args.entry == "ex":
            s1 = torch.empty(max(1, lib.vp3d_mpjpe_scratch_bytes(joints)), dtype=torch.uint8, device=dev)
            s2 = torch.empty(max(1, lib.vp3d_projected_mpjpe_scratch_bytes(n, t)), dtype=torch.uint8,
                             device=dev)
            calls = {
                "mpjpe": lambda: lib.vp3d_mpjpe_fwd_bwd_ex(
                    pred.data_ptr(), tgt.data_ptr(), None, joints, 3, loss.data_ptr(), dpred.data_ptr(),
                    s1.data_ptr(), s1.numel(), stream),
                "projected_mpjpe": lambda: lib.vp3d_projected_mpjpe_fwd_bwd_ex(
                    pred.data_ptr(), traj.data_ptr(), cam.data_ptr(), t2.data_ptr(), n, t, j, 0,
                    loss.data_ptr(), dpred.data_ptr(), dtraj.data_ptr(), s2.data_ptr(), s2.numel(),
                    stream)}
        else:
            calls = {
                "mpjpe": lambda: lib.vp3d_mpjpe_fwd_bwd(
                    pred.data_ptr(), tgt.data_ptr(), None, joints, 3, loss.data_ptr(), dpred.data_ptr(),
                    stream),
                "projected_mpjpe": lambda: lib.vp3d_projected_mpjpe_fwd_bwd(
                    pred.data_ptr(), traj.data_ptr(), cam.data_ptr(), t2.data_ptr(), n, t, j, 0,
                    loss.data_ptr(), dpred.data_ptr(), dtraj.data_ptr(), stream)}
        for name, call in calls.items():
            for _ in range(20):
                assert call() == 0
            torch.cuda.synchronize(dev)
            times = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    call()
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b) * 1000.0 / args.iters)
            times.sort()
            print(json.dumps({"kernel": name, "shape": [n, t, j], "entry": args.entry,
                              "lib": _capi.lib_path(), "us_median": round(times[len(times) // 2], 3),
                              "us_min": round(times[0], 3), "us_max": round(times[-1], 3),
                              "device": info}), flush=True)


if __name__ == "__main__":
    main()
