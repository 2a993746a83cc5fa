#!/usr/bin/env python
"""Streaming fed by a 2-D detector (StreamingSession.push_detections): what a call costs when the
session interpolates and normalises missed detections itself, against a plain push of frames the
user already normalised.

Arc 3,3,3,3,3, C = 1024, fp16, J = 17, F = 2, K = 1 (one video frame per slot and call), S in
{16, 256}.  Every slot misses a frame with probability p in {0, 0.1, 0.3}, in gaps of geometric
length (mean 3 frames), drawn before the loop; max_gap None (exact: a gap waits for the next
detection, then comes out as a burst of catch-up pushes) and 8.  CUDA events around every call,
median and p99 over --calls calls after --warmup warm-up calls, the two arms alternated in one loop:
  (a) plain: sess.push(x) of already-normalised frames, every slot full;
  (b) detections: sess.push_detections(kps_px, detected) of the same frames in pixels.
Per configuration also: launches, internal pushes per call and realigned (slot, push) pairs per
call, means over the timed calls.  The card's name and power limit are read in the same run.

    python tools/bench_stream_detections.py [--calls 500] [--warmup 50] > detections.jsonl
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import videopose3d_b200 as vp  # noqa: E402

ARC, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
STREAMS = [16, 256]
MISS = [0.0, 0.1, 0.3]
GAPS = [None, 8]
W, H = 1920, 1080


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [v.strip() for v in out.split(",")[:2]]
    return {"gpu": name, "power_limit": limit}


def draw_mask(rng, S, n, p):
    """(n, S) detected flags: after each detected frame a gap starts with probability p, its
    length geometric with mean 3 frames; frame 0 is detected."""
    det = np.ones((n, S), bool)
    for s in range(S):
        t = 1
        while t < n:
            if rng.rand() < p:
                g = int(rng.geometric(1 / 3))
                det[t:t + g, s] = False
                t += g
            t += 1
    return det


def stats(ms):
    t = np.sort(np.asarray(ms))
    return float(np.median(t)), float(t[min(len(t) - 1, int(math.ceil(0.99 * len(t))) - 1)])


def emit(**kw):
    print(json.dumps(kw), flush=True)


def bench(dev, calls, warmup):
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    info = card()
    total = warmup + calls
    for S in STREAMS:
        rng = np.random.RandomState(S)
        px = (torch.rand(S, 1, J, F, device=dev) * torch.tensor([W, H], device=dev)).contiguous()
        xn = px.clone()
        xn[..., 0] = px[..., 0] / W * 2 - 1
        xn[..., 1] = px[..., 1] / W * 2 - H / W
        res = [(W, H)] * S
        for p in MISS:
            mask = draw_mask(rng, S, total + 1, p)
            for gap in GAPS:
                a = m.streaming(streams=S, max_frames=1)
                b = m.streaming(streams=S, max_frames=1, detections=True, max_gap=gap)
                with torch.no_grad():
                    a.push(xn, start=[True] * S)
                    b.push_detections(px, mask[0][:, None], [True] * S, None, res)
                    ev = {"a": [], "b": []}
                    pushes = launches = realigned = 0
                    for i in range(total):
                        for n in ("a", "b"):
                            e0 = torch.cuda.Event(enable_timing=True)
                            e1 = torch.cuda.Event(enable_timing=True)
                            e0.record()
                            if n == "a":
                                a.push(xn)
                            else:
                                b.push_detections(px, mask[i + 1][:, None])
                            e1.record()
                            if i >= warmup:
                                ev[n].append((e0, e1))
                        if i >= warmup:
                            pushes += b.last_call_pushes
                            launches += b.last_call_launches
                            realigned += b.last_call_realigned
                    a.push(xn)
                    plain_launches = a.last_launch_count()
                torch.cuda.synchronize()
                med_a, p99_a = stats([e0.elapsed_time(e1) for e0, e1 in ev["a"]])
                med_b, p99_b = stats([e0.elapsed_time(e1) for e0, e1 in ev["b"]])
                emit(what="stream_detections", streams=S, k=1, p=p, max_gap=gap, precision="fp16",
                     arc=ARC, channels=C, calls=calls, warmup=warmup,
                     missed_fraction=float(1 - mask[1:total + 1].mean()),
                     plain_ms_median=med_a, plain_ms_p99=p99_a, plain_launches=plain_launches,
                     detections_ms_median=med_b, detections_ms_p99=p99_b,
                     launches_per_call=launches / calls, pushes_per_call=pushes / calls,
                     realigned_per_call=realigned / calls, over_plain_ms=med_b - med_a,
                     l2_flush="none", **info)
                del a, b
                torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_detections needs a CUDA device")
    bench(torch.device("cuda", 0), args.calls, args.warmup)


if __name__ == "__main__":
    main()
