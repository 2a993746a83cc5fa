#!/usr/bin/env python
"""Provisional poses in detector-fed sessions (push_detections(..., provisional=True)): what a call
costs when it also returns finish()'s rows for the look-ahead and for the frames pending after each
slot's last detection, against the same call without the request.

Arc 3,3,3,3,3 (look-ahead 121, receptive field 243), C = 1024, fp16, J = 17, F = 2, K = 1 (one
video frame per slot and call), S in {1, 16, 64}.  Every slot misses a frame with probability p in
{0, 0.2}, in gaps of geometric length (mean 3 frames), drawn before the loop; max_gap G in
{0, 15, 60}.  CUDA events around every call, median and p99 over --calls calls after --warmup
warm-up calls, the two arms alternated in one loop:
  (a) plain: push_detections on a session made without provisional=True;
  (b) provisional: push_detections(..., provisional=True) on a session made with it.
Per configuration also: launches per call of both arms, the mean and largest last_call_prov_rows
(tail rows computed: min(121 + max pending, 242)) and the state bytes of both sessions.  Before
timing, a fresh provisional session is driven through the first calls of the same mask and its
last provisional rows are checked bit for bit against finish() on a twin fed the same calls.
The card's name and power limit are read in the same run.

    python tools/bench_stream_detections_provisional.py [--calls 300] [--warmup 30] > out.jsonl
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
STREAMS = [1, 16, 64]
MISS = [0.0, 0.2]
GAPS = [0, 15, 60]
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


def session(m, S, gap, provisional):
    kw = dict(provisional=True) if provisional else {}
    return m.streaming(streams=S, max_frames=1, detections=True, max_gap=gap, **kw)


def check_exact(m, S, gap, px, mask, res, n):
    """Drive a provisional session and a twin without the flag through calls 0..n-1; the last
    call's provisional rows of slots 0, S // 2 and S - 1 must be the twin's finish() rows."""
    a, b = session(m, S, gap, True), session(m, S, gap, False)
    for i in range(n):
        st = [True] * S if i == 0 else None
        r = res if i == 0 else None
        _, _, yp, fp = a.push_detections(px, mask[i][:, None], st, None, r, provisional=True)
        b.push_detections(px, mask[i][:, None], st, None, r)
    yf, ff = b.finish()
    fp, ff = fp.cpu().numpy(), ff.cpu().numpy()
    checked = 0
    for s in sorted({0, S // 2, S - 1}):
        fin = {int(t): i for i, t in enumerate(ff[s]) if t >= 0}
        got = {int(t): i for i, t in enumerate(fp[s]) if t >= 0}
        assert sorted(got) == sorted(fin), (S, gap, s)
        for t, j in got.items():
            assert torch.equal(yp[s, j], yf[s, fin[t]]), (S, gap, s, t)
            checked += 1
    return checked


def bench(dev, calls, warmup):
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    info = card()
    total = warmup + calls
    for S in STREAMS:
        rng = np.random.RandomState(S)
        px = (torch.rand(S, 1, J, F, device=dev) * torch.tensor([W, H], device=dev)).contiguous()
        res = [(W, H)] * S
        for p in MISS:
            mask = draw_mask(rng, S, total + 1, p)
            for gap in GAPS:
                with torch.no_grad():
                    checked = check_exact(m, S, gap, px, mask, res, 160)
                    a, b = session(m, S, gap, False), session(m, S, gap, True)
                    a.push_detections(px, mask[0][:, None], [True] * S, None, res)
                    b.push_detections(px, mask[0][:, None], [True] * S, None, res,
                                      provisional=True)
                    ev = {"a": [], "b": []}
                    launches = {"a": 0, "b": 0}
                    prov_rows = []
                    for i in range(total):
                        for n in ("a", "b"):
                            e0 = torch.cuda.Event(enable_timing=True)
                            e1 = torch.cuda.Event(enable_timing=True)
                            e0.record()
                            if n == "a":
                                a.push_detections(px, mask[i + 1][:, None])
                            else:
                                b.push_detections(px, mask[i + 1][:, None], provisional=True)
                            e1.record()
                            if i >= warmup:
                                ev[n].append((e0, e1))
                                launches[n] += (a if n == "a" else b).last_call_launches
                        if i >= warmup:
                            prov_rows.append(b.last_call_prov_rows)
                torch.cuda.synchronize()
                med_a, p99_a = stats([e0.elapsed_time(e1) for e0, e1 in ev["a"]])
                med_b, p99_b = stats([e0.elapsed_time(e1) for e0, e1 in ev["b"]])
                emit(what="stream_detections_provisional", streams=S, k=1, p=p, max_gap=gap,
                     precision="fp16", arc=ARC, channels=C, calls=calls, warmup=warmup,
                     rows_checked=checked, missed_fraction=float(1 - mask[1:total + 1].mean()),
                     plain_ms_median=med_a, plain_ms_p99=p99_a,
                     provisional_ms_median=med_b, provisional_ms_p99=p99_b,
                     over_plain_ms=med_b - med_a,
                     plain_launches_per_call=launches["a"] / calls,
                     provisional_launches_per_call=launches["b"] / calls,
                     prov_rows_mean=float(np.mean(prov_rows)), prov_rows_max=int(max(prov_rows)),
                     plain_state_bytes=a._state.numel(), provisional_state_bytes=b._state.numel(),
                     l2_flush="none", **info)
                del a, b
                torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_detections_provisional needs a CUDA device")
    bench(torch.device("cuda", 0), args.calls, args.warmup)


if __name__ == "__main__":
    main()
