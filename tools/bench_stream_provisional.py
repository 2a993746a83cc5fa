#!/usr/bin/env python
"""Streaming with provisional outputs (push(..., provisional=True)): what a push costs that also
returns the look-ahead frames as finish() would give them now, against a plain push and against the
user's alternative of recomputing a window.

Arc 3,3,3,3,3 (look-ahead 121), C = 1024, fp16, J = 17, F = 2, k = 1, S in {1, 4, 16, 64, 256},
plain and with test-time flip augmentation.  CUDA events around every arm, median and p99 over
--pushes pushes after --warmup warm-up pushes, the arms alternated in one loop:
  (a) a plain push;
  (b) a push with provisional outputs (a session made with provisional=True);
  (c) what a user does without them: model(windows) on S windows of RF frames, the newest frame
      edge-padded over the look-ahead (the dependency-cone schedule of the offline forward; with
      augment the 2S plain and mirrored windows and the flip average), then a plain push.
FLOPs from shapes: a push computes k x P physical rows (P = S, 2S with augment) of the per-frame
chain, a provisional push (k + 121) x P, a window one output frame over its dependency cone.

Before timing, every configuration drives a fresh provisional session and checks the provisional
rows of up to four slots at three pushes bit for bit against the offline forward on the frames
pushed so far.  One JSON line per configuration and arm.

    python tools/bench_stream_provisional.py [--pushes 500] > provisional.jsonl
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
from videopose3d_b200 import metrics  # noqa: E402
from videopose3d_b200.generators import UnchunkedGenerator  # noqa: E402

ARC, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
STREAMS = [1, 4, 16, 64, 256]
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
LISTS = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [v.strip() for v in out.split(",")[:2]]
    return {"gpu": name, "power_limit": limit}


def stage_flops():
    """FLOPs of one output frame of each stage: the expand conv, every block (its k-tap conv and
    its 1x1 conv) and the shrink."""
    flops = [2 * ARC[0] * J * F * C]
    flops += [2 * w * C * C + 2 * C * C for w in ARC[1:]]
    flops.append(2 * C * J * 3)
    return flops


def frame_flops():
    return sum(stage_flops())


def cone_flops():
    """One output frame from RF input frames: stage i computes prod(ARC[i + 1:]) frames."""
    fl = stage_flops()
    return sum(fl[i] * math.prod(ARC[i + 1:]) for i in range(len(ARC))) + fl[-1]


def offline(m, x, augment):
    pad = (m.receptive_field() - 1) // 2
    if not augment:
        xp = np.pad(x.cpu().numpy(), ((pad, pad), (0, 0), (0, 0)), "edge")
        with torch.no_grad():
            return m(torch.from_numpy(xp)[None].to(x.device))[0]
    gen = UnchunkedGenerator(None, None, [x.cpu().numpy()], pad=pad, causal_shift=0, augment=True,
                             kps_left=LEFT, kps_right=RIGHT, device=x.device)
    with torch.no_grad():
        for _, _, b in gen.next_epoch():
            return metrics.flip_average(m(b), LEFT, RIGHT)[0]


def check_exact(m, dev, S, augment, at=(3, 60, 130)):
    """A fresh provisional session fed one frame per push; slots 0-3 at the pushes `at` against
    the offline forward on the frames pushed so far."""
    sess = m.streaming(streams=S, max_frames=1, augment=augment, provisional=True,
                       **(LISTS if augment else {}))
    xs = torch.rand(S, max(at) + 1, J, F, device=dev) * 2 - 1
    checked = 0
    for i in range(max(at) + 1):
        _, _, yp, fp = sess.push(xs[:, i:i + 1], start=[True] * S if i == 0 else None,
                                 provisional=True)
        if i not in at:
            continue
        fp = fp.cpu().numpy()
        for s in range(min(S, 4)):
            ref = offline(m, xs[s, :i + 1], augment)
            for j in np.nonzero(fp[s] >= 0)[0]:
                assert torch.equal(yp[s, j], ref[int(fp[s, j])]), (S, augment, i, s, j)
                checked += 1
    return checked


def stats(ms):
    t = np.sort(np.asarray(ms))
    return float(np.median(t)), float(t[min(len(t) - 1, int(math.ceil(0.99 * len(t))) - 1)])


def bench(dev, pushes, warmup):
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    rf = m.receptive_field()
    la = vp.streaming.lookahead(m)
    info = card()
    for augment in (False, True):
        lists = LISTS if augment else {}
        for S in STREAMS:
            n_checked = check_exact(m, dev, S, augment)
            emit(what="check", streams=S, augment=augment, frames_checked=n_checked,
                 bit_exact=True, **info)
            P = 2 * S if augment else S
            xs = torch.rand(S, 1, J, F, device=dev) * 2 - 1
            # the user's windows: the last RF - la frames, the newest repeated over the look-ahead
            win = torch.rand(S, rf, J, F, device=dev) * 2 - 1
            win[:, rf - la:] = win[:, rf - la - 1:rf - la]
            if augment:
                mir = win.clone()
                mir[..., 0] *= -1
                mir[:, :, LEFT + RIGHT] = mir[:, :, RIGHT + LEFT]
                win = torch.cat([win, mir])
            a = m.streaming(streams=S, max_frames=1, augment=augment, **lists)
            b = m.streaming(streams=S, max_frames=1, augment=augment, provisional=True, **lists)
            c = m.streaming(streams=S, max_frames=1, augment=augment, **lists)

            def window_arm():
                out = m(win)
                if augment:
                    metrics.flip_average(out.view(2, S, J, 3), LEFT, RIGHT)
                c.push(xs)

            arms = {"a": lambda: a.push(xs), "b": lambda: b.push(xs, provisional=True),
                    "c": window_arm}
            with torch.no_grad():
                for s in (a, b, c):
                    s.push(xs, start=[True] * S)
                ev = {n: [] for n in arms}
                for i in range(warmup + pushes):
                    for n, fn in arms.items():
                        e0 = torch.cuda.Event(enable_timing=True)
                        e1 = torch.cuda.Event(enable_timing=True)
                        e0.record()
                        fn()
                        e1.record()
                        if i >= warmup:
                            ev[n].append((e0, e1))
                launches = {}
                for n in ("a", "b"):
                    arms[n]()
                    launches[n] = a.last_launch_count()
                c.push(xs)
                launches["c"] = c.last_launch_count()
            torch.cuda.synchronize()
            flops = {"a": P * frame_flops(), "b": (1 + la) * P * frame_flops(),
                     "c": P * cone_flops() + P * frame_flops()}
            med_a, _ = stats([e0.elapsed_time(e1) for e0, e1 in ev["a"]])
            for n in arms:
                med, p99 = stats([e0.elapsed_time(e1) for e0, e1 in ev[n]])
                row = dict(what="stream_provisional", arm=n, streams=S, k=1, augment=augment,
                           precision="fp16", arc=ARC, channels=C, lookahead=la, pushes=pushes,
                           warmup=warmup, ms_median=med, ms_p99=p99, over_plain_ms=med - med_a,
                           gflop=flops[n] / 1e9, tflops_at_median=flops[n] / med / 1e9,
                           launches=launches[n] if n != "c" else None,
                           push_launches=launches[n] if n == "c" else None, **info)
                emit(**row)
            del a, b, c, arms
            torch.cuda.empty_cache()


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_provisional needs a CUDA device")
    bench(torch.device("cuda", 0), args.pushes, args.warmup)


if __name__ == "__main__":
    main()
