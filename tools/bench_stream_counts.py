#!/usr/bin/env python
"""Streaming with per-slot frame counts (StreamingSession.push's `count`): what a push costs when
some slots have fewer than k frames, against a plain push and against one session per arrival group.

Arc 3,3,3,3,3, C = 1024, fp16, J = 17, F = 2.  CUDA events around every push, median and p99 over
--pushes pushes after 50 warm-up pushes, the arms alternated in one loop:
  (a) a plain push, every slot full (count=None);
  (b) a counted push (count a device int32 tensor, drawn before the loop): at k = 1 a fraction p of
      the slots, a different random set every push, gets count 0 and the rest k; at k = 16 every
      slot's count is uniform in [0, 16];
  (c) for p > 0, what a user does without counts: one session per arrival group, timed as the
      pushes of the groups that have frames in this push.  At k = 1 that is one session of S - pS
      slots (the group without a frame waits); at k = 16 it is 16 sessions of ceil(S / 17) slots,
      session n pushing n frames.  This is a lower bound: real groups cannot be regrouped per push.
Realign bytes per realigned physical row, from shapes: 4 * sum_l H_l * ld_l * planes * 2 B.

Before timing, every configuration drives a fresh counted session for a few hundred pushes with the
same count policy and checks four slots bit for bit against the offline forward on the frames they
were fed.  One JSON line per configuration and arm.

    python tools/bench_stream_counts.py [--pushes 500] > counts.jsonl
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
from videopose3d_b200.streaming import ring_history  # noqa: E402

ARC, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
CONFIGS = [(16, 1), (256, 1), (1024, 1), (256, 16)]
FRACTIONS = [0.0, 0.1, 0.5]


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [v.strip() for v in out.split(",")[:2]]
    return {"gpu": name, "power_limit": limit}


def realign_bytes_per_row(planes=1):
    hist = ring_history(ARC)
    c_in = -(-J * F // 64) * 64
    c = -(-C // 64) * 64
    return sum(4 * h * (c_in if i == 0 else c) * planes * 2 for i, h in enumerate(hist))


def draw_counts(rng, S, k, p):
    """One push's counts: uniform in [0, k] for k > 1, else a random fraction p of the slots at 0."""
    if k > 1:
        return rng.randint(0, k + 1, S).astype(np.int32)
    n = np.full(S, k, np.int32)
    n[rng.permutation(S)[:int(round(p * S))]] = 0
    return n


def offline(m, x):
    pad = (m.receptive_field() - 1) // 2
    xp = np.pad(x.cpu().numpy(), ((pad, pad), (0, 0), (0, 0)), "edge")
    with torch.no_grad():
        return m(torch.from_numpy(xp)[None].to(x.device))[0]


def check_exact(m, dev, S, k, p, pushes, seed):
    """A fresh session under the count policy; slots 0-3 against the offline forward."""
    rng = np.random.RandomState(seed)
    la = vp.streaming.lookahead(m)
    sess = m.streaming(streams=S, max_frames=k)
    watch = 4
    fed = [[] for _ in range(watch)]
    got = [{} for _ in range(watch)]
    for i in range(pushes):
        x = torch.rand(S, k, J, F, device=dev) * 2 - 1
        n = draw_counts(rng, S, k, p)
        if i == 0:
            n[n == 0] = 1
        y, frame = sess.push(x, start=[True] * S if i == 0 else None,
                             count=torch.from_numpy(n).to(dev))
        fr = frame[:watch].cpu().numpy()
        for s in range(watch):
            fed[s].append(x[s, :int(n[s])])
            for f in np.nonzero(fr[s] >= 0)[0]:
                got[s][int(fr[s, f])] = y[s, f]
    checked = 0
    for s in range(watch):
        xs = torch.cat(fed[s])
        T = len(xs)
        assert sorted(got[s]) == list(range(T - la)), (S, k, p, s)
        if T - la > 0:
            ref = offline(m, xs)[:T - la]
            assert torch.equal(torch.stack([got[s][t] for t in range(T - la)]), ref), (S, k, p, s)
            checked += T - la
    return checked


def stats(ms):
    t = np.sort(np.asarray(ms))
    return float(np.median(t)), float(t[min(len(t) - 1, int(math.ceil(0.99 * len(t))) - 1)])


def bench(dev, pushes, warmup):
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    info = card()
    row_bytes = realign_bytes_per_row()
    for S, k in CONFIGS:
        fractions = FRACTIONS if k == 1 else [None]
        for p in fractions:
            n_checked = check_exact(m, dev, S, k, p or 0.0, 300 if k == 1 else 40, seed=S + k)
            emit(what="check", streams=S, k=k, p=p, frames_checked=n_checked, bit_exact=True,
                 **info)
        rng = np.random.RandomState(S * 100 + k)
        xs = torch.rand(S, k, J, F, device=dev) * 2 - 1
        a = m.streaming(streams=S, max_frames=k)
        b = m.streaming(streams=S, max_frames=k)
        arms = {}   # name -> fn(i), the arm's push i
        arms["a"] = lambda i: a.push(xs)
        groups = {}
        total = warmup + pushes
        for p in fractions:
            counts = [draw_counts(rng, S, k, p or 0.0) for _ in range(total)]
            dev_counts = [torch.from_numpy(n).to(dev) for n in counts]
            arms[f"b_{p}"] = (lambda dc: lambda i: b.push(xs, count=dc[i]))(dev_counts)
            arms[f"b_{p}"].rows = float(np.mean([(n < k).sum() for n in counts]))
            if p == 0.0:
                continue
            if k == 1:
                size = S - int(round(p * S))
                sessions = [(m.streaming(streams=size, max_frames=1), xs[:size])]
            else:
                size = -(-S // (k + 1))
                sessions = [(m.streaming(streams=size, max_frames=n), xs[:size, :n])
                            for n in range(1, k + 1)]
            groups[p] = sessions
            arms[f"c_{p}"] = (lambda ss: lambda i: [s.push(x) for s, x in ss])(sessions)
        with torch.no_grad():
            a.push(xs, start=[True] * S)
            b.push(xs, start=[True] * S)
            for ss in groups.values():
                for s, x in ss:
                    s.push(x, start=[True] * s.streams)
            names = list(arms)
            ev = {n: [] for n in names}
            for i in range(total):
                for n in names:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    arms[n](i)
                    e1.record()
                    if i >= warmup:
                        ev[n].append((e0, e1))
            # launches per arm, read right after each push: every session of the model shares
            # the plan, which counts the launches of the last push of any of them
            launches = {}
            for n in names:
                if n[0] == "c":
                    launches[n] = 0
                    for sess, x in groups[None if n.endswith("None") else float(n[2:])]:
                        sess.push(x)
                        launches[n] += sess.last_launch_count()
                else:
                    arms[n](total - 1)
                    launches[n] = a.last_launch_count()
        torch.cuda.synchronize()
        med_a, _ = stats([e0.elapsed_time(e1) for e0, e1 in ev["a"]])
        for n in names:
            med, p99 = stats([e0.elapsed_time(e1) for e0, e1 in ev[n]])
            row = dict(what="stream_counts", arm=n[0], streams=S, k=k, precision="fp16", arc=ARC,
                       channels=C, pushes=pushes, warmup=warmup, push_ms_median=med,
                       push_ms_p99=p99, l2_flush="none", **info)
            row["launches"] = launches[n]
            if n[0] != "a":
                p = None if n.endswith("None") else float(n[2:])
                row["p"] = p
            if n[0] == "b":
                rows = arms[n].rows
                row.update(realigned_rows_mean=rows,
                           realign_bytes_per_row=row_bytes,
                           realign_mb_per_push=rows * row_bytes / 1e6,
                           over_plain_ms=med - med_a)
            if n[0] == "c":
                row["sessions"] = len(groups[p])
            emit(**row)
        del a, b, groups, arms
        torch.cuda.empty_cache()


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_counts needs a CUDA device")
    bench(torch.device("cuda", 0), args.pushes, args.warmup)


if __name__ == "__main__":
    main()
