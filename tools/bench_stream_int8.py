#!/usr/bin/env python
"""int8 streaming sessions (model.streaming(..., int8=True)) against fp16 sessions of the same model.

Arc 3,3,3,3,3, C = 1024, J = 17, F = 2 (random weights, make_state_dict seed 0), int8 calibrated
(amax) on a (4, 400) random batch.  Pushes:
  * plain, (S, k) in (1, 1), (16, 1), (256, 1), (1024, 1), (256, 16);
  * provisional (k = 1 plus the 121 look-ahead rows), S in 16, 64, 256, without and with test-time
    flip augmentation.
Per configuration one fp16 and one int8 session, their pushes alternated in one loop, CUDA events
around every push: median and p99 over --pushes pushes after --warmup.  Launches per push, and the
work from shapes: fp16 GFLOP (expand, shrink and, in fp16, the blocks) and int8 GOP (the blocks
in int8), each over the median time.

Before timing, every configuration feeds a fresh int8 session 40 frames (k per push) and finish(),
and checks slots 0-3 bit for bit against the offline int8 forward on the edge-padded sequence (the
flip average with augment); once, the int8 forward's error against the float64 oracle on those
frames.  With --profile, torch.profiler then times each kernel of a few pushes of both sessions of
the compute-bound configurations (a separate phase, after every timing).  The card's name and power
limit are read in the same run.  One JSON line per row.

    python tools/bench_stream_int8.py [--pushes 300] [--warmup 30] [--profile] > int8.jsonl
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
from oracle import temporal_model_oracle as orc  # noqa: E402
from videopose3d_b200 import metrics  # noqa: E402
from videopose3d_b200.generators import UnchunkedGenerator  # noqa: E402

ARC, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
PLAIN = [(1, 1), (16, 1), (256, 1), (1024, 1), (256, 16)]
PROV = [16, 64, 256]
PROFILE = [("plain", 1024, 1, False), ("plain", 256, 16, False), ("provisional", 256, 1, False)]
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
LISTS = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [v.strip() for v in out.split(",")[:2]]
    return {"gpu": name, "power_limit": limit}


def work(rows):
    """(fp16 FLOPs, int8 ops) of `rows` physical frame rows of the chain of an int8 session: expand
    and shrink in fp16, every block (its k-tap and 1x1 convs) in int8."""
    edge = 2 * ARC[0] * J * F * C + 2 * C * J * 3
    blocks = sum(2 * w * C * C + 2 * C * C for w in ARC[1:])
    return rows * edge, rows * blocks


def offline(m, x, augment):
    pad = (m.receptive_field() - 1) // 2
    if not augment:
        xp = np.pad(x.cpu().numpy(), ((pad, pad), (0, 0), (0, 0)), "edge")
        with torch.no_grad():
            return m(torch.from_numpy(xp)[None].to(x.device))[0], xp
    gen = UnchunkedGenerator(None, None, [x.cpu().numpy()], pad=pad, causal_shift=0, augment=True,
                             kps_left=LEFT, kps_right=RIGHT, device=x.device)
    with torch.no_grad():
        for _, _, b in gen.next_epoch():
            return metrics.flip_average(m(b), LEFT, RIGHT)[0], None


def check_exact(m, dev, S, k, augment, T=40):
    """A fresh int8 session fed T frames k per push, then finish(); slots 0-3 against the offline
    int8 forward.  Returns the frames checked and the padded inputs of the plain slots."""
    sess = m.streaming(streams=S, max_frames=k, augment=augment, int8=True,
                       **(LISTS if augment else {}))
    xs = torch.rand(S, T, J, F, device=dev) * 2 - 1
    rows = {s: {} for s in range(min(S, 4))}

    def collect(y, frame):
        frame = frame.cpu().numpy()
        for s in rows:
            for f in np.nonzero(frame[s] >= 0)[0]:
                rows[s][int(frame[s, f])] = y[s, f]

    for i in range(0, T, k):
        collect(*sess.push(xs[:, i:i + k], start=[True] * S if i == 0 else None,
                           end=[T - i] * S if i + k >= T else None))
    collect(*sess.finish())
    padded = []
    for s in rows:
        ref, xp = offline(m, xs[s], augment)
        assert sorted(rows[s]) == list(range(T)), (S, k, augment, s)
        assert torch.equal(torch.stack([rows[s][t] for t in range(T)]), ref), (S, k, augment, s)
        padded.append(xp)
    return len(rows) * T, padded


def stats(ms):
    t = np.sort(np.asarray(ms))
    return float(np.median(t)), float(t[min(len(t) - 1, int(math.ceil(0.99 * len(t))) - 1)])


def configs():
    for S, k in PLAIN:
        yield "plain", S, k, False
    for augment in (False, True):
        for S in PROV:
            yield "provisional", S, 1, augment


def sessions(models, kind, S, k, augment):
    prov = kind == "provisional"
    kw = dict(streams=S, max_frames=k, augment=augment, provisional=prov,
              **(LISTS if augment else {}))
    return {p: models[p].streaming(int8=p == "int8", **kw) for p in ("fp16", "int8")}


def bench(dev, pushes, warmup, profile):
    sd = orc.make_state_dict(J, F, J, ARC, C, seed=0)
    models = {}
    for p in ("fp16", "int8"):
        m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C)
        m.load_state_dict(sd)
        models[p] = m.to(dev).eval()
    models["int8"].calibrate_int8(orc.make_input(4, 400, J, F, seed=1).to(dev))
    models["int8"].set_precision("int8")
    la = vp.streaming.lookahead(models["int8"])
    info = card()
    err_done = False
    for kind, S, k, augment in configs():
        n_checked, padded = check_exact(models["int8"], dev, S, k, augment)
        row = dict(what="check", kind=kind, streams=S, k=k, augment=augment,
                   frames_checked=n_checked, bit_exact=True, **info)
        if not err_done and padded[0] is not None:
            # the int8 (and fp16) forward on the checked frames against the float64 oracle
            xp = np.stack(padded)
            ref = orc.forward_numpy(sd, xp, ARC, dtype=np.float64)
            for p in ("fp16", "int8"):
                with torch.no_grad():
                    y = models[p](torch.from_numpy(xp).to(dev)).cpu().numpy()
                row[f"{p}_rel_err_max"] = float(np.abs(y - ref).max() / np.abs(ref).max())
                row[f"{p}_mean_joint_dist"] = float(np.linalg.norm(y - ref, axis=-1).mean())
            err_done = True
        emit(**row)
        sess = sessions(models, kind, S, k, augment)
        prov = kind == "provisional"
        xs = torch.rand(S, k, J, F, device=dev) * 2 - 1
        P = 2 * S if augment else S
        rows = (k + (la if prov else 0)) * P
        with torch.no_grad():
            for s in sess.values():
                s.push(xs, start=[True] * S)
            ev = {p: [] for p in sess}
            for i in range(warmup + pushes):
                for p, s in sess.items():
                    e0 = torch.cuda.Event(enable_timing=True)
                    e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    s.push(xs, provisional=prov)
                    e1.record()
                    if i >= warmup:
                        ev[p].append((e0, e1))
            torch.cuda.synchronize()
        for p, s in sess.items():
            med, p99 = stats([e0.elapsed_time(e1) for e0, e1 in ev[p]])
            f16, i8 = work(rows)
            if p == "fp16":
                f16, i8 = f16 + i8, 0
            emit(what="stream_int8", kind=kind, precision=p, streams=S, k=k, augment=augment,
                 lookahead=la if prov else 0, frame_rows=rows, arc=ARC, channels=C,
                 pushes=pushes, warmup=warmup, ms_median=med, ms_p99=p99,
                 launches=s.last_launch_count(), fp16_gflop=f16 / 1e9, int8_gop=i8 / 1e9,
                 fp16_tflops_at_median=f16 / med / 1e9, int8_tops_at_median=i8 / med / 1e9,
                 **info)
        del sess
        torch.cuda.empty_cache()
    if profile:
        for kind, S, k, augment in PROFILE:
            profile_kernels(models, dev, kind, S, k, augment, info)


def profile_kernels(models, dev, kind, S, k, augment, info, n=20):
    """Per-kernel device time of n pushes of each session (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    sess = sessions(models, kind, S, k, augment)
    prov = kind == "provisional"
    xs = torch.rand(S, k, J, F, device=dev) * 2 - 1
    with torch.no_grad():
        for p, s in sess.items():
            s.push(xs, start=[True] * S)
            for _ in range(5):
                s.push(xs, provisional=prov)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(n):
                    s.push(xs, provisional=prov)
                torch.cuda.synchronize()
            for e in prof.key_averages():
                if e.device_type.name != "CUDA" or e.count == 0:
                    continue
                emit(what="kernel", kind=kind, precision=p, streams=S, k=k, augment=augment,
                     kernel=e.key[:120], calls_per_push=e.count / n,
                     us_per_push=e.self_device_time_total / n, **info)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_int8 needs a CUDA device")
    bench(torch.device("cuda", 0), args.pushes, args.warmup, args.profile)


if __name__ == "__main__":
    main()
