#!/usr/bin/env python
"""Offline inference on a list of clips: model.predict (a few long GEMM chains over the
concatenated, edge-padded clips) against the per-clip forward that metrics.evaluate runs.

Workloads (arc 3^5, C = 1024, J = 17, test-time flip augmentation, fp16 and int8):
  * metrics: the 240 clips of `bench_extra.py --what stream_seq`, lengths
    RandomState(0).randint(1000, 4001) -- the final evaluation's size;
  * short:   2000 clips, lengths RandomState(0).randint(30, 301) -- in-the-wild 2-D tracks.
Arms:
  (a) per clip: model(b) on the padded (2, T + RF - 1, J, F) batch of the device
      UnchunkedGenerator, then metrics.flip_average, as bench_stream_seq runs it;
  (b) model.predict(clips, augment=True, ...) with the default max_rows.
Per arm: wall time ending in a device synchronise (median of --reps runs after one warm-up, the
two arms alternated in one process), frames/s, launches, TFLOP executed from shapes ((b) counts
every row a chain computes, the discarded rows between clips included), TFLOP/s, workspace bytes,
and whether every clip's output is bit-identical between the arms.  The card's name and power
limit are read in the same run and printed with every line.

    python tools/bench_predict.py [--reps 5] [--what metrics,short] [--precision fp16,int8]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import videopose3d_b200 as vp  # noqa: E402
from bench_extra import ARC, C, F, J, card, emit, offline_flops  # noqa: E402
from videopose3d_b200 import metrics  # noqa: E402
from videopose3d_b200.clips import DEFAULT_MAX_ROWS, clip_tables  # noqa: E402
from videopose3d_b200.generators import UnchunkedGenerator  # noqa: E402

LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
WORKLOADS = {"metrics": (240, 1000, 4001), "short": (2000, 30, 301)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bench(dev, what, precision, reps, info):
    n, lo, hi = WORKLOADS[what]
    lens = np.random.RandomState(0).randint(lo, hi, n)
    frames = int(lens.sum())
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval()
    rf = m.receptive_field()
    pad = (rf - 1) // 2
    rng = np.random.RandomState(1)
    p2 = [rng.uniform(-1, 1, (T, J, F)).astype(np.float32) for T in lens]
    clips = [torch.from_numpy(x).to(dev) for x in p2]
    gen = UnchunkedGenerator(None, None, p2, pad=pad, causal_shift=0, augment=True, kps_left=LEFT,
                             kps_right=RIGHT, device=dev)
    batches = [b for _, _, b in gen.next_epoch()]
    if precision == "int8":
        m.calibrate_int8(batches[:16])
    m.set_precision(precision)
    outs = {}

    def per_clip():
        with torch.no_grad():
            outs["a"] = [metrics.flip_average(m(b), LEFT, RIGHT)[0] for b in batches]

    def chains():
        with torch.no_grad():
            outs["b"] = m.predict(clips, augment=True, kps_left=LEFT, kps_right=RIGHT,
                                  joints_left=LEFT, joints_right=RIGHT)

    per_clip()
    chains()
    ta, tb = [], []
    for _ in range(reps):   # the arms alternate
        ta.append(timed(per_clip))
        tb.append(timed(chains))
    t_a, t_b = float(np.median(ta)), float(np.median(tb))
    launches_a = 0
    ws_a = 0
    lib = vp._capi.load()
    for b in batches:
        with torch.no_grad():
            m(b)
        launches_a += m.last_launch_count() + 1   # + the flip average
        ws_a = max(ws_a, lib.vp3d_workspace_bytes(m._plan, 2, int(b.shape[1])))
    _, _, rows = clip_tables([int(T) for T in lens], rf, True, DEFAULT_MAX_ROWS)
    ws_b = max(lib.vp3d_clips_workspace_bytes(m._plan, r, vp._capi.VP3D_CLIPS_AUGMENT)
               for r in rows)
    fl_a = sum(2 * offline_flops(ARC, C, J * F, J * 3, int(T) + rf - 1) for T in lens)
    fl_b = sum(offline_flops(ARC, C, J * F, J * 3, r) for r in rows)
    equal = all(torch.equal(a, b) for a, b in zip(outs["a"], outs["b"]))
    common = dict(what=what, clips=n, frames=frames, arc=ARC, channels=C, precision=precision,
                  tta=True, reps=reps, bit_equal=equal, **info)
    emit(arm="per_clip_forward_flip_average", seconds=t_a, frames_per_s=frames / t_a,
         launches=launches_a, tflop_executed=fl_a / 1e12, tflops=fl_a / t_a / 1e12,
         workspace_bytes=ws_a, **common)
    emit(arm="predict", chains=len(rows), max_rows=DEFAULT_MAX_ROWS, seconds=t_b,
         frames_per_s=frames / t_b, launches=m.last_predict_launches, tflop_executed=fl_b / 1e12,
         tflops=fl_b / t_b / 1e12, workspace_bytes=ws_b, speedup_over_per_clip=t_a / t_b, **common)
    del outs, batches, clips
    m._engine.workspace = None
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--what", default="metrics,short")
    ap.add_argument("--precision", default="fp16,int8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for what in args.what.split(","):
        for precision in args.precision.split(","):
            bench(dev, what, precision, args.reps, info)


if __name__ == "__main__":
    main()
