#!/usr/bin/env python
"""Moving streaming slots between sessions (StreamingSession.export_slots / import_slots): what an
export and an import of n slots cost, against the bytes they have to move.

Arc 3,3,3,3,3, C = 1024, J = 17, F = 2, in fp16 and in int8 with augment (every block int8).  The
source session has S = 256 slots and K = 1, the destination S = 256 and K = 4; both have pushed
enough frames to hold history in every slot.  n in {1, 16, 256} slots.  CUDA events around each call
(export: vp3d_stream_export, one launch; import: vp3d_stream_import, one launch), median and p90
over --reps calls after --warmup warm-up calls.  Bytes from shapes: a slot record is
vp3d_stream_slot_bytes; export reads the record's history once and writes the record, import reads
the record and writes both mirror copies of the history.  Achieved GB/s is those bytes over the
median time, shown against the 3.35 TB/s of an H100 SXM's HBM3.  The card's name and power limit are
read in the same run.

    python tools/bench_stream_migrate.py [--reps 200] [--warmup 20] > migrate.jsonl
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import videopose3d_b200 as vp  # noqa: E402
from videopose3d_b200 import _capi  # noqa: E402

ARC, C, J, F = [3, 3, 3, 3, 3], 1024, 17, 2
S_SRC, K_SRC, S_DST, K_DST = 256, 1, 256, 4
NS = [1, 16, 256]
HBM = 3.35e12
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
MODES = {"fp16": dict(precision="fp16", augment=False), "int8_augment": dict(precision="int8",
                                                                              augment=True)}


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [v.strip() for v in out.split(",")[:2]]
    return {"gpu": name, "power_limit": limit}


def model(dev, precision):
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, causal=False, dropout=0.0, channels=C)
    m = m.to(dev).eval()
    if precision == "int8":
        m.calibrate_int8(torch.rand(2, m.receptive_field() + 16, J, F, device=dev) * 2 - 1)
    return m.set_precision(precision)


def session(m, S, K, augment, int8):
    lists = dict(kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT) \
        if augment else {}
    sess = m.streaming(streams=S, max_frames=K, augment=augment, int8=int8, **lists)
    dev = m.expand_conv.weight.device
    for i in range(8):
        sess.push(torch.rand(S, K, J, F, device=dev) * 2 - 1, start=[i == 0] * S)
    return sess


def history_bytes(m, augment, int8):
    """Bytes of one slot's history (every ring, plane and physical row), from shapes."""
    hist = vp.streaming.ring_history(ARC)
    c_in = -(-J * F // 64) * 64
    planes = 2 if m.precision == "bf16x3" else 1
    b = sum(h * (c_in if i == 0 else C) * 2 * planes + (h * C if int8 and i > 0 else 0)
            for i, h in enumerate(hist))
    return b * (2 if augment else 1)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
          for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = np.array([a.elapsed_time(b) for a, b in ev]) * 1e-3
    return float(np.median(t)), float(np.percentile(t, 90))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_migrate needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = card()
    lib = _capi.load()
    with torch.no_grad():
        for name, mode in MODES.items():
            int8 = mode["precision"] == "int8"
            m = model(dev, mode["precision"])
            src = session(m, S_SRC, K_SRC, mode["augment"], int8)
            dst = session(m, S_DST, K_DST, mode["augment"], int8)
            slot = lib.vp3d_stream_slot_bytes(src._plan, src._flags)
            hist = history_bytes(m, mode["augment"], int8)
            assert slot == 32 + hist, (slot, hist)
            for n in NS:
                slots = list(range(n))
                state = src.export_slots(slots)
                assert src.last_launch_count() == 1
                ex = timed(lambda: src.export_slots(slots), args.reps, args.warmup)
                im = timed(lambda: dst.import_slots(state, slots), args.reps, args.warmup)
                assert dst.last_launch_count() == 1
                for op, (med, p90), moved in (("export", ex, n * (hist + slot)),
                                              ("import", im, n * (slot + 2 * hist))):
                    print(json.dumps(dict(
                        info, mode=name, op=op, slots=n, slot_bytes=slot, bytes=moved,
                        median_ms=round(med * 1e3, 4), p90_ms=round(p90 * 1e3, 4),
                        gb_s=round(moved / med / 1e9, 1),
                        share_of_hbm=round(moved / med / HBM, 3))), flush=True)


if __name__ == "__main__":
    main()
