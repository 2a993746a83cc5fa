#!/usr/bin/env python
"""Speed and accuracy of the int8 precision per block set (set_int8_blocks) on the bench model.

    python tools/bench_int8_blocks.py [--steps 10] [--warmup 3] [--rounds 3] [--json OUT]

TemporalModel arc 3,3,3,3,3, C = 1024 (bench.py's model and seeds), calibrated with "amax" on the
N = 1024, T = 243 batch.  Block sets: all (the default int8), none (fp16 blocks, int8 plan), every
"all but block b", and the prefixes {1}, {1,2}, {1,2,3}.  Per set:
- forward time of the N = 1024 batch: CUDA events around each forward, L2 flushed before each (a
  256 MB write), `steps` forwards per set and round, the sets alternated within each of `rounds`
  rounds in one process;
- launches of that forward;
- max|y - ref| / max|ref| and mean joint distance / mean joint norm against the float64 forward
  (oracle) on 64 held-out windows (another seed than the calibration batch), as
  tools/bench_int8.py and tests/test_int8_cpu.py measure them.
The card's name and power limit are read in the same run.  A random-init model: how the error
splits over the blocks of a trained checkpoint is not measured here.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def block_sets(nb):
    all_ = tuple(range(1, nb + 1))
    sets = {"all": all_, "none": ()}
    for b in all_:
        sets[f"all_but_{b}"] = tuple(i for i in all_ if i != b)
    for k in (1, 2, 3):
        sets["prefix_" + "".join(map(str, all_[:k]))] = all_[:k]
    return sets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import videopose3d_b200 as vp
    from eval_launch_times import card_info
    from oracle import temporal_model_oracle as orc

    if not torch.cuda.is_available():
        raise SystemExit("bench_int8_blocks.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    J, F, C, N, T, ARC = bench.J, bench.F, bench.C, bench.N_PER_GPU, bench.T, bench.ARC
    name, power = card_info()
    sd = orc.make_state_dict(J, F, J, ARC, C, seed=0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, causal=False, dropout=0.25, channels=C)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = orc.make_input(N, T, J, F, seed=1).to(dev)
    m.calibrate_int8(x, method="amax")
    m.set_precision("int8")
    sets = block_sets(len(ARC) - 1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(blocks):
        m.set_int8_blocks(blocks)
        ms = []
        with torch.no_grad():
            for _ in range(args.warmup):
                m(x)
            for _ in range(args.steps):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                m(x)
                b.record()
                b.synchronize()
                ms.append(a.elapsed_time(b))
        return float(np.mean(ms)), m.last_launch_count()

    times = {k: [] for k in sets}
    launches = {}
    for _ in range(args.rounds):
        for k, blocks in sets.items():
            t, launches[k] = timed(blocks)
            times[k].append(t)

    xh = orc.make_input(64, T, J, F, seed=78)
    ref = orc.forward_numpy(sd, xh.numpy(), ARC, strided=True)
    xh = xh.to(dev)
    rows = []
    for k, blocks in sets.items():
        with torch.no_grad():
            y = m.set_int8_blocks(blocks)(xh).double().cpu().numpy()
        rel_max = float(np.abs(y - ref).max() / np.abs(ref).max())
        rel_joint = float(np.linalg.norm(y - ref, axis=-1).mean() / np.linalg.norm(ref, axis=-1).mean())
        rows.append({"set": k, "blocks": list(blocks), "forward_ms": times[k],
                     "forward_ms_mean": float(np.mean(times[k])), "launches": launches[k],
                     "rel_max": rel_max, "rel_joint": rel_joint})
    out = {"card": name, "power_limit_w": power, "N": N, "T": T, "C": C, "arc": ARC,
           "steps": args.steps, "rounds": args.rounds, "sets": rows}
    base = rows[0]["forward_ms_mean"]
    print(f"{name}, power limit {power} W; N={N} T={T} C={C} arc={ARC}")
    print(f"{'set':<12} {'blocks':<16} {'ms':>8} {'x all':>6} {'launches':>8} {'max|d|/max':>11} "
          f"{'joint':>9}")
    for r in rows:
        print(f"{r['set']:<12} {str(r['blocks']):<16} {r['forward_ms_mean']:8.3f} "
              f"{r['forward_ms_mean'] / base:6.3f} {r['launches']:8d} {r['rel_max']:11.2e} "
              f"{r['rel_joint']:9.2e}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
