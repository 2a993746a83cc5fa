#!/usr/bin/env python
"""Data-parallel training benchmark (BASELINE configs[3] shape): TemporalModelOptimized1f, arc
3,3,3,3,3, N = 1024 windows per GPU (weak scaling), forward + backward + gradient all-reduce +
Adam(amsgrad), one process per GPU over NCCL.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29541 tools/bench_train_dp.py [--steps 30] [--no-overlap] [--check]

Rank 0 prints one JSON line: total frames/s (max over ranks of the CUDA-event time), per-step ms,
and — with --check — the maximum difference between the averaged gradients and a reference average
computed with a plain all_reduce of per-rank gradients (parity of the staged / overlapped path).

--sync-bn: the step with and without synchronized BatchNorm (GradientReducer(sync_bn=...)),
alternated --rounds times in one run, with the forward / backward launch counts of each and the
card's name and power limit.  Also runs on one GPU, where it measures the cost of the synchronized
kernels alone (one rank: the exchange moves nothing).
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import videopose3d_b200 as vp  # noqa: E402

ARC, C, J, F, N, T = [3, 3, 3, 3, 3], 1024, 17, 2, 1024, 243


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-overlap", action="store_true")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--sync-bn", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    torch.manual_seed(0)  # identical initial weights on every rank
    m = vp.TemporalModelOptimized1f(J, F, J, filter_widths=ARC, channels=C).to(dev).train()
    m.set_train_precision(args.precision)
    red = vp.GradientReducer(overlap=not args.no_overlap).attach(m) if world > 1 else None
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)
    g = torch.Generator().manual_seed(1000 + rank)  # each rank its own batches
    x = (torch.rand(N, T, J, F, generator=g) * 2 - 1).to(dev)
    tgt = (torch.randn(N, 1, J, 3, generator=g) * 0.3).to(dev)

    if args.sync_bn:
        sync_bn_compare(args, m, opt, x, tgt, world, rank, dev)
        return

    check = None
    if args.check and world > 1:
        # The BatchNorm batch sums use fp32 atomics, so two runs of the *same* step differ by ReLU
        # mask flips; the noise floor (two plain runs) is reported next to the staged-path check.
        def plain_avg():
            torch.manual_seed(7)  # same dropout seed draw on every rank is fine; data differs
            object.__setattr__(m, "_grad_reducer", None)
            opt.zero_grad()
            torch.mean(torch.norm(m(x) - tgt, dim=-1)).backward()
            out = [p.grad.clone() for p in m.parameters()]
            for t in out:
                dist.all_reduce(t, op=dist.ReduceOp.AVG)
            return out

        def rel_l2(a, b):
            return max(float((p - r).norm() / r.norm().clamp_min(1e-20)) for p, r in zip(a, b))

        ref, ref2 = plain_avg(), plain_avg()
        object.__setattr__(m, "_grad_reducer", red)
        torch.manual_seed(7)
        opt.zero_grad()
        torch.mean(torch.norm(m(x) - tgt, dim=-1)).backward()
        torch.cuda.synchronize()
        staged = [p.grad for p in m.parameters()]
        check = {"staged_vs_plain_rel_l2": rel_l2(staged, ref),
                 "plain_vs_plain_rel_l2_noise_floor": rel_l2(ref2, ref)}

    def step():
        opt.zero_grad()
        loss = torch.mean(torch.norm(m(x) - tgt, dim=-1))
        loss.backward()
        opt.step()
        return loss

    for _ in range(args.warmup):
        step()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        total_ms = float(ms[0])
        print(json.dumps({
            "what": "train_step_dp", "n_gpus": world, "precision": args.precision,
            "overlap": not args.no_overlap, "ms_per_step": total_ms / args.steps,
            "frames_per_s": N * world * args.steps / (total_ms * 1e-3), "scaling": "weak",
            "grad_allreduce_mb": sum(p.numel() for p in m.parameters()) * 4 / 1e6,
            "staged_vs_plain_allreduce_max_rel": check, "final_loss": float(loss.detach()),
        }), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def card():
    """Name and power limit of the current GPU (read-only query)."""
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        idx = str(torch.cuda.current_device())
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        info["power_limit"] = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = None
    return info


def sync_bn_compare(args, m, opt, x, tgt, world, rank, dev):
    reducers = {False: vp.GradientReducer(overlap=not args.no_overlap),
                True: vp.GradientReducer(overlap=not args.no_overlap, sync_bn=True)}
    times = {False: [], True: []}
    launches = {}

    def step():
        opt.zero_grad()
        loss = torch.mean(torch.norm(m(x) - tgt, dim=-1))
        fwd = m.last_launch_count()
        loss.backward()
        bwd = m.last_launch_count()
        opt.step()
        return fwd, bwd

    for _ in range(args.rounds):
        for sync in (False, True):
            reducers[sync].attach(m)
            for _ in range(args.warmup):
                launches[sync] = step()
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1) / args.steps], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            times[sync].append(float(ms[0]))
    if rank == 0:
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        print(json.dumps({
            "what": "train_step_dp_sync_bn", "n_gpus": world, "precision": args.precision,
            "overlap": not args.no_overlap, "n_per_rank": N, **card(),
            "ms_per_step": {"plain": med[False], "sync_bn": med[True]},
            "ms_per_step_rounds": {"plain": times[False], "sync_bn": times[True]},
            "sync_bn_overhead": med[True] / med[False] - 1.0,
            "launches_fwd_bwd": {"plain": launches[False], "sync_bn": launches[True]},
            "bn_exchanges_per_step": reducers[True].exchanges // (args.rounds * (args.warmup + args.steps)),
        }), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
