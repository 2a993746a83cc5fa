#!/usr/bin/env python
"""Secondary measurements that bench.py's single JSON line does not carry (1 GPU):

  * the number north_star asks to beat: the reference network executed by stock PyTorch/cuDNN on the
    same GPU (fp32 with TF32 convolutions = PyTorch default, TF32 off, bf16 autocast), for the
    eval forward of BASELINE configs[1] and the training step of configs[2];
  * this repo's eval forward in all three precision modes and its Optimized1f training step
    (forward + backward + Adam(amsgrad) as in run.py:252, 409-420);
  * `--what stream`: streaming sessions (videopose3d_b200.streaming) against a user recomputing the
    receptive-field window per new frame, per-push latency over >= 500 pushes (see bench_stream);
  * `--what stream_tta`: the same with test-time flip augmentation -- an augmented session against a
    plain session of twice the slots and against model(windows) + metrics.flip_average (see
    bench_stream_tta);
  * `--what stream_seq`: the 240 sequences of the metrics workload through a session's predict()
    (sequences ending on their own slot, longest first) against what metrics.evaluate runs, one
    padded TTA batch per sequence (see bench_stream_seq);
  * `--what metrics`: the final evaluation of run.py (run.py:652-721) on a Human3.6M-test-sized
    workload, the fused metrics kernel (videopose3d_b200.metrics) against the path run.py runs
    (torch mpjpe / n_mpjpe with .item(), .cpu(), NumPy p_mpjpe / mean_velocity_error of the staged
    reference), for the metrics alone and for the whole evaluate() with test-time augmentation.

The cuDNN baseline is built here from plain torch.nn modules following common/model.py:85-138 /
151-197 (it is a measurement target, not the product and not the oracle).  CUDA-event timing,
10 warm-up + N timed iterations, cudnn.benchmark on, GPU-resident synthetic inputs.

    python tools/bench_extra.py [--iters 30] [--what eval,train,seq,metrics,stream,stream_tta,stream_seq] > extra.jsonl
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import videopose3d_b200 as vp  # noqa: E402

ARC, C, J, F, N, T = [3, 3, 3, 3, 3], 1024, 17, 2, 1024, 243


class CudnnTemporal(nn.Module):
    """Stock-PyTorch execution of the reference architecture (dilated or strided)."""

    def __init__(self, strided, dropout=0.25):
        super().__init__()
        self.strided = strided
        fw = ARC
        self.expand = nn.Conv1d(J * F, C, fw[0], stride=fw[0] if strided else 1, bias=False)
        self.expand_bn = nn.BatchNorm1d(C, momentum=0.1)
        convs, bns = [], []
        d = fw[0]
        self.pads = []
        for w in fw[1:]:
            self.pads.append((w - 1) * d // 2)
            convs.append(nn.Conv1d(C, C, w, stride=w, bias=False) if strided
                         else nn.Conv1d(C, C, w, dilation=d, bias=False))
            bns.append(nn.BatchNorm1d(C, momentum=0.1))
            convs.append(nn.Conv1d(C, C, 1, bias=False))
            bns.append(nn.BatchNorm1d(C, momentum=0.1))
            d *= w
        self.convs, self.bns = nn.ModuleList(convs), nn.ModuleList(bns)
        self.shrink = nn.Conv1d(C, J * 3, 1)
        self.drop, self.relu = nn.Dropout(dropout), nn.ReLU(inplace=True)

    def forward(self, x):
        n = x.shape[0]
        x = x.view(n, x.shape[1], -1).permute(0, 2, 1)
        x = self.drop(self.relu(self.expand_bn(self.expand(x))))
        for i, w in enumerate(ARC[1:]):
            if self.strided:
                res = x[:, :, w // 2:: w]
            else:
                p = self.pads[i]
                res = x[:, :, p: x.shape[2] - p]
            x = self.drop(self.relu(self.bns[2 * i](self.convs[2 * i](x))))
            x = res + self.drop(self.relu(self.bns[2 * i + 1](self.convs[2 * i + 1](x))))
        x = self.shrink(x)
        return x.permute(0, 2, 1).reshape(n, -1, J, 3)


def timeit(fn, iters, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
          for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2], ms[0]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    """Name and power limit of the GPU, read in the run that measures."""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                              "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in out.split(",")[:2]]
    except Exception:
        name, limit = torch.cuda.get_device_name(0), "not read"
    return {"gpu": name, "power_limit": limit}


def host_time(fn, reps):
    """Median wall time (s) of fn(), each rep ending in a device synchronise."""
    import time
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def bench_metrics(dev, reps):
    """run.py's final evaluation (run.py:652-721, called per action at :825-861): 240 test sequences
    of 1000-4000 frames (about the Human3.6M S9/S11 test split), J = 17, test-time augmentation on."""
    import numpy as np
    from videopose3d_b200 import metrics
    from videopose3d_b200.generators import UnchunkedGenerator
    sys.path.insert(0, ROOT)
    from oracle import stage_ref
    info = card()
    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    lens = np.random.RandomState(0).randint(1000, 4001, 240)
    frames = int(lens.sum())
    g = torch.Generator().manual_seed(0)
    preds = [(torch.randn(2, n, J, 3, generator=g) * 0.25).to(dev) for n in lens]
    batches = [(torch.randn(2, n, J, 3, generator=g) * 0.25).to(dev) for n in lens]
    ref = stage_ref.reference_dir()
    ref_loss = None
    if ref is not None:
        sys.path.insert(0, ref)
        import common.loss as ref_loss

    def runpy_metrics(pred, batch):
        """run.py:674-704 with the reference's metrics; returns (frames weight, 4 errors)."""
        pred = pred.clone()
        pred[1, :, :, 0] *= -1
        pred[1, :, left + right] = pred[1, :, right + left]
        pred = torch.mean(pred, dim=0, keepdim=True)
        inputs_3d = batch.clone()
        inputs_3d[:, :, 0] = 0
        inputs_3d = inputs_3d[:1]
        w = inputs_3d.shape[0] * inputs_3d.shape[1]
        e1 = ref_loss.mpjpe(pred, inputs_3d).item()
        e3 = ref_loss.n_mpjpe(pred, inputs_3d).item()
        inputs = inputs_3d.cpu().numpy().reshape(-1, J, 3)
        p = pred.cpu().numpy().reshape(-1, J, 3)
        return w, (e1, ref_loss.p_mpjpe(p, inputs), e3, ref_loss.mean_velocity_error(p, inputs))

    def fused_metrics(pred, batch):
        tgt = batch[:1].clone()
        tgt[:, :, 0] = 0
        return metrics.pose_errors(pred, tgt, left, right, return_averaged=False)[0]

    def run_fused():
        acc = None
        for pred, batch in zip(preds, batches):
            m = fused_metrics(pred, batch) * pred.shape[1]
            acc = m if acc is None else acc + m
        return (acc / frames * 1000).tolist()

    ref_mm = {}

    def run_ref():
        acc = np.zeros(4)
        for pred, batch in zip(preds, batches):
            w, e = runpy_metrics(pred, batch)
            acc += w * np.array(e)
        ref_mm["metrics"] = (acc / frames * 1000).tolist()

    run_fused()
    t_fused = host_time(run_fused, reps)
    res = dict(what="eval_metrics", sequences=len(lens), frames=frames, joints=J, tta=True, **info,
               fused_s=t_fused, fused_frames_per_s=frames / t_fused, fused_mm=run_fused())
    if ref_loss is not None:
        for p, b in zip(preds[:4], batches[:4]):
            runpy_metrics(p, b)
        t_ref = host_time(run_ref, 1)
        res.update(reference_s=t_ref, reference_frames_per_s=frames / t_ref, reference_mm=ref_mm["metrics"],
                   speedup=t_ref / t_fused)
    else:
        res.update(reference_s="not measured", reference_frames_per_s="not measured")
    emit(**res)

    # the whole evaluate(): model forward (fp16 inference) + flip average + metrics, per sequence
    del preds
    torch.cuda.empty_cache()
    model = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval()
    pad = model.receptive_field() // 2
    rng = np.random.RandomState(1)
    p2 = [rng.uniform(-1, 1, (n, J, F)).astype(np.float32) for n in lens]
    p3 = [rng.normal(0, 0.25, (n, J, 3)).astype(np.float32) for n in lens]
    gen = UnchunkedGenerator(None, p3, p2, pad=pad, causal_shift=0, augment=True, kps_left=left,
                             kps_right=right, joints_left=left, joints_right=right, device=dev)

    def eval_fused():
        return metrics.evaluate(model, gen, left, right)

    def eval_ref():
        acc, n = np.zeros(4), 0
        with torch.no_grad():
            for _, batch, batch_2d in gen.next_epoch():
                w, e = runpy_metrics(model(batch_2d), batch)
                acc += w * np.array(e)
                n += w
        ref_mm["evaluate"] = (acc / n * 1000).tolist()

    def forward_only():
        with torch.no_grad():
            for _, _, batch_2d in gen.next_epoch():
                model(batch_2d)

    forward_only()
    t_fwd = host_time(forward_only, reps)
    t_eval = host_time(eval_fused, reps)
    res = dict(what="evaluate_tta", sequences=len(lens), frames=frames, arc=ARC, channels=C,
               precision=model.precision, **info, forward_only_s=t_fwd, fused_s=t_eval,
               fused_mm=eval_fused())
    if ref_loss is not None:
        t_ref = host_time(eval_ref, 1)
        res.update(reference_s=t_ref, reference_mm=ref_mm["evaluate"], speedup=t_ref / t_eval,
                   metrics_share_of_reference=(t_ref - t_fwd) / t_ref)
    else:
        res.update(reference_s="not measured")
    emit(**res)


def stream_flops_per_frame(fw, C, c_in, c_out):
    """Executed FLOPs per output frame, from shapes: (streaming session, dependency-cone forward of
    one receptive field).  A session computes one new row per layer; the cone forward (model(x)
    with T = RF) computes L_0 = RF / w_0 expand rows and L_i = L_{i-1} / w_i rows in block i."""
    rf = 1
    for w in fw:
        rf *= w
    stream = 2 * c_in * fw[0] * C + sum(2 * C * C * (w + 1) for w in fw[1:]) + 2 * C * c_out
    rows = rf // fw[0]
    cone = rows * 2 * c_in * fw[0] * C
    for w in fw[1:]:
        rows //= w
        cone += rows * 2 * C * C * (w + 1)
    cone += rows * 2 * C * c_out
    return stream, cone


def bench_stream(dev, pushes):
    """Per-push latency of a streaming session at arc 3^5, C = 1024, fp16, against the baseline a
    real-time user has without it: model(window) on the last receptive field of every stream
    (N = S * k windows, T = RF, the dependency-cone schedule), alternated with the session in the
    same loop.  CUDA events around every push / baseline call; no L2 flush in between (a live
    stream keeps its weights hot)."""
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    rf = m.receptive_field()
    st_fl, cone_fl = stream_flops_per_frame(ARC, C, J * F, J * 3)
    info = card()
    for S, k in ((1, 1), (16, 1), (256, 1), (1024, 1), (256, 16)):
        sess = m.streaming(streams=S, max_frames=k)
        xs = (torch.rand(S, k, J, F, device=dev) * 2 - 1)
        win = (torch.rand(S * k, rf, J, F, device=dev) * 2 - 1)
        with torch.no_grad():
            sess.push(xs, start=[True] * S)
            for _ in range(50):
                sess.push(xs)
                m(win)
        torch.cuda.synchronize()
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(pushes)]
        with torch.no_grad():
            for e in ev:
                e[0].record()
                sess.push(xs)
                e[1].record()
                e[2].record()
                m(win)
                e[3].record()
        torch.cuda.synchronize()
        t_s = np.sort([e[0].elapsed_time(e[1]) for e in ev])
        t_b = np.sort([e[2].elapsed_time(e[3]) for e in ev])
        p99 = lambda t: float(t[min(len(t) - 1, int(np.ceil(0.99 * len(t))) - 1)])
        med_s, med_b = float(np.median(t_s)), float(np.median(t_b))
        emit(what="stream_push", streams=S, k=k, precision="fp16", arc=ARC, channels=C,
             pushes=pushes, push_ms_median=med_s, push_ms_p99=p99(t_s),
             frames_per_s=S * k / med_s * 1e3, push_launches=sess.last_launch_count(),
             baseline_ms_median=med_b, baseline_ms_p99=p99(t_b),
             baseline_frames_per_s=S * k / med_b * 1e3, speedup_median=med_b / med_s,
             mflop_per_frame_stream=st_fl / 1e6, mflop_per_frame_baseline=cone_fl / 1e6,
             stream_tflops=st_fl * S * k / med_s / 1e9, l2_flush="none", **info)
        del sess, xs, win
        torch.cuda.empty_cache()


def bench_stream_tta(dev, pushes):
    """Streaming with test-time flip augmentation (run.py's default), same model, configs and loop
    as bench_stream.  Three arms alternate in one loop, CUDA events around each:
      * the augmented session, S slots (plain + mirrored rows in the same launches, flip average on
        the device);
      * a plain session with 2S slots: the same GEMM rows, so the difference is the cost of
        mirroring and averaging;
      * what a TTA user has without it: model(windows) on the S*k plain and S*k mirrored
        receptive-field windows, then metrics.flip_average."""
    from videopose3d_b200 import metrics
    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    lists = dict(kps_left=left, kps_right=right, joints_left=left, joints_right=right)
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    rf = m.receptive_field()
    st_fl, cone_fl = stream_flops_per_frame(ARC, C, J * F, J * 3)
    info = card()
    p99 = lambda t: float(t[min(len(t) - 1, int(np.ceil(0.99 * len(t))) - 1)])  # noqa: E731
    for S, k in ((1, 1), (16, 1), (256, 1), (1024, 1), (256, 16)):
        aug = m.streaming(streams=S, max_frames=k, augment=True, **lists)
        plain = m.streaming(streams=2 * S, max_frames=k)
        xs = (torch.rand(S, k, J, F, device=dev) * 2 - 1)
        x2 = (torch.rand(2 * S, k, J, F, device=dev) * 2 - 1)
        win = (torch.rand(2 * S * k, rf, J, F, device=dev) * 2 - 1)   # [plain; mirrored] windows

        def baseline():
            return metrics.flip_average(m(win).view(2, S * k, J, 3), left, right)

        arms = (("augmented", lambda: aug.push(xs)), ("plain_2S", lambda: plain.push(x2)),
                ("model_windows_flip_average", baseline))
        with torch.no_grad():
            aug.push(xs, start=[True] * S)
            plain.push(x2, start=[True] * 2 * S)
            for _ in range(50):
                for _, fn in arms:
                    fn()
        torch.cuda.synchronize()
        ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
               for _ in arms] for _ in range(pushes)]
        with torch.no_grad():
            for n, e in enumerate(ev):
                for j in range(len(arms)):   # rotated, so that no arm always follows the same one
                    i = (j + n) % len(arms)
                    e[i][0].record()
                    arms[i][1]()
                    e[i][1].record()
            # the sessions share the model's plan and its launch counter: read it after each call
            launches = {}
            for (name, fn), count in zip(arms, (aug.last_launch_count, plain.last_launch_count,
                                                lambda: m.last_launch_count() + 1)):
                fn()
                launches[name] = count()
        torch.cuda.synchronize()
        res = dict(what="stream_tta_push", streams=S, k=k, precision="fp16", arc=ARC, channels=C,
                   pushes=pushes, l2_flush="none", **info)
        for i, (name, _) in enumerate(arms):
            t = np.sort([e[i][0].elapsed_time(e[i][1]) for e in ev])
            med = float(np.median(t))
            res[name] = dict(ms_median=med, ms_p99=p99(t), frames_per_s=S * k / med * 1e3,
                             launches=launches[name],
                             mflop_per_frame=2 * (cone_fl if i == 2 else st_fl) / 1e6)
        res["augmented_over_plain_2S"] = res["augmented"]["ms_median"] / res["plain_2S"]["ms_median"]
        res["speedup_over_windows"] = (res["model_windows_flip_average"]["ms_median"]
                                       / res["augmented"]["ms_median"])
        emit(**res)
        del aug, plain, xs, x2, win
        torch.cuda.empty_cache()


def offline_flops(fw, C, c_in, c_out, t_in):
    """Executed FLOPs of the offline dilated forward on one padded sequence of t_in frames."""
    rows = t_in - (fw[0] - 1)
    fl = rows * 2 * c_in * fw[0] * C
    d = fw[0]
    for w in fw[1:]:
        rows -= (w - 1) * d
        fl += rows * 2 * C * C * (w + 1)
        d *= w
    return fl + rows * 2 * C * c_out


def bench_stream_seq(dev, reps):
    """The metrics workload's 240 sequences (lengths RandomState(0).randint(1000, 4001), J = 17) at
    arc 3^5, C = 1024, fp16, test-time augmentation, two ways:
      (a) what metrics.evaluate runs: per sequence model(b) on the padded (2, T + 2 pad, J, F) batch
          of the device UnchunkedGenerator, then metrics.flip_average;
      (b) sess.predict(seqs) of an augmented session at a few (S, K), the session reused.
    Wall time ending in a device synchronise (median of `reps`, after one warm-up), frames/s,
    launches, FLOPs executed (from shapes: (b) counts every row a push computes, drain frames and
    idle slots included, and the start v-passes), session state bytes, and whether all 240 outputs
    of every arm are bit-identical to (a)'s."""
    from videopose3d_b200 import metrics
    from videopose3d_b200.generators import UnchunkedGenerator
    from videopose3d_b200.streaming import predict_schedule
    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    lists = dict(kps_left=left, kps_right=right, joints_left=left, joints_right=right)
    info = card()
    lens = np.random.RandomState(0).randint(1000, 4001, 240)
    frames = int(lens.sum())
    torch.manual_seed(0)
    m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval().set_precision("fp16")
    pad = (m.receptive_field() - 1) // 2
    la = vp.streaming.lookahead(m)
    rng = np.random.RandomState(1)
    p2 = [rng.uniform(-1, 1, (n, J, F)).astype(np.float32) for n in lens]
    seqs = [torch.from_numpy(x).to(dev) for x in p2]
    gen = UnchunkedGenerator(None, None, p2, pad=pad, causal_shift=0, augment=True, kps_left=left,
                             kps_right=right, device=dev)
    batches = [b for _, _, b in gen.next_epoch()]
    outs = {}

    def per_sequence():
        with torch.no_grad():
            outs["a"] = [metrics.flip_average(m(b), left, right)[0] for b in batches]

    per_sequence()
    t_a = host_time(per_sequence, reps)
    launches_a = 0
    for b in batches:
        with torch.no_grad():
            m(b)
        launches_a += m.last_launch_count() + 1   # + the flip average
    fl_a = sum(2 * offline_flops(ARC, C, J * F, J * 3, int(n) + 2 * pad) for n in lens)
    rows = [dict(arm="model_per_sequence_flip_average", seconds=t_a, frames_per_s=frames / t_a,
                 launches=launches_a, tflop_executed=fl_a / 1e12, tflops=fl_a / t_a / 1e12)]
    st_fl, _ = stream_flops_per_frame(ARC, C, J * F, J * 3)
    v_fl = st_fl - 2 * C * J * 3        # a start's v-pass: every layer but the shrink, one row
    for S, K in ((240, 16), (128, 32), (64, 64)):
        sess = m.streaming(streams=S, max_frames=K, augment=True, **lists)
        got = {}

        def run():
            with torch.no_grad():
                got["b"] = sess.predict(seqs)

        run()
        t_b = host_time(run, reps)
        pushes = predict_schedule(lens, S, K, la)
        P = 2 * S
        fl_b = sum(p["k"] * P * st_fl + (P * v_fl if p["start"].any() else 0) for p in pushes)
        equal = all(torch.equal(a, b) for a, b in zip(outs["a"], got["b"]))
        rows.append(dict(arm="predict", streams=S, max_frames=K, seconds=t_b,
                         frames_per_s=frames / t_b, launches=sess.last_predict_launches,
                         pushes=len(pushes), tflop_executed=fl_b / 1e12, tflops=fl_b / t_b / 1e12,
                         state_bytes=sess._state.numel(), bit_equal_to_per_sequence=equal,
                         speedup_over_per_sequence=t_a / t_b))
        del sess, got
        torch.cuda.empty_cache()
    for r in rows:
        emit(what="stream_seq", sequences=len(lens), frames=frames, arc=ARC, channels=C,
             precision="fp16", tta=True, **info, **r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--what", default="eval,train")
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of the metrics arms")
    ap.add_argument("--pushes", type=int, default=500, help="timed pushes per streaming config")
    args = ap.parse_args()
    what = set(args.what.split(","))
    dev = torch.device("cuda:0")
    if "stream" in what:
        bench_stream(dev, args.pushes)
    if "stream_tta" in what:
        bench_stream_tta(dev, args.pushes)
    if "stream_seq" in what:
        bench_stream_seq(dev, args.reps)
    if "metrics" in what:
        bench_metrics(dev, args.reps)
    torch.backends.cudnn.benchmark = True
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(N, T, J, F, generator=g) * 2 - 1).to(dev)
    tgt = (torch.randn(N, 1, J, 3, generator=g) * 0.3).to(dev)

    if "eval" in what:
        m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval()
        for prec in ("mixed", "bf16", "bf16x3"):
            m.set_precision(prec)
            with torch.no_grad():
                med, best = timeit(lambda: m(x), args.iters)
            emit(what="eval_forward", impl="vp3d_b200", precision=prec, ms_median=med, ms_best=best,
                 frames_per_s=N / med * 1e3, launches=m.last_launch_count())
        del m
        ref = CudnnTemporal(strided=False).to(dev).eval()
        for name, tf32, autocast in (("fp32_tf32", True, False), ("fp32_ieee", False, False),
                                     ("bf16_autocast", True, True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32

            def run():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    return ref(x)
            med, best = timeit(run, max(5, args.iters // 3), warmup=3)
            emit(what="eval_forward", impl="pytorch_cudnn_reference_arch", precision=name,
                 ms_median=med, ms_best=best, frames_per_s=N / med * 1e3)
        del ref
        torch.cuda.empty_cache()

    if "seq" in what:
        # the reference's inference use (UnchunkedGenerator + evaluate(), run.py:652-721): one whole
        # video per forward, test-time flip augmentation -> batch of 2 sequences, every frame
        # predicted.  This is the dilated schedule (no cone pruning possible).
        frames = 6000
        xs = (torch.rand(2, frames + 242, J, F, generator=g) * 2 - 1).to(dev)
        m = vp.TemporalModel(J, F, J, filter_widths=ARC, channels=C).to(dev).eval()
        for prec in ("mixed", "bf16", "bf16x3"):
            m.set_precision(prec)
            with torch.no_grad():
                med, best = timeit(lambda: m(xs), args.iters)
            emit(what="eval_sequence_2x6000", impl="vp3d_b200", precision=prec, ms_median=med,
                 ms_best=best, frames_per_s=2 * frames / med * 1e3, launches=m.last_launch_count())
        del m
        ref = CudnnTemporal(strided=False).to(dev).eval()
        for name, tf32, autocast in (("fp32_tf32", True, False), ("bf16_autocast", True, True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32

            def run_seq():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    return ref(xs)
            med, best = timeit(run_seq, max(5, args.iters // 3), warmup=3)
            emit(what="eval_sequence_2x6000", impl="pytorch_cudnn_reference_arch", precision=name,
                 ms_median=med, ms_best=best, frames_per_s=2 * frames / med * 1e3)
        del ref
        torch.cuda.empty_cache()

    if "train" in what:
        for prec in ("bf16", "bf16x3"):
            m = vp.TemporalModelOptimized1f(J, F, J, filter_widths=ARC, channels=C).to(dev).train()
            m.set_train_precision(prec)
            opt = torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)

            def step():
                opt.zero_grad()
                loss = torch.mean(torch.norm(m(x) - tgt, dim=-1))
                loss.backward()
                opt.step()
            med, best = timeit(step, args.iters)

            def fwd_bwd():
                opt.zero_grad()
                torch.mean(torch.norm(m(x) - tgt, dim=-1)).backward()
            med_fb, _ = timeit(fwd_bwd, args.iters, warmup=3)
            emit(what="train_step", impl="vp3d_b200", precision=prec, ms_median=med, ms_best=best,
                 ms_fwd_bwd=med_fb, frames_per_s=N / med * 1e3)
            del m, opt
            torch.cuda.empty_cache()
        for name, tf32, autocast in (("fp32_tf32", True, False), ("bf16_autocast", True, True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ref = CudnnTemporal(strided=True).to(dev).train()
            opt = torch.optim.Adam(ref.parameters(), lr=1e-3, amsgrad=True)

            def step():
                opt.zero_grad()
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                    out = ref(x)
                loss = torch.mean(torch.norm(out.float() - tgt, dim=-1))
                loss.backward()
                opt.step()
            med, best = timeit(step, args.iters)
            emit(what="train_step", impl="pytorch_cudnn_reference_arch", precision=name, ms_median=med,
                 ms_best=best, frames_per_s=N / med * 1e3)
            del ref, opt
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
