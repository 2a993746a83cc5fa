"""GPU: synchronized BatchNorm (GradientReducer(sync_bn=True)).

One rank: the synchronized kernels (slot store, exchange callback, rank-ordered merge and sums)
give the unsynchronized path's outputs, running statistics, parameter gradients and input
gradient bit for bit, for every training golden in both training precisions.

Several ranks: W processes share the one GPU over gloo (or, with two GPUs, one process per GPU
over NCCL), each runs its shard of a golden's batch -- ragged where N does not divide -- and
together they must reproduce the single-process golden: running statistics bit-identical across
ranks and within the G1 gate (1e-3) of the golden's, concatenated outputs within 1e-3 of the
golden's y, and W times the averaged gradients of the sum loss within 1e-3 of the golden's
gradients (test_gpu_train.py's gates, now met by a sharded step)."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN_DIR, golden_names, load_golden
import videopose3d_b200 as vp
from videopose3d_b200.data_parallel import GradientReducer

pytestmark = pytest.mark.gpu

TRAIN_CASES = [n for n in golden_names() if n.startswith(("opt", "tm")) and "train" in n]
JOIN_TIMEOUT_S = 900


def _build(meta, sd, dev, precision):
    kw = dict(filter_widths=meta["fw"], causal=meta["causal"], dropout=0.0, channels=meta["C"])
    if meta["cls"] == "TemporalModel":
        m = vp.TemporalModel(meta["J"], meta["F"], meta["Jout"], dense=meta["dense"], **kw)
    else:
        m = vp.TemporalModelOptimized1f(meta["J"], meta["F"], meta["Jout"], **kw)
    m.load_state_dict(sd)
    m = m.to(dev).train().set_train_precision(precision)
    m.set_bn_momentum(meta.get("momentum", 0.1))
    return m


def _rel(a, b):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    b = b.detach().cpu().numpy() if hasattr(b, "detach") else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _rel_l2(a, b):
    a = a.detach().cpu().double() if hasattr(a, "detach") else torch.as_tensor(a).double()
    b = b.detach().cpu().double() if hasattr(b, "detach") else torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _load_case(name):
    """(meta, state_dict, x, y_ref, new) of a small golden or of the cfg3-shape fixture."""
    if not name.startswith("big_"):
        return load_golden(name)
    from oracle import temporal_model_oracle as orc
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    sd = orc.make_state_dict(meta["J"], meta["F"], meta["Jout"], meta["fw"], meta["C"], seed=meta["seed"])
    x = orc.make_input(meta["N"], meta["T"], meta["J"], meta["F"], seed=meta["seed"] + 1)
    new = {k: z[k] for k in z.files if k.startswith(("new/", "gidx/", "gval/", "gnorm/"))}
    new["gy"] = z["gy"]
    return meta, sd, x, z["y"], new


def _step(m, x, gy, loss_div=1.0):
    """One training step with the sum loss (y * gy).sum() / loss_div; returns y, dx."""
    x = x.clone().requires_grad_(True)
    y = m(x)
    ((y * gy).sum() / loss_div).backward()
    return y.detach(), x.grad


# ---------------------------------------------------------------------------------------------
# one rank: bit identity with the unsynchronized path
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name", TRAIN_CASES)
def test_one_rank_sync_bn_is_bit_identical(cuda_device, name, precision):
    assert not dist.is_initialized()
    meta, sd, x, _, new = load_golden(name)
    x = x.to(cuda_device)
    gy = torch.from_numpy(new["gy"]).to(cuda_device)
    ref = _build(meta, sd, cuda_device, precision)
    y0, dx0 = _step(ref, x, gy)
    launches_plain = ref.last_launch_count()

    m = _build(meta, sd, cuda_device, precision)
    red = GradientReducer(sync_bn=True).attach(m)
    assert red.world == 1
    n_bn = 1 + len(m.layers_bn)
    xg = x.clone().requires_grad_(True)
    y1 = m(xg)
    assert red.exchanges == n_bn            # one exchange per training BatchNorm in the forward
    (y1 * gy).sum().backward()
    assert red.exchanges == 2 * n_bn        # ... and one per BatchNorm backward
    # the backward adds a slot memset and one rank-ordered sum per BatchNorm
    assert m.last_launch_count() == launches_plain + 1 + n_bn

    assert torch.equal(y1.detach(), y0)
    assert torch.equal(xg.grad, dx0)
    for (k, b0), (_, b1) in zip(ref.named_buffers(), m.named_buffers()):
        assert torch.equal(b0, b1), k
    for (k, p0), (_, p1) in zip(ref.named_parameters(), m.named_parameters()):
        assert torch.equal(p0.grad, p1.grad), k

    # switching the reducer's sync off restores the plain path on the same plan
    red.sync_bn = False
    before = red.exchanges
    m.load_state_dict(sd)
    for p in m.parameters():
        p.grad = None
    y2, _ = _step(m, x, gy)
    assert red.exchanges == before
    assert torch.equal(y2, y0)


def test_frozen_batchnorm_backward_never_exchanges(cuda_device):
    meta, sd, x, _, new = load_golden("opt_333_c64_train")
    m = _build(meta, sd, cuda_device, "bf16x3")
    red = GradientReducer(sync_bn=True).attach(m)
    gy = torch.from_numpy(new["gy"]).to(cuda_device)
    _step(m, x.to(cuda_device), gy)      # the training plan now has synchronisation configured
    done = red.exchanges
    assert done == 2 * (1 + len(m.layers_bn))
    m.eval()                             # eval-mode autograd: frozen BatchNorm on the same plan
    xg = x.to(cuda_device).requires_grad_(True)
    (m(xg) * gy).sum().backward()
    assert red.exchanges == done and xg.grad is not None


# ---------------------------------------------------------------------------------------------
# several ranks
# ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _bounds(n, world, rank):
    """Rows [lo, hi) of rank `rank`: the first n % world ranks take one row more."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def _shard_worker(rank, world, port, backend, name, precision, sync_bn, mean_loss, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        meta, sd, x, _, new = _load_case(name)
        m = _build(meta, sd, dev, precision)
        red = GradientReducer(sync_bn=sync_bn).attach(m)
        lo, hi = _bounds(int(meta["N"]), world, rank)
        gy = torch.from_numpy(new["gy"][lo:hi]).to(dev)
        if mean_loss:
            red.set_step_rows(hi - lo, int(meta["N"]))
        y, _ = _step(m, x[lo:hi].to(dev), gy, loss_div=float(hi - lo) if mean_loss else 1.0)
        torch.cuda.synchronize()
        torch.save({"y": y.cpu(),
                    "buffers": {k: b.detach().cpu() for k, b in m.named_buffers()},
                    "grads": {k: p.grad.detach().cpu() for k, p in m.named_parameters()},
                    "exchanges": red.exchanges},
                   os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _run_sharded(tmp_path, world, name, precision="bf16x3", sync_bn=True, mean_loss=False,
                 backend="gloo"):
    """Run `world` processes of _shard_worker; returns their results in rank order."""
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker,
                         args=(r, world, port, backend, name, precision, sync_bn, mean_loss,
                               str(tmp_path)))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(JOIN_TIMEOUT_S)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
            if p.is_alive():
                p.kill()
                p.join()
    assert [p.exitcode for p in procs] == [0] * world
    return [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]


def _check_ranks_agree(res):
    for r in res[1:]:
        for k, b in res[0]["buffers"].items():
            assert torch.equal(r["buffers"][k], b), k
        for k, g in res[0]["grads"].items():   # the gradient all-reduce leaves the mean everywhere
            assert torch.equal(r["grads"][k], g), k


SHARDED = [("opt_35_c128_train_causal", 3),   # N = 70: rows 24 / 23 / 23
           ("tm_333_c128_train", 2),          # N = 3: 2 / 1 sequences, dilated
           ("opt_333_c128_train", 2),         # N = 40: equal shards
           ("opt_337_c64_train", 4),          # N = 6: 2 / 2 / 1 / 1, a width-7 block
           ("opt_733_c64_train", 2),          # N = 6: expand width 7
           ("tm_337_c64_t202_train", 2)]      # N = 2: one 140-frame sequence each, dilated


@pytest.mark.parametrize("name,world", SHARDED)
def test_sharded_step_matches_single_process_golden(cuda_device, tmp_path, name, world):
    meta, sd, x, y_ref, new = load_golden(name)
    res = _run_sharded(tmp_path, world, name)
    n_bn = 1 + 2 * (len(meta["fw"]) - 1)
    assert all(r["exchanges"] == 2 * n_bn for r in res)
    _check_ranks_agree(res)
    y = torch.cat([r["y"] for r in res])
    assert _rel(y, y_ref) <= 1e-3
    for k, v in new.items():
        if k == "gy" or k.startswith("grad/"):
            continue
        got = res[0]["buffers"][k]
        if k.endswith("num_batches_tracked"):
            assert int(got) == int(v)
        else:
            assert _rel(got, v) <= 1e-3, k
    bad = {k: _rel(world * g, new["grad/" + k]) for k, g in res[0]["grads"].items()}
    bad = {k: v for k, v in bad.items() if not v <= 1e-3}
    assert not bad, f"gradient mismatch: {bad}"


def test_sharded_mean_loss_with_ragged_rows(cuda_device, tmp_path):
    """Each rank's loss is its own mean; set_step_rows weights dY so that the averaged gradient is
    the gradient of the global mean loss: the golden's (sum-loss) gradient / N."""
    name, world = "opt_35_c128_train_causal", 3
    meta, sd, x, y_ref, new = load_golden(name)
    res = _run_sharded(tmp_path, world, name, mean_loss=True)
    _check_ranks_agree(res)
    n = int(meta["N"])
    bad = {k: _rel(g, new["grad/" + k] / n) for k, g in res[0]["grads"].items()}
    bad = {k: v for k, v in bad.items() if not v <= 1e-3}
    assert not bad, f"gradient mismatch: {bad}"


def test_sharded_bf16_step_matches_single_process_bf16(cuda_device, tmp_path):
    """Default bf16 kernels: the sharded step against one process on the whole batch, with the
    bf16 gates of test_gpu_train.py (ReLU-mask flips make a tighter bf16 comparison ill-posed)."""
    name, world = "opt_35_c128_train_causal", 3
    meta, sd, x, _, new = load_golden(name)
    m = _build(meta, sd, cuda_device, "bf16")
    y1, _ = _step(m, x.to(cuda_device), torch.from_numpy(new["gy"]).to(cuda_device))
    res = _run_sharded(tmp_path, world, name, precision="bf16")
    _check_ranks_agree(res)
    assert _rel(torch.cat([r["y"] for r in res]), y1) <= 3e-2
    worst = {k: _rel_l2(world * res[0]["grads"][k], p.grad) for k, p in m.named_parameters()}
    assert max(worst.values()) <= 5e-2, worst
    for k, b in m.named_buffers():
        if not k.endswith("num_batches_tracked"):
            assert _rel(res[0]["buffers"][k], b) <= 1e-2, k


def test_unsynchronized_shards_miss_the_golden_statistics(cuda_device, tmp_path):
    """Control: the same shards with sync_bn off normalise over their own rows, so their running
    statistics differ from rank to rank and miss the golden's."""
    name, world = "opt_35_c128_train_causal", 3
    meta, sd, x, y_ref, new = load_golden(name)
    res = _run_sharded(tmp_path, world, name, sync_bn=False)
    assert all(r["exchanges"] == 0 for r in res)
    stats = [k for k in new if k.endswith(("running_mean", "running_var"))]
    worst = max(_rel(res[0]["buffers"][k], new[k]) for k in stats)
    assert worst > 1e-3, worst
    assert any(not torch.equal(res[0]["buffers"][k], res[1]["buffers"][k]) for k in stats)


def test_cfg3_shape_sharded_over_four_ranks(cuda_device, tmp_path):
    """big_opt_33333_c1024_train (arc 3^5, C = 1024, N = 1024) over 4 ranks of 256 rows, against
    the gates of test_gpu_train.py::test_cfg3_shape_train_step_matches_reference."""
    name, world = "big_opt_33333_c1024_train", 4
    meta, sd, x, y_ref, z = _load_case(name)
    res = _run_sharded(tmp_path, world, name)
    _check_ranks_agree(res)
    assert _rel(torch.cat([r["y"] for r in res]), y_ref) <= 1e-3
    med, l2, fn = {}, {}, {}
    for k, g in res[0]["grads"].items():
        g = (world * g).reshape(-1).double()
        ref = z["gval/" + k].astype(np.float64)
        norm, total, gmax = z["gnorm/" + k]
        err = np.abs(g[torch.from_numpy(z["gidx/" + k])].numpy() - ref)
        med[k] = float(np.median(err) / gmax)
        l2[k] = float(np.linalg.norm(err) / max(np.linalg.norm(ref), 1e-30))
        fn[k] = max(abs(float(g.norm()) - norm) / norm,
                    abs(float(g.sum()) - total) / (norm * np.sqrt(g.numel())))
    assert max(med.values()) <= 3e-3, med
    assert max(l2.values()) <= 2e-2, l2
    assert max(fn.values()) <= 2e-3, fn
    for k in z:
        if not k.startswith("new/"):
            continue
        got = res[0]["buffers"][k[4:]]
        if k.endswith("num_batches_tracked"):
            assert int(got) == int(z[k])
        else:
            assert _rel(got, z[k]) <= 1e-3, k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_over_nccl(cuda_device, tmp_path):
    name, world = "opt_35_c128_train_causal", 2
    meta, sd, x, y_ref, new = load_golden(name)
    res = _run_sharded(tmp_path, world, name, backend="nccl")
    _check_ranks_agree(res)
    assert _rel(torch.cat([r["y"] for r in res]), y_ref) <= 1e-3
    bad = {k: _rel(world * g, new["grad/" + k]) for k, g in res[0]["grads"].items()}
    assert not {k: v for k, v in bad.items() if not v <= 1e-3}, bad
