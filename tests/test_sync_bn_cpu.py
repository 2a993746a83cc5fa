"""CPU: the arithmetic of synchronized BatchNorm (GradientReducer(sync_bn=True)) and its exchange.

A float64 restatement of one training BatchNorm layer sharded over W ranks, as the kernels split
it: each rank reduces its rows to (n, mean, M2), the ranks' triples are merged in rank order
(Chan et al.); in the backward each rank's sum dY and sum dY * xhat are summed over ranks, dZ uses
the global sums and row count, d weight / d bias the rank's own sums, and the gradient all-reduce
averages.  Then the exchange itself over gloo with 2 and 3 ranks."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import videopose3d_b200 as vp
from videopose3d_b200.data_parallel import GradientReducer

EPS = 1e-5


def _bounds(n, world):
    base, extra = divmod(n, world)
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def _moments(x):
    n = x.shape[0]
    mean = x.mean(0)
    return float(n), mean, ((x - mean) ** 2).sum(0)


def _merge(a, b):
    """Chan et al. in the kernels' form (merge of b into the accumulator a)."""
    if b[0] <= 0:
        return a
    if a[0] <= 0:
        return b
    n = a[0] + b[0]
    d = b[1] - a[1]
    f = b[0] / n
    return n, a[1] + d * f, a[2] + b[2] + d * d * a[0] * f


def _bn_backward_global(z, gamma, dy):
    """Reference: dZ, d weight, d bias of y = gamma * (z - mean) * invstd + beta over all rows."""
    n = z.shape[0]
    mean = z.mean(0)
    invstd = 1.0 / np.sqrt(((z - mean) ** 2).mean(0) + EPS)
    xhat = (z - mean) * invstd
    dgamma = (dy * xhat).sum(0)
    dbeta = dy.sum(0)
    dz = gamma * invstd / n * (n * dy - dbeta - xhat * dgamma)
    return dz, dgamma, dbeta


def _bn_backward_sharded(z, gamma, dys, bounds):
    """The synchronized kernels' split: global statistics from the rank-ordered merge, local sums
    exchanged and summed in rank order, dZ from the global sums and count, d weight / d bias from
    the local sums, then the 1/W average of the gradient all-reduce."""
    world = len(bounds)
    acc = (0.0, 0.0, 0.0)
    for lo, hi in bounds:
        acc = _merge(acc, _moments(z[lo:hi]))
    n, mean, m2 = acc
    invstd = 1.0 / np.sqrt(m2 / n + EPS)
    local = []
    for (lo, hi), dy in zip(bounds, dys):
        xhat = (z[lo:hi] - mean) * invstd
        local.append((dy.sum(0), (dy * xhat).sum(0)))
    s1 = sum(s[0] for s in local)
    s2 = sum(s[1] for s in local)
    dz = []
    for (lo, hi), dy in zip(bounds, dys):
        xhat = (z[lo:hi] - mean) * invstd
        dz.append(gamma * invstd * (dy - s1 / n - xhat * s2 / n))
    dgamma = sum(s[1] for s in local) / world
    dbeta = sum(s[0] for s in local) / world
    return np.concatenate(dz), dgamma, dbeta


@pytest.mark.parametrize("n,world", [(64, 4), (70, 3), (3, 2), (9, 8)])
def test_rank_ordered_merge_equals_global_moments(n, world):
    rng = np.random.default_rng(n * 10 + world)
    z = rng.normal(2.0, 3.0, size=(n, 16))
    acc = (0.0, 0.0, 0.0)
    for lo, hi in _bounds(n, world):
        if hi > lo:
            acc = _merge(acc, _moments(z[lo:hi]))
    assert acc[0] == n
    np.testing.assert_allclose(acc[1], z.mean(0), rtol=0, atol=1e-12)
    np.testing.assert_allclose(acc[2] / n, z.var(0), rtol=1e-12, atol=1e-12)
    # one rank: merging one slot into the empty accumulator is a copy
    one = _moments(z)
    assert _merge((0.0, 0.0, 0.0), one) is one


@pytest.mark.parametrize("n,world", [(64, 4), (70, 3), (3, 2)])
@pytest.mark.parametrize("loss", ["sum", "mean"])
def test_sharded_batchnorm_backward_gives_the_global_gradient(n, world, loss):
    rng = np.random.default_rng(7 * n + world)
    c = 12
    z = rng.normal(0.5, 2.0, size=(n, c))
    gamma = rng.normal(1.0, 0.3, size=c)
    g = rng.normal(size=(n, c))            # dL/dy of the sum loss (y * g).sum()
    bounds = _bounds(n, world)
    if loss == "sum":
        dy_global = g
        dys = [g[lo:hi] for lo, hi in bounds]
        scale = world                     # W x the averaged gradient is the global one
    else:
        # global mean loss: dL/dy = g / N.  Each rank's own mean loss gives g / n_r; the
        # set_step_rows weight n_r * W / N is applied to dY before the backward
        dy_global = g / n
        dys = [g[lo:hi] / (hi - lo) * ((hi - lo) * world / n) for lo, hi in bounds]
        scale = 1.0                       # after the 1/W average: the global mean-loss gradient
    dz_ref, dgamma_ref, dbeta_ref = _bn_backward_global(z, gamma, dy_global)
    dz, dgamma, dbeta = _bn_backward_sharded(z, gamma, dys, bounds)
    if loss == "mean":
        dz = dz / world   # dZ of each rank carries the W of its weight; the average removes it
    np.testing.assert_allclose(dz, dz_ref, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(scale * dgamma, dgamma_ref, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(scale * dbeta, dbeta_ref, rtol=1e-10, atol=1e-12)


def test_global_sums_instead_of_averaged_sums_would_be_w_times_too_large():
    """Why d weight / d bias come from the local sums: the all-reduce averages over W ranks."""
    rng = np.random.default_rng(3)
    n, world = 60, 3
    z = rng.normal(size=(n, 4))
    g = rng.normal(size=(n, 4))
    bounds = _bounds(n, world)
    _, dgamma_ref, _ = _bn_backward_global(z, np.ones(4), g)
    _, dgamma, _ = _bn_backward_sharded(z, np.ones(4), [g[lo:hi] for lo, hi in bounds], bounds)
    np.testing.assert_allclose(world * dgamma, dgamma_ref, rtol=1e-10)


# ---------------------------------------------------------------------------------------------
# the exchange over gloo
# ---------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _slot_values(rank, floats):
    return torch.arange(floats, dtype=torch.float32) * 0.5 + 1000.0 * rank - 3.25


def _exchange_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m = vp.TemporalModelOptimized1f(17, 2, 17, [3, 3], channels=64)
        red = GradientReducer(sync_bn=True).attach(m)
        assert red.world == world and red.rank == rank
        assert red.bn_group is not None
        assert dist.get_process_group_ranks(red.bn_group) == list(range(world))
        for floats in (3 * 64, 2 * 64):          # forward moments, backward sums
            slots = torch.zeros(world * floats)
            slots[rank * floats:(rank + 1) * floats] = _slot_values(rank, floats)
            red.exchange(slots)
            want = torch.cat([_slot_values(r, floats) for r in range(world)])
            assert torch.equal(slots, want)
            # every rank holds the same bits
            got = [torch.empty_like(slots) for _ in range(world)]
            dist.all_gather(got, slots)
            assert all(torch.equal(g, slots) for g in got)
        assert red.exchanges == 2
        # with sync_bn the ragged weight goes to dY before the backward, not into reduce_flat
        red.set_step_rows(rank + 1, world * (world + 1) // 2)
        v = torch.full((8,), float(rank + 1))
        red.reduce_flat(v)
        assert torch.allclose(v, torch.full((8,), sum(range(1, world + 1)) / world), atol=1e-6)
        out[rank] = "ok"
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_exchange_fills_every_slot_identically_gloo(world):
    port = _free_port()
    with mp.Manager() as mgr:
        out = mgr.dict()
        mp.spawn(_exchange_worker, args=(world, port, out), nprocs=world, join=True)
        assert dict(out) == {r: "ok" for r in range(world)}


def test_one_rank_exchange_is_a_no_op_that_counts():
    red = GradientReducer(sync_bn=True)
    assert red.world == 1 and red.rank == 0
    slots = torch.arange(12, dtype=torch.float32)
    assert torch.equal(red.exchange(slots.clone()), slots)
    assert red.exchanges == 1
    assert GradientReducer().sync_bn is False
