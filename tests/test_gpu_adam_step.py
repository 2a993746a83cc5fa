"""GPU: the optimizer step bit for bit against adam_reference.py, the exact float32 restatement of
csrc/step_ops.cu's ``adam_update``.

1. ``vp3d_adam_step`` (through the C entry and through FusedAdam): every size around the float4
   path, the scalar tail and the 8192-element chunk edges; each of the five streams misaligned on
   its own (the kernel's alignment check then takes the scalar path); lists of 63 to 130 tensors,
   split into launches of 64; amsgrad on and off, weight decay, steps 1, 2 and 10 000 with the lr
   decayed in between; zero, tiny, huge and non-finite gradients, the non-finite ones also against
   torch.optim.Adam.  Every tensor sits inside a larger buffer whose guard bands must come back
   with their bits unchanged.
2. ``vp3d_adam_step_packed`` on the architectures of test_gpu_train_layers plus an 8-width model
   (15 conv weights in one launch): a model stepped with the fused update + re-pack and a twin
   stepped with the plain update + separate re-pack.  The parameters and optimizer states equal
   the restatement; the next training step -- which reads every forward and transposed pack --
   is the same in both models bit for bit.
3. The optimizer's bookkeeping: two models in one optimizer, parameter groups with different step
   counts, and conv weights changed outside the optimizer between the forward and the step.
"""
import time

import numpy as np
import pytest
import torch

import adam_reference as ar
from oracle import temporal_model_oracle as orc
from test_gpu_train_layers import CASES, OPT, _build, _cfg, _key, _resolve, _state_dict
from videopose3d_b200 import _capi
from videopose3d_b200.optim import FusedAdam

pytestmark = pytest.mark.gpu

CHUNK = 8192            # kAdamChunk: elements per block of adam_step_kernel
MAX_TENSORS = 64        # VP3D_ADAM_MAX_TENSORS: tensors per launch
GUARD = 64              # sentinel floats on either side of every tensor (256 B keeps the alignment)
SENTINEL = 0x7FA5A5A5   # a NaN bit pattern no update produces
BETAS, EPS = (0.9, 0.999), 1e-8
COUNT = {"cases": 0}
T0 = time.perf_counter()


def _report():
    COUNT["cases"] += 1
    print(f"\n[test_gpu_adam_step] {COUNT['cases']} cases, {time.perf_counter() - T0:.1f} s so far")


# ------------------------------------------------------------------------------ guarded tensors
class Slab:
    """n floats at `off` floats past a 256-byte aligned guard band, inside one larger buffer."""

    def __init__(self, n, off, dev, values=None):
        self.n, self.lo = n, GUARD + off
        self.buf = torch.full((self.lo + n + GUARD,), SENTINEL, dtype=torch.int32, device=dev)
        self.t = self.buf.view(torch.float32)[self.lo:self.lo + n]
        if values is not None:
            self.t.copy_(torch.from_numpy(np.ascontiguousarray(values, np.float32)))

    def guards_intact(self):
        b = self.buf.cpu()
        return bool((b[:self.lo] == SENTINEL).all() and (b[self.lo + self.n:] == SENTINEL).all())

    def np(self):
        return self.t.cpu().numpy()


def _mismatch(got, want):
    """Number of elements whose bits differ (any NaN equals any NaN) and the first index."""
    got, want = np.asarray(got, np.float32).ravel(), np.asarray(want, np.float32).ravel()
    ok = (got.view(np.int32) == want.view(np.int32)) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(~ok)
    return len(bad), (int(bad[0]) if len(bad) else None)


def _assert_same(got, want, what):
    n, i = _mismatch(got, want)
    assert n == 0, (f"{what}: {n} of {np.asarray(want).size} elements differ from the restatement; "
                    f"first at {i}: got {np.asarray(got).ravel()[i]!r}, "
                    f"exact {np.asarray(want).ravel()[i]!r}")


class Entry:
    """One tensor of a vp3d_adam_step call: five guarded streams (vmax None without amsgrad) and
    the restatement's copy of p, m, v, vmax."""

    def __init__(self, n, offsets, amsgrad, dev, rng, p_scale=1.0):
        p0 = (rng.standard_normal(n) * p_scale).astype(np.float32)
        self.p, self.g = Slab(n, offsets[0], dev, p0), Slab(n, offsets[1], dev)
        self.m, self.v = Slab(n, offsets[2], dev, np.zeros(n)), Slab(n, offsets[3], dev, np.zeros(n))
        self.x = Slab(n, offsets[4], dev, np.zeros(n)) if amsgrad else None
        self.ref = ar.State(p0, amsgrad)
        self.n, self.offsets = n, offsets

    def slabs(self):
        return [s for s in (self.p, self.g, self.m, self.v, self.x) if s is not None]

    def check(self, where):
        for name, got, want in (("param", self.p, self.ref.p), ("exp_avg", self.m, self.ref.m),
                                ("exp_avg_sq", self.v, self.ref.v),
                                ("max_exp_avg_sq", self.x, self.ref.vmax)):
            if got is not None:
                _assert_same(got.np(), want, f"{where}: {name}")
        assert all(s.guards_intact() for s in self.slabs()), f"{where}: a guard band was written"


def _c_step(entries, step, lr, wd):
    table = (_capi.AdamTensor * max(len(entries), 1))()
    for row, e in zip(table, entries):
        row.param, row.grad = e.p.t.data_ptr(), e.g.t.data_ptr()
        row.exp_avg, row.exp_avg_sq = e.m.t.data_ptr(), e.v.t.data_ptr()
        row.max_exp_avg_sq = e.x.t.data_ptr() if e.x is not None else None
        row.numel = e.n
    stream = torch.cuda.current_stream().cuda_stream
    _capi.check(_capi.load().vp3d_adam_step(table, len(entries), step, lr, BETAS[0], BETAS[1], EPS,
                                            wd, stream), "vp3d_adam_step")


class FusedPath:
    """The same entries stepped by FusedAdam: parameters, gradients and optimizer states are the
    guarded views themselves, so the optimizer writes into the guarded buffers."""

    def __init__(self, entries, amsgrad, wd):
        self.entries = entries
        self.params = [torch.nn.Parameter(e.p.t) for e in entries]
        for prm, e in zip(self.params, entries):
            assert prm.data_ptr() == e.p.t.data_ptr()
        self.opt = FusedAdam(self.params, lr=1.0, betas=BETAS, eps=EPS, weight_decay=wd,
                             amsgrad=amsgrad)
        for prm, e in zip(self.params, entries):
            st = self.opt.state[prm]
            st["step"] = torch.tensor(0.0)
            st["exp_avg"], st["exp_avg_sq"] = e.m.t, e.v.t
            if amsgrad:
                st["max_exp_avg_sq"] = e.x.t

    def step(self, step, lr):
        for prm, e in zip(self.params, self.entries):
            prm.grad = e.g.t
            self.opt.state[prm]["step"].fill_(step - 1)
        self.opt.param_groups[0]["lr"] = lr
        self.opt.step()


def _run(entries, path, amsgrad, wd, schedule, grads):
    """Steps the entries through `path` ('c' or 'fused') and the restatement; checks every step."""
    fused = FusedPath(entries, amsgrad, wd) if path == "fused" else None
    for (step, lr), gen in zip(schedule, grads):
        for e in entries:
            g = gen(e).astype(np.float32)
            e.g.t.copy_(torch.from_numpy(g))
            e.ref.step(g, ar.hyper(step, lr, BETAS[0], BETAS[1], EPS, wd))
        if fused is not None:
            fused.step(step, lr)
        else:
            _c_step(entries, step, lr, wd)
        torch.cuda.synchronize()
        for e in entries:
            e.check(f"{path} numel {e.n} offsets {e.offsets} step {step}")
    return fused


SCHEDULE = [(1, 1e-3), (2, 9e-4), (10000, 8.1e-4)]
SIZES = [0, 1, 3, 4, 5, 8191, 8192, 8193, 3 * CHUNK + 7]


def _normal_grads(rng):
    return lambda e: rng.standard_normal(e.n) * rng.choice([1e-3, 1.0, 30.0])


@pytest.mark.parametrize("path", ["c", "fused"])
@pytest.mark.parametrize("amsgrad,wd", [(True, 0.0), (False, 0.0), (True, 0.01), (False, 0.01)])
def test_adam_step_sizes_and_alignment(cuda_device, path, amsgrad, wd):
    """The float4 path with its scalar tail (numel % 4 != 0) and the chunk edges, all streams
    aligned; then each stream alone offset by 1, 2 and 3 floats, so that the block takes the
    scalar path, at a size with a partial last chunk and numel % 4 != 0."""
    rng = np.random.default_rng(0)
    entries = [Entry(n, (0,) * 5, amsgrad, cuda_device, rng) for n in SIZES]
    for s in range(5 if amsgrad else 4):
        for off in (1, 2, 3):
            offs = tuple(off if k == s else 0 for k in range(5))
            entries.append(Entry(2 * CHUNK + 5, offs, amsgrad, cuda_device, rng))
    if wd:   # subnormal and tiny parameters through the weight-decay fma
        entries[-1].p.t[:4] = torch.tensor([1e-40, -1e-42, 1e-30, 0.0])
        entries[-1].ref.p[:4] = np.array([1e-40, -1e-42, 1e-30, 0.0], np.float32)
    _run(entries, path, amsgrad, wd, SCHEDULE, [_normal_grads(rng)] * len(SCHEDULE))
    _report()


MARKER = "FillFunctor"   # in the name of the kernel of Tensor.fill_ on the device


def _kernel_launches(fn, name, restore, tries=3):
    """Kernels called `name` among the CUDA activity the profiler records while fn() runs.  A
    marker kernel launched right after fn() must be among the records: a capture without it lost
    its CUDA activity records and says nothing about fn, so restore() puts fn's inputs back and fn
    runs again (at most `tries` captures).  A capture with the marker counts what fn launched."""
    from torch.profiler import ProfilerActivity, profile
    marker = torch.empty(1, device="cuda")
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            marker.fill_(1.0)
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events()]
        if any(MARKER in n for n in names):
            return sum(1 for n in names if name in n)
        print(f"\nprofiler capture lost its CUDA activity ({len(names)} records); running again")
        restore()
    raise AssertionError(f"the profiler recorded no CUDA activity in {tries} captures")


@pytest.mark.parametrize("path", ["c", "fused"])
@pytest.mark.parametrize("count", [63, 64, 65, 130])
def test_adam_step_split_launches(cuda_device, path, count):
    """Lists longer than 64 tensors go out in launches of 64; each launch's tensor-to-block scan
    must find every tensor's first block, with chunk-crossing tensors in between."""
    rng = np.random.default_rng(count)
    sizes = [int(s) for s in rng.integers(1, 300, count)]
    sizes[::9] = [CHUNK + 3] * len(sizes[::9])
    entries = [Entry(n, (0,) * 5, True, cuda_device, rng) for n in sizes]
    fused = _run(entries, path, True, 0.0, SCHEDULE[:1], [_normal_grads(rng)])
    for e in entries:
        e.g.t.copy_(torch.from_numpy(rng.standard_normal(e.n).astype(np.float32)))
        e.ref.step(e.g.np(), ar.hyper(2, 9e-4, BETAS[0], BETAS[1], EPS, 0.0))
    step = (lambda: fused.step(2, 9e-4)) if fused else (lambda: _c_step(entries, 2, 9e-4, 0.0))
    before = [(s.buf, s.buf.clone()) for e in entries for s in e.slabs()]

    def restore():
        for buf, saved in before:
            buf.copy_(saved)
    launches = _kernel_launches(step, "adam_step_kernel", restore)
    assert launches == -(-count // MAX_TENSORS), launches
    for e in entries:
        e.check(f"{path} {count} tensors, numel {e.n}, step 2")
    _report()


def _special(kind, n, rng):
    g = rng.standard_normal(n)
    if kind == "zero":
        return np.zeros(n)
    if kind == "tiny":
        return g * 1e-30
    if kind == "huge":
        return g * 1e30
    g[::3] = np.inf
    g[1::3] = -np.inf
    g[2::6] = np.nan
    return g


@pytest.mark.parametrize("path", ["c", "fused"])
@pytest.mark.parametrize("amsgrad", [True, False])
def test_adam_step_special_gradients(cuda_device, path, amsgrad):
    """Zero gradients, gradients of 1e-30 (g^2 underflows) and 1e30 (g^2 overflows), +-inf and NaN,
    then one ordinary step: bit for bit against the restatement; the non-finite pattern of every
    tensor (NaN, +inf, -inf) also against torch.optim.Adam on the GPU, foreach and not: torch's
    maximum keeps NaN, so after a NaN gradient max_exp_avg_sq holds NaN in both."""
    rng = np.random.default_rng(5)
    kinds = ("zero", "tiny", "huge", "nonfinite")
    entries = [Entry(8 * 257 + 3, (0,) * 5, amsgrad, cuda_device, rng) for _ in kinds] + \
              [Entry(1027, (1, 0, 0, 0, 0), amsgrad, cuda_device, rng)]   # the scalar path
    kinds = kinds + ("nonfinite",)
    g1 = {id(e): _special(k, e.n, rng).astype(np.float32) for e, k in zip(entries, kinds)}
    g2 = {id(e): rng.standard_normal(e.n).astype(np.float32) for e in entries}
    p0 = [e.p.np().copy() for e in entries]
    _run(entries, path, amsgrad, 0.0, SCHEDULE[:2], [lambda e: g1[id(e)], lambda e: g2[id(e)]])
    for foreach in (False, True):
        ps = [torch.nn.Parameter(torch.from_numpy(p).to(cuda_device)) for p in p0]
        opt = torch.optim.Adam(ps, lr=SCHEDULE[0][1], betas=BETAS, eps=EPS, amsgrad=amsgrad,
                               foreach=foreach)
        for (step, lr), g in zip(SCHEDULE[:2], (g1, g2)):
            opt.param_groups[0]["lr"] = lr
            for prm, e in zip(ps, entries):
                prm.grad = torch.from_numpy(g[id(e)]).to(cuda_device)
            opt.step()
        for prm, e, k in zip(ps, entries, kinds):
            st = opt.state[prm]
            pairs = [("param", e.p, prm), ("exp_avg", e.m, st["exp_avg"]),
                     ("exp_avg_sq", e.v, st["exp_avg_sq"])]
            if amsgrad:
                pairs.append(("max_exp_avg_sq", e.x, st["max_exp_avg_sq"]))
            for name, ours, theirs in pairs:
                a, b = ours.np(), theirs.detach().cpu().numpy()
                for test in (np.isnan, np.isposinf, np.isneginf):
                    assert np.array_equal(test(a), test(b)), \
                        f"{k} gradients, foreach={foreach}: {name} {test.__name__} differs from torch"
    if amsgrad:   # the case that separates a NaN-dropping maximum from torch's
        assert np.isnan(entries[3].x.np()).any()
    _report()


# ------------------------------------------------------------------- fused re-pack on the models
# The architectures of test_gpu_train_layers.  Left out: the frozen-BatchNorm cases (eval-mode
# steps, no training packs to keep current) and the wave-edge shapes, whose channel counts are
# multiples of 32 on the strided 3,3,3 model -- the pack geometry of opt_333_c256 -- and which
# differ only in the GEMM tiling.  Added: an 8-width model, 7 blocks, whose 14 layer convs and the
# shrink are 15 tensors of one packed launch (at most 16), on two receptive-field windows.
REPACK_CASES = [c for c in CASES if not c[4].get("frozen") and not c[0].startswith("wave_")]
REPACK_CASES.append(("opt_3x8_c64_two_windows", _cfg(OPT, [3] * 8, 64), 2, 3 ** 8, {}))
REPACK = [pytest.param(c[0], c[1], c[2], c[3], prec, p, id=f"{c[0]}-{prec}-p{p}")
          for c in REPACK_CASES for prec in ("bf16", "bf16x3") for p in (0.0, 0.25)]
LR = 1e-3


def _bits_equal(a, b):
    a, b = a.detach().contiguous(), b.detach().contiguous().reshape(a.shape)
    if a.dtype != torch.float32:   # num_batches_tracked
        return torch.equal(a, b)
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _gy(shape, dev):
    """The output gradient of a step: fixed for a given output shape."""
    return torch.randn(shape, generator=torch.Generator().manual_seed(5 + shape[2])).to(dev)


def _train_step(models, xs, seed, want_dx=False):
    """One training forward + backward of each model on its input, ``(y * gy).sum()`` with the
    dropout seed fixed; returns y, dx and the forward's and the backward's launch counts."""
    out = []
    for m, x in zip(models, xs):
        xin = x.clone().requires_grad_(want_dx)
        torch.manual_seed(seed)
        y = m(xin)
        fwd = m.last_launch_count()
        (y * _gy(y.shape, y.device)).sum().backward()
        torch.cuda.synchronize()
        out.append((y.detach(), xin.grad, fwd, m.last_launch_count()))
    return out


def _restate(refs, named, grads, opt, k, lr, where):
    """Steps the restatement with the captured gradients and compares the parameters and every
    optimizer state tensor of `named` (name -> parameter) bit for bit."""
    h = ar.hyper(k, lr, BETAS[0], BETAS[1], EPS, 0.0)
    for name, prm in named.items():
        st, ref = opt.state[prm], refs[name]
        ref.step(grads[name], h)
        _assert_same(prm.detach().cpu().numpy(), ref.p, f"{where}: {name}")
        _assert_same(st["exp_avg"].cpu().numpy(), ref.m, f"{where}: {name} exp_avg")
        _assert_same(st["exp_avg_sq"].cpu().numpy(), ref.v, f"{where}: {name} exp_avg_sq")
        _assert_same(st["max_exp_avg_sq"].cpu().numpy(), ref.vmax, f"{where}: {name} max_exp_avg_sq")
        assert float(st["step"]) == k, (where, name, float(st["step"]))


def _tie(a, b, what):
    """Model `a`'s step (y, dx, launches) and its parameter gradients equal model `b`'s."""
    (ya, dxa, fa, ba), (yb, dxb, fb, bb) = a[1], b[1]
    assert _bits_equal(ya, yb), f"{what}: y differs in {int((ya != yb).sum())} of {ya.numel()}"
    if dxa is not None or dxb is not None:
        assert _bits_equal(dxa, dxb), f"{what}: dx differs"
    assert (fa, ba) == (fb, bb), f"{what}: launches {fa}+{ba} vs {fb}+{bb}"
    pa, pb = dict(a[0].named_parameters()), dict(b[0].named_parameters())
    for name, prm in pa.items():
        if prm.grad is None:
            assert pb[name].grad is None, f"{what}: {name}"
            continue
        assert _bits_equal(prm.grad, pb[name].grad), f"{what}: {name}.grad differs"


@pytest.mark.parametrize("case,cfg,N,T,precision,p", REPACK)
def test_fused_repack_matches_plain_update(cuda_device, case, cfg, N, T, precision, p):
    """Three AMSGrad steps (lr decayed between them) of a model whose optimizer re-packs the conv
    weights inside the update and of a twin that updates and re-packs separately, on the same
    data and dropout seeds.  Every step: the twins' y and gradients equal bit for bit, and the
    fused model's parameters and optimizer states equal the restatement of the captured
    gradients.  Then a fourth step with dx, and an eval forward against a fresh model."""
    dev = cuda_device
    cfg, N = _resolve(cfg, N)
    sd = _state_dict(_key(cfg))
    fused, plain = (_build(cfg, sd, dev, precision, p) for _ in range(2))
    opts = []
    for m, fuse in ((fused, True), (plain, False)):
        opt = FusedAdam(m.parameters(), lr=LR, betas=BETAS, eps=EPS, amsgrad=True)
        opt.fuse_repack = fuse
        opts.append(opt)
    refs = {name: ar.State(prm.detach().cpu().numpy(), True)
            for name, prm in fused.named_parameters()}
    named = dict(fused.named_parameters())
    xs = [orc.make_input(N, T, cfg["J"], cfg["F"], seed=1 + k).to(dev) for k in range(4)]
    lr = LR
    tag = f"{case}-{precision}-p{p}"
    for k in range(1, 4):
        for o in opts:
            o.zero_grad()
        res = _train_step((fused, plain), (xs[k - 1],) * 2, seed=100 + k)
        _tie((fused, res[0]), (plain, res[1]), f"{tag} step {k}")
        grads = {name: prm.grad.detach().cpu().numpy() for name, prm in named.items()}
        for o in opts:
            o.step()
        assert [o.last_launches for o in opts] == [1 + 1 + 2, 1], [o.last_launches for o in opts]
        _restate(refs, named, grads, opts[0], k, lr, f"{tag} step {k}")
        for (name, a), b in zip(fused.state_dict().items(), plain.state_dict().values()):
            assert _bits_equal(a, b), f"{tag} step {k}: {name} differs between the twins"
        lr *= 0.9
        for o in opts:
            o.param_groups[0]["lr"] = lr
    # the next step reads every forward and transposed pack; dx the expand's transposed pack
    for o in opts:
        o.zero_grad()
    res = _train_step((fused, plain), (xs[3],) * 2, seed=104, want_dx=True)
    _tie((fused, res[0]), (plain, res[1]), f"{tag} next step")
    for (name, a), b in zip(fused.state_dict().items(), plain.state_dict().values()):
        assert _bits_equal(a, b), f"{tag} next step: {name} differs between the twins"
    # the eval forward packs from the fp32 masters: the same as a fresh model's
    fresh = _build(cfg, {k: v.cpu() for k, v in fused.state_dict().items()}, dev, precision, p)
    with torch.no_grad():
        ye, yf = fused.eval()(xs[0]), fresh.eval()(xs[0])
    assert _bits_equal(ye, yf), f"{tag}: eval forward differs from a fresh model's"
    _report()


# --------------------------------------------------------------------------------- bookkeeping
def _model(dev, precision, Jout=17, C=64, fw=(3, 3, 3), seed=0):
    cfg = _cfg(OPT, list(fw), C, Jout=Jout)
    sd = orc.make_state_dict(17, 2, Jout, list(fw), C, seed=seed)
    return cfg, sd, _build(cfg, sd, dev, precision, 0.0)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_two_models_one_optimizer(cuda_device, precision):
    """run.py's semi-supervised training: one AMSGrad optimizer over the position model and the
    trajectory model (Jout = 1).  Each model gets its own fused launch set (4 launches each)."""
    dev = cuda_device
    twins = []
    for fuse in (True, False):
        (_, _, pos), (_, _, traj) = _model(dev, precision), _model(dev, precision, Jout=1, seed=1)
        opt = FusedAdam(list(pos.parameters()) + list(traj.parameters()), lr=LR, betas=BETAS,
                        eps=EPS, amsgrad=True)
        opt.fuse_repack = fuse
        twins.append((pos, traj, opt))
    named = {f"pos.{n}": q for n, q in twins[0][0].named_parameters()}
    named.update({f"traj.{n}": q for n, q in twins[0][1].named_parameters()})
    refs = {n: ar.State(q.detach().cpu().numpy(), True) for n, q in named.items()}
    x = [orc.make_input(64, 27, 17, 2, seed=10 + k).to(dev) for k in range(4)]
    for k in range(1, 5):
        outs = []
        for pos, traj, opt in twins:
            opt.zero_grad()
            outs.append(_train_step((pos, traj), (x[k - 1],) * 2, seed=k, want_dx=k == 4))
        for i, what in ((0, "pos"), (1, "traj")):
            _tie((twins[0][i], outs[0][i]), (twins[1][i], outs[1][i]), f"{what} step {k}")
        if k == 4:
            break
        grads = {n: q.grad.detach().cpu().numpy() for n, q in named.items()}
        for _, _, opt in twins:
            opt.step()
        assert [t[2].last_launches for t in twins] == [2 * (1 + 1 + 2), 1]
        _restate(refs, named, grads, twins[0][2], k, LR, f"two models step {k}")
    _report()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_param_groups_with_different_steps(cuda_device, precision):
    """Two parameter groups of one model (C = 40: padded packs): the first holds the expand, the
    first block and the shrink, the second -- the last block, added after the first step -- has
    its own lr and is one step behind.  Each group is its own set of launches in one step()."""
    dev = cuda_device
    twins = []
    for fuse in (True, False):
        cfg, sd, m = _model(dev, precision, C=40)
        late = [m.layers_conv[2].weight, m.layers_conv[3].weight] + \
               [t for bn in m.layers_bn[2:] for t in (bn.weight, bn.bias)]
        early = [q for q in m.parameters() if all(q is not r for r in late)]
        opt = FusedAdam(early, lr=LR, betas=BETAS, eps=EPS, amsgrad=True)
        opt.fuse_repack = fuse
        twins.append((m, opt, late))
    m, opt, late = twins[0]
    named = dict(m.named_parameters())
    group_of = {n: (1 if any(q is r for r in late) else 0) for n, q in named.items()}
    refs = {n: ar.State(q.detach().cpu().numpy(), True) for n, q in named.items()}
    lrs = (LR, 3 * LR)
    x = [orc.make_input(96, 27, 17, 2, seed=30 + k).to(dev) for k in range(4)]
    for k in range(1, 5):
        for mm, o, _ in twins:
            o.zero_grad()
            mm.zero_grad()   # the late group's gradients before it joins the optimizer
        res = _train_step([t[0] for t in twins], (x[k - 1],) * 2, seed=k, want_dx=k == 4)
        _tie((twins[0][0], res[0]), (twins[1][0], res[1]), f"groups step {k}")
        if k == 4:
            break
        grads = {n: q.grad.detach().cpu().numpy() for n, q in named.items()}
        for _, o, _ in twins:
            o.step()
        want = [1 + 1 + 2, 1] if k == 1 else [(1 + 1 + 2) + (1 + 1), 2]
        assert [t[1].last_launches for t in twins] == want, (k, [t[1].last_launches for t in twins])
        for gi in (0, 1):
            steps = k if gi == 0 else k - 1
            if steps:
                sub = {n: q for n, q in named.items() if group_of[n] == gi}
                _restate(refs, sub, grads, opt, steps, lrs[gi], f"group {gi} step {steps}")
        if k == 1:
            for _, o, lt in twins:
                o.add_param_group(dict(params=lt, lr=lrs[1]))
    _report()


def _edit_shrink_by_sgd(m):
    sgd = torch.optim.SGD([m.shrink.weight], lr=0.1)
    return [q for q in m.parameters() if q is not m.shrink.weight], lambda: sgd.step(), None


def _edit_frozen_conv(m):
    w = m.layers_conv[1].weight
    w.requires_grad_(False)

    def edit():
        with torch.no_grad():
            w.mul_(0.5)
    return [q for q in m.parameters() if q.requires_grad], edit, w


def _edit_frozen_expand(m):
    w = m.expand_conv.weight
    w.requires_grad_(False)

    def edit():
        with torch.no_grad():
            w.add_(0.01)
    return [q for q in m.parameters() if q.requires_grad], edit, w


@pytest.mark.parametrize("form", ["second_optimizer", "frozen_conv", "frozen_expand"])
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_weights_changed_outside_the_step_are_repacked(cuda_device, form, precision):
    """A conv weight changes between the training forward and the fused step without going through
    this optimizer: stepped by a second optimizer, or frozen and edited in place.  The fused step
    re-packs only what it updated, so the next training forward must notice the other change and
    re-pack it: its y and gradients equal those of a fresh model loaded with the current
    parameters."""
    dev = cuda_device
    cfg, sd, m = _model(dev, precision)
    params, edit, frozen = {"second_optimizer": _edit_shrink_by_sgd, "frozen_conv": _edit_frozen_conv,
                            "frozen_expand": _edit_frozen_expand}[form](m)
    opt = FusedAdam(params, lr=LR, amsgrad=True)
    x = [orc.make_input(64, 27, 17, 2, seed=40 + k).to(dev) for k in range(3)]
    for k in range(2):
        opt.zero_grad()
        m.zero_grad()
        _train_step((m,), (x[k],), seed=k)
        edit()
        opt.step()
        assert opt.last_launches == 1 + 1 + (0 if form == "frozen_expand" else 2)
        fresh = _build(cfg, {n: v.cpu() for n, v in m.state_dict().items()}, dev, precision, 0.0)
        if frozen is not None:
            name = next(n for n, q in m.named_parameters() if q is frozen)
            fresh.get_parameter(name).requires_grad_(False)
        m.zero_grad()
        res = _train_step((m, fresh), (x[k + 1],) * 2, seed=10 + k)
        _tie((m, res[0]), (fresh, res[1]), f"{form} after step {k + 1}")
        m.zero_grad()
    _report()
