"""Generate input-gradient golden vectors from the REAL reference implementation.

Run in the build container only (needs the reference checkout):

    python tests/golden/make_input_grad_golden.py

Imports ``common.model`` from the reference unchanged, loads seeded state dicts with randomised
BatchNorm parameters and running statistics (``oracle.make_state_dict``), converts the module to
float64 on the CPU, sets ``x.requires_grad_()`` and back-propagates ``(y * gy).sum()``.  Eval-mode
cases run the module in ``eval()`` (BatchNorm on running statistics, the gradient of test-time
refinement and frozen-BatchNorm fine-tuning); train-mode cases run ``train()`` with dropout 0
(BatchNorm batch statistics).  Each fixture in ``input_grad/`` stores x, gy, y, x.grad and every
parameter gradient; gradients with more than SAMPLE_ABOVE entries are stored as a fixed sample of
entries plus their L2 norm.  The state dict is not stored: ``make_state_dict(seed)`` regenerates it.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import stage_ref  # noqa: E402
from oracle import temporal_model_oracle as orc  # noqa: E402

OUT = os.path.join(HERE, "input_grad")
SAMPLE_ABOVE = 4096
SAMPLES = 1024
MIN_PREACT = 2e-5   # smallest |pre-activation| a fixture may have (away from the ReLU kink)

_TM, _OPT = "TemporalModel", "TemporalModelOptimized1f"
CASES = {
    # eval mode (BatchNorm on running statistics)
    "tm_333_c64_rf": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=3, T=27),
    "tm_333_c64_long": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=2, T=40),
    "tm_333_c64_causal": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=2, T=35,
                              causal=True),
    "tm_33_c64_dense": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3], C=64, N=2, T=12, dense=True),
    "tm_353_c128_traj": dict(cls=_TM, J=17, F=2, Jout=1, fw=[3, 5, 3], C=128, N=2, T=50),
    "tm_333_c64_f3": dict(cls=_TM, J=16, F=3, Jout=16, fw=[3, 3, 3], C=64, N=2, T=30),
    "tm_333_c100_j15": dict(cls=_TM, J=15, F=2, Jout=15, fw=[3, 3, 3], C=100, N=2, T=30),
    "opt_333_c64_rf": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=4, T=27),
    "opt_333_c64_t30": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=3, T=30),
    # expand width 7: the tap-merged transposed expand and the strided tail (68 = 7 * 9 + 5);
    # 16 channels keep every gradient whole and the fixture small
    "opt_733_c16_t68": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[7, 3, 3], C=16, N=3, T=68),
    # train mode, dropout 0 (BatchNorm batch statistics)
    "train_opt_333_c64": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=6, T=27,
                              train=True),
    "train_opt_333_c64_t29": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=6, T=29,
                                  train=True),
    "train_opt_35_c64_causal": dict(cls=_OPT, J=17, F=2, Jout=17, fw=[3, 5], C=64, N=8, T=15,
                                    causal=True, train=True),
    "train_tm_333_c64": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3, 3], C=64, N=3, T=30,
                             train=True),
    "train_tm_33_c64_causal": dict(cls=_TM, J=17, F=2, Jout=17, fw=[3, 3], C=64, N=3, T=20,
                                   causal=True, train=True),
}


def case_inputs(name, cfg, seed):
    """State dict (torch float32, BatchNorm randomised), x and gy of a case for a given seed."""
    sd = orc.make_state_dict(cfg["J"], cfg["F"], cfg["Jout"], cfg["fw"], cfg["C"],
                             dense=bool(cfg.get("dense")), seed=seed)
    x = orc.make_input(cfg["N"], cfg["T"], cfg["J"], cfg["F"], seed=seed + 1)
    return sd, x


def sample_index(name, size):
    """Fixed entries stored for a large gradient (depends on the case name only)."""
    g = np.random.RandomState(sum(ord(c) for c in name) + size)
    return np.sort(g.choice(size, SAMPLES, replace=False))


def build_case(name, cfg):
    ref = stage_ref.import_reference()
    seed = sum(ord(c) for c in name)
    causal, dense = bool(cfg.get("causal")), bool(cfg.get("dense"))
    strided = cfg["cls"] == _OPT
    train = bool(cfg.get("train"))
    for _ in range(400):
        sd, x = case_inputs(name, cfg, seed)
        probe = {}
        orc.forward_numpy(sd, x.numpy(), cfg["fw"], causal=causal, dense=dense, strided=strided,
                          training=train, probe=probe)
        if probe["min_abs_preact"] >= MIN_PREACT:
            break
        seed += 1000
    else:
        raise AssertionError(f"{name}: no seed keeps every pre-activation away from the ReLU kink")
    kw = dict(filter_widths=cfg["fw"], causal=causal, dropout=0.0, channels=cfg["C"])
    if strided:
        model = ref.TemporalModelOptimized1f(cfg["J"], cfg["F"], cfg["Jout"], **kw)
    else:
        model = ref.TemporalModel(cfg["J"], cfg["F"], cfg["Jout"], dense=dense, **kw)
    model.load_state_dict(sd)
    model = model.double()
    model.train(train)
    xd = x.double().requires_grad_()
    y = model(xd)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed + 2), dtype=torch.float64)
    (y * gy).sum().backward()
    out = {"x": x.numpy(), "gy": gy.numpy(), "y": y.detach().numpy(), "grad/x": xd.grad.numpy()}
    for k, prm in model.named_parameters():
        g = prm.grad.numpy().reshape(-1)
        if g.size > SAMPLE_ABOVE:
            out["gidx/" + k] = sample_index(name + k, g.size)
            out["gval/" + k] = g[out["gidx/" + k]]
            out["gnorm/" + k] = np.array(np.linalg.norm(g))
        else:
            out["grad/" + k] = prm.grad.numpy()
    meta = dict(cfg, name=name, seed=seed, causal=causal, dense=dense, train=train,
                min_abs_preact=probe["min_abs_preact"], receptive_field=model.receptive_field(),
                torch=torch.__version__)
    out["meta"] = np.array(json.dumps(meta))
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(OUT, exist_ok=True)
    only = set(sys.argv[1:])
    for name, cfg in CASES.items():
        if only and name not in only:
            continue
        data = build_case(name, cfg)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **data)
        meta = json.loads(str(data["meta"]))
        print(f"{name}: y{tuple(data['y'].shape)} min|preact| {meta['min_abs_preact']:.1e} "
              f"-> {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
