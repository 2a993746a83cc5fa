"""CPU: the fp64 oracle of the input gradient against the reference's own goldens, and the error
paths of the input-gradient C entry points without a GPU.

The fixtures in golden/input_grad/ come from the reference classes in float64 with x requiring grad
(tests/golden/make_input_grad_golden.py): eval() mode (BatchNorm on running statistics) and train()
mode with dropout 0.  float64 autograd through oracle.forward_torch must reproduce each one to
1e-10 -- it is the reference the GPU tests use for cases beyond the fixtures."""
import ctypes
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import temporal_model_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "input_grad")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


def load_case(name):
    """(meta, state_dict (torch float32), x, gy, y, grads) of a fixture; grads maps 'x' and every
    parameter name to either a full array or a (index, values, norm) sample."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    sd = orc.make_state_dict(meta["J"], meta["F"], meta["Jout"], meta["fw"], meta["C"],
                             dense=meta["dense"], seed=meta["seed"])
    grads = {}
    for k in z.files:
        if k.startswith("grad/"):
            grads[k[5:]] = z[k]
        elif k.startswith("gidx/"):
            n = k[5:]
            grads[n] = (z[k], z["gval/" + n], float(z["gnorm/" + n]))
    return meta, sd, torch.from_numpy(z["x"]), torch.from_numpy(z["gy"]), z["y"], grads


def oracle_grads(meta, sd, x, gy, masks=None):
    """float64 autograd through forward_torch in the fixture's mode: (y, {'x': dx, name: grad})."""
    sd = {k: v.double().clone() if v.is_floating_point() else v.clone() for k, v in sd.items()}
    leaves = {k: v.requires_grad_(True) for k, v in sd.items()
              if v.is_floating_point() and "running_" not in k}
    xd = x.double().clone().requires_grad_(True)
    y = orc.forward_torch(sd, xd, meta["fw"], causal=meta["causal"], dense=meta["dense"],
                          strided=meta["cls"] == "TemporalModelOptimized1f",
                          training=meta["train"], masks=masks)
    (y * gy.double()).sum().backward()
    out = {k: v.grad for k, v in leaves.items()}
    out["x"] = xd.grad
    return y.detach(), out


def compare(got, want):
    """Max |got - want| / max |want| over a stored gradient (full or sampled: the sampled entries
    and the L2 norm)."""
    got = torch.as_tensor(got).double()
    if isinstance(want, tuple):
        idx, val, norm = want
        flat = got.reshape(-1)
        e = float((flat[torch.from_numpy(idx)] - torch.from_numpy(val)).abs().max()
                  / np.abs(val).max())
        return max(e, abs(float(flat.norm()) - norm) / norm)
    want = torch.from_numpy(np.asarray(want)).double()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


def test_fixture_set():
    assert len(NAMES) == 15
    total = sum(os.path.getsize(os.path.join(GOLDEN, n + ".npz")) for n in NAMES)
    assert total < 2 * 1024 * 1024


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_input_gradients(name):
    meta, sd, x, gy, y_ref, grads = load_case(name)
    y, got = oracle_grads(meta, sd, x, gy)
    assert y.shape == y_ref.shape
    assert float(np.abs(y.numpy() - y_ref).max() / np.abs(y_ref).max()) <= 1e-10
    assert set(got) == set(grads)
    for k, want in grads.items():
        assert compare(got[k], want) <= 1e-10, k
    # frames past the strided prefix get no gradient
    if meta["cls"] == "TemporalModelOptimized1f":
        used = y_ref.shape[1] * int(np.prod(meta["fw"]))
        if used < x.shape[1]:
            assert float(got["x"][:, used:].abs().max()) == 0.0


# ---- C-ABI error paths (no GPU needed: every check runs before any device work) ---------------
def _lib():
    from videopose3d_b200 import _capi
    try:
        return _capi, _capi.load()
    except RuntimeError as e:
        pytest.skip(str(e))


def test_new_entries_reject_null_plan():
    capi, lib = _lib()
    w = capi.Weights()
    g = capi.Grads()
    assert lib.vp3d_forward_train_ex(None, 1, 1, 1, 27, ctypes.byref(w), None, 0.0, 0,
                                     capi.VP3D_TRAIN_FROZEN_BN, 1, 1, None) == -1
    assert lib.vp3d_backward_ex(None, 1, ctypes.byref(g), 1, 1, 1, None, None, None) == -1
    assert lib.vp3d_backward_ex(None, 1, None, 1, 1, 1, None, None, None) == -1
    # neither parameter nor input gradients
    assert lib.vp3d_backward_ex(None, 1, None, None, 1, 1, None, None, None) == -1
    assert b"neither" in lib.vp3d_last_error()


def test_frozen_bn_rejects_dropout_and_unknown_flags():
    capi, lib = _lib()
    w = capi.Weights()
    fake_plan = ctypes.c_void_p(1)   # the flag checks come before the plan is read
    assert lib.vp3d_forward_train_ex(fake_plan, 1, 1, 1, 27, ctypes.byref(w), None, 0.25, 0,
                                     capi.VP3D_TRAIN_FROZEN_BN, 1, 1, None) == -1
    assert b"dropout" in lib.vp3d_last_error()
    assert lib.vp3d_forward_train_ex(fake_plan, 1, 1, 1, 27, ctypes.byref(w), None, 0.0, 0, 6,
                                     1, 1, None) == -1
    assert b"unknown flags" in lib.vp3d_last_error()
    # without FROZEN_BN the momenta are required, as by vp3d_forward_train
    assert lib.vp3d_forward_train_ex(fake_plan, 1, 1, 1, 27, ctypes.byref(w), None, 0.0, 0, 0,
                                     1, 1, None) == -1
