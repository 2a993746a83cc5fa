"""Byte counts of every caller-sized device buffer, over a grid of plans.

    python tests/golden/make_workspace_layouts.py [OUT]      (needs a CUDA device)

Writes `tests/golden/workspace_layouts.json` (or OUT): what the library returns for
vp3d_workspace_bytes, vp3d_train_workspace_bytes, vp3d_stream_state_bytes_ex (flags 0 and
VP3D_STREAM_AUGMENT) and vp3d_clips_workspace_bytes on each plan of PLANS, and
vp3d_int8_thresholds_scratch_bytes for every layer count.  A zero is recorded as it is returned (a
size the entry refuses).  tests/test_gpu_workspace_layouts.py asserts that the library still returns
every one of these numbers: each layout carves its buffers in a fixed order, and a caller that sized
a buffer with one build must be able to hand it to the next.
"""
import ctypes
import itertools
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "workspace_layouts.json")

ARCS = ([3], [3, 3, 3], [3, 5, 3], [3, 3, 3, 3, 3])
CHANNELS = (64, 100, 1024)
PRECISIONS = ("bf16", "bf16x3", "fp16", "int8")
# (variant, dense): TemporalModel, its dense ablation, TemporalModelOptimized1f
MODELS = (("dilated", 0), ("dilated", 1), ("strided", 0))
PLANS = [dict(variant=v, dense=d, causal=c, arc=a, channels=ch, precision=pr)
         for (v, d), c, a, ch, pr in itertools.product(MODELS, (0, 1), ARCS, CHANNELS, PRECISIONS)]
J_IN, FEATURES, J_OUT = 17, 2, 17


def _capi():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from videopose3d_b200 import _capi
    return _capi


def create_plan(lib, case):
    """The plan of one PLANS entry, or None where vp3d_plan_create refuses it (int8 blocks whose
    int32 sums could overflow)."""
    capi = _capi()
    cfg = capi.Config()
    cfg.num_joints_in, cfg.in_features, cfg.num_joints_out = J_IN, FEATURES, J_OUT
    cfg.num_widths = len(case["arc"])
    for i, w in enumerate(case["arc"]):
        cfg.filter_widths[i] = w
    cfg.causal, cfg.channels, cfg.dense = case["causal"], case["channels"], case["dense"]
    cfg.variant = capi.VP3D_VARIANT_STRIDED if case["variant"] == "strided" else capi.VP3D_VARIANT_DILATED
    cfg.precision = getattr(capi, "VP3D_PRECISION_" + case["precision"].upper())
    h = ctypes.c_void_p()
    rc = lib.vp3d_plan_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == -2:
        return None
    capi.check(rc, "vp3d_plan_create")
    return h


def measure(lib, plan):
    """Every size of one plan, as lists of [arguments..., bytes]."""
    rf = lib.vp3d_receptive_field(plan)
    frames = (rf - 1, rf, rf + 7, 2 * rf + 100)
    out = {"workspace": [], "train_workspace": [], "stream_state": [], "clips_workspace": []}
    for n, t in itertools.product((1, 5, 1024), frames):
        out["workspace"].append([n, t, lib.vp3d_workspace_bytes(plan, n, t)])
        out["train_workspace"].append([n, t, lib.vp3d_train_workspace_bytes(plan, n, t)])
    for s, k, flags in itertools.product((1, 5, 64), (1, 8, 300), (0, 1)):
        out["stream_state"].append([s, k, flags, lib.vp3d_stream_state_bytes_ex(plan, s, k, flags)])
    for rows, flags in itertools.product((rf, 2 * rf + 2, 9000, 250000), (0, 1)):
        out["clips_workspace"].append([rows, flags, lib.vp3d_clips_workspace_bytes(plan, rows, flags)])
    return out


def scratch_sizes(lib):
    """[layers, vp3d_int8_thresholds_scratch_bytes(layers)] for layers 0 .. VP3D_MAX_LAYERS + 1."""
    return [[n, lib.vp3d_int8_thresholds_scratch_bytes(n)]
            for n in range(_capi().VP3D_MAX_LAYERS + 2)]


def main(path):
    lib = _capi().load()
    plans = []
    for case in PLANS:
        plan = create_plan(lib, case)
        if plan is None:
            continue
        plans.append(dict(case, **measure(lib, plan)))
        lib.vp3d_plan_destroy(plan)
    table = {"int8_thresholds_scratch": scratch_sizes(lib), "plans": plans}
    with open(path, "w") as f:
        json.dump(table, f, separators=(",", ":"))
        f.write("\n")
    print(f"{path}: {len(plans)} plans")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
