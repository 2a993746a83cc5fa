"""Every caller-sized buffer keeps its byte count: the library must return exactly the sizes recorded
in tests/golden/workspace_layouts.json (tests/golden/make_workspace_layouts.py) for the eval, clip
and training workspaces, the streaming state and the int8 threshold scratch, over a grid of plans
(both variants, causal and dense, channels 64 / 100 / 1024, bf16 / bf16x3 / fp16 / int8) and
shapes, refusals (0) included."""
import json
import os
import sys

import pytest

from videopose3d_b200 import _capi

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
try:
    import make_workspace_layouts as mk
finally:
    sys.path.pop(0)

with open(mk.OUT) as f:
    TABLE = json.load(f)
SIZES = ("workspace", "train_workspace", "stream_state", "clips_workspace")


def test_int8_thresholds_scratch_bytes():
    assert mk.scratch_sizes(_capi.load()) == TABLE["int8_thresholds_scratch"]


def test_fixture_covers_the_plan_grid():
    stored = [{k: p[k] for k in mk.PLANS[0]} for p in TABLE["plans"]]
    missing = [c for c in mk.PLANS if c not in stored]
    # only plans vp3d_plan_create refuses: int8 dense blocks whose int32 sums could overflow
    assert len(stored) + len(missing) == len(mk.PLANS)
    assert missing and all(c["precision"] == "int8" and c["dense"] for c in missing)


@pytest.mark.gpu
def test_plan_sizes_match_the_fixture(cuda_device):
    lib = _capi.load()
    wrong = []
    for case in TABLE["plans"]:
        plan = mk.create_plan(lib, case)
        assert plan is not None, case
        try:
            got = mk.measure(lib, plan)
        finally:
            lib.vp3d_plan_destroy(plan)
        for k in SIZES:
            wrong += [(case, k, want, new) for want, new in zip(case[k], got[k]) if want != new]
            assert len(got[k]) == len(case[k])
    assert not wrong, f"{len(wrong)} sizes differ, first: {wrong[0]}"
