"""GPU: both instances of the pose kernel (csrc/pose_loss.cu, procrustes.cuh) element by element
against float64, with the bounds derived in tests/pose_bounds.py.

Loss instance (`vp3d_pose_loss_fwd_bwd` through `loss.pose_loss`): every term alone and all four
weighted together; each gradient element, each term and the loss within its bound; the degenerate
count equal to Horn's rule (except for poses within 10x of the threshold); the forward without a
gradient bit-identical to the forward with one.  Sizes: fewer than 8 poses, 1024 x 1, the training
shape 64 x 243 (several grid-stride passes unlimited), and 32k + a few poses on a grid capped to
2 SMs (hundreds of passes, ragged for one and two blocks per SM); J in {1, 2, 3, 15, 17, 32};
F in {1, 2, 27, 243}, so velocity neighbours straddle sequence, block and pass boundaries.  The
largest case is run twice and must give the same bits.  P-MPJPE rotations: reflected poses,
exactly collinear ones, exactly planar ones whose gap falls on both sides of the threshold,
improper H with s2 = s3, identical prediction and target, and zero-spread poses (NaN where the
reference gives NaN).

Metrics instance (`vp3d_pose_errors`): F in {1, 2, 100 001}, one copy or two with and without a
mirror map, J in {15, 17, 32}; each `which` bit alone and all four; unselected slots 0; the means
within the fp64 bound of oracle/metrics_oracle.py on the kernel's own flip average, which must be
bit-identical to run.py:677-680's torch expression; the loss's fp32 term equal to the metric rounded
where both grids are equal and within one fp32 ulp of it elsewhere.

Prints the worst ratio to its bound per gate, the case count and the wall time.
"""
import time
import warnings

import numpy as np
import pytest
import torch

import pose_bounds as pb
from oracle import pose_loss_oracle as po
from videopose3d_b200 import _capi
from videopose3d_b200 import loss as vloss
from videopose3d_b200 import metrics

pytestmark = pytest.mark.gpu

WEIGHTS = [(1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 1.0, 0.0), (0.0, 0.0, 0.0, 1.0),
           (1.0, 0.5, 0.25, 2.0)]
WORST = {}            # gate -> (ratio, case)
COUNT = {"cases": 0, "multi_pass": 0}
T0 = time.time()


@pytest.fixture
def sm_limit():
    """Caps the cooperative grid of the pose kernel; always restores the default."""
    lib = _capi.load()

    def set_limit(n):
        _capi.check(lib.vp3d_set_sm_limit(n), "vp3d_set_sm_limit")
    try:
        yield set_limit
    finally:
        _capi.check(lib.vp3d_set_sm_limit(0), "vp3d_set_sm_limit")


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _note(gate, r, where):
    assert r <= 1.0, f"{where}: {gate} off by {r:.3g} of its bound"
    if gate not in WORST or r > WORST[gate][0]:
        WORST[gate] = (r, where)


def _report(tag):
    print(f"\n{tag}: {COUNT['cases']} cases ({COUNT['multi_pass']} with the pass loop run more than "
          f"once with gradients on), {time.time() - T0:.1f} s; worst ratio per gate: "
          + ", ".join(f"{k} {v[0]:.3g} ({v[1]})" for k, v in sorted(WORST.items())))


def _loss(p, t, w, grad):
    pd = torch.from_numpy(p).cuda().requires_grad_(grad)
    loss, terms, deg = vloss.pose_loss(pd, torch.from_numpy(t).cuda(), *w, return_degenerate=True)
    if grad:
        loss.backward()
    torch.cuda.synchronize()
    return (loss.detach().cpu().numpy(), terms.cpu().numpy(), int(deg),
            pd.grad.cpu().numpy() if grad else None)


def _check_loss(p, t, sms, tag, weights=WEIGHTS):
    """Every gate on one (seqs, F, J, 3) batch; returns the last run's outputs."""
    ref = pb.Reference(p, t)
    depth = pb.sum_depth(ref.poses, sms)
    near = pb.near_threshold(ref.gap_rel)
    deg_clear = int((ref.horn["degenerate"] & ~near).sum())
    COUNT["cases"] += 1
    if pb.min_passes(ref.poses, sms) > 1:
        COUNT["multi_pass"] += 1
    out = None
    for w in weights:
        where = f"{tag} w={w}"
        loss, terms, deg, g = _loss(p, t, w, True)
        name = "+".join(pb.NAMES[k] for k in range(4) if w[k]) if sum(map(bool, w)) == 1 else "combined"
        _note(f"grad {name}", pb.ratio(g, ref.grad_ref(w), ref.grad_bound(w)), where)
        for k in range(4):
            if w[k]:
                _note(f"term {pb.NAMES[k]}", pb.ratio(terms[k], ref.value[k], ref.term_bound(k, depth)), where)
            else:
                assert terms[k] == 0, f"{where}: unselected term {k} is {terms[k]}"
        _note("loss", pb.ratio(loss, ref.loss_ref(w), ref.loss_bound(w, depth)), where)
        if w[2]:
            assert deg_clear <= deg <= deg_clear + int(near.sum()), \
                f"{where}: {deg} degenerate poses, Horn's rule gives {ref.degenerate} ({int(near.sum())} near)"
        else:
            assert deg == 0
        f_loss, f_terms, f_deg, _ = _loss(p, t, w, False)
        assert f_loss.tobytes() == loss.tobytes() and f_terms.tobytes() == terms.tobytes() and f_deg == deg, \
            f"{where}: the forward without a gradient differs"
        out = (loss, terms, deg, g)
    return ref, out


# (J, F, seqs, SM limit): < 8 poses; 1024 x 1; the training shape; 32k + a few poses on 2 SMs
LOSS_CASES = [
    (1, 1, 5, 0), (2, 2, 3, 0), (3, 1, 7, 0), (15, 2, 3, 0), (17, 1, 5, 0), (32, 2, 3, 0),
    (17, 1, 1024, 0), (32, 1, 1024, 0), (2, 2, 512, 0),
    (17, 243, 64, 0), (15, 27, 576, 0),
    (1, 1, 32769, 2), (2, 2, 16385, 2), (3, 27, 1214, 2), (17, 27, 1214, 2), (15, 243, 135, 2),
    (32, 243, 135, 2),
]


@pytest.mark.parametrize("J,F,seqs,limit", LOSS_CASES,
                         ids=[f"j{c[0]}_f{c[1]}_s{c[2]}_lim{c[3]}" for c in LOSS_CASES])
def test_loss_against_float64(cuda_device, sm_limit, J, F, seqs, limit):
    sm_limit(limit)
    sms = limit or _sms()
    p, t = pb.random_poses(np.random.RandomState(J * 1000 + F + seqs), seqs, F, J)
    tag = f"J={J} F={F} seqs={seqs} limit={limit} passes>={pb.min_passes(F * seqs, sms)}"
    ref, (loss, terms, deg, g) = _check_loss(p, t, sms, tag)
    if J == 2:
        assert deg == F * seqs                       # two joints are always collinear
    if J == 1:
        assert np.isnan(terms[2]) and np.isnan(g).all()   # P-MPJPE of one joint: 0 / 0
    if (J, F, seqs, limit) == max(LOSS_CASES, key=lambda c: c[0] * c[1] * c[2]):
        again = _loss(p, t, WEIGHTS[-1], True)
        assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes()
                   for a, b in zip(again, (loss, terms, deg, g))), "two runs differ"
        # the gates reject a gradient rounded toward zero or one pose swapped with its neighbour
        for name, wrong in pb.demonstrations(ref, 2)[:2]:
            w = (0.0, 0.0, 1.0, 0.0)
            assert pb.ratio(wrong, ref.grad_ref(w), ref.grad_bound(w)) > 1.0, name
    _report(tag)


@pytest.mark.parametrize("name", ["reflected", "collinear", "improper_s2_eq_s3", "identical",
                                  "zero_spread", "planar"])
def test_p_mpjpe_rotations(cuda_device, name):
    rng = np.random.RandomState(31)
    (_, p, t), = [c for c in pb.rotation_cases(rng) if c[0] == name]
    ref, (loss, terms, deg, g) = _check_loss(p, t, _sms(), name,
                                             weights=[(0.0, 0.0, 1.0, 0.0), WEIGHTS[-1]])
    hs = ref.horn
    P = ref.poses
    print(f"\n{name}: Horn degenerate {ref.degenerate}, kernel {deg}; gap_rel of the special poses: "
          + np.array2string(np.sort(hs["gap_rel"][np.isfinite(hs["gap_rel"])])[:10], precision=2))
    g3 = g.reshape(P, ref.J, 3)
    if name == "collinear":
        assert ref.degenerate == 5 and deg == 5
    elif name == "improper_s2_eq_s3":
        assert ref.degenerate == 5 and deg == 5
        assert np.isfinite(g).all()
    elif name == "identical":     # zero errors: mpjpe and N-MPJPE have zero gradients there
        for w in ((1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0)):
            _, _, _, gz = _loss(p, t, w, True)
            assert (gz.reshape(P, ref.J, 3)[::3] == 0).all()
    elif name == "zero_spread":
        assert np.isnan(terms[2]) and np.isnan(loss)
        bad = ~hs["finite"]
        assert bad.sum() == 3 and np.isnan(g3[bad]).all() and np.isfinite(g3[~bad]).all()
    elif name == "planar":
        gaps = hs["gap_rel"][:2 * len(pb.PLANAR_EPS)]
        assert (gaps[:4] < po.DEGENERATE_GAP / 10).all() and (gaps[6:8] > po.DEGENERATE_GAP * 10).all()
        print("planar gap_rel per eps:", {e: gaps[2 * i:2 * i + 2].tolist()
                                          for i, e in enumerate(pb.PLANAR_EPS)})
    _report(name)


LR15 = ([2, 3, 4, 8, 9, 10], [5, 6, 7, 11, 12, 13])
LR17 = ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16])
LR32 = (list(range(1, 16)), list(range(16, 31)))
MIRROR = {15: LR15, 17: LR17, 32: LR32}


def _torch_flip_average(pred, lists):
    want = pred.clone()                                     # run.py:677-680, literally
    want[1, :, :, 0] *= -1
    if lists is not None:
        jl, jr = lists
        want[1, :, jl + jr] = want[1, :, jr + jl]
    return torch.mean(want, dim=0, keepdim=True)


METRIC_CASES = [(F, mode, J) for F in (1, 2, 100_001) for mode in ("one", "two", "two_mirror")
                for J in (15, 17, 32)]


@pytest.mark.parametrize("F,mode,J", METRIC_CASES, ids=[f"f{c[0]}_{c[1]}_j{c[2]}" for c in METRIC_CASES])
def test_metrics_against_float64(cuda_device, F, mode, J):
    rng = np.random.RandomState(F + J)
    copies = 1 if mode == "one" else 2
    p, t = pb.random_poses(rng, 1, F, J)
    pred = torch.from_numpy(p[0]).cuda()
    if copies == 2:    # the mirrored copy of a slightly different prediction
        q = torch.from_numpy((p[0] + rng.normal(0, 0.02, p[0].shape)).astype(np.float32)).cuda()
        pred = torch.stack([pred, q])
    else:
        pred = pred[None]
    tgt = torch.from_numpy(t[0]).cuda()
    lists = MIRROR[J] if mode == "two_mirror" else None
    src = metrics._mirror_src(J, *lists, pred.device) if lists else None
    want_avg = _torch_flip_average(pred, lists) if copies == 2 else pred
    sms = _sms()
    depth = pb.sum_depth(F, sms)
    ref = None
    COUNT["cases"] += 1
    for which in (1, 2, 4, 8, 15):
        avg = torch.full((1, F, J, 3), float("nan"), device=pred.device)
        means = metrics._launch(pred, copies, src, tgt, F, J, which, avg).cpu().numpy()
        assert torch.equal(avg, want_avg), f"F={F} {mode} J={J}: averaged differs from torch"
        if ref is None:
            a = avg.cpu().numpy()
            ref = pb.Reference(a[None, 0], t[None, 0])
            want = pb.metric_means(a[0], t[0])
        for k in range(4):
            slot = pb.EVAL_SLOT[k]
            where = f"F={F} {mode} J={J} which={which}"
            if which >> slot & 1:
                assert abs(want[slot] - ref.value[k]) <= ref.value_fp64_err(k, 1) or np.isnan(want[slot])
                _note(f"mean {pb.NAMES[k]}", pb.ratio(means[slot], want[slot], ref.value_fp64_err(k, depth)),
                      where)
            else:
                assert means[slot] == 0, f"{where}: unselected slot {slot} is {means[slot]}"
    # the loss instance on the same averaged poses: its fp32 terms are the metrics rounded
    _, terms, _, _ = _loss(want_avg.cpu().numpy(), t, (1.0, 1.0, 1.0, 1.0), False)
    same_grid = F <= pb.POSE_WARPS * sms                   # one block per 8 poses in both instances
    for k in range(4):
        m = means[pb.EVAL_SLOT[k]]
        if np.isnan(m):
            assert np.isnan(terms[k])
        elif same_grid:
            assert np.float32(m) == terms[k], (k, float(terms[k]), m)
        else:
            assert abs(float(terms[k]) - m) <= np.spacing(np.float32(m)), (k, float(terms[k]), m)
    _report(f"metrics F={F} {mode} J={J}")
