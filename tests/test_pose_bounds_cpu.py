"""CPU: the float64 references and error bounds of tests/pose_bounds.py, which gate the pose-loss
and metrics kernel in test_gpu_pose_kernels.py.  The reference rounded to nearest fp32 passes its
own gates, every wrong answer the gates exist to catch fails them, and the two P-MPJPE routes
(autograd through the SVD, Horn's quaternion form) agree within the fp64 term at every gap the GPU
test uses."""
import math
import warnings

import numpy as np
import pytest
import torch

import pose_bounds as pb
from oracle import pose_loss_oracle as po

WEIGHTS = [(1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 1.0, 0.0), (0.0, 0.0, 0.0, 1.0),
           (1.0, 0.5, 0.25, 2.0)]


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


@pytest.mark.parametrize("J,F,seqs", [(1, 1, 5), (2, 2, 9), (3, 27, 2), (15, 1, 40), (17, 27, 3),
                                      (32, 243, 1)])
def test_rounded_reference_passes_its_own_gate(J, F, seqs):
    p, t = pb.random_poses(np.random.RandomState(J), seqs, F, J)
    ref = pb.Reference(p, t)
    depth = pb.sum_depth(ref.poses, 132)
    for w in WEIGHTS:
        g64 = ref.grad_ref(w)
        assert pb.ratio(pb.round_nearest(g64), g64, ref.grad_bound(w)) <= 1.0, w
        loss = ref.loss_ref(w)
        assert pb.ratio(np.float32(loss), loss, ref.loss_bound(w, depth)) <= 1.0, w
    for k in range(4):
        assert pb.ratio(np.float32(ref.value[k]), ref.value[k], ref.term_bound(k, depth)) <= 1.0, k


@pytest.mark.parametrize("J", [3, 17, 32])
def test_every_wrong_answer_fails_the_gate(J):
    p, t = pb.random_poses(np.random.RandomState(100 + J), 4, 27, J)
    ref = pb.Reference(p, t)
    seen = set()
    for k in range(4):
        w = [float(i == k) for i in range(4)]
        g64, bound = ref.grad_ref(w), ref.grad_bound(w)
        for name, wrong in pb.demonstrations(ref, k):
            r = pb.ratio(wrong, g64, bound)
            assert r > 1.0, f"{pb.NAMES[k]}: the gate accepts the gradient with {name} ({r:.3f})"
            seen.add(name)
    assert seen == {"rounded toward zero", "one pose swapped with its neighbour", "scale detached",
                    "rotation detached", "no start difference"}


def test_round_toward_zero_differs_from_nearest():
    x = np.array([1.0 + 2.0 ** -24 + 2.0 ** -30, -(1.0 + 2.0 ** -24 + 2.0 ** -30), 1.0, -3.0])
    assert pb.round_toward_zero(x).tolist() == [1.0, -1.0, 1.0, -3.0]
    assert pb.round_nearest(x)[0] == np.float32(1.0 + 2.0 ** -23)


def _horn_vs_svd(p, t):
    """Worst ratio of |g_horn - g_svd| to the fp64 gradient term over the finite non-degenerate
    poses, and of the two values' difference to the fp64 value term."""
    ref = pb.Reference(p, t)
    hs = ref.horn
    keep = hs["finite"] & ~hs["degenerate"]
    P, J = ref.poses, ref.J
    p3, t3 = ref.p.reshape(P, J, 3)[keep], ref.t.reshape(P, J, 3)[keep]
    x = torch.from_numpy(p3).requires_grad_(True)
    v_svd = po.p_mpjpe(x, torch.from_numpy(t3))
    v_svd.backward()
    v_horn, g_horn, _ = po.p_mpjpe_horn(p3, t3)
    n = keep.sum()
    g0 = ref.G[2].reshape(P, J)[keep] * pb.K_GRAD[2] / (1 + 1 / hs["gap_rel"][keep]
                                                         + np.where(hs["svd_cond"][keep] <= pb.SVD_COND_MAX,
                                                                    hs["svd_cond"][keep],
                                                                    1 / hs["gap_rel"][keep]))[:, None]
    cond = 1 + 1 / hs["gap_rel"][keep] + hs["svd_cond"][keep]
    bound = pb.E * g0 * cond[:, None] * ref.count[2] / (n * J)
    r_grad = pb.ratio(g_horn, x.grad.numpy(), bound[..., None])
    sub = pb.Reference(p.reshape(P, 1, J, 3)[keep][None, :, 0], t.reshape(P, 1, J, 3)[keep][None, :, 0])
    r_val = abs(float(v_svd.detach()) - v_horn) / sub.value_fp64_err(2, 1)
    return r_grad, r_val, hs["gap_rel"][keep]


def test_horn_and_svd_agree_at_every_gap_the_gpu_test_uses():
    rng = np.random.RandomState(7)
    gaps = []
    for name, p, t in pb.rotation_cases(rng) + [("random_j3", *pb.random_poses(rng, 2, 27, 3)),
                                                ("random_j32", *pb.random_poses(rng, 2, 27, 32))]:
        r_grad, r_val, g = _horn_vs_svd(p, t)
        print(f"{name}: gradient {r_grad:.3g}, value {r_val:.3g} of the fp64 term; "
              f"smallest gap_rel {g.min():.3g}")
        assert r_grad <= 1.0 and r_val <= 1.0, name
        gaps.append(g)
    gaps = np.concatenate(gaps)
    assert gaps.min() < 1e-9 and (gaps < 1e-6).sum() >= 2    # the planar poses above the threshold


def test_planar_constructions_straddle_the_threshold():
    rng = np.random.RandomState(11)
    (_, p, t), = [c for c in pb.rotation_cases(rng) if c[0] == "planar"]
    hs = pb.horn_stats(p[0].astype(np.float64), t[0].astype(np.float64))
    gap = hs["gap_rel"][:2 * len(pb.PLANAR_EPS)].reshape(-1, 2)
    print("planar gap_rel per eps:", {e: g.tolist() for e, g in zip(pb.PLANAR_EPS, gap)})
    assert (gap[0] == 0).all() and (gap[1] < po.DEGENERATE_GAP / 10).all()
    assert (gap[3] > po.DEGENERATE_GAP * 10).all() and (gap[3] < 1e-9).all()
    assert (gap[4] > 1e-8).all()
    assert (hs["sv"][:2 * len(pb.PLANAR_EPS), 2] == 0).all()


def test_sum_depth_and_passes():
    assert pb.sum_depth(5, 132) == 1 + 5 + 8 + 1 + 1
    assert pb.min_passes(64 * 243, 132) == math.ceil(64 * 243 / (8 * 264))
    assert pb.min_passes(32 * 1024 + 1, 2) == math.ceil((32 * 1024 + 1) / 32)
