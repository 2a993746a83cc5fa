"""Golden values of the differentiable pose losses, produced by the REAL reference.

    python tests/golden/make_pose_loss_golden.py [--reference DIR]

Writes `tests/golden/pose_loss/*.npz`.  Each file holds a seeded input, the four term values from
the reference's own functions in common/loss.py, and the float64 gradient of the weighted sum.
Entries:
  pred, target  (..., frames, J, 3) float32
  terms         [mpjpe, n_mpjpe, p_mpjpe, mean_velocity_error] of the reference on the float32
                inputs taken to float64 (NaN where the reference gives NaN or, for p_mpjpe on a pose
                with no spread, where its SVD raises)
  weights       the term weights of the combined loss
  grad          float64 d (sum_k weights[k] terms[k]) / d pred, autograd through the torch
                restatement oracle/pose_loss_oracle.py (NaN-filled when that loss is NaN but for the
                velocity of a single frame, whose empty mean has a zero gradient)
  degenerate    poses whose top two Horn eigenvalues are closer than 1e-12 relative
  meta          json: shape, seed, what the case exercises
The reference's functions take (frames, J, 3) for p_mpjpe and mean_velocity_error and
(N, T, J, 3) for n_mpjpe; a batch is scored as run.py does (flattened frames for p_mpjpe) and the
velocity along T within each sample (the mean over samples of equal length).
`make_case(name, reference_dir)` regenerates one case (used by the CPU test that checks the files).
"""
import argparse
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "pose_loss")

WEIGHTS = (1.0, 0.5, 0.25, 2.0)

# name -> (seed, shape, kind)
CASES = {
    "seq_j17": (21, (60, 17, 3), "noisy"),
    "seq_j15": (22, (50, 15, 3), "rigid"),
    "seq_j1": (23, (40, 1, 3), "noisy"),
    "batch_n4_t243_j17": (24, (4, 243, 17, 3), "noisy"),
    "batch_n1024_t1_j17": (25, (1024, 1, 17, 3), "rigid"),
    "batch_n8_t1_j15": (26, (8, 1, 15, 3), "noisy"),
    "mirrored_j17": (27, (30, 17, 3), "mirrored"),
    "near_degenerate_j17": (28, (2, 12, 17, 3), "near_collinear"),
    "zero_pred_j17": (29, (3, 8, 17, 3), "zero"),
}


def _rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def _inputs(name):
    seed, shape, kind = CASES[name]
    rng = np.random.RandomState(seed)
    frames = int(np.prod(shape[:-2]))
    J = shape[-2]
    base = rng.normal(0.0, 0.25, (J, 3))
    motion = np.cumsum(rng.normal(0.0, 0.01, (frames, J, 3)), axis=0)
    t = base[None] + motion + np.array([0.1, -0.2, 4.5])
    if kind == "noisy":
        p = t + rng.normal(0, 0.03, t.shape)
    elif kind == "rigid":
        p = rng.uniform(0.8, 1.2, (frames, 1, 1)) * np.einsum("fja,fab->fjb", t, _rotations(rng, frames))
        p += rng.normal(0, 0.5, (frames, 1, 3)) + rng.normal(0, 0.02, t.shape)
    elif kind == "mirrored":
        p = t * np.array([-1.0, 1.0, 1.0]) + rng.normal(0, 0.01, t.shape)
    elif kind == "near_collinear":
        # joints spread along one line with a small transverse scatter: the two largest eigenvalues
        # of Horn's matrix are close (an ill-conditioned but differentiable rotation)
        line = rng.normal(size=3)
        line /= np.linalg.norm(line)
        s = rng.uniform(-0.5, 0.5, (frames, J, 1))
        p = s * line + rng.normal(0, 2e-3, (frames, J, 3)) + np.array([0.0, 0.0, 4.0])
    else:   # zero
        p = np.zeros_like(t)
    return p.reshape(shape).astype(np.float32), t.reshape(shape).astype(np.float32)


def _reference_loss(reference_dir):
    if reference_dir not in sys.path:
        sys.path.insert(0, reference_dir)
    import common.loss as ref_loss
    return ref_loss


def reference_terms(ref_loss, pred, target):
    """The four terms from common/loss.py on float64 copies of the inputs."""
    import torch
    p, t = pred.astype(np.float64), target.astype(np.float64)
    J = p.shape[-2]
    p4 = p if p.ndim == 4 else p.reshape((1,) * (4 - p.ndim) + p.shape)
    t4 = t if t.ndim == 4 else t.reshape(p4.shape)
    e1 = ref_loss.mpjpe(torch.from_numpy(p), torch.from_numpy(t)).item()
    e3 = ref_loss.n_mpjpe(torch.from_numpy(p4), torch.from_numpy(t4)).item()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        try:
            e2 = float(ref_loss.p_mpjpe(p.reshape(-1, J, 3).copy(), t.reshape(-1, J, 3).copy()))
        except np.linalg.LinAlgError:   # no spread: NaN in the normalisation, the SVD refuses it
            e2 = float("nan")
        seqs_p = p.reshape((-1,) + p.shape[-3:])
        seqs_t = t.reshape(seqs_p.shape)
        ev = float(np.mean([ref_loss.mean_velocity_error(a, b) for a, b in zip(seqs_p, seqs_t)]))
    return np.array([e1, e2, e3, ev])[[0, 2, 1, 3]]   # -> [mpjpe, n_mpjpe, p_mpjpe, velocity]


def oracle_grad(pred, target, weights):
    """float64 gradient of the weighted sum through the torch restatement, or None when the
    restatement has none (the SVD of a NaN matrix)."""
    import torch
    sys.path.insert(0, ROOT)
    from oracle import pose_loss_oracle as po
    p = torch.tensor(pred, dtype=torch.float64, requires_grad=True)
    t = torch.tensor(target, dtype=torch.float64)
    try:
        loss, _ = po.pose_loss(p, t, weights)
    except RuntimeError:
        return None
    loss.backward()
    return p.grad.numpy()


def make_case(name, reference_dir):
    sys.path.insert(0, ROOT)
    from oracle import pose_loss_oracle as po
    ref_loss = _reference_loss(reference_dir)
    seed, shape, kind = CASES[name]
    pred, target = _inputs(name)
    terms = reference_terms(ref_loss, pred, target)
    grad = oracle_grad(pred, target, WEIGHTS)
    if grad is None:
        grad = np.full(pred.shape, np.nan)
    with np.errstate(all="ignore"):
        _, _, degenerate = po.p_mpjpe_horn(pred, target)
    meta = dict(seed=seed, shape=list(shape), kind=kind)
    return {"pred": pred, "target": target, "terms": terms, "weights": np.array(WEIGHTS),
            "grad": grad, "degenerate": np.int64(degenerate), "meta": np.array(json.dumps(meta))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None)
    args = ap.parse_args()
    ref = args.reference
    if ref is None:
        sys.path.insert(0, ROOT)
        from oracle import stage_ref
        ref = stage_ref.reference_dir()
    if ref is None:
        raise SystemExit("no reference checkout: pass --reference")
    os.makedirs(OUT, exist_ok=True)
    for name in CASES:
        case = make_case(name, ref)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **case)
        print(f"{path}: terms {case['terms']}, degenerate {int(case['degenerate'])}, "
              f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
