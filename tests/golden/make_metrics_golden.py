"""Golden values of the evaluation metrics, produced by the REAL reference.

    python tests/golden/make_metrics_golden.py [--reference DIR]

Writes `tests/golden/metrics/*.npz`.  Each file holds a seeded input and what the reference computes
from it: `common/loss.py` (mpjpe, n_mpjpe, p_mpjpe, mean_velocity_error) applied as run.py:674-704
does, test-time flip averaging included, once in float32 (the dtype run.py computes in) and once
with the same code on float64 inputs.  Entries:
  pred      (copies, frames, J, 3) float32   model output (row 1 = mirrored copy when copies = 2)
  batch_3d  (copies, frames, J, 3) float32   3-D batch as the generator yields it (root = trajectory)
  ref32, ref64  [P1, P2, P3, MPJVE] in metres ("kind" = "sequence"), or [P1, P3] ("kind" =
            "n_mpjpe": a multi-sample 4-D input scored by mpjpe and n_mpjpe only)
  det_h_negative  frames whose Procrustes cross-covariance has det < 0 (the reflection branch)
  meta      json: kind, seed, J, copies, joints_left / joints_right (None = x negation only)
`make_case(name, reference_dir)` regenerates one case (used by the CPU test that checks the files).
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "metrics")

H36M_LEFT, H36M_RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]   # run.py:104-105, 17 joints

# name -> (kind, seed, J, frames, copies, mirror lists)
CASES = {
    "near_identity_j17": ("sequence", 11, 17, 240, 1, None),
    "rigid_j17": ("sequence", 12, 17, 240, 1, None),
    "mirrored_j15": ("sequence", 13, 15, 200, 1, None),
    "rigid_j15": ("sequence", 14, 15, 200, 1, None),
    "tta_h36m_j17": ("sequence", 15, 17, 300, 2, (H36M_LEFT, H36M_RIGHT)),
    "tta_trajectory_j17": ("sequence", 16, 17, 120, 2, None),
    "n_mpjpe_multi_j17": ("n_mpjpe", 17, 17, 60, 4, None),
}


def _poses(rng, frames, joints):
    """Smooth pose sequence (metres) with a moving root (joint 0 = global trajectory)."""
    base = rng.normal(0.0, 0.25, (joints, 3))
    motion = np.cumsum(rng.normal(0.0, 0.004, (frames, joints, 3)), axis=0)
    root = np.array([0.1, -0.2, 4.5]) + np.cumsum(rng.normal(0.0, 0.01, (frames, 3)), axis=0)
    p = base[None] + motion
    p[:, 0] = root
    return p


def _rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def _inputs(name):
    kind, seed, J, F, copies, lists = CASES[name]
    rng = np.random.RandomState(seed)
    t = _poses(rng, F, J)
    tz = t.copy()
    tz[:, 0] = 0
    if kind == "n_mpjpe":
        batch = np.stack([_poses(rng, F, J) for _ in range(copies)])
        pred = batch * rng.uniform(0.7, 1.3, (copies, F, 1, 1)) + rng.normal(0, 0.02, batch.shape)
        return pred.astype(np.float32), batch.astype(np.float32)
    if name.startswith("near_identity"):
        p = tz + rng.normal(0, 0.002, tz.shape)
    elif name.startswith("rigid"):
        r = _rotations(rng, F)
        p = rng.uniform(0.8, 1.2, (F, 1, 1)) * np.einsum("fja,fab->fjb", tz, r)
        p += rng.normal(0, 0.5, (F, 1, 3)) + rng.normal(0, 0.01, tz.shape)
    elif name.startswith("mirrored"):
        p = tz * np.array([-1.0, 1.0, 1.0]) + rng.normal(0, 0.005, tz.shape)
    else:   # TTA: the model's output on the plain and on the mirrored input
        p0 = tz + rng.normal(0, 0.01, tz.shape)
        p1 = tz + rng.normal(0, 0.01, tz.shape)
        p1[..., 0] *= -1
        if lists is not None:
            left, right = lists
            p1[:, left + right] = p1[:, right + left]
        p = np.stack([p0, p1])
    pred = p if copies == 2 else p[None]
    batch = np.stack([t] * copies)
    if copies == 2:
        batch[1, ..., 0] *= -1
    return pred.astype(np.float32), batch.astype(np.float32)


def _reference_loss(reference_dir):
    if reference_dir not in sys.path:
        sys.path.insert(0, reference_dir)
    import common.loss as ref_loss
    return ref_loss


def _run_py(ref_loss, pred_np, batch_np, lists, dtype):
    """run.py:674-704 verbatim (the TTA branch runs when the batch holds two copies)."""
    import torch
    predicted_3d_pos = torch.from_numpy(pred_np.astype(dtype))
    augment = predicted_3d_pos.shape[0] == 2
    if augment:
        predicted_3d_pos[1, :, :, 0] *= -1
        if lists is not None:
            joints_left, joints_right = lists
            predicted_3d_pos[1, :, joints_left + joints_right] = \
                predicted_3d_pos[1, :, joints_right + joints_left]
        predicted_3d_pos = torch.mean(predicted_3d_pos, dim=0, keepdim=True)
    inputs_3d = torch.from_numpy(batch_np.astype(dtype))
    inputs_3d[:, :, 0] = 0
    if augment:
        inputs_3d = inputs_3d[:1]
    e1 = ref_loss.mpjpe(predicted_3d_pos, inputs_3d).item()
    e3 = ref_loss.n_mpjpe(predicted_3d_pos, inputs_3d).item()
    inputs = inputs_3d.cpu().numpy().reshape(-1, inputs_3d.shape[-2], inputs_3d.shape[-1])
    pred = predicted_3d_pos.cpu().numpy().reshape(-1, inputs_3d.shape[-2], inputs_3d.shape[-1])
    e2 = ref_loss.p_mpjpe(pred, inputs)
    ev = ref_loss.mean_velocity_error(pred, inputs)
    det = _det_h(pred.astype(np.float64), inputs.astype(np.float64))
    return np.array([e1, e2, e3, ev], dtype=np.float64), int((det < 0).sum())


def _det_h(pred, target):
    x0 = target - target.mean(axis=1, keepdims=True)
    y0 = pred - pred.mean(axis=1, keepdims=True)
    return np.linalg.det(np.einsum("fja,fjb->fab", x0, y0))


def make_case(name, reference_dir):
    import torch
    ref_loss = _reference_loss(reference_dir)
    kind, seed, J, F, copies, lists = CASES[name]
    pred, batch = _inputs(name)
    out = {"pred": pred, "batch_3d": batch}
    if kind == "n_mpjpe":
        for tag, dt in (("ref32", np.float32), ("ref64", np.float64)):
            p, t = torch.from_numpy(pred.astype(dt)), torch.from_numpy(batch.astype(dt))
            out[tag] = np.array([ref_loss.mpjpe(p, t).item(), ref_loss.n_mpjpe(p, t).item()])
        out["det_h_negative"] = np.int64(0)
    else:
        out["ref32"], _ = _run_py(ref_loss, pred, batch, lists, np.float32)
        out["ref64"], neg = _run_py(ref_loss, pred, batch, lists, np.float64)
        out["det_h_negative"] = np.int64(neg)
    meta = dict(kind=kind, seed=seed, J=J, copies=copies,
                joints_left=lists[0] if lists else None, joints_right=lists[1] if lists else None)
    out["meta"] = np.array(json.dumps(meta))
    return out


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
        print(f"{path}: ref32 {case['ref32']}, det<0 frames {int(case['det_h_negative'])}, "
              f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
