"""float64 NumPy statement of the evaluation metrics (TEST ORACLE for the metrics of csrc/pose_loss.cu).

Written from the definitions, not from the reference's code:
  * P1, MPJPE: mean over frames and joints of the Euclidean distance;
  * P2, P-MPJPE: per frame, the similarity transform (translation, isotropic scale, proper
    rotation) of the prediction that best fits the target in least squares (orthogonal
    Procrustes by SVD with the det = +1 constraint), then P1;
  * P3, N-MPJPE: per frame, the least-squares scale <t, p> / <p, p> of the prediction, then P1;
  * MPJVE: P1 of the first differences along the frame axis;
  * the test-time flip average: mean of the prediction and its mirrored copy with x negated and
    left / right joints exchanged back.
Frames are indexed by every axis but the last two (joints, xyz).
"""
import numpy as np


def _frames(a):
    a = np.asarray(a, dtype=np.float64)
    return a.reshape(-1, a.shape[-2], a.shape[-1])


def mpjpe(pred, target):
    return float(np.mean(np.linalg.norm(_frames(pred) - _frames(target), axis=-1)))


def procrustes_align(pred, target):
    """Per frame: s * (p - mean p) @ R + mean t, minimising the squared distance to t."""
    p, t = _frames(pred), _frames(target)
    pc = p - p.mean(axis=1, keepdims=True)
    tc = t - t.mean(axis=1, keepdims=True)
    # maximise tr(R^T M), M = pc^T tc (3x3 per frame): R = U diag(1, 1, d) V^T
    m = np.einsum("fja,fjb->fab", pc, tc)
    u, sv, vt = np.linalg.svd(m)
    d = np.sign(np.linalg.det(np.einsum("fab,fbc->fac", u, vt)))
    dd = np.ones_like(sv)
    dd[:, 2] = d
    r = np.einsum("fab,fb,fbc->fac", u, dd, vt)
    scale = (sv * dd).sum(axis=1) / np.einsum("fja,fja->f", pc, pc)
    return scale[:, None, None] * np.einsum("fja,fab->fjb", pc, r) + t.mean(axis=1, keepdims=True)


def p_mpjpe(pred, target):
    return mpjpe(procrustes_align(pred, target), target)


def n_mpjpe(pred, target):
    p, t = _frames(pred), _frames(target)
    s = np.einsum("fja,fja->f", t, p) / np.einsum("fja,fja->f", p, p)
    return mpjpe(s[:, None, None] * p, t)


def mean_velocity_error(pred, target):
    p, t = _frames(pred), _frames(target)
    return mpjpe(np.diff(p, axis=0), np.diff(t, axis=0))


def mirror_map(joints, left, right):
    """src[j]: the joint of the mirrored copy that lands on joint j (later pairs win)."""
    src = np.arange(joints)
    for dst, s in zip(list(left) + list(right), list(right) + list(left)):
        src[dst] = s
    return src


def flip_average(pred, left=None, right=None):
    """(2, frames, joints, 3) -> (1, frames, joints, 3) in float64."""
    pred = np.asarray(pred, dtype=np.float64)
    m = pred[1].copy()
    m[..., 0] *= -1
    if left is not None and right is not None:
        m = m[:, mirror_map(pred.shape[2], left, right)]
    return ((pred[0] + m) / 2)[None]


def sequence_errors(pred, batch_3d, left=None, right=None):
    """One evaluated sequence: pred (1 or 2, frames, joints, 3) model output, batch_3d the 3-D
    batch as the generator yields it.  Returns ([P1, P2, P3, MPJVE] in metres, frames weight)."""
    pred = np.asarray(pred, dtype=np.float64)
    tgt = np.array(batch_3d, dtype=np.float64)[:1]
    tgt[:, :, 0] = 0
    avg = flip_average(pred, left, right) if pred.shape[0] == 2 else pred
    e = [mpjpe(avg, tgt), p_mpjpe(avg, tgt), n_mpjpe(avg, tgt), mean_velocity_error(avg, tgt)]
    return np.array(e), tgt.shape[0] * tgt.shape[1]
