"""Evaluation metrics on the device (run.py:652-721, common/loss.py:11-89).

The reference computes its four evaluation protocols per test sequence with an `.item()` sync for
each torch metric, a copy of prediction and target to the host, and NumPy for Protocol #2 (batched
3x3 SVD per frame) and the velocity error.  Here one launch (`vp3d_pose_errors`,
csrc/pose_loss.cu) flip-averages the test-time-augmented prediction and produces all four
per-sequence means in float64; `evaluate()` keeps the frame-weighted sums on the device and syncs
once at the end.

  * `p_mpjpe`, `n_mpjpe`, `mean_velocity_error`: the reference's signatures and
    semantics, returning 0-d CUDA float64 tensors without syncing;
  * `flip_average`: run.py:675-680 (undo the mirroring of batch row 1, average with row 0);
  * `pose_errors`: [P1, P2, P3, MPJVE] of one sequence and the averaged prediction;
  * `evaluate`: run.py's evaluate() loop over a device `UnchunkedGenerator`.

CUDA float32 tensors only; there is no host or torch fallback.
"""
import torch

from . import _capi
from .generators import mirror_source

__all__ = ["p_mpjpe", "n_mpjpe", "mean_velocity_error", "flip_average", "pose_errors", "evaluate"]

_ALL = (_capi.VP3D_EVAL_MPJPE | _capi.VP3D_EVAL_P_MPJPE | _capi.VP3D_EVAL_N_MPJPE
        | _capi.VP3D_EVAL_VELOCITY)


def _check(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        got = f"{t.device}, {t.dtype}" if isinstance(t, torch.Tensor) else type(t).__name__
        raise RuntimeError(f"videopose3d_b200.metrics: {what} must be a CUDA float32 tensor "
                           f"(got {got}); there is no fallback path")


_src_cache = {}


def _mirror_src(joints, left, right, device):
    if left is None or right is None:
        return None
    key = (joints, tuple(left), tuple(right), device)
    if key not in _src_cache:
        _src_cache[key] = torch.from_numpy(mirror_source(joints, left, right)).to(device)
    return _src_cache[key]


def _launch(pred, copies, src, target, frames, joints, which, averaged):
    """One vp3d_pose_errors call; returns the (4,) float64 device tensor of means (or None)."""
    lib = _capi.load()
    dev = pred.device
    means = scratch = None
    if which:
        means = torch.empty(4, dtype=torch.float64, device=dev)
        scratch = torch.empty(max(1, lib.vp3d_pose_errors_scratch_bytes(frames)), dtype=torch.uint8,
                              device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _capi.check(lib.vp3d_pose_errors(
            pred.data_ptr(), copies, ptr(src), ptr(target), frames, joints, which, ptr(averaged),
            ptr(means), ptr(scratch), scratch.numel() if scratch is not None else 0, stream),
            "vp3d_pose_errors")
    if means is not None and frames == 0:
        means.fill_(float("nan"))   # torch.mean / np.mean of nothing
    return means


def _single(predicted, target, bit, ndim, name):
    _check(predicted, "predicted")
    _check(target, "target")
    assert predicted.shape == target.shape
    if predicted.dim() != ndim or predicted.shape[-1] != 3:
        raise ValueError(f"{name}: expected a {ndim}-D (..., joints, 3) tensor, got "
                         f"{tuple(predicted.shape)}")
    joints = predicted.shape[-2]
    frames = predicted.numel() // (3 * joints) if joints else 0
    m = _launch(predicted.contiguous(), 1, None, target.contiguous(), frames, joints, bit, None)
    return m[bit.bit_length() - 1]


def p_mpjpe(predicted, target):
    """Protocol #2: MPJPE after per-frame rigid alignment with scale (loss.py:27-66).
    (frames, joints, 3) tensors, as run.py:697-701 passes them."""
    return _single(predicted, target, _capi.VP3D_EVAL_P_MPJPE, 3, "p_mpjpe")


def n_mpjpe(predicted, target):
    """Protocol #3: MPJPE after per-frame least-squares scale (loss.py:68-78).
    (batch, frames, joints, 3) tensors."""
    return _single(predicted, target, _capi.VP3D_EVAL_N_MPJPE, 4, "n_mpjpe")


def mean_velocity_error(predicted, target):
    """MPJVE: mean distance of the first differences along axis 0 (loss.py:80-89).
    (frames, joints, 3) tensors, as run.py:697-704 passes them."""
    return _single(predicted, target, _capi.VP3D_EVAL_VELOCITY, 3, "mean_velocity_error")


def _pred_shape(pred):
    _check(pred, "predicted")
    if pred.dim() != 4 or pred.shape[0] not in (1, 2) or pred.shape[-1] != 3:
        raise ValueError(f"expected a (copies, frames, joints, 3) prediction with copies 1 or 2, got "
                         f"{tuple(pred.shape)}")
    return pred.shape[0], pred.shape[1], pred.shape[2]


def flip_average(pred, joints_left=None, joints_right=None):
    """run.py:675-680 on a (2, frames, joints, 3) prediction: negate x of row 1, swap its left and
    right joints (skipped when the lists are None: the trajectory model, run.py:678) and average
    with row 0.  Returns (1, frames, joints, 3), bit-identical to the torch expression."""
    copies, frames, joints = _pred_shape(pred)
    if copies != 2:
        raise ValueError("flip_average needs the plain and the mirrored copy (batch of 2)")
    pred = pred.contiguous()
    out = torch.empty((1, frames, joints, 3), dtype=torch.float32, device=pred.device)
    _launch(pred, 2, _mirror_src(joints, joints_left, joints_right, pred.device), None, frames, joints,
            0, out)
    return out


def pose_errors(pred, target, joints_left=None, joints_right=None, return_averaged=True):
    """[P1, P2, P3, MPJVE] in metres (float64 CUDA tensor of 4) of one sequence, and the averaged
    prediction (1, frames, joints, 3) (None unless `return_averaged`).

    pred: (1 or 2, frames, joints, 3); with 2 rows, row 1 is the mirrored copy and is flip-averaged
    first (run.py:675-680; `joints_left` / `joints_right` None = negate x only).  target:
    (frames, joints, 3) or (1, frames, joints, 3), used as given (run.py zeroes its root joint
    first, :688)."""
    copies, frames, joints = _pred_shape(pred)
    _check(target, "target")
    if tuple(target.shape[-3:]) != (frames, joints, 3) or target.numel() != frames * joints * 3:
        raise ValueError(f"target {tuple(target.shape)} does not match prediction {tuple(pred.shape)}")
    pred = pred.contiguous()
    out = None
    if return_averaged:
        out = pred if copies == 1 else torch.empty((1, frames, joints, 3), dtype=torch.float32,
                                                   device=pred.device)
    src = _mirror_src(joints, joints_left, joints_right, pred.device) if copies == 2 else None
    means = _launch(pred, copies, src, target.contiguous(), frames, joints, _ALL,
                    out if copies == 2 else None)
    return means, out


def evaluate(model, generator, joints_left=None, joints_right=None, return_predictions=False):
    """run.py's evaluate() (run.py:652-721) on a device `UnchunkedGenerator`: Protocols #1-#3 and
    MPJVE in mm, each sequence weighted by its frame count, summed on the device; one host sync at
    the end.  With test-time augmentation the mirrored copy is averaged in (joints swapped through
    `joints_left` / `joints_right`; None = trajectory model) and target row 0 is scored, with its
    root joint zeroed (run.py:686-690).  `return_predictions`: like run.py, returns the first
    sequence's averaged prediction, (frames, joints, 3), here as a CUDA tensor."""
    model.eval()
    tta = generator.augment_enabled()
    acc = None
    n = 0
    with torch.no_grad():
        for _, batch_3d, batch_2d in generator.next_epoch():
            pred = model(batch_2d)
            if return_predictions:
                if tta:
                    return flip_average(pred, joints_left, joints_right).squeeze(0)
                return pred.squeeze(0)
            target = batch_3d[:1] if tta else batch_3d
            target[:, :, 0] = 0
            w = target.shape[0] * target.shape[1]
            means, _ = pose_errors(pred, target, joints_left, joints_right, return_averaged=False)
            acc = means * w if acc is None else acc.add_(means, alpha=w)
            n += w
    if acc is None:
        raise ValueError("evaluate(): the generator yielded no sequence")
    e1, e2, e3, ev = (acc / n * 1000).tolist()
    return e1, e2, e3, ev
