"""Fused losses (SURVEY §8 row f2).

`mpjpe` and `weighted_mpjpe` with the reference's signatures and values (common/loss.py:11-17,
:19-25; used at run.py:359, 413, 452, 501): the loss and its gradient with respect to the
prediction come out of ONE launch (`vp3d_mpjpe_fwd_bwd_ex`, csrc/step_ops.cu) instead of the
subtract / norm / mean kernels and their four backward kernels.  `projected_mpjpe` is the
re-projection loss of the semi-supervised branch (run.py:374-379): camera projection of
`predicted_pos + predicted_traj` (common/camera.py:37-88) and the 2-D mpjpe, with the gradients for
both model outputs, in one launch (`vp3d_projected_mpjpe_fwd_bwd_ex`).  `semi_supervised_loss` is the
whole loss head of the semi-supervised step -- 3-D loss, depth-weighted trajectory loss,
re-projection loss and the bone-length penalty (run.py:350-390) with the gradients for both model
outputs -- in one cooperative launch (`vp3d_semi_loss_fwd_bwd`, csrc/semi_loss.cu);
`bone_length_penalty` is that kernel with only the penalty enabled.  `pose_loss` is any weighted
combination of mpjpe, `n_mpjpe`, `p_mpjpe` and `mean_velocity_error` (loss.py:27-89, NumPy or
gradient-free in the reference) with the gradient of the sum, in one cooperative launch
(`vp3d_pose_loss_fwd_bwd`, csrc/pose_loss.cu); the three named functions are that kernel with one
term enabled.  CUDA float32 only, no fallback.
"""
import torch

from . import _capi

__all__ = ["mpjpe", "weighted_mpjpe", "projected_mpjpe", "bone_length_penalty",
           "semi_supervised_loss", "n_mpjpe", "p_mpjpe", "mean_velocity_error", "pose_loss"]


def _scratch(nbytes, dev):
    """Device scratch of the block-ordered loss sums (None when one block does the whole sum)."""
    return torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _numel(t):
    return t.numel() if t is not None else 0


class _Mpjpe(torch.autograd.Function):
    @staticmethod
    def forward(ctx, predicted, target, weights):
        for t, what in ((predicted, "predicted"), (target, "target")):
            if not (t.is_cuda and t.dtype == torch.float32):
                raise RuntimeError(f"videopose3d_b200.loss: {what} must be a CUDA float32 tensor "
                                   f"(got {t.device}, {t.dtype}); there is no fallback path")
        lib = _capi.load()
        pred = predicted.contiguous()
        tgt = target.contiguous()
        dims = pred.shape[-1]
        joints = pred.numel() // dims if dims else 0
        w = None
        if weights is not None:
            w = weights.to(device=pred.device, dtype=torch.float32).expand(pred.shape[:-1]).contiguous()
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        need_grad = ctx.needs_input_grad[0]
        dpred = torch.empty_like(pred) if need_grad else None
        scratch = _scratch(lib.vp3d_mpjpe_scratch_bytes(joints), pred.device)
        with torch.cuda.device(pred.device):
            stream = torch.cuda.current_stream(pred.device).cuda_stream
            _capi.check(lib.vp3d_mpjpe_fwd_bwd_ex(pred.data_ptr(), tgt.data_ptr(),
                                                  w.data_ptr() if w is not None else None, joints,
                                                  dims, loss.data_ptr(),
                                                  dpred.data_ptr() if need_grad else None,
                                                  _ptr(scratch), _numel(scratch), stream),
                        "vp3d_mpjpe_fwd_bwd_ex")
        # kept for the lifetime of the graph: a second backward (retain_graph=True, or the loss
        # feeding two backward passes) gets the same gradient again, as with the torch expression
        ctx.dpred = dpred
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        dpred = ctx.dpred
        return (dpred * grad_out if dpred is not None else None), None, None


def mpjpe(predicted, target):
    """Mean Euclidean distance between predicted and target joints (loss.py:11-17)."""
    assert predicted.shape == target.shape
    return _Mpjpe.apply(predicted, target, None)


def weighted_mpjpe(predicted, target, w):
    """Weighted mean Euclidean distance, `w` broadcast over the joint axis (loss.py:19-25)."""
    assert predicted.shape == target.shape
    assert w.shape[0] == predicted.shape[0]
    return _Mpjpe.apply(predicted, target, w)


class _ProjectedMpjpe(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, traj, cam, target, linear):
        for t, what in ((pos, "predicted_pos"), (traj, "predicted_traj"), (cam, "camera_params"),
                        (target, "target_2d")):
            if not (t.is_cuda and t.dtype == torch.float32):
                raise RuntimeError(f"videopose3d_b200.loss: {what} must be a CUDA float32 tensor "
                                   f"(got {t.device}, {t.dtype}); there is no fallback path")
        n, frames, joints = pos.shape[0], pos.shape[1], pos.shape[2]
        assert pos.dim() == 4 and pos.shape[-1] == 3
        assert traj.shape == (n, frames, 1, 3), traj.shape
        assert cam.shape == (n, 9), cam.shape                      # camera.py:47-49
        assert target.shape == (n, frames, joints, 2), target.shape
        lib = _capi.load()
        pos_c, traj_c, cam_c, tgt_c = (t.contiguous() for t in (pos, traj, cam, target))
        loss = torch.empty((), dtype=torch.float32, device=pos.device)
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        dpos = torch.empty_like(pos_c) if need_grad else None
        dtraj = torch.empty_like(traj_c) if need_grad else None
        scratch = _scratch(lib.vp3d_projected_mpjpe_scratch_bytes(n, frames), pos.device)
        with torch.cuda.device(pos.device):
            stream = torch.cuda.current_stream(pos.device).cuda_stream
            _capi.check(lib.vp3d_projected_mpjpe_fwd_bwd_ex(
                pos_c.data_ptr(), traj_c.data_ptr(), cam_c.data_ptr(), tgt_c.data_ptr(), n, frames,
                joints, int(bool(linear)), loss.data_ptr(),
                dpos.data_ptr() if need_grad else None, dtraj.data_ptr() if need_grad else None,
                _ptr(scratch), _numel(scratch), stream), "vp3d_projected_mpjpe_fwd_bwd_ex")
        ctx.grads = (dpos, dtraj)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        dpos, dtraj = ctx.grads
        if dpos is None:
            return None, None, None, None, None
        return dpos * grad_out, dtraj * grad_out, None, None, None


def projected_mpjpe(predicted_pos, predicted_traj, camera_params, target_2d, linear=False):
    """`mpjpe(project_to_2d(predicted_pos + predicted_traj, camera_params), target_2d)` -- the
    reconstruction loss of run.py:374-379 (`project_to_2d_linear` when `linear`)."""
    return _ProjectedMpjpe.apply(predicted_pos, predicted_traj, camera_params, target_2d, linear)


def _checked_parents(parents, joints):
    """The skeleton's parent list as ints; every entry after the root must index the pose, because
    the kernel reads pos[parent] unchecked.  The root's parent (-1 in the reference's list) is
    never read: bones start at joint 1."""
    plist = [int(p) for p in parents]
    bad = [(j, p) for j, p in enumerate(plist) if j >= 1 and not 0 <= p < joints]
    if len(plist) != joints or bad:
        raise ValueError(f"videopose3d_b200.loss: parents must give each of the {joints} joints after "
                         f"the root a parent in [0, {joints}) (got {len(plist)} entries; out of range "
                         f"(joint, parent): {bad[:4]})")
    return plist


class _SemiLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, traj, target_3d, cam, target_2d, parents, n_labeled, linear, terms, which):
        if terms & _capi.VP3D_SEMI_BONE:
            parents = _checked_parents(parents, pos.shape[2])
        for t, what in ((pos, "predicted_3d_pos"), (traj, "predicted_traj")):
            if not (t.is_cuda and t.dtype == torch.float32):
                raise RuntimeError(f"videopose3d_b200.loss: {what} must be a CUDA float32 tensor "
                                   f"(got {t.device}, {t.dtype}); there is no fallback path")
        n, frames, joints = pos.shape[0], pos.shape[1], pos.shape[2]
        n_unl = n - n_labeled
        assert pos.dim() == 4 and pos.shape[-1] == 3 and 0 <= n_labeled <= n
        assert traj.shape == (n, frames, 1, 3), traj.shape
        dev = pos.device

        def prep(t, shape, what):
            if t is None:
                return None
            t = t.to(device=dev, dtype=torch.float32).contiguous()
            assert tuple(t.shape) == shape, (what, tuple(t.shape), shape)
            return t
        tgt3 = prep(target_3d, (n_labeled, frames, joints, 3), "inputs_3d")
        cam_c = prep(cam, (n_unl, 9), "cam")
        tgt2 = prep(target_2d, (n_unl, frames, joints, 2), "target_2d")
        par = None
        if terms & _capi.VP3D_SEMI_BONE:
            par = torch.as_tensor(parents, dtype=torch.int32).clamp_min(0).to(dev)
        lib = _capi.load()
        pos_c, traj_c = pos.contiguous(), traj.contiguous()
        losses = torch.empty(5, dtype=torch.float32, device=dev)
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        dpos = torch.empty_like(pos_c) if need_grad else None
        dtraj = torch.empty_like(traj_c) if need_grad else None
        scratch = torch.empty(lib.vp3d_semi_loss_scratch_bytes(), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _capi.check(lib.vp3d_semi_loss_fwd_bwd(
                pos_c.data_ptr(), traj_c.data_ptr(), _ptr(tgt3), _ptr(cam_c), _ptr(tgt2), _ptr(par),
                n_labeled, n_unl, frames, joints, int(bool(linear)), int(terms), losses.data_ptr(),
                _ptr(dpos), _ptr(dtraj), scratch.data_ptr(), scratch.numel(), stream),
                "vp3d_semi_loss_fwd_bwd")
        ctx.grads = (dpos, dtraj)
        ctx.mark_non_differentiable(losses)
        return losses[which].clone(), losses

    @staticmethod
    def backward(ctx, grad_out, _grad_terms):
        dpos, dtraj = ctx.grads
        if dpos is None:
            return (None,) * 10
        return (dpos * grad_out, dtraj * grad_out) + (None,) * 8


def semi_supervised_loss(predicted_3d_pos_cat, predicted_traj_cat, inputs_3d, cam_semi, target_2d_semi,
                         parents, linear_projection=False, no_proj=False, bone_length_term=True):
    """The loss head of run.py's semi-supervised step in one launch.

    predicted_3d_pos_cat / predicted_traj_cat: the two models' outputs on `cat(labeled, unlabeled)`
    (run.py:350, 358); inputs_3d: the labeled batch's 3-D poses AS THE GENERATOR YIELDS THEM (root
    joint = global trajectory: the kernel zeroes it for the pose loss and uses it as the trajectory
    target, run.py:335-336), its length is the split index; cam_semi / target_2d_semi: intrinsics
    and 2-D targets of the unlabeled part (run.py:329, 368-371); parents:
    `dataset.skeleton().parents()`.  Returns (loss_total, terms) with terms = [loss_3d_pos,
    loss_traj, loss_reconstruction, penalty, loss_total] (detached, for the logging lines
    run.py:353, 360, 377).  loss_total = what run.py accumulates in `loss_total` (:354, 361, 380, 388)."""
    n_labeled = int(inputs_3d.shape[0])
    mask = _capi.VP3D_SEMI_POS | _capi.VP3D_SEMI_TRAJ
    if predicted_3d_pos_cat.shape[0] > n_labeled:
        mask |= 0 if no_proj else _capi.VP3D_SEMI_PROJ
        mask |= _capi.VP3D_SEMI_BONE if bone_length_term else 0
    total, terms = _SemiLoss.apply(predicted_3d_pos_cat, predicted_traj_cat, inputs_3d, cam_semi,
                                   target_2d_semi, parents, n_labeled, linear_projection, mask, 4)
    return total, terms


def bone_length_penalty(predicted_3d_pos_cat, split_idx, parents):
    """Bone-length consistency term of run.py:383-387 through the fused kernel with only the penalty
    selected: mean over bones of |mean labeled bone length - mean unlabeled bone length|."""
    n, frames = predicted_3d_pos_cat.shape[0], predicted_3d_pos_cat.shape[1]
    traj = torch.zeros(n, frames, 1, 3, dtype=torch.float32, device=predicted_3d_pos_cat.device)
    pen, _ = _SemiLoss.apply(predicted_3d_pos_cat, traj, None, None, None, parents, int(split_idx),
                             False, _capi.VP3D_SEMI_BONE, 3)
    return pen


class _PoseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, predicted, target, weights):
        for t, what in ((predicted, "predicted"), (target, "target")):
            if not (t.is_cuda and t.dtype == torch.float32):
                raise RuntimeError(f"videopose3d_b200.loss: {what} must be a CUDA float32 tensor "
                                   f"(got {t.device}, {t.dtype}); there is no fallback path")
        assert predicted.shape == target.shape, (tuple(predicted.shape), tuple(target.shape))
        if predicted.dim() < 2 or predicted.shape[-1] != 3:
            raise ValueError(f"videopose3d_b200.loss: expected (..., frames, joints, 3) poses, got "
                             f"{tuple(predicted.shape)}")
        lib = _capi.load()
        dev = predicted.device
        pred, tgt = predicted.contiguous(), target.contiguous()
        joints = pred.shape[-2]
        frames = pred.shape[-3] if pred.dim() >= 3 else 1
        seqs = pred.numel() // (3 * joints * frames) if joints * frames else 0
        out = torch.empty(6, dtype=torch.float32, device=dev)      # loss, 4 terms, degenerate count
        need_grad = ctx.needs_input_grad[0]
        dpred = torch.empty_like(pred) if need_grad else None
        w = (_capi.ctypes.c_double * 4)(*weights)
        scratch = torch.empty(max(1, lib.vp3d_pose_loss_scratch_bytes(max(frames, 1), seqs)),
                              dtype=torch.uint8, device=dev)
        if seqs == 0 or joints == 0:
            out.fill_(float("nan"))            # torch.mean / np.mean of nothing
            out[5] = 0
            if need_grad:
                dpred.zero_()
        else:
            degenerate = out[5:].view(torch.int32)
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream(dev).cuda_stream
                _capi.check(lib.vp3d_pose_loss_fwd_bwd(
                    pred.data_ptr(), tgt.data_ptr(), frames, seqs, joints, w, out[1:5].data_ptr(),
                    out.data_ptr(), dpred.data_ptr() if need_grad else None, degenerate.data_ptr(),
                    scratch.data_ptr(), scratch.numel(), stream), "vp3d_pose_loss_fwd_bwd")
        # kept for the lifetime of the graph, as in _Mpjpe (retain_graph=True gets it again)
        ctx.dpred = dpred
        terms = out[1:5].clone()
        n_degenerate = out[5:].view(torch.int32).clone().squeeze(0)
        ctx.mark_non_differentiable(terms, n_degenerate)
        return out[0].clone(), terms, n_degenerate

    @staticmethod
    def backward(ctx, grad_out, _grad_terms, _grad_degenerate):
        dpred = ctx.dpred
        return (dpred * grad_out if dpred is not None else None), None, None


def _one_term(predicted, target, k):
    weights = [0.0] * 4
    weights[k] = 1.0
    loss, _, _ = _PoseLoss.apply(predicted, target, tuple(weights))
    return loss


def n_mpjpe(predicted, target):
    """Normalized MPJPE (loss.py:68-78): per pose (one (..., frame) slice of joints) the prediction
    is scaled by the least-squares factor mean <t, p> / mean <p, p>, then mpjpe.  The gradient
    includes the scale's own derivative."""
    assert predicted.shape == target.shape
    return _one_term(predicted, target, 1)


def p_mpjpe(predicted, target):
    """Procrustes-aligned MPJPE (loss.py:27-66) with a gradient: per pose, the similarity transform
    (rotation, scale, translation) fitted to the target, then mpjpe.  The gradient flows through the
    alignment itself.  (frames, joints, 3) as the reference takes it, or any (..., joints, 3)."""
    assert predicted.shape == target.shape
    return _one_term(predicted, target, 2)


def mean_velocity_error(predicted, target):
    """Mean per-joint velocity error (loss.py:80-89) with a gradient: mpjpe of the first differences
    along dim -3 -- the reference's axis 0 for (frames, joints, 3); along T within each sample for a
    (N, T, joints, 3) batch.  NaN for a single frame, like np.mean of nothing."""
    assert predicted.shape == target.shape
    return _one_term(predicted, target, 3)


def pose_loss(predicted, target, mpjpe=1.0, n_mpjpe=0.0, p_mpjpe=0.0, velocity=0.0,
              return_degenerate=False):
    """Weighted sum of mpjpe, n_mpjpe, p_mpjpe and mean_velocity_error (dim -3) and its gradient in
    ONE launch.  Terms with weight 0 are not evaluated.  Returns (loss, terms) with terms a detached
    (4,) tensor [mpjpe, n_mpjpe, p_mpjpe, velocity] (0 for a term not evaluated); with
    `return_degenerate`, also the 0-d int32 count of poses whose Procrustes rotation is not
    differentiable (the two largest eigenvalues of Horn's matrix closer than 1e-12 relative: their
    gradient holds the rotation fixed)."""
    weights = tuple(float(w) for w in (mpjpe, n_mpjpe, p_mpjpe, velocity))
    if not any(weights):
        raise ValueError("pose_loss: every term weight is 0")
    loss, terms, n_degenerate = _PoseLoss.apply(predicted, target, weights)
    return (loss, terms, n_degenerate) if return_degenerate else (loss, terms)
