"""float64 statement of the training loss kernels (TEST ORACLE for csrc/step_ops.cu's mpjpe and
projected-mpjpe kernels and csrc/semi_loss.cu).

  * `mpjpe`, `weighted_mpjpe`: common/loss.py:11-25.
  * `project_to_2d`, `project_to_2d_linear`: common/camera.py:37-88 (camera of sample n broadcast
    over every frame and joint of that sample).
  * `bone_length_penalty`: run.py:383-387.
  * `semi_loss_head`: run.py:329-390 between the two model outputs and `loss_total` -- 3-D loss
    with the root zeroed, depth-weighted trajectory loss, re-projection loss and bone-length
    penalty, with `no_proj` / `bone_length_term` deciding what enters the total.

Everything is plain torch on whatever dtype it is given (float64 in the tests); autograd gives the
gradients for both model outputs.  `*_scale` helpers give the magnitudes the fp32 round-off of the
kernels is measured against (the same expressions with absolute values).
"""
import torch


def mpjpe(predicted, target):
    return torch.mean(torch.norm(predicted - target, dim=len(target.shape) - 1))


def weighted_mpjpe(predicted, target, w):
    return torch.mean(w * torch.norm(predicted - target, dim=len(target.shape) - 1))


def _cam(camera_params, X):
    while camera_params.dim() < X.dim():
        camera_params = camera_params.unsqueeze(1)
    return camera_params


def project_to_2d(X, camera_params):
    cp = _cam(camera_params, X)
    f, c, k, p = cp[..., :2], cp[..., 2:4], cp[..., 4:7], cp[..., 7:]
    XX = torch.clamp(X[..., :2] / X[..., 2:], min=-1, max=1)
    r2 = torch.sum(XX ** 2, dim=-1, keepdim=True)
    radial = 1 + torch.sum(k * torch.cat((r2, r2 ** 2, r2 ** 3), dim=-1), dim=-1, keepdim=True)
    tan = torch.sum(p * XX, dim=-1, keepdim=True)
    return f * (XX * (radial + tan) + p * r2) + c


def project_to_2d_linear(X, camera_params):
    cp = _cam(camera_params, X)
    return cp[..., :2] * torch.clamp(X[..., :2] / X[..., 2:], min=-1, max=1) + cp[..., 2:4]


def projected_mpjpe(pos, traj, cam, target_2d, linear=False):
    proj = project_to_2d_linear if linear else project_to_2d
    return mpjpe(proj(pos + traj, cam), target_2d)


def bone_length_penalty(pos, split_idx, parents):
    dists = pos[:, :, 1:] - pos[:, :, list(parents)[1:]]
    bone_lengths = torch.mean(torch.norm(dists, dim=3), dim=1)
    return torch.mean(torch.abs(torch.mean(bone_lengths[:split_idx], dim=0)
                                - torch.mean(bone_lengths[split_idx:], dim=0)))


def semi_loss_head(pos, traj, inputs_3d, cam, target_2d, parents, linear=False, no_proj=False,
                   bone_length_term=True):
    """run.py:334-388 with skip = False.  inputs_3d as the generator yields it (joint 0 = global
    root trajectory).  Returns (loss_total, [loss_3d_pos, loss_traj, loss_reconstruction,
    penalty]); the last two are None without unlabeled samples."""
    inputs_3d = inputs_3d.clone()
    inputs_traj = inputs_3d[:, :, :1].clone()
    inputs_3d[:, :, 0] = 0
    split_idx = inputs_3d.shape[0]
    loss_3d_pos = mpjpe(pos[:split_idx], inputs_3d)
    w = 1 / inputs_traj[:, :, :, 2]
    loss_traj = weighted_mpjpe(traj[:split_idx], inputs_traj, w)
    total = loss_3d_pos + loss_traj
    rec = pen = None
    if pos.shape[0] > split_idx:
        rec = projected_mpjpe(pos[split_idx:], traj[split_idx:], cam, target_2d, linear)
        if not no_proj:
            total = total + rec
        pen = bone_length_penalty(pos, split_idx, parents)
        if bone_length_term:
            total = total + pen
    return total, [loss_3d_pos, loss_traj, rec, pen]


# ---- magnitudes for the round-off bounds --------------------------------------------------------

def projection_scale(X, camera_params, target_2d, linear=False):
    """Per point (shape of target_2d[..., 0]): sum over both image axes of |f * proj| + |c| + |t|
    evaluated with absolute values (clamped ratio |x| / |z| taken as is): the size of what the
    fp32 residual f * proj + c - t cancels, which bounds its absolute round-off / 2^-24."""
    cp = _cam(camera_params, X).abs()
    f, c, k, p = cp[..., :2], cp[..., 2:4], cp[..., 4:7], cp[..., 7:]
    XX = torch.clamp(X[..., :2].abs() / X[..., 2:].abs(), max=1)
    if linear:
        o = XX
    else:
        r2 = torch.sum(XX ** 2, dim=-1, keepdim=True)
        radial = 1 + r2 * (k[..., :1] + r2 * (k[..., 1:2] + r2 * k[..., 2:]))
        o = XX * (radial + torch.sum(p * XX, dim=-1, keepdim=True)) + p * r2
    return (f * o + c + target_2d.abs()).sum(-1)
