"""float64 statements of the differentiable pose losses (TEST ORACLE for csrc/pose_loss.cu).

Two independent routes to the same numbers:
  * torch, differentiable through `torch.linalg.svd`: `mpjpe`, `n_mpjpe`, `p_mpjpe` and
    `mean_velocity_error` restate common/loss.py:11-17, :68-78, :27-66 and :80-89 on (..., J, 3)
    tensors -- a pose is one (..., frame) slice; the velocity differences run along dim -3, so a
    (frames, J, 3) input is the reference's `np.diff(axis=0)` and a (N, T, J, 3) batch is
    differenced along T within each sample.  Autograd gives their gradients.
  * NumPy, Horn's quaternion form with the reverse-mode eigenvector formula the kernel uses:
    `p_mpjpe_horn` returns P-MPJPE, its gradient with respect to the prediction and the number of
    poses whose rotation is not differentiable (top eigenvalue gap <= 1e-12 max(|lambda_0|, 1);
    those get the gradient with the rotation held fixed).
"""
import numpy as np
import torch

DEGENERATE_GAP = 1e-12


def _poses(x):
    return x.reshape(-1, x.shape[-2], x.shape[-1])


def mpjpe(predicted, target):
    return torch.linalg.norm(predicted - target, dim=-1).mean()


def n_mpjpe(predicted, target):
    """loss.py:75-78 on every pose of a (..., J, 3) tensor."""
    norm_predicted = torch.mean(torch.sum(predicted ** 2, dim=-1, keepdim=True), dim=-2, keepdim=True)
    norm_target = torch.mean(torch.sum(target * predicted, dim=-1, keepdim=True), dim=-2, keepdim=True)
    return mpjpe(norm_target / norm_predicted * predicted, target)


def p_mpjpe(predicted, target):
    """loss.py:34-66 per pose, with torch ops (the SVD's backward carries the gradient)."""
    p, t = _poses(predicted), _poses(target)
    mu_x = t.mean(dim=1, keepdim=True)
    mu_y = p.mean(dim=1, keepdim=True)
    x0, y0 = t - mu_x, p - mu_y
    norm_x = torch.sqrt(torch.sum(x0 ** 2, dim=(1, 2), keepdim=True))
    norm_y = torch.sqrt(torch.sum(y0 ** 2, dim=(1, 2), keepdim=True))
    x0, y0 = x0 / norm_x, y0 / norm_y
    h = x0.transpose(1, 2) @ y0
    u, s, vt = torch.linalg.svd(h)
    v = vt.transpose(1, 2)
    r = v @ u.transpose(1, 2)
    sign = torch.sign(torch.linalg.det(r)).detach()          # reflection fix, loss.py:51-55
    ones = torch.ones_like(sign)
    d = torch.stack([ones, ones, sign], dim=-1)
    v = v * d[:, None, :]
    s = s * d
    r = v @ u.transpose(1, 2)
    tr = s.sum(dim=1)[:, None, None]
    a = tr * norm_x / norm_y
    shift = mu_x - a * (mu_y @ r)
    aligned = a * (p @ r) + shift
    return torch.linalg.norm(aligned - t, dim=-1).mean()


def mean_velocity_error(predicted, target):
    """loss.py:86-89 with the first difference along dim -3 (NaN for a single frame)."""
    vp = torch.diff(predicted, dim=-3)
    vt = torch.diff(target, dim=-3)
    return torch.linalg.norm(vp - vt, dim=-1).mean()


TERMS = (mpjpe, n_mpjpe, p_mpjpe, mean_velocity_error)


def pose_loss(predicted, target, weights):
    """(sum_k w_k term_k over the terms with w_k != 0, [term_k or 0])."""
    total = predicted.new_zeros(())
    values = []
    for w, fn in zip(weights, TERMS):
        if w != 0:
            v = fn(predicted, target)
            total = total + w * v
            values.append(v.detach())
        else:
            values.append(predicted.new_zeros(()).detach())
    return total, torch.stack(values)


# ---------------------------------------------------------------- Horn's form and its reverse mode

def horn_matrix(h):
    """Horn's symmetric 4x4 N(H) for H = X0^T Y0 (batched): its top eigenpair is the optimal trace
    and the unit quaternion of the rotation."""
    s = np.swapaxes(h, -1, -2)   # S = H^T
    sxx, sxy, sxz = s[:, 0, 0], s[:, 0, 1], s[:, 0, 2]
    syx, syy, syz = s[:, 1, 0], s[:, 1, 1], s[:, 1, 2]
    szx, szy, szz = s[:, 2, 0], s[:, 2, 1], s[:, 2, 2]
    n = np.stack([
        np.stack([sxx + syy + szz, syz - szy, szx - sxz, sxy - syx], -1),
        np.stack([syz - szy, sxx - syy - szz, sxy + syx, szx + sxz], -1),
        np.stack([szx - sxz, sxy + syx, -sxx + syy - szz, syz + szy], -1),
        np.stack([sxy - syx, szx + sxz, syz + szy, -sxx - syy + szz], -1)], -2)
    return n


def horn_matrix_transpose(b):
    """Adjoint of H -> N(H): the H-gradient of <B, N(H)> for a symmetric B."""
    sb = np.empty(b.shape[:-2] + (3, 3))
    sb[:, 0, 0] = b[:, 0, 0] + b[:, 1, 1] - b[:, 2, 2] - b[:, 3, 3]
    sb[:, 1, 1] = b[:, 0, 0] - b[:, 1, 1] + b[:, 2, 2] - b[:, 3, 3]
    sb[:, 2, 2] = b[:, 0, 0] - b[:, 1, 1] - b[:, 2, 2] + b[:, 3, 3]
    sb[:, 1, 2] = 2 * (b[:, 0, 1] + b[:, 2, 3])
    sb[:, 2, 1] = 2 * (-b[:, 0, 1] + b[:, 2, 3])
    sb[:, 2, 0] = 2 * (b[:, 0, 2] + b[:, 1, 3])
    sb[:, 0, 2] = 2 * (-b[:, 0, 2] + b[:, 1, 3])
    sb[:, 0, 1] = 2 * (b[:, 0, 3] + b[:, 1, 2])
    sb[:, 1, 0] = 2 * (-b[:, 0, 3] + b[:, 1, 2])
    return np.swapaxes(sb, -1, -2)   # H-bar = S-bar^T


def quat_rotation(q):
    """Row-major rotation Q (applied as Q y) of unit quaternions q = (w, x, y, z); R = Q^T."""
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([
        np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        np.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
        np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1)], -2)


def quat_rotation_transpose(q, b):
    """q-gradient of <B, Q(q)> (Q's entries are quadratic forms in q)."""
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    B = lambda i, j: b[:, i, j]  # noqa: E731
    gw = w * (B(0, 0) + B(1, 1) + B(2, 2)) + z * (B(1, 0) - B(0, 1)) + y * (B(0, 2) - B(2, 0)) \
        + x * (B(2, 1) - B(1, 2))
    gx = x * (B(0, 0) - B(1, 1) - B(2, 2)) + y * (B(0, 1) + B(1, 0)) + z * (B(0, 2) + B(2, 0)) \
        + w * (B(2, 1) - B(1, 2))
    gy = y * (-B(0, 0) + B(1, 1) - B(2, 2)) + x * (B(0, 1) + B(1, 0)) + w * (B(0, 2) - B(2, 0)) \
        + z * (B(1, 2) + B(2, 1))
    gz = z * (-B(0, 0) - B(1, 1) + B(2, 2)) + w * (B(1, 0) - B(0, 1)) + x * (B(0, 2) + B(2, 0)) \
        + y * (B(1, 2) + B(2, 1))
    return 2 * np.stack([gw, gx, gy, gz], -1)


def p_mpjpe_horn(predicted, target):
    """(P-MPJPE, d P-MPJPE / d predicted, degenerate pose count) in float64 NumPy.

    Forward: centre, normalise, H = X0^T Y0, top eigenpair (lambda_0, q_0) of N(H): trace =
    lambda_0, rotation Q = Q(q_0); per joint the aligned error is |X0| (lambda_0 Q y0_j - x0_j).
    Reverse: the eigenvalue takes lambda-bar q0 q0^T, the eigenvector
    sum_{k>=1} (q_k^T q0-bar) / (lambda_0 - lambda_k) q_k q0^T (dropped for a degenerate pose),
    symmetrised, mapped back to H through the adjoint of N(.), then through the normalisation and
    the centring of the prediction."""
    shape = np.shape(predicted)
    p = _poses(np.asarray(predicted, dtype=np.float64))
    t = _poses(np.asarray(target, dtype=np.float64))
    P, J, _ = p.shape
    with np.errstate(invalid="ignore", divide="ignore"):
        x0 = t - t.mean(axis=1, keepdims=True)
        z = p - p.mean(axis=1, keepdims=True)
        nx = np.sqrt((x0 ** 2).sum(axis=(1, 2)))
        ny = np.sqrt((z ** 2).sum(axis=(1, 2)))
        x0 = x0 / nx[:, None, None]
        y0 = z / ny[:, None, None]
        h = np.einsum("pja,pjb->pab", x0, y0)
        n = horn_matrix(h)
        ok = np.isfinite(n).all(axis=(1, 2))
        lam = np.full((P, 4), np.nan)
        vec = np.full((P, 4, 4), np.nan)
        if ok.any():
            lam_ok, vec_ok = np.linalg.eigh(n[ok])
            lam[ok], vec[ok] = lam_ok[:, ::-1], vec_ok[:, :, ::-1]   # descending
        q = vec[:, :, 0]
        tr = lam[:, 0]
        Q = quat_rotation(q)
        qy = np.einsum("pab,pjb->pja", Q, y0)
        e = nx[:, None, None] * (tr[:, None, None] * qy - x0)
        d = np.linalg.norm(e, axis=-1)
        value = float(d.mean())
        M = P * J
        u = np.where(d[..., None] > 0, e / np.where(d > 0, d, 1)[..., None], 0.0) / M
        tr_bar = nx * np.einsum("pja,pja->p", u, qy)
        q_bar_mat = (nx * tr)[:, None, None] * np.einsum("pja,pjb->pab", u, y0)
        y0_bar = (nx * tr)[:, None, None] * np.einsum("pab,pja->pjb", Q, u)
        q_bar = quat_rotation_transpose(q, q_bar_mat)
        gap = lam[:, 0] - lam[:, 1]
        degenerate = gap <= DEGENERATE_GAP * np.maximum(np.abs(lam[:, 0]), 1.0)
        nbar = tr_bar[:, None, None] * np.einsum("pa,pb->pab", q, q)
        for k in range(1, 4):
            qk = vec[:, :, k]
            c = np.einsum("pa,pa->p", qk, q_bar) / (lam[:, 0] - lam[:, k])
            c = np.where(degenerate, 0.0, c)
            nbar = nbar + c[:, None, None] * np.einsum("pa,pb->pab", qk, q)
        nbar = 0.5 * (nbar + np.swapaxes(nbar, -1, -2))
        h_bar = horn_matrix_transpose(nbar)
        y0_bar = y0_bar + np.einsum("pab,pja->pjb", h_bar, x0)
        z_bar = (y0_bar - np.einsum("pja,pja->p", y0_bar, y0)[:, None, None] * y0) / ny[:, None, None]
        g = z_bar - z_bar.mean(axis=1, keepdims=True)
    return value, g.reshape(shape), int(degenerate[ok].sum())
