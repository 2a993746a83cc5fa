"""float64 references and per-element error bounds of the pose-loss / metrics kernel
(csrc/pose_loss.cu with procrustes.cuh), shared by test_pose_bounds_cpu.py and
test_gpu_pose_kernels.py.

The kernel reads fp32 poses, works in fp64 and rounds once to fp32 for every term, the loss and
every gradient element (the metrics instance keeps fp64 means).  The references here are float64
statements of the same mathematics on the same fp32 inputs widened to float64: autograd through
oracle/pose_loss_oracle.py for the gradients (the SVD route for P-MPJPE), the SVD route of
oracle/metrics_oracle.py for the metric means.  u = 2^-24 (one fp32 rounding to nearest), E = 2^-53
(one fp64 rounding).

Gradient, per element:   |g - g64| <= u |g64| + E sum_k |w_k| K_k G_k  (+ 4 E sum_k |w_k g64_k|).
  * u |g64| is the one rounding of the kernel's fp64 value x to fp32: |fl(x) - g64| <= u |x| +
    |x - g64|, and u |x| <= u |g64| + u |x - g64| is inside the fp64 term's slack.
  * E K_k G_k bounds the fp64 error of term k along both routes (the kernel and the reference each
    contribute at most half of K_k).  G_k is the term's per-element magnitude scale: the sum of the
    absolute values of what the computation adds, per unit E.  gw = w / count (the kernel's
    gradient scale).  kappa = 1 + max_j Ee_j / max(|e_j|, K E Ee_j) is the conditioning of the unit
    vector u_j = e_j / |e_j| when e_j is computed with an absolute error of order E Ee_j: its
    direction moves by |de| / |e|.  Ee_j = 0 for mpjpe and velocity (e is the exact difference of
    fp32 values, or one rounding of it, so u is accurate to a few E whatever |e|).
    - mpjpe: G = gw.  K = 16: |e|^2 (3 products, 2 additions), sqrt, reciprocal, 3 products, the
      weight and the addition into g: 9 roundings in the kernel, 7 in torch's norm backward.
    - velocity: G = gw.  K = 48: two unit vectors per element (the differences ending and starting
      at the frame), each 10 roundings after the one of (p - p') - (t - t'), both routes.
    - N-MPJPE: s = <t, p> / <p, p> from two warp sums of 3 J products (8 levels: the product, two
      lane additions, the 5-level butterfly), so |ds| <= 17 E A with A = sum_i |t_i||p_i| / pp;
      e_j = s p_j - t_j has |de_j| <= 19 E Ee_j, Ee_j = A |p_j| + |t_j|; c = sum u.p / pp has
      |c| <= Cp = sum_i |p_i| / pp; g = gw (s u_j + c (t_j - 2 s p_j)).  Per pose
      G = gw (1 + A) (1 + Cp max_j (|t_j| + 2 A |p_j|)) kappa, and K = 64 (the 19 above, the
      13 roundings of u, c and g, both routes).
    - P-MPJPE: the gradient is z-bar / ny with z-bar built from nx tr Q^T u_j (size nx tr <= nx) and
      H-bar^T x0_j, whose entries are sums over the J joints of |u_j||y0_j| (<= sqrt J, as
      sum |y0_j|^2 = 1) times nx.  So G0 = gw (1 + sqrt(J) nx / ny) kappa, with
      Ee_j = nx (|y0_j| + |x0_j|) (e_j = nx (tr Q y0_j - x0_j)).  The rounding errors of N(H) and of
      its eigenpairs are E times ||N|| <= 2 times the operation count; an eigenvector moves by that
      over the gap lambda_0 - lambda_1, and the reverse mode divides by the gaps again, so the
      conditioning factor is 1 + 1 / gap_rel, gap_rel = (lambda_0 - lambda_1) / max(|lambda_0|, 1)
      (the kernel's degeneracy test).  The SVD reference has its own factor max_{i<j}
      1 / |s_i - s_j| (torch's SVD backward divides by s_i^2 - s_j^2); it is used where that
      factor is at most SVD_COND_MAX, Horn's form (the kernel's algorithm restated in NumPy)
      elsewhere, and always for the poses the rule calls degenerate (the rotation held fixed, as
      the kernel does).  K = 4096: centring, normalising and H take 16 roundings, N(H) 2, the 12
      sweeps of 6 Jacobi rotations 12 each (72 x 12 = 864), the reverse mode about as many again;
      2 x 1024 per route rounded up, two routes.
      G = K G0 (1 + 1 / gap_rel + cond_ref), cond_ref the reference's own factor.
      For a degenerate pose the rotation is an arbitrary vector of a (nearly) repeated eigenspace;
      holding it fixed keeps 1 / gap out of the reverse mode, and an orientation error of the
      rotation cannot exceed 2, so G = G0 min(K (1 + 1 / gap_rel), 2 / E).
Terms and loss:   |v - v64| <= u |v64| + E (depth sum d + K_d sum d + sum_j K Ee_j c_j) / count.
  * depth: additions along the longest path of the kernel's sum -- one per grid-stride pass in each
    lane, the 5-level warp butterfly, the 8 warps in order, the blocks in order, the division by
    count (`sum_depth`).  Recursive summation of non-negative terms errs by at most depth E sum d.
  * K_d = 8: the roundings of one distance |e| (3 products, 2 additions, sqrt), both routes.
  * sum_j K Ee_j c_j: e_j's own error (the cancellation it carries), with c_j the conditioning:
    1 for N-MPJPE, min(1 + 1 / gap_rel, 2 / (K E)) for P-MPJPE (a rotation error of at most 2).
    The depth term alone is not a bound: where the distances are round-off themselves (an
    identical prediction and target gives P-MPJPE distances of order E nx, computed differently by
    every route) only the per-distance terms cover the difference.
  * the loss is sum_k w_k v_k in fp64 rounded once: u |loss64| + sum_k |w_k| (fp64 part of term k)
    + 4 E sum_k |w_k v_k|.
Metric means (fp64 out): the same fp64 part, with no u term.

`demonstrations` builds five plausible wrong gradients (N-MPJPE with its scale detached, P-MPJPE
with the rotation detached, velocity without the difference that starts at the frame, the fp64
value rounded toward zero, one pose's gradient swapped with its neighbour's); each must fail the
gate.
"""
import math

import numpy as np
import torch

from oracle import metrics_oracle as mo
from oracle import pose_loss_oracle as po

U = 2.0 ** -24
E = 2.0 ** -53
K_GRAD = (16.0, 64.0, 4096.0, 48.0)     # mpjpe, n_mpjpe, p_mpjpe, velocity
K_DIST = 8.0
SVD_COND_MAX = 1e6
POSE_WARPS, MAX_BLOCKS = 8, 1024
NAMES = ("mpjpe", "n_mpjpe", "p_mpjpe", "velocity")


def sum_depth(poses, sms, per_sm_max=2):
    """Upper bound of the additions along the longest path of the kernel's block-ordered sum, for a
    grid of one or `per_sm_max` blocks per SM on `sms` SMs."""
    blocks = max(1, math.ceil(poses / POSE_WARPS))
    lo = min(blocks, MAX_BLOCKS, sms)
    hi = min(blocks, MAX_BLOCKS, per_sm_max * sms)
    passes = math.ceil(poses / (POSE_WARPS * lo))
    return passes + 5 + POSE_WARPS + hi + 1


def min_passes(poses, sms, per_sm_max=2):
    """Grid-stride passes the busiest warp makes at least, whatever the occupancy."""
    hi = min(max(1, math.ceil(poses / POSE_WARPS)), MAX_BLOCKS, per_sm_max * sms)
    return math.ceil(poses / (POSE_WARPS * hi))


def _kappa(ee, e_norm, k):
    floor = np.maximum(e_norm, k * E * ee)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(ee > 0, ee / np.where(floor > 0, floor, 1.0), 0.0)
    return 1.0 + r.max(axis=-1)


def horn_stats(p, t):
    """Per pose (P, J, 3) float64: Horn's eigenvalues (descending), gap_rel, the degeneracy rule,
    the SVD's conditioning, nx, ny, x0, y0 and the aligned errors e."""
    P, J, _ = p.shape
    with np.errstate(invalid="ignore", divide="ignore"):
        x0 = t - t.mean(axis=1, keepdims=True)
        y0 = p - p.mean(axis=1, keepdims=True)
        nx = np.sqrt((x0 ** 2).sum(axis=(1, 2)))
        ny = np.sqrt((y0 ** 2).sum(axis=(1, 2)))
        x0 = x0 / nx[:, None, None]
        y0 = y0 / ny[:, None, None]
        h = np.einsum("pja,pjb->pab", x0, y0)
    finite = np.isfinite(h).all(axis=(1, 2))
    lam = np.full((P, 4), np.nan)
    vec = np.full((P, 4, 4), np.nan)
    sv = np.full((P, 3), np.nan)
    if finite.any():
        w, v = np.linalg.eigh(po.horn_matrix(h[finite]))
        lam[finite], vec[finite] = w[:, ::-1], v[:, :, ::-1]
        sv[finite] = np.linalg.svd(h[finite], compute_uv=False)
    with np.errstate(invalid="ignore", divide="ignore"):
        gap_rel = (lam[:, 0] - lam[:, 1]) / np.maximum(np.abs(lam[:, 0]), 1.0)
        degenerate = finite & (lam[:, 0] - lam[:, 1] <= po.DEGENERATE_GAP * np.maximum(np.abs(lam[:, 0]), 1.0))
        d01, d02, d12 = sv[:, 0] - sv[:, 1], sv[:, 0] - sv[:, 2], sv[:, 1] - sv[:, 2]
        svd_cond = 1.0 / np.minimum(np.minimum(np.abs(d01), np.abs(d02)), np.abs(d12))
        Q = po.quat_rotation(vec[:, :, 0])
        e = nx[:, None, None] * (lam[:, :1, None] * np.einsum("pab,pjb->pja", Q, y0) - x0)
    return dict(lam=lam, gap_rel=gap_rel, degenerate=degenerate, finite=finite, svd_cond=svd_cond,
                nx=nx, ny=ny, x0=x0, y0=y0, e=e, sv=sv)


def _autograd(fn, p, t, scale=1.0):
    x = torch.from_numpy(p).requires_grad_(True)
    v = fn(x, torch.from_numpy(t)) * scale
    v.backward()
    return float(v.detach()), x.grad.numpy()


def _velocity_missing_start(predicted, target):
    """Wrong: only the difference ending at each frame reaches its gradient."""
    vp = predicted[..., 1:, :, :] - predicted[..., :-1, :, :].detach()
    return torch.linalg.norm(vp - torch.diff(target, dim=-3), dim=-1).mean()


def _n_mpjpe_scale_detached(predicted, target):
    """Wrong: the envelope-theorem mistake -- the least-squares scale treated as a constant."""
    pp = torch.mean(torch.sum(predicted ** 2, dim=-1, keepdim=True), dim=-2, keepdim=True)
    tp = torch.mean(torch.sum(target * predicted, dim=-1, keepdim=True), dim=-2, keepdim=True)
    return po.mpjpe((tp / pp).detach() * predicted, target)


def _p_mpjpe_rotation_detached(predicted, target):
    """Wrong: po.p_mpjpe with R (and the sign) held fixed on every pose."""
    p, t = po._poses(predicted), po._poses(target)
    mu_x, mu_y = t.mean(dim=1, keepdim=True), p.mean(dim=1, keepdim=True)
    x0, y0 = t - mu_x, p - mu_y
    norm_x = torch.sqrt(torch.sum(x0 ** 2, dim=(1, 2), keepdim=True))
    norm_y = torch.sqrt(torch.sum(y0 ** 2, dim=(1, 2), keepdim=True))
    u, s, vt = torch.linalg.svd((x0 / norm_x).transpose(1, 2) @ (y0 / norm_y))
    v = vt.transpose(1, 2)
    sign = torch.sign(torch.linalg.det(v @ u.transpose(1, 2))).detach()
    ones = torch.ones_like(sign)
    d = torch.stack([ones, ones, sign], dim=-1)
    r = ((v * d[:, None, :]) @ u.transpose(1, 2)).detach()
    a = (s * d).sum(dim=1)[:, None, None] * norm_x / norm_y
    aligned = a * (p @ r) + (mu_x - a * (mu_y @ r))
    return torch.linalg.norm(aligned - t, dim=-1).mean()


class Reference:
    """float64 values, gradients and bound ingredients of the four terms on fp32 poses
    (seqs, F, J, 3) (the loss) -- every per-term gradient is the gradient of the term's mean over
    the whole batch, so a weighted sum of them is the combined loss's."""

    def __init__(self, pred, target):
        assert pred.dtype == np.float32 and target.dtype == np.float32 and pred.ndim == 4
        self.shape = pred.shape
        S, F, J, _ = pred.shape
        self.J, self.F, self.seqs = J, F, S
        P = S * F
        self.poses = P
        p = pred.astype(np.float64)
        t = target.astype(np.float64)
        self.p, self.t = p, t
        p3, t3 = p.reshape(P, J, 3), t.reshape(P, J, 3)
        self.count = np.array([P * J, P * J, P * J, (F - 1) * S * J], dtype=np.float64)
        gw = np.where(self.count > 0, 1.0 / np.maximum(self.count, 1), 0.0)
        value = np.zeros(4)
        grad = np.zeros((4,) + pred.shape)
        G = np.zeros((4, P, J))               # per element scale, xyz share it
        dsum = np.zeros(4)                    # sum of the distances
        esum = np.zeros(4)                    # sum_j K Ee_j c_j
        # mpjpe
        value[0], grad[0] = _autograd(po.mpjpe, p, t)
        dsum[0] = np.linalg.norm(p3 - t3, axis=-1).sum()
        G[0] = gw[0]
        # N-MPJPE
        value[1], grad[1] = _autograd(po.n_mpjpe, p, t)
        with np.errstate(invalid="ignore", divide="ignore"):
            pn, tn = np.linalg.norm(p3, axis=-1), np.linalg.norm(t3, axis=-1)
            pp = (p3 * p3).sum(axis=(1, 2))
            s = (t3 * p3).sum(axis=(1, 2)) / pp
            A = (tn * pn).sum(axis=1) / pp
            Cp = pn.sum(axis=1) / pp
            e = s[:, None, None] * p3 - t3
            en = np.linalg.norm(e, axis=-1)
            ee = A[:, None] * pn + tn
            kap = _kappa(ee, en, K_GRAD[1])
            G[1] = (gw[1] * (1 + A) * (1 + Cp * (tn + 2 * A[:, None] * pn).max(axis=1)) * kap)[:, None]
        dsum[1] = en.sum()
        esum[1] = K_GRAD[1] * ee.sum()
        # P-MPJPE
        hs = horn_stats(p3, t3)
        self.horn = hs
        self.degenerate = int(hs["degenerate"].sum())
        fin = hs["finite"]
        use_svd = fin & ~hs["degenerate"] & (hs["svd_cond"] <= SVD_COND_MAX)
        use_horn = fin & ~use_svd
        self.svd_poses, self.horn_poses = int(use_svd.sum()), int(use_horn.sum())
        g2 = np.full((P, J, 3), np.nan)
        if use_svd.any():
            _, g2[use_svd] = _autograd(po.p_mpjpe, p3[use_svd], t3[use_svd], use_svd.sum() / P)
        if use_horn.any():
            _, gh, _ = po.p_mpjpe_horn(p3[use_horn], t3[use_horn])
            g2[use_horn] = gh * (use_horn.sum() / P)
        grad[2] = g2.reshape(pred.shape)
        value[2] = float(po.p_mpjpe(torch.from_numpy(p3), torch.from_numpy(t3))) if fin.all() else math.nan
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            en = np.linalg.norm(hs["e"], axis=-1)
            ee = hs["nx"][:, None] * (np.linalg.norm(hs["y0"], axis=-1) + np.linalg.norm(hs["x0"], axis=-1))
            kap = _kappa(ee, en, K_GRAD[2])
            g0 = gw[2] * (1 + math.sqrt(J) * hs["nx"] / hs["ny"]) * kap
            inv_gap = 1.0 / hs["gap_rel"]
            cond_ref = np.where(use_svd, hs["svd_cond"], inv_gap)
            full = K_GRAD[2] * g0 * (1 + inv_gap + cond_ref)
            fixed = g0 * np.minimum(K_GRAD[2] * (1 + inv_gap), 2 / E)
            G[2] = np.where(hs["degenerate"], fixed, full)[:, None] / K_GRAD[2]
            c = np.minimum(1 + inv_gap, 2 / (K_GRAD[2] * E))
            dsum[2] = en.sum()
            esum[2] = K_GRAD[2] * (ee * c[:, None]).sum()
        self.gap_rel = hs["gap_rel"]
        # velocity
        if F > 1:
            value[3], grad[3] = _autograd(po.mean_velocity_error, p, t)
            dsum[3] = np.linalg.norm(np.diff(p, axis=1) - np.diff(t, axis=1), axis=-1).sum()
        else:
            value[3] = math.nan
        G[3] = gw[3]
        self.value, self.grad, self.G, self.dsum, self.esum = value, grad, G, dsum, esum

    # ---- gates -----------------------------------------------------------------------------------
    def grad_ref(self, w):
        return sum(w[k] * self.grad[k] for k in range(4) if w[k] != 0)

    def grad_bound(self, w):
        """Per-element bound of |g - g64| for term weights w (NaN where g64 is NaN)."""
        g64 = self.grad_ref(w)
        fp64 = np.zeros(self.shape[:-1])
        adds = np.zeros(self.shape)
        for k in range(4):
            if w[k] != 0:
                fp64 = fp64 + abs(w[k]) * K_GRAD[k] * self.G[k].reshape(self.shape[:-1])
                adds = adds + np.abs(w[k] * self.grad[k])
        return U * np.abs(g64) + E * fp64[..., None] + 4 * E * adds

    def value_fp64_err(self, k, depth):
        if self.count[k] == 0:
            return math.nan
        return E * ((depth + K_DIST) * self.dsum[k] + self.esum[k]) / self.count[k]

    def term_bound(self, k, depth):
        return U * abs(self.value[k]) + self.value_fp64_err(k, depth)

    def loss_ref(self, w):
        return sum(w[k] * self.value[k] for k in range(4) if w[k] != 0)

    def loss_bound(self, w, depth):
        fp64 = sum(abs(w[k]) * self.value_fp64_err(k, depth) + 4 * E * abs(w[k] * self.value[k])
                   for k in range(4) if w[k] != 0)
        return U * abs(self.loss_ref(w)) + fp64


def ratio(got, want, bound):
    """Worst |got - want| / bound over the elements; NaN must meet NaN (ratio inf otherwise)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), want.shape)
    nan_w, nan_g = np.isnan(want), np.isnan(got)
    if (nan_w != nan_g).any():
        return math.inf
    ok = ~nan_w
    if not ok.any():
        return 0.0
    d = np.abs(got[ok] - want[ok])
    b = bound[ok]
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(d == 0, 0.0, d / b)
    return float(np.nan_to_num(r, nan=0.0).max())


def round_nearest(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32)


def round_toward_zero(x):
    x = np.asarray(x, dtype=np.float64)
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    return np.where(over, np.nextafter(f, np.float32(0)), f)


def demonstrations(ref, k):
    """[(name, wrong fp32 gradient of term k alone)] for term k of `ref` (a Reference)."""
    w = [0.0] * 4
    w[k] = 1.0
    g64 = ref.grad_ref(w)
    out = [("rounded toward zero", round_toward_zero(g64))]
    swapped = round_nearest(g64).reshape(ref.poses, ref.J, 3).copy()
    i = int(np.argmax(np.abs(swapped).sum(axis=(1, 2))[:-1]))
    swapped[[i, i + 1]] = swapped[[i + 1, i]]
    out.append(("one pose swapped with its neighbour", swapped.reshape(ref.shape)))
    wrong = {1: _n_mpjpe_scale_detached, 2: _p_mpjpe_rotation_detached, 3: _velocity_missing_start}
    if k in wrong:
        _, g = _autograd(wrong[k], ref.p, ref.t)
        name = {1: "scale detached", 2: "rotation detached", 3: "no start difference"}[k]
        if k == 2:   # degenerate poses hold the rotation fixed already: compare on the others
            keep = ~ref.horn["degenerate"].reshape(ref.shape[:2])
            g = np.where(keep[..., None, None], g, g64)
        out.append((name, round_nearest(g)))
    return out


def metric_means(avg, target):
    """float64 [mpjpe, p_mpjpe, n_mpjpe, velocity] (VP3D_EVAL_* order) of one sequence: avg, target
    (frames, J, 3) fp32 (avg the kernel's own flip average)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        vel = mo.mean_velocity_error(avg, target) if avg.shape[0] > 1 else math.nan
    return np.array([mo.mpjpe(avg, target), mo.p_mpjpe(avg, target), mo.n_mpjpe(avg, target), vel])


EVAL_SLOT = (0, 2, 1, 3)   # term k of the loss -> VP3D_EVAL_* slot


# ---- inputs ---------------------------------------------------------------------------------------

def random_poses(rng, seqs, F, J):
    """fp32 (seqs, F, J, 3) target and prediction: noise on the target, half of the poses rotated,
    scaled and shifted, every fourth of those reflected (an improper H)."""
    t = rng.normal(0, 0.3, (seqs * F, J, 3))
    p = t + rng.normal(0, 0.05, t.shape)
    half = (seqs * F) // 2
    r, _ = np.linalg.qr(rng.normal(size=(half, 3, 3)))
    r[::4, :, 0] *= -1
    p[:half] = np.einsum("fja,fab->fjb", p[:half], r) * rng.uniform(0.7, 1.3, (half, 1, 1)) + 0.2
    shape = (seqs, F, J, 3)
    return p.reshape(shape).astype(np.float32), t.reshape(shape).astype(np.float32)


# gap_rel of order 1e-14 (2^-24), near 1e-12 (2^-21), 1e-10 (2^-17) and 1e-6 (2^-10)
PLANAR_EPS = (0.0, 2.0 ** -24, 2.0 ** -21, 2.0 ** -17, 2.0 ** -10)


def planar_pose(rng, J, eps):
    """Target and prediction with z = 0 and a y-spread of eps in fp32-exact steps: s3 = 0 exactly
    and lambda_0 - lambda_1 = 2 s2, of order eps^2."""
    x = rng.uniform(-1, 1, J).astype(np.float32)
    xp = (x + rng.normal(0, 0.05, J)).astype(np.float32)
    t = np.zeros((J, 3), np.float32)
    p = np.zeros((J, 3), np.float32)
    t[:, 0], p[:, 0] = x, xp
    t[:, 1] = np.float32(eps) * rng.randint(-4, 5, J).astype(np.float32)
    p[:, 1] = np.float32(eps) * rng.randint(-4, 5, J).astype(np.float32)
    return p, t


def improper_equal_pose(J, alpha=0.75, beta=0.375):
    """H = diag(a, b, -b) up to normalisation: singular values s2 = s3 with det H < 0, Horn's gap
    2 (s2 - s3) = 0.  Target: +-alpha e1, +-beta e2, +-beta e3 (repeated, the rest at the origin);
    prediction: the target with z negated."""
    pts = [alpha * np.eye(3)[0], beta * np.eye(3)[1], beta * np.eye(3)[2]]
    t = np.zeros((J, 3), np.float32)
    j = 0
    while j + 6 <= J:
        for v in pts:
            t[j], t[j + 1] = v, -v
            j += 2
    p = t.copy()
    p[:, 2] *= -1
    return p, t


def collinear_pose(rng, J):
    """Prediction on one line (H of rank 1, lambda_0 = lambda_1) against a random target."""
    t = rng.normal(0, 0.3, (J, 3)).astype(np.float32)
    m = rng.randint(-8, 9, J).astype(np.float32) / 16          # fp32-exact products: exactly on a line
    p = np.outer(m, np.array([0.75, 0.0, 0.5], np.float32)).astype(np.float32) + np.float32(0.125)
    return p, t


def rotation_cases(rng, J=17):
    """(name, pred, target) of (1, F, J, 3) batches: every special construction among random
    poses, so each batch also has a spread of ordinary poses."""
    out = []
    for name, make in (("reflected", None), ("collinear", lambda: collinear_pose(rng, J)),
                       ("improper_s2_eq_s3", lambda: improper_equal_pose(J)),
                       ("identical", None), ("zero_spread", None)):
        p, t = random_poses(rng, 1, 24, J)
        if name == "reflected":
            p[0, ::2] = p[0, ::2] * np.array([-1, 1, 1], np.float32)
        elif name == "identical":
            p[0, ::3] = t[0, ::3]
        elif name == "zero_spread":
            p[0, 3] = p[0, 3, :1]           # every joint the same point: ny = 0
            t[0, 7] = 0.25                  # a point target: nx = 0
            p[0, 11] = 0.0                  # all-zero prediction: <p, p> = 0 too
        else:
            for f in range(0, 24, 5):
                p[0, f], t[0, f] = make()
        out.append((name, p, t))
    p, t = random_poses(rng, 1, 2 * len(PLANAR_EPS), J)
    for i, eps in enumerate(PLANAR_EPS):
        for f in (2 * i, 2 * i + 1):
            p[0, f], t[0, f] = planar_pose(rng, J, eps)
    out.append(("planar", p, t))
    return out


def near_threshold(gap_rel):
    """Poses whose gap is within 10x of the degeneracy threshold, either side."""
    g = np.asarray(gap_rel)
    return (g > po.DEGENERATE_GAP / 10) & (g < po.DEGENERATE_GAP * 10)
