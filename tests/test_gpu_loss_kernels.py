"""GPU: the training loss kernels against the float64 oracle (oracle/loss_head_oracle.py) at the
shapes where they can go wrong -- one partial block, a ragged last block, tens and more than a
thousand blocks, several frames per sample (camera per sample, bone lengths averaged over frames),
1 / 15 / 17 / 32 joints, points on and beyond the projection's clamp, bone deltas of exactly zero,
the semi-supervised head's grid barrier and grid-stride passes -- and the bit reproducibility of
all three entry points.

Tolerances.  u = 2^-24.  A loss is a sum of non-negative terms: its fp32 error is at most
(per-term error + summation depth) u S, where S is the oracle's value with absolute values taken
through the same expression (for the projection: |f proj| + |c| + |target| per point, what the
residual cancels).  The summation depth follows from the launch geometry (per-thread loop, the
8-level block tree, the partials in block order).  Each gradient element is bounded by its own
magnitude scale G (|e / d| <= 1 times the term's weight, or the projection chain's size): the error
is k u (|g| + G).  Every bound is doubled for second-order terms.  A wrong camera, a missing block
or a skipped grid-stride pass moves values by orders of magnitude more.
"""
import math

import pytest
import torch

from oracle import loss_head_oracle as lo
from videopose3d_b200 import _capi
from videopose3d_b200 import loss as vloss

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
THREADS, MAX_BLOCKS = 256, 4096
H36M_PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]
HE_PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 7, 11, 12, 7]     # HumanEva-I, 15 joints


def _parents(j):
    if j == 17:
        return H36M_PARENTS
    if j == 15:
        return HE_PARENTS
    return [-1] + [(i - 1) // 2 for i in range(1, j)]              # a binary tree (j = 1, 32)


def _sum_depth(items):
    """Additions along the longest path of the block-ordered loss sum of the mpjpe kernels."""
    blocks = max(1, min(math.ceil(items / THREADS), MAX_BLOCKS))
    per_thread = max(1, math.ceil(items / (blocks * THREADS)))
    return per_thread + 8 + math.ceil(blocks / THREADS) + 8 + 2


@pytest.fixture
def sm_limit():
    """Caps the cooperative grid of the semi-supervised kernel; always restores the default."""
    lib = _capi.load()

    def set_limit(n):
        _capi.check(lib.vp3d_set_sm_limit(n), "vp3d_set_sm_limit")
    try:
        yield set_limit
    finally:
        _capi.check(lib.vp3d_set_sm_limit(0), "vp3d_set_sm_limit")


# ---- mpjpe / weighted_mpjpe ---------------------------------------------------------------------

def _check_mpjpe(pred, tgt, w, dev):
    """pred / tgt: fp32 CPU tensors (..., dims); w: None or broadcastable to pred.shape[:-1]."""
    dims = pred.shape[-1]
    items = pred.numel() // dims
    p32 = pred.to(dev).requires_grad_(True)
    got = vloss.mpjpe(p32, tgt.to(dev)) if w is None else vloss.weighted_mpjpe(p32, tgt.to(dev), w.to(dev))
    got.backward()
    p64 = pred.double().requires_grad_(True)
    ref = lo.mpjpe(p64, tgt.double()) if w is None else lo.weighted_mpjpe(p64, tgt.double(), w.double())
    ref.backward()
    # loss: per term dims fma + sqrt + weight product; S = ref (every term >= 0)
    k = 2 * (dims + 4 + _sum_depth(items))
    assert abs(got.item() - ref.item()) <= k * U * ref.item(), (got.item(), ref.item(), k)
    # gradient: w_j / N * (e / d), |e / d| <= 1
    wj = (torch.ones(pred.shape[:-1], dtype=torch.float64) if w is None
          else w.double().expand(pred.shape[:-1]))[..., None].abs() / items
    err = (p32.grad.cpu().double() - p64.grad).abs()
    bound = 2 * (dims + 8) * U * (p64.grad.abs() + wj)
    assert bool((err <= bound).all()), float((err / bound).max())
    return p32.grad


@pytest.mark.parametrize("dims", [1, 2, 3, 16])
@pytest.mark.parametrize("items", [100, 1000, 1024 * 17, 64 * 243 * 17])
def test_mpjpe_matches_oracle(cuda_device, dims, items):
    """One partial block, a ragged last block (1000 = 3 x 256 + 232), 68 blocks, 1033 blocks."""
    g = torch.Generator().manual_seed(items + dims)
    pred = torch.randn(items, dims, generator=g) * 0.5
    tgt = torch.randn(items, dims, generator=g) * 0.5
    tgt[items // 3] = pred[items // 3]
    tgt[-1] = pred[-1]                                     # zero-length error vectors
    grad = _check_mpjpe(pred, tgt, None, cuda_device)
    assert float(grad[items // 3].abs().max()) == 0.0 and float(grad[-1].abs().max()) == 0.0
    w = torch.rand(items, generator=g) + 0.25
    _check_mpjpe(pred, tgt, w, cuda_device)


def test_weighted_mpjpe_with_broadcast_weight(cuda_device):
    """run.py:359: w of shape (n, F, 1) against (n, F, J, 3) poses; a ragged multi-block size."""
    g = torch.Generator().manual_seed(3)
    pred = torch.randn(37, 27, 17, 3, generator=g)
    tgt = torch.randn(37, 27, 17, 3, generator=g)
    w = 1 / (torch.rand(37, 27, 1, generator=g) * 3 + 3)
    _check_mpjpe(pred, tgt, w, cuda_device)


def test_mpjpe_of_non_contiguous_inputs(cuda_device):
    g = torch.Generator().manual_seed(4)
    pred = torch.randn(17, 300, 3, generator=g).transpose(0, 1)          # a transposed view
    tgt = torch.randn(300, 3, 17, generator=g).transpose(1, 2)
    assert not pred.is_contiguous() and not tgt.is_contiguous()
    assert not pred.to(cuda_device).is_contiguous()
    _check_mpjpe(pred, tgt, None, cuda_device)
    _check_mpjpe(pred, tgt, torch.rand(17, 300, generator=g).t(), cuda_device)


def test_mpjpe_of_an_empty_batch_is_nan(cuda_device):
    """torch.mean over nothing (common/loss.py:17) is NaN; so is the kernel's."""
    p = torch.zeros(0, 1, 17, 3, device=cuda_device, requires_grad=True)
    t = torch.zeros(0, 1, 17, 3, device=cuda_device)
    got = vloss.mpjpe(p, t)
    assert torch.isnan(got).item() and torch.isnan(lo.mpjpe(p.detach().double(), t.double())).item()
    got.backward()
    assert p.grad.shape == p.shape
    assert torch.isnan(vloss.weighted_mpjpe(p, t, torch.zeros(0, 1, 1, device=cuda_device))).item()


# ---- projected mpjpe ----------------------------------------------------------------------------

def _projection_case(seed, n, f, j, on_clamp=True):
    g = torch.Generator().manual_seed(seed)
    q = 1 / 4096.0                        # a grid on which the sums below are exact in fp32
    pos = torch.round(torch.randn(n, f, j, 3, generator=g) * 0.3 / q) * q
    traj = torch.round((torch.randn(n, f, 1, 3, generator=g) * 0.3 + torch.tensor([0., 0., 4.5])) / q) * q
    pos[0, 0, 1, 0] = 9.0                                  # beyond the clamp: no gradient through x
    pos[-1, -1, j - 1, 1] = -9.0
    if on_clamp:                                           # exactly on it: u = 1, v = -1
        z = pos[..., 2] + traj[..., 2]
        pos[:, :, 0, 0] = z[:, :, 0] - traj[:, :, 0, 0]
        pos[:, :, j // 2, 1] = -z[:, :, j // 2] - traj[:, :, 0, 1]
        X = pos + traj
        assert bool((X[:, :, 0, 0] == X[:, :, 0, 2]).all())
        assert bool((X[:, :, j // 2, 1] == -X[:, :, j // 2, 2]).all())
    cam = torch.cat([torch.rand(n, 2, generator=g) + 1.0, torch.randn(n, 2, generator=g) * 0.1,
                     torch.randn(n, 3, generator=g) * 0.1, torch.randn(n, 2, generator=g) * 0.01], dim=1)
    tgt = torch.randn(n, f, j, 2, generator=g) * 0.3
    return pos, traj, cam, tgt


def _projection_grad_scale(pos, traj, cam, tgt, linear, weight):
    """Per point: a bound on |d loss / d pos| (f / z times the clamp-and-distortion chain) and on the
    error of the residual's direction e / d (|f proj| + |c| + |t|) / d."""
    X = (pos + traj).double()
    cp = cam.double().abs()[:, None, None, :]
    z = X[..., 2].abs()
    uv = (X[..., :2].abs() / z[..., None]).clamp(max=1.0).sum(-1)
    chain = 1 + uv
    if not linear:
        chain = chain * (1 + 3 * cp[..., 4:7].sum(-1) + 4 * cp[..., 7:].sum(-1)) * 2
    with torch.no_grad():
        proj = (lo.project_to_2d_linear if linear else lo.project_to_2d)(X, cam.double())
        d = torch.norm(proj - tgt.double(), dim=-1)
    scale = lo.projection_scale(X, cam.double(), tgt.double(), linear)
    return weight * (cp[..., 0] + cp[..., 1]) * chain / z * (1 + scale / d), scale


@pytest.mark.parametrize("linear", [False, True])
@pytest.mark.parametrize("n,f", [(1024, 1), (64, 27), (64, 243)])
def test_projected_mpjpe_matches_oracle(cuda_device, linear, n, f):
    """A different camera per sample: indexing it by frame fails at F > 1."""
    j = 17
    pos, traj, cam, tgt = _projection_case(n + f, n, f, j)
    dev = cuda_device
    pa, ta = pos.to(dev).requires_grad_(True), traj.to(dev).requires_grad_(True)
    got = vloss.projected_mpjpe(pa, ta, cam.to(dev), tgt.to(dev), linear=linear)
    got.backward()
    pb, tb = pos.double().requires_grad_(True), traj.double().requires_grad_(True)
    ref = lo.projected_mpjpe(pb, tb, cam.double(), tgt.double(), linear)
    ref.backward()
    items = n * f * j
    G, scale = _projection_grad_scale(pos, traj, cam, tgt, linear, 1.0 / items)
    # loss: ~20 roundings in the projection and residual per point, relative to `scale`; the norm and
    # the sum (per thread J points + the block-ordered sum) relative to the value
    bound = 2 * U * (24 * float(scale.mean()) + (4 + j + _sum_depth(n * f)) * ref.item())
    assert abs(got.item() - ref.item()) <= bound, (got.item(), ref.item(), bound)
    assert float(pa.grad[0, 0, 1, 0]) == 0.0 and float(pa.grad[-1, -1, j - 1, 1]) == 0.0
    # on the clamp the gradient passes, as torch.clamp's does
    assert bool((pb.grad[:, :, 0, 0] != 0).all()) and bool((pa.grad[:, :, 0, 0] != 0).all())
    err = (pa.grad.cpu().double() - pb.grad).abs()
    lim = 2 * 32 * U * (pb.grad.abs() + G[..., None])
    assert bool((err <= lim).all()), float((err / lim).max())
    err_t = (ta.grad.cpu().double() - tb.grad).abs()
    lim_t = 2 * 32 * U * (tb.grad.abs() + G.sum(-1, keepdim=True)[..., None] * 3)
    assert bool((err_t <= lim_t).all()), float((err_t / lim_t).max())


def test_projected_mpjpe_of_no_samples_is_nan(cuda_device):
    z = torch.zeros(0, 1, 17, 3, device=cuda_device)
    got = vloss.projected_mpjpe(z, torch.zeros(0, 1, 1, 3, device=cuda_device),
                                torch.zeros(0, 9, device=cuda_device),
                                torch.zeros(0, 1, 17, 2, device=cuda_device))
    assert torch.isnan(got).item()


def test_entry_points_without_scratch_match_the_scratch_ones(cuda_device):
    """The ABI-compatible entry points run one block: the same numbers, the sum in another order
    (the same bits when one block is all the scratch-taking grid needs)."""
    lib = _capi.load()
    dev = cuda_device
    stream = torch.cuda.current_stream(dev).cuda_stream
    for n, f, j in ((5, 3, 17), (64, 243, 17)):
        pos, traj, cam, tgt = (t.to(dev) for t in _projection_case(7, n, f, j))
        tgt3 = (pos + traj).contiguous()
        ref_p = lo.mpjpe(pos.double(), tgt3.double()).item()
        ref_r = lo.projected_mpjpe(pos.double(), traj.double(), cam.double(), tgt.double()).item()
        out = torch.empty(2, device=dev)
        dpos, dtraj, dpred = torch.empty_like(pos), torch.empty_like(traj), torch.empty_like(pos)
        _capi.check(lib.vp3d_mpjpe_fwd_bwd(pos.data_ptr(), tgt3.data_ptr(), None, n * f * j, 3,
                                           out.data_ptr(), dpred.data_ptr(), stream), "mpjpe")
        _capi.check(lib.vp3d_projected_mpjpe_fwd_bwd(
            pos.data_ptr(), traj.data_ptr(), cam.data_ptr(), tgt.data_ptr(), n, f, j, 0,
            out[1:].data_ptr(), dpos.data_ptr(), dtraj.data_ptr(), stream), "projected")
        p = pos.clone().requires_grad_(True)
        ex_p = vloss.mpjpe(p, tgt3)
        ex_p.backward()
        pa, ta = pos.clone().requires_grad_(True), traj.clone().requires_grad_(True)
        ex_r = vloss.projected_mpjpe(pa, ta, cam, tgt)
        ex_r.backward()
        got = out.cpu().tolist()
        # one block: per thread n f j / 256 terms in order, then the tree
        depth = math.ceil(n * f * j / THREADS) + 8 + 2
        assert abs(got[0] - ref_p) <= 2 * U * (3 + 4 + depth) * ref_p
        _, scale = _projection_grad_scale(pos.cpu(), traj.cpu(), cam.cpu(), tgt.cpu(), False, 1.0)
        assert abs(got[1] - ref_r) <= 2 * U * (24 * float(scale.mean())
                                               + (4 + j * math.ceil(n * f / THREADS) + 10) * ref_r)
        assert torch.equal(dpred, p.grad) and torch.equal(dpos, pa.grad) and torch.equal(dtraj, ta.grad)
        if n * f <= THREADS:
            assert got[1] == ex_r.item()
        if n * f * j <= THREADS:
            assert got[0] == ex_p.item()


# ---- semi-supervised head -----------------------------------------------------------------------

def _semi_inputs(seed, n_lab, n_unl, f, j, identical=False):
    g = torch.Generator().manual_seed(seed)
    n = n_lab + n_unl
    pos = torch.randn(n, f, j, 3, generator=g) * 0.3
    traj = torch.randn(n, f, 1, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 4.5])
    pos[n_lab, 0, 0, 0] = 9.0                              # beyond the clamp
    if j > 1:
        pos[0, 0, 1] = pos[0, 0, _parents(j)[1]]           # one bone of length exactly 0
    if identical:                                          # every bone delta exactly 0
        pos[n_lab:] = pos[:n_lab]
    in3 = torch.randn(n_lab, f, j, 3, generator=g) * 0.4
    in3[:, :, 0, 2] = torch.rand(n_lab, f, generator=g) * 3 + 3
    cam = torch.cat([torch.rand(n_unl, 2, generator=g) + 1.0, torch.randn(n_unl, 2, generator=g) * 0.1,
                     torch.randn(n_unl, 3, generator=g) * 0.1, torch.randn(n_unl, 2, generator=g) * 0.01],
                    dim=1)
    t2 = torch.randn(n_unl, f, j, 2, generator=g) * 0.3
    return pos, traj, in3, cam, t2


def _semi_grid(units, limit):
    sms = min(132, limit) if limit else 132
    return max(1, min(math.ceil(units / THREADS), sms))


def _check_semi(dev, n_lab, n_unl, f, j, linear=False, no_proj=False, bone=True, identical=False,
                limit=0, seed=0):
    pos, traj, in3, cam, t2 = _semi_inputs(seed + 31 * j + f, n_lab, n_unl, f, j, identical)
    parents = _parents(j)
    pa, ta = pos.to(dev).requires_grad_(True), traj.to(dev).requires_grad_(True)
    total, terms = vloss.semi_supervised_loss(pa, ta, in3.to(dev), cam.to(dev), t2.to(dev), parents,
                                              linear_projection=linear, no_proj=no_proj,
                                              bone_length_term=bone)
    total.backward()
    pb, tb = pos.double().requires_grad_(True), traj.double().requires_grad_(True)
    ref_total, ref_terms = lo.semi_loss_head(pb, tb, in3.double(), cam.double(), t2.double(), parents,
                                             linear=linear, no_proj=no_proj, bone_length_term=bone)
    ref_total.backward()
    got = terms.cpu().double()
    units_lab, units_unl = n_lab * f, n_unl * f
    grid = _semi_grid(units_lab + units_unl, limit)
    passes = math.ceil(max(units_lab, units_unl) / (grid * THREADS))
    depth = passes * j + 8 + grid + 2            # per-thread units x joints, block tree, block order
    # 3-D and trajectory terms: non-negative sums, S = value
    for i in (0, 1):
        r = ref_terms[i].item()
        assert abs(got[i].item() - r) <= 2 * U * (16 + depth) * r, (i, got[i].item(), r)
    _, scale = _projection_grad_scale(pos[n_lab:], traj[n_lab:], cam, t2, linear, 1.0)
    r = ref_terms[2].item()
    assert abs(got[2].item() - r) <= 2 * U * (24 * float(scale.mean()) + (4 + depth) * r), (got[2].item(), r)
    # penalty: each delta cancels the two mean lengths (S = their sum), then the bone mean
    with torch.no_grad():
        lengths = torch.norm(pb[:, :, 1:] - pb[:, :, parents[1:]], dim=3).mean(1)
        s_pen = float((lengths[:n_lab].mean(0) + lengths[n_lab:].mean(0)).mean()) if j > 1 else 0.0
    r = ref_terms[3].item()
    if not bone:                                           # run.py:382 does not evaluate the term
        assert got[3].item() == 0.0
    elif j == 1:
        assert math.isnan(r) and math.isnan(got[3].item())
    else:
        assert abs(got[3].item() - r) <= 2 * U * ((8 + depth) * s_pen + 8 * r), (got[3].item(), r)
    if identical:
        assert r == 0.0 and got[3].item() == 0.0
    rt = ref_total.item()
    if math.isnan(rt):
        assert math.isnan(total.item())
    else:
        assert abs(total.item() - rt) <= 2 * U * (
            (16 + depth) * (ref_terms[0].item() + ref_terms[1].item()
                             + (0 if no_proj else ref_terms[2].item()))
            + 24 * float(scale.mean()) + (8 + depth) * s_pen + 4 * rt)
    # gradient scales per element: 3-D term 1 / (lab units J); trajectory w / lab units; projection
    # chain; bone term (1 + children) / ((J - 1) units of its side)
    G = torch.zeros(pos.shape, dtype=torch.float64)
    G[:n_lab] += 1.0 / (units_lab * j)
    if not no_proj:
        Gp, _ = _projection_grad_scale(pos[n_lab:], traj[n_lab:], cam, t2, linear, 1.0 / (units_unl * j))
        G[n_lab:] += Gp[..., None]
    if bone and j > 1:
        fan = torch.ones(j, dtype=torch.float64)
        for c in range(1, j):
            fan[parents[c]] += 1
        G[:n_lab] += fan[:, None] / ((j - 1) * units_lab)
        G[n_lab:] += fan[:, None] / ((j - 1) * units_unl)
    err = (pa.grad.cpu().double() - pb.grad).abs()
    lim = 2 * 32 * U * (pb.grad.abs() + G)
    assert bool((err <= lim).all()), float((err / lim).max())
    Gt = torch.zeros(traj.shape, dtype=torch.float64)
    Gt[:n_lab] += 1.0 / (in3[:, :, :1, 2:].double().abs() * units_lab)
    if not no_proj:
        Gt[n_lab:] += G[n_lab:].sum(2, keepdim=True).amax(-1, keepdim=True) * 3
    err_t = (ta.grad.cpu().double() - tb.grad).abs()
    lim_t = 2 * 32 * U * (tb.grad.abs() + Gt)
    assert bool((err_t <= lim_t).all()), float((err_t / lim_t).max())
    if no_proj and not bone:                               # --no-proj: logged, not optimised
        assert float(pa.grad[n_lab:].abs().max()) == 0.0
    return pa.grad


@pytest.mark.parametrize("j", [1, 15, 17, 32])
@pytest.mark.parametrize("f", [1, 27])
def test_semi_head_one_block(cuda_device, j, f):
    _check_semi(cuda_device, 5, 4, f, j)                   # 9 f <= 243 units


@pytest.mark.parametrize("j,f,linear,no_proj,bone", [
    (17, 27, False, False, True), (17, 27, True, False, True), (15, 27, False, True, True),
    (32, 1, False, False, False), (1, 27, True, False, True), (17, 1, False, True, False)])
def test_semi_head_several_blocks(cuda_device, j, f, linear, no_proj, bone):
    """About the semi-supervised config's size: several blocks, one pass."""
    n = 512 if f > 1 else 4000                             # 55 / 16 blocks
    _check_semi(cuda_device, n // 2 + 3, n // 2 - 2, f, j, linear, no_proj, bone)


@pytest.mark.parametrize("j,f,n_lab,n_unl", [(17, 1, 1000, 700), (32, 27, 37, 29), (15, 1, 555, 1500)])
def test_semi_head_grid_stride_passes(cuda_device, sm_limit, j, f, n_lab, n_unl):
    """A grid of 3 blocks (768 threads): several passes, lab_units a multiple of neither 256 nor
    768, so pass 2 revisits unlabeled units from other threads and blocks than pass 1."""
    sm_limit(3)
    assert (n_lab * f) % 256 and (n_lab * f) % 768
    _check_semi(cuda_device, n_lab, n_unl, f, j, limit=3)
    _check_semi(cuda_device, n_lab, n_unl, f, j, linear=True, limit=3)


def test_semi_head_full_grid_many_passes(cuda_device):
    """More than 132 x 256 units with no cap: every SM's block strides over several units."""
    _check_semi(cuda_device, 20011, 17003, 1, 17)


@pytest.mark.parametrize("f", [1, 27])
def test_semi_head_identical_poses_have_no_bone_gradient(cuda_device, f):
    """Labeled and unlabeled poses equal (and as many): every bone delta is exactly 0, its sign 0,
    and the abs() gradient of the reference is 0 -- the head's gradient is that without the term."""
    n = 300 if f == 1 else 20
    g_with = _check_semi(cuda_device, n, n, f, 17, identical=True)
    g_without = _check_semi(cuda_device, n, n, f, 17, bone=False, identical=True)
    assert torch.equal(g_with, g_without)


def test_semi_head_refuses_33_joints_and_bad_parents(cuda_device):
    pos, traj, in3, cam, t2 = (t.to(cuda_device) for t in _semi_inputs(1, 3, 3, 1, 33))
    with pytest.raises(ValueError, match="at most 32 joints"):
        vloss.semi_supervised_loss(pos, traj, in3, cam, t2, [-1] + list(range(32)))
    pos, traj, in3, cam, t2 = (t.to(cuda_device) for t in _semi_inputs(1, 3, 3, 1, 17))
    bad = list(H36M_PARENTS)
    bad[9] = 17
    for call in (lambda: vloss.semi_supervised_loss(pos, traj, in3, cam, t2, bad),
                 lambda: vloss.bone_length_penalty(pos, 3, bad)):
        with pytest.raises(ValueError, match="parents"):
            call()


def test_bone_length_penalty_multi_frame_multi_block(cuda_device, sm_limit):
    sm_limit(3)
    g = torch.Generator().manual_seed(9)
    pred = torch.randn(120, 27, 17, 3, generator=g)
    a = pred.to(cuda_device).requires_grad_(True)
    got = vloss.bone_length_penalty(a, 47, H36M_PARENTS)
    got.backward()
    b = pred.double().requires_grad_(True)
    ref = lo.bone_length_penalty(b, 47, H36M_PARENTS)
    ref.backward()
    with torch.no_grad():
        lengths = torch.norm(b[:, :, 1:] - b[:, :, H36M_PARENTS[1:]], dim=3).mean(1)
        s = float((lengths[:47].mean(0) + lengths[47:].mean(0)).mean())
    depth = math.ceil(73 * 27 / 768) * 17 + 8 + 3 + 2
    assert abs(got.item() - ref.item()) <= 2 * U * ((8 + depth) * s + 8 * ref.item())
    fan = torch.ones(17, dtype=torch.float64)
    for c in range(1, 17):
        fan[H36M_PARENTS[c]] += 1
    G = torch.zeros(pred.shape, dtype=torch.float64)
    G[:47] += fan[:, None] / (16 * 47 * 27)
    G[47:] += fan[:, None] / (16 * 73 * 27)
    err = (a.grad.cpu().double() - b.grad).abs()
    assert bool((err <= 2 * 32 * U * (b.grad.abs() + G)).all())


# ---- reproducibility ----------------------------------------------------------------------------

def _run_all(dev, data):
    pos, traj, cam, tgt, in3, cam_s, t2, mp, mt = data
    out = []
    p = mp.clone().requires_grad_(True)
    l1 = vloss.mpjpe(p, mt)
    l1.backward()
    out += [l1.detach(), p.grad]
    pa, ta = pos.clone().requires_grad_(True), traj.clone().requires_grad_(True)
    l2 = vloss.projected_mpjpe(pa, ta, cam, tgt)
    l2.backward()
    out += [l2.detach(), pa.grad, ta.grad]
    pa, ta = pos.clone().requires_grad_(True), traj.clone().requires_grad_(True)
    l3, terms = vloss.semi_supervised_loss(pa, ta, in3, cam_s, t2, H36M_PARENTS)
    l3.backward()
    out += [terms, pa.grad, ta.grad]
    return [t.clone() for t in out]


def test_same_input_gives_same_bits(cuda_device):
    """More than 100 blocks in every kernel: two calls in a row, a call on a second stream and a
    call after an unrelated launch of another size give identical bits.  (The order-fixed sums make
    this hold by construction; the atomics they replaced could also pass by chance.)"""
    dev = cuda_device
    g = torch.Generator().manual_seed(12)
    n, f, j = 128, 243, 17                                 # 31104 frames: 122 blocks
    pos = (torch.randn(n, f, j, 3, generator=g) * 0.3).to(dev)
    traj = (torch.randn(n, f, 1, 3, generator=g) * 0.3 + torch.tensor([0., 0., 4.5])).to(dev)
    cam = torch.cat([torch.rand(n, 2, generator=g) + 1, torch.randn(n, 7, generator=g) * 0.05], 1).to(dev)
    tgt = (torch.randn(n, f, j, 2, generator=g) * 0.3).to(dev)
    in3 = torch.randn(n // 2, f, j, 3, generator=g) * 0.4
    in3[:, :, 0, 2] = torch.rand(n // 2, f, generator=g) * 3 + 3
    data = (pos, traj, cam, tgt, in3.to(dev), cam[n // 2:].contiguous(), tgt[n // 2:].contiguous(),
            torch.randn(n * 2, f, j, 3, generator=g).to(dev),     # 1.06 M joints: 4096 blocks
            torch.randn(n * 2, f, j, 3, generator=g).to(dev))
    base = _run_all(dev, data)
    again = _run_all(dev, data)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        other = _run_all(dev, data)
    torch.cuda.current_stream(dev).wait_stream(side)
    small = torch.randn(3, 5, 17, 3, device=dev)
    vloss.mpjpe(small, small * 0.5).item()                 # an unrelated launch of another size
    after = _run_all(dev, data)
    torch.cuda.synchronize(dev)
    for run in (again, other, after):
        for a, b in zip(base, run):
            assert torch.equal(a, b)
