// Differentiable pose losses in ONE launch: any weighted subset of
//   [0] mpjpe      mean ||p - t||                                            common/loss.py:11-17
//   [1] n_mpjpe    mean ||s p - t||, s = sum <t, p> / sum <p, p> per pose    loss.py:68-78
//   [2] p_mpjpe    mean ||a p R + t0 - t|| after per-pose similarity Procrustes   loss.py:27-66
//   [3] velocity   mean ||diff(p) - diff(t)||, first differences along the frame axis   loss.py:80-89
// and the gradient of their weighted sum with respect to the prediction.  A pose is one
// (sequence, frame) slice of J <= 32 joints: one warp per pose, one lane per joint, fp64 inside,
// rounded once to fp32 for the terms, the loss and the gradient.
//
// Gradients (per pose, u_j = e_j / ||e_j||, 0 for a zero error as autograd's norm backward gives):
//   mpjpe     u_j
//   n_mpjpe   s u_j + (sum_i u_i . p_i) (t_j - 2 s p_j) / sum <p, p>   (the scale's own derivative is
//             kept: the loss is an unsquared distance, so the envelope theorem does not apply)
//   p_mpjpe   e_j = |X0| (tr Q y0_j - x0_j) with y0 the centred, normalised prediction, Q = R^T the
//             rotation of the top eigenvector q0 of Horn's N(H) and tr = lambda_0 (procrustes.cuh).
//             Reverse mode: tr-bar and Q-bar from the errors, q0-bar through Q(q), then
//             N-bar = tr-bar q0 q0^T + sum_{k>=1} (q_k . q0-bar) / (lambda_0 - lambda_k) q_k q0^T,
//             symmetrised, mapped to H-bar by the adjoint of H -> N, and through the normalisation
//             and centring of the prediction.  A pose with lambda_0 - lambda_1 <= 1e-12 max(|lambda_0|, 1)
//             has no differentiable rotation: it gets the gradient with the rotation held fixed (the
//             eigenvector sum dropped) and is counted in `degenerate`.
//   velocity  v_f - v_{f+1}, v_f = u of the difference ending at frame f (each warp recomputes its
//             neighbours' differences, so no two warps write one gradient row).
// Reductions: per-lane sums in a fixed pose order, warp sums, warps in order, a grid-wide barrier,
// then blocks in order -- no floating-point atomics, so the same input gives the same bits.
#include <cooperative_groups.h>

#include "internal.cuh"
#include "procrustes.cuh"

namespace cg = cooperative_groups;

namespace vp3d {
namespace {

constexpr int kPoseWarps = 8;
constexpr int kPoseThreads = 32 * kPoseWarps;
constexpr int kPoseMaxJoints = 32;
constexpr int kPoseMaxBlocks = 1024;
constexpr int kPartStride = 5;  // four term sums and the degenerate count of one block
constexpr double kDegenerateGap = 1e-12;

struct PoseLossArgs {
  const float* pred;    // [poses][J][3], poses = seqs * F
  const float* target;  // same
  float* dpred;         // same, or null (no backward)
  float* terms;         // [4]
  float* loss;          // [1]
  int* degenerate;      // [1] or null
  double* part;         // [grid][kPartStride]
  double w[4];          // term weights; 0 = term not evaluated
  double gw[4];         // w_k / (number of distances averaged by term k): gradient scales
  double count[4];      // number of distances averaged by term k
  long long poses;
  int F, J;
};

__device__ __forceinline__ double warp_sum(double v) {  // butterfly: every lane ends with the same bits
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void load3(const float* base, long long pose, int J, int j, double* v) {
  const float* s = base + (pose * J + j) * 3;
  v[0] = s[0]; v[1] = s[1]; v[2] = s[2];
}

// u = e / ||e|| (0 for a zero vector); returns ||e||.
__device__ __forceinline__ double unit(const double* e, double* u) {
  const double d = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
  const double r = d > 0.0 ? 1.0 / d : 0.0;
  u[0] = e[0] * r; u[1] = e[1] * r; u[2] = e[2] * r;
  return d;
}

// P-MPJPE of one pose (this lane's joint): returns the lane's aligned distance and, when `grads`,
// adds scale * d distance-sum / d p (this lane's joint) to g.  *degenerate: the rotation's gap test.
__device__ __forceinline__ double p_mpjpe_pose(const double* p, const double* t, bool on, int J,
                                               bool grads, double scale, double* g, bool* degenerate) {
  const double inv_j = 1.0 / J;
  const double mx0 = warp_sum(t[0]) * inv_j, mx1 = warp_sum(t[1]) * inv_j, mx2 = warp_sum(t[2]) * inv_j;
  const double my0 = warp_sum(p[0]) * inv_j, my1 = warp_sum(p[1]) * inv_j, my2 = warp_sum(p[2]) * inv_j;
  double x0[3] = {on ? t[0] - mx0 : 0.0, on ? t[1] - mx1 : 0.0, on ? t[2] - mx2 : 0.0};
  double y0[3] = {on ? p[0] - my0 : 0.0, on ? p[1] - my1 : 0.0, on ? p[2] - my2 : 0.0};
  const double nx = sqrt(warp_sum(x0[0] * x0[0] + x0[1] * x0[1] + x0[2] * x0[2]));
  const double ny = sqrt(warp_sum(y0[0] * y0[0] + y0[1] * y0[1] + y0[2] * y0[2]));
#pragma unroll
  for (int c = 0; c < 3; ++c) { x0[c] /= nx; y0[c] /= ny; }
  double H[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) H[r][c] = warp_sum(x0[r] * y0[c]);
  double A[4][4], V[4][4];
  horn_eigen(H, A, V);
  double lam[4] = {A[0][0], A[1][1], A[2][2], A[3][3]};
  int k0 = 0;
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (lam[k] > lam[k0]) k0 = k;
  double q[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) q[r] = V[r][0];
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (k == k0) {
#pragma unroll
      for (int r = 0; r < 4; ++r) q[r] = V[r][k];
    }
  const double lam0 = lam[k0];
  {
    const double n = rsqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
    for (int r = 0; r < 4; ++r) q[r] *= n;
  }
  double Q[3][3];
  quat_rotation(q[0], q[1], q[2], q[3], Q);
  const double tr = lam0;
  double qy[3], e[3], u[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    qy[r] = Q[r][0] * y0[0] + Q[r][1] * y0[1] + Q[r][2] * y0[2];
    e[r] = nx * (tr * qy[r] - x0[r]);
  }
  const double d = on ? unit(e, u) : 0.0;
  if (!on) u[0] = u[1] = u[2] = 0.0;
  double lam1 = -INFINITY;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (k != k0 && lam[k] > lam1) lam1 = lam[k];
  *degenerate = lam0 - lam1 <= kDegenerateGap * fmax(fabs(lam0), 1.0);
  if (!grads) return d;

  // e = nx (tr Q y0 - x0): tr-bar, Q-bar and the direct y0-bar
  const double tr_bar = nx * warp_sum(u[0] * qy[0] + u[1] * qy[1] + u[2] * qy[2]);
  const double ntr = nx * tr;
  double B[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) B[a][b] = ntr * warp_sum(u[a] * y0[b]);
  double yb[3];
#pragma unroll
  for (int b = 0; b < 3; ++b) yb[b] = ntr * (Q[0][b] * u[0] + Q[1][b] * u[1] + Q[2][b] * u[2]);
  // q-bar: Q's entries are quadratic forms in q = (w, x, y, z)
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  double qb[4];
  qb[0] = 2.0 * (w * (B[0][0] + B[1][1] + B[2][2]) + z * (B[1][0] - B[0][1]) + y * (B[0][2] - B[2][0]) +
                 x * (B[2][1] - B[1][2]));
  qb[1] = 2.0 * (x * (B[0][0] - B[1][1] - B[2][2]) + y * (B[0][1] + B[1][0]) + z * (B[0][2] + B[2][0]) +
                 w * (B[2][1] - B[1][2]));
  qb[2] = 2.0 * (y * (-B[0][0] + B[1][1] - B[2][2]) + x * (B[0][1] + B[1][0]) + w * (B[0][2] - B[2][0]) +
                 z * (B[1][2] + B[2][1]));
  qb[3] = 2.0 * (z * (-B[0][0] - B[1][1] + B[2][2]) + w * (B[1][0] - B[0][1]) + x * (B[0][2] + B[2][0]) +
                 y * (B[1][2] + B[2][1]));
  // N-bar = tr-bar q q^T + sum_{k != k0} c_k v_k q^T, c_k = (v_k . q-bar) / (lambda_0 - lambda_k)
  double col[4];  // N-bar = (tr-bar q + sum c_k v_k) q^T = col q^T
#pragma unroll
  for (int r = 0; r < 4; ++r) col[r] = tr_bar * q[r];
  if (!*degenerate) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k == k0) continue;
      const double ck = (V[0][k] * qb[0] + V[1][k] * qb[1] + V[2][k] * qb[2] + V[3][k] * qb[3]) /
                        (lam0 - lam[k]);
#pragma unroll
      for (int r = 0; r < 4; ++r) col[r] += ck * V[r][k];
    }
  }
  double N[4][4];  // symmetrised
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) N[r][c] = 0.5 * (col[r] * q[c] + col[c] * q[r]);
  // adjoint of H -> N(H) (S = H^T, see horn_eigen)
  const double sxx = N[0][0] + N[1][1] - N[2][2] - N[3][3];
  const double syy = N[0][0] - N[1][1] + N[2][2] - N[3][3];
  const double szz = N[0][0] - N[1][1] - N[2][2] + N[3][3];
  const double syz = 2.0 * (N[0][1] + N[2][3]), szy = 2.0 * (N[2][3] - N[0][1]);
  const double szx = 2.0 * (N[0][2] + N[1][3]), sxz = 2.0 * (N[1][3] - N[0][2]);
  const double sxy = 2.0 * (N[0][3] + N[1][2]), syx = 2.0 * (N[1][2] - N[0][3]);
  const double Hb[3][3] = {{sxx, syx, szx}, {sxy, syy, szy}, {sxz, syz, szz}};  // H-bar = S-bar^T
  // H = sum_j x0_j y0_j^T: y0-bar_j += H-bar^T x0_j
#pragma unroll
  for (int b = 0; b < 3; ++b) yb[b] += Hb[0][b] * x0[0] + Hb[1][b] * x0[1] + Hb[2][b] * x0[2];
  // y0 = (p - mean p) / |p - mean p|
  const double gy = warp_sum(yb[0] * y0[0] + yb[1] * y0[1] + yb[2] * y0[2]);
  double zb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) zb[c] = on ? (yb[c] - gy * y0[c]) / ny : 0.0;
  const double m0 = warp_sum(zb[0]) * inv_j, m1 = warp_sum(zb[1]) * inv_j, m2 = warp_sum(zb[2]) * inv_j;
  g[0] += scale * (zb[0] - m0); g[1] += scale * (zb[1] - m1); g[2] += scale * (zb[2] - m2);
  return d;
}

__global__ void __launch_bounds__(kPoseThreads) pose_loss_kernel(const PoseLossArgs a) {
  __shared__ double sm[kPoseWarps][kPartStride];
  __shared__ double tot[kPartStride];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool on = lane < a.J;
  const bool grads = a.dpred != nullptr;
  const bool t_mp = a.w[0] != 0.0, t_n = a.w[1] != 0.0, t_p = a.w[2] != 0.0, t_v = a.w[3] != 0.0;
  const long long n_warps = (long long)gridDim.x * kPoseWarps;
  double acc[4] = {0.0, 0.0, 0.0, 0.0}, n_degenerate = 0.0;

  for (long long f = (long long)blockIdx.x * kPoseWarps + warp; f < a.poses; f += n_warps) {
    double p[3] = {0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0};
    if (on) {
      load3(a.pred, f, a.J, lane, p);
      load3(a.target, f, a.J, lane, t);
    }
    if (t_mp) {
      const double e[3] = {p[0] - t[0], p[1] - t[1], p[2] - t[2]};
      double u[3];
      const double d = unit(e, u);
      if (on) acc[0] += d;
      if (grads) { g[0] += a.gw[0] * u[0]; g[1] += a.gw[0] * u[1]; g[2] += a.gw[0] * u[2]; }
    }
    if (t_n) {
      const double tp = warp_sum(t[0] * p[0] + t[1] * p[1] + t[2] * p[2]);
      const double pp = warp_sum(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
      const double s = tp / pp;
      const double e[3] = {s * p[0] - t[0], s * p[1] - t[1], s * p[2] - t[2]};
      double u[3];
      const double d = unit(e, u);
      if (on) acc[1] += d;
      if (grads) {
        const double c = warp_sum(on ? u[0] * p[0] + u[1] * p[1] + u[2] * p[2] : 0.0) / pp;
#pragma unroll
        for (int k = 0; k < 3; ++k) g[k] += a.gw[1] * (s * u[k] + c * (t[k] - 2.0 * s * p[k]));
      }
    }
    if (t_p) {
      bool deg = false;
      const double d = p_mpjpe_pose(p, t, on, a.J, grads, a.gw[2], g, &deg);
      if (on) acc[2] += d;
      if (lane == 0 && deg) n_degenerate += 1.0;
    }
    if (t_v && on) {
      const int fr = (int)(f % a.F);
      if (fr > 0) {  // the difference ending at this frame
        double pq[3], tq[3], u[3];
        load3(a.pred, f - 1, a.J, lane, pq);
        load3(a.target, f - 1, a.J, lane, tq);
        const double e[3] = {(p[0] - pq[0]) - (t[0] - tq[0]), (p[1] - pq[1]) - (t[1] - tq[1]),
                             (p[2] - pq[2]) - (t[2] - tq[2])};
        acc[3] += unit(e, u);
        if (grads) { g[0] += a.gw[3] * u[0]; g[1] += a.gw[3] * u[1]; g[2] += a.gw[3] * u[2]; }
      }
      if (grads && fr + 1 < a.F) {  // the one starting at it (its distance is the next warp's)
        double pn[3], tn[3], u[3];
        load3(a.pred, f + 1, a.J, lane, pn);
        load3(a.target, f + 1, a.J, lane, tn);
        const double e[3] = {(pn[0] - p[0]) - (tn[0] - t[0]), (pn[1] - p[1]) - (tn[1] - t[1]),
                             (pn[2] - p[2]) - (tn[2] - t[2])};
        unit(e, u);
        g[0] -= a.gw[3] * u[0]; g[1] -= a.gw[3] * u[1]; g[2] -= a.gw[3] * u[2];
      }
    }
    if (grads && on) {
      float* o = a.dpred + (f * a.J + lane) * 3;
      o[0] = (float)g[0]; o[1] = (float)g[1]; o[2] = (float)g[2];
    }
  }

  const double w0 = warp_sum(acc[0]), w1 = warp_sum(acc[1]), w2 = warp_sum(acc[2]), w3 = warp_sum(acc[3]);
  if (lane == 0) {
    sm[warp][0] = w0; sm[warp][1] = w1; sm[warp][2] = w2; sm[warp][3] = w3; sm[warp][4] = n_degenerate;
  }
  __syncthreads();
  if (threadIdx.x < kPartStride) {
    double s = 0.0;
    for (int w = 0; w < kPoseWarps; ++w) s += sm[w][threadIdx.x];
    a.part[(size_t)blockIdx.x * kPartStride + threadIdx.x] = s;
  }
  __threadfence();
  cg::this_grid().sync();
  if (blockIdx.x != 0) return;
  if (threadIdx.x < kPartStride) {
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(a.part + (size_t)b * kPartStride + threadIdx.x);
    tot[threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double loss = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double v = a.w[k] != 0.0 ? tot[k] / a.count[k] : 0.0;  // 0 / 0 = NaN: mean of nothing
      a.terms[k] = (float)v;
      if (a.w[k] != 0.0) loss += a.w[k] * v;
    }
    *a.loss = (float)loss;
    if (a.degenerate) *a.degenerate = (int)tot[4];
  }
}

int pose_blocks(long long poses) {
  const long long b = (poses + kPoseWarps - 1) / kPoseWarps;
  return (int)(b < kPoseMaxBlocks ? b : kPoseMaxBlocks);
}

}  // namespace
}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) size_t vp3d_pose_loss_scratch_bytes(int32_t frames_per_seq,
                                                                                       int64_t seqs) {
  if (frames_per_seq < 1 || seqs < 1) return 0;
  return (size_t)vp3d::pose_blocks((long long)frames_per_seq * seqs) * vp3d::kPartStride * sizeof(double);
}

extern "C" __attribute__((visibility("default"))) int vp3d_pose_loss_fwd_bwd(
    const float* pred, const float* target, int32_t frames_per_seq, int64_t seqs, int32_t joints,
    const double* term_weights, float* terms_out, float* loss_out, float* dpred, int32_t* degenerate_out,
    void* scratch, size_t scratch_bytes, void* stream) {
  using namespace vp3d;
  if (joints > kPoseMaxJoints)
    return fail(VP3D_ERR_UNSUPPORTED, "pose_loss: %d joints (at most %d)", joints, kPoseMaxJoints);
  if (joints < 1 || frames_per_seq < 1 || seqs < 0)
    return fail(VP3D_ERR_INVALID, "pose_loss: bad sizes (frames %d, seqs %lld, joints %d)", frames_per_seq,
                (long long)seqs, joints);
  if (!term_weights) return fail(VP3D_ERR_INVALID, "pose_loss: null term_weights");
  bool any = false;
  for (int k = 0; k < 4; ++k) any |= term_weights[k] != 0.0;
  if (!any) return fail(VP3D_ERR_INVALID, "pose_loss: every term weight is 0: nothing to compute");
  if (seqs == 0) return VP3D_OK;
  if (!pred || !target || !terms_out || !loss_out || !scratch)
    return fail(VP3D_ERR_INVALID, "pose_loss: null pred / target / terms / loss / scratch pointer");
  const long long poses = (long long)frames_per_seq * seqs;
  if (poses > 0x7fffffffll * 32) return fail(VP3D_ERR_UNSUPPORTED, "pose_loss: too many poses");
  int grid = pose_blocks(poses);
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pose_loss_kernel, kPoseThreads, 0));
  if (per_sm < 1) return fail(VP3D_ERR_UNSUPPORTED, "pose_loss: kernel does not fit on an SM");
  if (grid > per_sm * num_sms()) grid = per_sm * num_sms();  // cooperative launch: all blocks resident
  if ((size_t)grid * kPartStride * sizeof(double) > scratch_bytes)
    return fail(VP3D_ERR_WORKSPACE, "pose_loss: scratch too small (%zu bytes)", scratch_bytes);
  PoseLossArgs a;
  a.pred = pred; a.target = target; a.dpred = dpred; a.terms = terms_out; a.loss = loss_out;
  a.degenerate = degenerate_out; a.part = static_cast<double*>(scratch);
  a.poses = poses; a.F = frames_per_seq; a.J = joints;
  const double n_pose = (double)poses * joints, n_vel = (double)(frames_per_seq - 1) * seqs * joints;
  for (int k = 0; k < 4; ++k) {
    a.w[k] = term_weights[k];
    a.count[k] = k == 3 ? n_vel : n_pose;
    a.gw[k] = a.count[k] > 0.0 ? a.w[k] / a.count[k] : 0.0;
  }
  void* params[] = {&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)pose_loss_kernel, dim3(grid), dim3(kPoseThreads), params, 0,
                                       static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}
