// Per-pose errors of common/loss.py in ONE launch, as two instances of one kernel:
//   [0] mpjpe      mean ||p - t||                                            common/loss.py:11-17
//   [1] n_mpjpe    mean ||s p - t||, s = sum <t, p> / sum <p, p> per pose    loss.py:68-78
//   [2] p_mpjpe    mean ||a p R + t0 - t|| after per-pose similarity Procrustes   loss.py:27-66
//   [3] velocity   mean ||diff(p) - diff(t)||, first differences along the frame axis   loss.py:80-89
//  * the loss (vp3d_pose_loss_fwd_bwd): any weighted subset of the terms and the gradient of their
//    weighted sum with respect to the prediction, rounded once to fp32 for the terms, the loss and
//    the gradient;
//  * the metrics (vp3d_pose_errors, run.py's evaluate(), run.py:674-704): the selected terms as fp64
//    means of one sequence, after the test-time flip average avg = (pred[0] + mirror(pred[1])) * 0.5
//    (run.py:677-680), formed in fp32 with the rounding of the torch expression and optionally
//    stored.  No gradient code is compiled into this instance.
// A pose is one (sequence, frame) slice of J <= 32 joints: one warp per pose, one lane per joint,
// fp64 after the fp32 inputs.  Both instances run the same per-pose code, so a metric rounded to
// fp32 is the loss's term whenever the two grids are equal.
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
constexpr double kDegenerateGap = 1e-12;

// Per-block partials: the four term sums, and for the loss the degenerate count.
constexpr int part_stride(bool metrics) { return metrics ? 4 : 5; }
// means[] slot (VP3D_EVAL_* order: mpjpe, p_mpjpe, n_mpjpe, velocity) of term k.
constexpr int eval_slot(int k) { return k == 1 ? 2 : k == 2 ? 1 : k; }

struct PoseArgs {
  const float* pred;      // [copies][poses][J][3], poses = seqs * F
  const int* mirror_src;  // metrics with two copies: [J] or null
  const float* target;    // [poses][J][3]
  float* averaged;        // metrics: [poses][J][3] or null
  float* dpred;           // loss: [poses][J][3], or null (no backward)
  float* terms;           // loss: [4]
  float* loss;            // loss: [1]
  int* degenerate;        // loss: [1] or null
  double* means;          // metrics: [4]
  double* part;           // [grid][part_stride]
  double w[4];            // term weights; 0 = term not evaluated
  double gw[4];           // w_k / (number of distances averaged by term k): gradient scales
  double count[4];        // number of distances averaged by term k
  long long poses, F;
  int J, copies;
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

// The prediction of joint j of pose f as the terms see it: the loss reads it as given, the metrics
// flip-average two copies first (flip_average, internal.cuh).
template <bool kMetrics>
__device__ __forceinline__ void load_pred(const PoseArgs& a, long long f, int j, float* out) {
  const float* p0 = a.pred + (f * a.J + j) * 3;
  if (!kMetrics || a.copies == 1) {
    out[0] = p0[0]; out[1] = p0[1]; out[2] = p0[2];
    return;
  }
  const int s = a.mirror_src ? a.mirror_src[j] : j;
  const float* p1 = a.pred + ((a.poses + f) * a.J + s) * 3;
  out[0] = flip_average(p0[0], p1[0], 0);
  out[1] = flip_average(p0[1], p1[1], 1);
  out[2] = flip_average(p0[2], p1[2], 2);
}

template <bool kMetrics>
__device__ __forceinline__ void load_pred(const PoseArgs& a, long long f, int j, double* out) {
  float v[3];
  load_pred<kMetrics>(a, f, j, v);
  out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
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
  // The centroids divide by J, as np.mean does: J copies of one fp32 value sum exactly in fp64, so a
  // pose with every joint at one point centres to exactly 0 and gives NaN (0 / 0) like the
  // reference.  Multiplying by 1.0 / J instead leaves a spread of round-off and a finite answer.
  const double inv_j = 1.0 / J;
  const double mx0 = warp_sum(t[0]) / J, mx1 = warp_sum(t[1]) / J, mx2 = warp_sum(t[2]) / J;
  const double my0 = warp_sum(p[0]) / J, my1 = warp_sum(p[1]) / J, my2 = warp_sum(p[2]) / J;
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
  const double lam[4] = {A[0][0], A[1][1], A[2][2], A[3][3]};
  int k0 = 0;
  double lam0 = lam[0];  // the top eigenpair: the first largest eigenvalue
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (lam[k] > lam0) { k0 = k; lam0 = lam[k]; }
  double q[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) q[r] = V[r][0];
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (k == k0) {
#pragma unroll
      for (int r = 0; r < 4; ++r) q[r] = V[r][k];
    }
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

// The loss instance runs one block per SM.  The metrics instance, with no gradient code, fits two
// (at most 128 registers), which fixes its grid and with it the order of its sums.
template <bool kMetrics>
__global__ void __launch_bounds__(kPoseThreads, kMetrics ? 2 : 1) pose_kernel(const PoseArgs a) {
  constexpr int kParts = part_stride(kMetrics);
  __shared__ double sm[kPoseWarps][kParts];
  __shared__ double tot[kParts];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool on = lane < a.J;
  const bool grads = !kMetrics && a.dpred != nullptr;
  const bool t_mp = a.w[0] != 0.0, t_n = a.w[1] != 0.0, t_p = a.w[2] != 0.0, t_v = a.w[3] != 0.0;
  const bool any = t_mp || t_n || t_p || t_v;  // the metrics may only average
  const long long n_warps = (long long)gridDim.x * kPoseWarps;
  double acc[4] = {0.0, 0.0, 0.0, 0.0}, n_degenerate = 0.0;

  for (long long f = (long long)blockIdx.x * kPoseWarps + warp; f < a.poses; f += n_warps) {
    double p[3] = {0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0};
    if (on) {
      float v[3];
      load_pred<kMetrics>(a, f, lane, v);
      if (kMetrics && a.averaged) {
        float* o = a.averaged + (f * a.J + lane) * 3;
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
      }
      p[0] = v[0]; p[1] = v[1]; p[2] = v[2];
      if (any) load3(a.target, f, a.J, lane, t);
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
      const long long fr = kMetrics ? f : f % a.F;  // frame in its sequence; the metrics see one sequence
      if (fr > 0) {  // the difference ending at this frame
        double pq[3], tq[3], u[3];
        load_pred<kMetrics>(a, f - 1, lane, pq);
        load3(a.target, f - 1, a.J, lane, tq);
        const double e[3] = {(p[0] - pq[0]) - (t[0] - tq[0]), (p[1] - pq[1]) - (t[1] - tq[1]),
                             (p[2] - pq[2]) - (t[2] - tq[2])};
        acc[3] += unit(e, u);
        if (grads) { g[0] += a.gw[3] * u[0]; g[1] += a.gw[3] * u[1]; g[2] += a.gw[3] * u[2]; }
      }
      if (grads && fr + 1 < a.F) {  // the one starting at it (its distance is the next warp's)
        double pn[3], tn[3], u[3];
        load_pred<kMetrics>(a, f + 1, lane, pn);
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
  if (!any) return;  // nothing to sum: no scratch either

  const double w0 = warp_sum(acc[0]), w1 = warp_sum(acc[1]), w2 = warp_sum(acc[2]), w3 = warp_sum(acc[3]);
  if (lane == 0) {
    sm[warp][0] = w0; sm[warp][1] = w1; sm[warp][2] = w2; sm[warp][3] = w3;
    if constexpr (!kMetrics) sm[warp][4] = n_degenerate;
  }
  __syncthreads();
  if (threadIdx.x < kParts) {
    double s = 0.0;
    for (int w = 0; w < kPoseWarps; ++w) s += sm[w][threadIdx.x];
    a.part[(size_t)blockIdx.x * kParts + threadIdx.x] = s;
  }
  __threadfence();
  cg::this_grid().sync();
  if (blockIdx.x != 0) return;
  if (threadIdx.x < kParts) {
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(a.part + (size_t)b * kParts + threadIdx.x);
    tot[threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double loss = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double v = a.w[k] != 0.0 ? tot[k] / a.count[k] : 0.0;  // 0 / 0 = NaN: mean of nothing
      if constexpr (kMetrics) {
        a.means[eval_slot(k)] = v;
      } else {
        a.terms[k] = (float)v;
        if (a.w[k] != 0.0) loss += a.w[k] * v;
      }
    }
    if constexpr (!kMetrics) {
      *a.loss = (float)loss;
      if (a.degenerate) *a.degenerate = (int)tot[4];
    }
  }
}

int pose_blocks(long long poses) {
  const long long b = (poses + kPoseWarps - 1) / kPoseWarps;
  return (int)(b < kPoseMaxBlocks ? b : kPoseMaxBlocks);
}

// Term weights w (0 = not evaluated) and the number of distances each term averages over `seqs`
// sequences of a.F frames.
void set_terms(PoseArgs& a, const double* w, long long seqs) {
  const double n_pose = (double)a.poses * a.J, n_vel = (double)(a.F - 1) * seqs * a.J;
  for (int k = 0; k < 4; ++k) {
    a.w[k] = w[k];
    a.count[k] = k == 3 ? n_vel : n_pose;
    a.gw[k] = a.count[k] > 0.0 ? a.w[k] / a.count[k] : 0.0;
  }
}

// Cooperative launch of one instance: every block must be resident, so the grid is capped by that
// instance's own occupancy.  `sums`: the launch reduces into the caller's scratch.
template <bool kMetrics>
int launch_pose_kernel(const char* who, PoseArgs& a, bool sums, size_t scratch_bytes, void* stream) {
  int grid = pose_blocks(a.poses);
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pose_kernel<kMetrics>, kPoseThreads, 0));
  if (per_sm < 1) return fail(VP3D_ERR_UNSUPPORTED, "%s: kernel does not fit on an SM", who);
  if (grid > per_sm * num_sms()) grid = per_sm * num_sms();
  if (sums && (size_t)grid * part_stride(kMetrics) * sizeof(double) > scratch_bytes)
    return fail(VP3D_ERR_WORKSPACE, "%s: scratch too small (%zu bytes)", who, scratch_bytes);
  void* params[] = {&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)pose_kernel<kMetrics>, dim3(grid), dim3(kPoseThreads),
                                       params, 0, static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}

}  // namespace
}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) size_t vp3d_pose_loss_scratch_bytes(int32_t frames_per_seq,
                                                                                       int64_t seqs) {
  if (frames_per_seq < 1 || seqs < 1) return 0;
  return (size_t)vp3d::pose_blocks((long long)frames_per_seq * seqs) * vp3d::part_stride(false) *
         sizeof(double);
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
  PoseArgs a = {};
  a.pred = pred; a.target = target; a.dpred = dpred; a.terms = terms_out; a.loss = loss_out;
  a.degenerate = degenerate_out; a.part = static_cast<double*>(scratch);
  a.poses = poses; a.F = frames_per_seq; a.J = joints; a.copies = 1;
  set_terms(a, term_weights, seqs);
  return launch_pose_kernel<false>("pose_loss", a, true, scratch_bytes, stream);
}

extern "C" __attribute__((visibility("default"))) size_t vp3d_pose_errors_scratch_bytes(int64_t frames) {
  return frames > 0 ? (size_t)vp3d::pose_blocks(frames) * vp3d::part_stride(true) * sizeof(double) : 0;
}

extern "C" __attribute__((visibility("default"))) int vp3d_pose_errors(
    const float* pred, int32_t copies, const int32_t* mirror_src, const float* target, int64_t frames,
    int32_t joints, int32_t which, float* averaged, double* means, void* scratch, size_t scratch_bytes,
    void* stream) {
  using namespace vp3d;
  if (joints > kPoseMaxJoints)
    return fail(VP3D_ERR_UNSUPPORTED, "pose_errors: %d joints (at most %d)", joints, kPoseMaxJoints);
  if (joints < 1 || frames < 0 || (copies != 1 && copies != 2))
    return fail(VP3D_ERR_INVALID, "pose_errors: bad sizes (copies %d, frames %lld, joints %d)", copies,
                (long long)frames, joints);
  if (which < 0 || which > 15) return fail(VP3D_ERR_INVALID, "pose_errors: which must be a 4-bit mask");
  if (frames == 0) return VP3D_OK;
  if (!pred) return fail(VP3D_ERR_INVALID, "pose_errors: null pred pointer");
  if (which && (!target || !means || !scratch))
    return fail(VP3D_ERR_INVALID, "pose_errors: null target / means / scratch pointer");
  if (!which && !averaged) return fail(VP3D_ERR_INVALID, "pose_errors: nothing to compute");
  if (frames > 0x7fffffffll * 32) return fail(VP3D_ERR_UNSUPPORTED, "pose_errors: too many frames");
  PoseArgs a = {};
  a.pred = pred; a.mirror_src = mirror_src; a.target = target; a.averaged = averaged;
  a.means = means; a.part = static_cast<double*>(scratch);
  a.poses = frames; a.F = frames; a.J = joints; a.copies = copies;
  double w[4];  // one sequence; a selected term has weight 1
  for (int k = 0; k < 4; ++k) w[k] = (which >> eval_slot(k)) & 1 ? 1.0 : 0.0;
  set_terms(a, w, 1);
  return launch_pose_kernel<true>("pose_errors", a, which != 0, scratch_bytes, stream);
}
