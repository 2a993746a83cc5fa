// Per-sequence evaluation metrics of run.py's evaluate() (run.py:674-704) in ONE launch:
//   avg  = (pred[0] + mirror(pred[1])) * 0.5        test-time flip averaging, run.py:677-680
//   P1   = mean ||avg - target||                     mpjpe, common/loss.py:11-17
//   P2   = P1 after per-frame similarity Procrustes  p_mpjpe, loss.py:27-66
//   P3   = P1 after per-frame least-squares scale    n_mpjpe, loss.py:68-78
//   MPJVE= mean ||diff(avg) - diff(target)|| along the flattened frame axis, loss.py:80-89
// One warp per frame, one lane per joint (J <= 32).  Inputs are fp32; the flip average is formed in
// fp32 with the rounding of the torch expression (and optionally stored); everything after it is
// fp64.  Procrustes uses Horn's closed form (procrustes.cuh): the largest eigenpair of the 4x4 symmetric matrix built
// from H = X0^T Y0 (cyclic Jacobi in fp64) gives the optimal trace s1 + s2 + sign(det H) s3 of the
// reference's SVD as the eigenvalue and the rotation as a unit quaternion.  Reductions: per-lane
// running sums in a fixed frame order, warp sums, warps in order, a grid-wide barrier, then blocks
// in order -- no floating-point atomics, so the same input gives the same bits.
#include <cooperative_groups.h>

#include "internal.cuh"
#include "procrustes.cuh"

namespace cg = cooperative_groups;

namespace vp3d {
namespace {

constexpr int kWarps = 8;
constexpr int kThreads = 32 * kWarps;
constexpr int kMaxJoints = 32;
constexpr int kMaxBlocks = 1024;

struct EvalArgs {
  const float* pred;      // [copies][frames][J][3]
  const int* mirror_src;  // [J] or null
  const float* target;    // [frames][J][3]
  float* averaged;        // [frames][J][3] or null
  double* means;          // [4]
  double* part;           // [grid][4]
  long long frames;
  int J, copies, which;
};

__device__ __forceinline__ double warp_sum(double v) {  // butterfly: every lane ends with the same bits
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Flip-averaged prediction of joint j of frame f (flip_average, internal.cuh).
__device__ __forceinline__ void load_avg(const EvalArgs& a, long long f, int j, float* out) {
  const float* p0 = a.pred + (f * a.J + j) * 3;
  if (a.copies == 1) {
    out[0] = p0[0]; out[1] = p0[1]; out[2] = p0[2];
    return;
  }
  const int s = a.mirror_src ? a.mirror_src[j] : j;
  const float* p1 = a.pred + ((a.frames + f) * a.J + s) * 3;
  out[0] = flip_average(p0[0], p1[0], 0);
  out[1] = flip_average(p0[1], p1[1], 1);
  out[2] = flip_average(p0[2], p1[2], 2);
}

__global__ void __launch_bounds__(kThreads) pose_errors_kernel(const EvalArgs a) {
  __shared__ double sm[kWarps][4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool on = lane < a.J;
  const bool p1 = a.which & VP3D_EVAL_MPJPE, p2 = a.which & VP3D_EVAL_P_MPJPE;
  const bool p3 = a.which & VP3D_EVAL_N_MPJPE, vel = a.which & VP3D_EVAL_VELOCITY;
  const long long n_warps = (long long)gridDim.x * kWarps;
  double acc1 = 0.0, acc2 = 0.0, acc3 = 0.0, accv = 0.0;  // this lane's joint, this warp's frames

  for (long long f = (long long)blockIdx.x * kWarps + warp; f < a.frames; f += n_warps) {
    float pf[3] = {0.0f, 0.0f, 0.0f}, tf[3] = {0.0f, 0.0f, 0.0f};
    if (on) {
      load_avg(a, f, lane, pf);
      if (a.averaged) {
        float* o = a.averaged + (f * a.J + lane) * 3;
        o[0] = pf[0]; o[1] = pf[1]; o[2] = pf[2];
      }
      if (a.which) {
        const float* t = a.target + (f * a.J + lane) * 3;
        tf[0] = t[0]; tf[1] = t[1]; tf[2] = t[2];
      }
    }
    if (!a.which) continue;
    const double px = pf[0], py = pf[1], pz = pf[2];
    const double tx = tf[0], ty = tf[1], tz = tf[2];
    if (p1) {
      const double ex = px - tx, ey = py - ty, ez = pz - tz;
      if (on) acc1 += sqrt(ex * ex + ey * ey + ez * ez);
    }
    if (p3) {  // scale = sum <t, p> / sum <p, p> over the frame's joints
      const double tp = warp_sum(tx * px + ty * py + tz * pz);
      const double pp = warp_sum(px * px + py * py + pz * pz);
      const double s = tp / pp;
      const double ex = s * px - tx, ey = s * py - ty, ez = s * pz - tz;
      if (on) acc3 += sqrt(ex * ex + ey * ey + ez * ez);
    }
    if (p2) {
      const double inv_j = 1.0 / a.J;
      const double mxx = warp_sum(tx) * inv_j, mxy = warp_sum(ty) * inv_j, mxz = warp_sum(tz) * inv_j;
      const double myx = warp_sum(px) * inv_j, myy = warp_sum(py) * inv_j, myz = warp_sum(pz) * inv_j;
      double x0[3] = {on ? tx - mxx : 0.0, on ? ty - mxy : 0.0, on ? tz - mxz : 0.0};
      double y0[3] = {on ? px - myx : 0.0, on ? py - myy : 0.0, on ? pz - myz : 0.0};
      const double norm_x = sqrt(warp_sum(x0[0] * x0[0] + x0[1] * x0[1] + x0[2] * x0[2]));
      const double norm_y = sqrt(warp_sum(y0[0] * y0[0] + y0[1] * y0[1] + y0[2] * y0[2]));
#pragma unroll
      for (int c = 0; c < 3; ++c) { x0[c] /= norm_x; y0[c] /= norm_y; }
      double H[3][3];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) H[r][c] = warp_sum(x0[r] * y0[c]);
      double Q[3][3], tr;
      procrustes(H, Q, &tr);
      // aligned - target = a (p - muY) R + muX - t = norm_x (tr (Q y0) - x0), a = tr norm_x / norm_y
      double e2 = 0.0;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double e = tr * (Q[r][0] * y0[0] + Q[r][1] * y0[1] + Q[r][2] * y0[2]) - x0[r];
        e2 += e * e;
      }
      if (on) acc2 += norm_x * sqrt(e2);
    }
    if (vel && f > 0 && on) {
      float qf[3];
      load_avg(a, f - 1, lane, qf);
      const float* t = a.target + ((f - 1) * a.J + lane) * 3;
      const double ex = (px - (double)qf[0]) - (tx - (double)t[0]);
      const double ey = (py - (double)qf[1]) - (ty - (double)t[1]);
      const double ez = (pz - (double)qf[2]) - (tz - (double)t[2]);
      accv += sqrt(ex * ex + ey * ey + ez * ez);
    }
  }
  if (!a.which) return;

  const double w1 = warp_sum(acc1), w2 = warp_sum(acc2), w3 = warp_sum(acc3), wv = warp_sum(accv);
  if (lane == 0) { sm[warp][0] = w1; sm[warp][1] = w2; sm[warp][2] = w3; sm[warp][3] = wv; }
  __syncthreads();
  if (threadIdx.x < 4) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += sm[w][threadIdx.x];
    a.part[(size_t)blockIdx.x * 4 + threadIdx.x] = s;
  }
  __threadfence();
  cg::this_grid().sync();
  if (blockIdx.x == 0 && threadIdx.x < 4) {
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(a.part + (size_t)b * 4 + threadIdx.x);
    const double n = threadIdx.x == 3 ? (double)(a.frames - 1) * a.J : (double)a.frames * a.J;
    a.means[threadIdx.x] = (a.which >> threadIdx.x) & 1 ? s / n : 0.0;
  }
}

int blocks_for(long long frames) {
  const long long b = (frames + kWarps - 1) / kWarps;
  return (int)(b < kMaxBlocks ? b : kMaxBlocks);
}

}  // namespace
}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) size_t vp3d_pose_errors_scratch_bytes(int64_t frames) {
  return frames > 0 ? (size_t)vp3d::blocks_for(frames) * 4 * sizeof(double) : 0;
}

extern "C" __attribute__((visibility("default"))) int vp3d_pose_errors(
    const float* pred, int32_t copies, const int32_t* mirror_src, const float* target, int64_t frames,
    int32_t joints, int32_t which, float* averaged, double* means, void* scratch, size_t scratch_bytes,
    void* stream) {
  using namespace vp3d;
  if (joints > kMaxJoints)
    return fail(VP3D_ERR_UNSUPPORTED, "pose_errors: %d joints (at most %d)", joints, kMaxJoints);
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
  int grid = blocks_for(frames);
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pose_errors_kernel, kThreads, 0));
  if (per_sm < 1) return fail(VP3D_ERR_UNSUPPORTED, "pose_errors: kernel does not fit on an SM");
  if (grid > per_sm * num_sms()) grid = per_sm * num_sms();  // cooperative launch: all blocks resident
  if (which && (size_t)grid * 4 * sizeof(double) > scratch_bytes)
    return fail(VP3D_ERR_WORKSPACE, "pose_errors: scratch too small (%zu bytes)", scratch_bytes);
  EvalArgs a;
  a.pred = pred; a.mirror_src = mirror_src; a.target = target; a.averaged = averaged;
  a.means = means; a.part = static_cast<double*>(scratch);
  a.frames = frames; a.J = joints; a.copies = copies; a.which = which;
  void* params[] = {&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)pose_errors_kernel, dim3(grid), dim3(kThreads),
                                       params, 0, static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}
