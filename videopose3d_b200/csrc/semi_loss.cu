// Loss head of the semi-supervised training step (SURVEY §8 row f2, BASELINE configs[4]) in ONE
// launch: everything run.py:350-390 computes between the two model outputs and `loss_total` --
//   loss_3d_pos        = mpjpe(pred_pos[:split], inputs_3d with the root joint zeroed)      run.py:352, 336
//   loss_traj          = weighted_mpjpe(pred_traj[:split], root trajectory, w = 1 / z_root) run.py:358-360
//   loss_reconstruction= mpjpe(project_to_2d(pred_pos[split:] + pred_traj[split:], cam), target_2d)
//                        (common/camera.py:37-88, distortion-aware or linear)                 run.py:374-379
//   penalty            = mean_bone | mean_labeled(bone length) - mean_unlabeled(bone length) |,
//                        bone length = mean over frames of ||joint - parent||               run.py:383-387
// -- plus d loss_total / d pred_pos and d pred_traj.  The reference spends ~40 elementwise /
// reduction kernels forward and as many backward on this; here one cooperative grid does a first
// pass (all per-frame terms and the per-bone length sums), a grid-wide barrier, and a second pass
// that adds the bone-length gradient (its sign needs the global means).  All reductions are
// per-block partials summed in block order: reproducible.
#include <cooperative_groups.h>

#include "internal.cuh"
#include "camera.cuh"

namespace cg = cooperative_groups;

namespace vp3d {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxJoints = 32;
constexpr int kPartStride = 3 + 2 * kMaxJoints;  // pos, traj, recon sums + per-bone sums (lab, unl)

struct SemiArgs {
  const float* pos;        // [n_lab + n_unl][F][J][3]
  const float* traj;       // [n_lab + n_unl][F][1][3]
  const float* target_3d;  // [n_lab][F][J][3], joint 0 = global root trajectory
  const float* cam;        // [n_unl][9]
  const float* target_2d;  // [n_unl][F][J][2]
  const int* parents;      // [J]
  float* dpos;             // like pos, or null
  float* dtraj;            // like traj, or null
  float* losses;           // [5]: pos, traj, reconstruction, penalty, total
  float* part;             // [grid][kPartStride]
  int n_lab, n_unl, F, J;
  int linear, use_pos, use_traj, use_proj, use_bone;   // which terms enter the total / gradients
};

__device__ __forceinline__ float block_sum(float v, float* sm) {  // ordered: warp tree, then warps 0..7
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.0f;
  for (int w = 0; w < kThreads / 32; ++w) t += sm[w];
  return t;
}

__global__ void __launch_bounds__(kThreads) semi_loss_kernel(const SemiArgs a) {
  __shared__ float sm[kThreads / 32];
  __shared__ float s_sign[kMaxJoints];
  const int J = a.J, F = a.F;
  const long long lab_units = (long long)a.n_lab * F, unl_units = (long long)a.n_unl * F;
  const long long stride = (long long)gridDim.x * kThreads;
  const long long first = (long long)blockIdx.x * kThreads + threadIdx.x;
  const float w_pos = lab_units > 0 ? 1.0f / ((float)lab_units * J) : 0.0f;
  const float w_traj = lab_units > 0 ? 1.0f / (float)lab_units : 0.0f;
  const float w_pos_g = a.use_pos ? w_pos : 0.0f, w_traj_g = a.use_traj ? w_traj : 0.0f;
  const bool have_t3 = a.target_3d != nullptr;   // penalty-only calls pass no 3-D targets
  const float w_rec = unl_units > 0 ? 1.0f / ((float)unl_units * J) : 0.0f;
  const bool grads = a.dpos != nullptr;
  float* my_part = a.part + (size_t)blockIdx.x * kPartStride;

  float acc_pos = 0.0f, acc_traj = 0.0f, acc_rec = 0.0f;
  float bone[kMaxJoints];
  // ---------------------------------------------------------------- pass 1, labeled units
#pragma unroll
  for (int j = 0; j < kMaxJoints; ++j) bone[j] = 0.0f;
  for (long long u = first; u < lab_units; u += stride) {
    const float* p = a.pos + u * J * 3;
    const float* q = have_t3 ? a.target_3d + u * J * 3 : p;
    const float rx = have_t3 ? q[0] : 0.0f, ry = have_t3 ? q[1] : 0.0f, rz = have_t3 ? q[2] : 1.0f;
    for (int j = 0; j < J; ++j) {                            // (rx, ry, rz): root trajectory, run.py:335
      const float px = p[j * 3], py = p[j * 3 + 1], pz = p[j * 3 + 2];
      const float ex = px - (j ? q[j * 3] : 0.0f), ey = py - (j ? q[j * 3 + 1] : 0.0f),
                  ez = pz - (j ? q[j * 3 + 2] : 0.0f);       // inputs_3d[:, :, 0] = 0 (run.py:336)
      const float d = sqrtf(ex * ex + ey * ey + ez * ez);
      acc_pos += d;
      if (grads) {
        const float s = d > 0.0f ? w_pos_g / d : 0.0f;
        float* g = a.dpos + (u * J + j) * 3;
        g[0] = ex * s; g[1] = ey * s; g[2] = ez * s;
      }
      if (j > 0 && a.use_bone) {
        const int pa = a.parents[j];
        const float bx = px - p[pa * 3], by = py - p[pa * 3 + 1], bz = pz - p[pa * 3 + 2];
        bone[j] += sqrtf(bx * bx + by * by + bz * bz);
      }
    }
    const float* t = a.traj + u * 3;
    const float ex = t[0] - rx, ey = t[1] - ry, ez = t[2] - rz;
    const float d = sqrtf(ex * ex + ey * ey + ez * ez);
    const float w = 1.0f / rz;                               // run.py:359
    acc_traj += w * d;
    if (grads) {
      const float s = d > 0.0f ? w_traj_g * w / d : 0.0f;
      float* g = a.dtraj + u * 3;
      g[0] = ex * s; g[1] = ey * s; g[2] = ez * s;
    }
  }
  for (int j = 1; j < J; ++j) {
    const float t = block_sum(bone[j], sm);
    if (threadIdx.x == 0) my_part[3 + j] = t;
  }
  // ---------------------------------------------------------------- pass 1, unlabeled units
#pragma unroll
  for (int j = 0; j < kMaxJoints; ++j) bone[j] = 0.0f;
  const float w_rec_g = a.use_proj ? w_rec : 0.0f;          // --no-proj: logged, not optimised
  for (long long v = first; v < unl_units; v += stride) {
    const long long u = lab_units + v;
    const float* p = a.pos + u * J * 3;
    const bool have_cam = a.cam != nullptr && a.target_2d != nullptr;   // else intrinsics and target read as 0
    const Camera c = have_cam ? load_camera(a.cam + (v / F) * 9) : Camera{};
    const float tx = a.traj[u * 3], ty = a.traj[u * 3 + 1], tz = a.traj[u * 3 + 2];
    float gtx = 0.0f, gty = 0.0f, gtz = 0.0f;
    for (int j = 0; j < J; ++j) {
      const float px = p[j * 3], py = p[j * 3 + 1], pz = p[j * 3 + 2];
      const Projection P = project(c, px + tx, py + ty, pz + tz, a.linear);
      const float* tg = have_cam ? a.target_2d + (v * J + j) * 2 : nullptr;
      const float ex = have_cam ? P.x - tg[0] : 0.0f, ey = have_cam ? P.y - tg[1] : 0.0f;
      const float d = sqrtf(ex * ex + ey * ey);
      acc_rec += d;
      if (grads) {
        const float3 gp = project_backward(c, P, ex, ey, d > 0.0f ? w_rec_g / d : 0.0f, a.linear);
        float* g = a.dpos + (u * J + j) * 3;
        g[0] = gp.x; g[1] = gp.y; g[2] = gp.z;
        gtx += gp.x; gty += gp.y; gtz += gp.z;
      }
      if (j > 0 && a.use_bone) {
        const int pa = a.parents[j];
        const float bx = px - p[pa * 3], by = py - p[pa * 3 + 1], bz = pz - p[pa * 3 + 2];
        bone[j] += sqrtf(bx * bx + by * by + bz * bz);
      }
    }
    if (grads) {
      float* g = a.dtraj + u * 3;
      g[0] = gtx; g[1] = gty; g[2] = gtz;
    }
  }
  for (int j = 1; j < J; ++j) {
    const float t = block_sum(bone[j], sm);
    if (threadIdx.x == 0) my_part[3 + kMaxJoints + j] = t;
  }
  {
    const float s0 = block_sum(acc_pos, sm), s1 = block_sum(acc_traj, sm), s2 = block_sum(acc_rec, sm);
    if (threadIdx.x == 0) { my_part[0] = s0; my_part[1] = s1; my_part[2] = s2; }
  }
  __threadfence();
  cg::this_grid().sync();

  // ---------------------------------------------------------------- global sums (every block, block order)
  float delta_sign = 0.0f, abs_delta = 0.0f;
  if (a.use_bone && threadIdx.x >= 1 && threadIdx.x < J) {
    float bl = 0.0f, bu = 0.0f;
    for (unsigned b = 0; b < gridDim.x; ++b) {
      bl += __ldcg(a.part + (size_t)b * kPartStride + 3 + threadIdx.x);
      bu += __ldcg(a.part + (size_t)b * kPartStride + 3 + kMaxJoints + threadIdx.x);
    }
    const float delta = bl / (float)lab_units - bu / (float)unl_units;
    abs_delta = fabsf(delta);
    delta_sign = delta > 0.0f ? 1.0f : (delta < 0.0f ? -1.0f : 0.0f);
  }
  if (threadIdx.x < kMaxJoints) s_sign[threadIdx.x] = delta_sign;
  const float pen_sum = block_sum(abs_delta, sm);            // also orders s_sign for everyone
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float t0 = 0.0f, t1 = 0.0f, t2 = 0.0f;
    for (unsigned b = 0; b < gridDim.x; ++b) {
      t0 += __ldcg(a.part + (size_t)b * kPartStride);
      t1 += __ldcg(a.part + (size_t)b * kPartStride + 1);
      t2 += __ldcg(a.part + (size_t)b * kPartStride + 2);
    }
    const float l_pos = t0 * w_pos, l_traj = t1 * w_traj, l_rec = t2 * w_rec;
    const float pen = a.use_bone ? pen_sum / (float)(J - 1) : 0.0f;
    a.losses[0] = l_pos; a.losses[1] = l_traj; a.losses[2] = l_rec; a.losses[3] = pen;
    a.losses[4] = (a.use_pos ? l_pos : 0.0f) + (a.use_traj ? l_traj : 0.0f) +
                  (a.use_proj ? l_rec : 0.0f) + pen;
  }
  if (!a.use_bone || !grads) return;

  // ---------------------------------------------------------------- pass 2: bone-length gradient
  // d penalty / d p_j = sign_j / (J-1) * (+1/(n_lab F) | -1/(n_unl F)) * (p_j - p_parent) / len_j,
  // and the opposite on the parent; a unit's joints live in one thread, so plain read-modify-write
  const float c_lab = 1.0f / ((float)(J - 1) * (float)lab_units);
  const float c_unl = -1.0f / ((float)(J - 1) * (float)unl_units);
  for (long long u = first; u < lab_units + unl_units; u += stride) {
    const float c = u < lab_units ? c_lab : c_unl;
    const float* p = a.pos + u * J * 3;
    float* g = a.dpos + u * J * 3;
    for (int j = 1; j < J; ++j) {
      const float sg = s_sign[j];
      if (sg == 0.0f) continue;
      const int pa = a.parents[j];
      const float bx = p[j * 3] - p[pa * 3], by = p[j * 3 + 1] - p[pa * 3 + 1],
                  bz = p[j * 3 + 2] - p[pa * 3 + 2];
      const float len = sqrtf(bx * bx + by * by + bz * bz);
      if (len <= 0.0f) continue;
      const float f = sg * c / len;
      g[j * 3] += bx * f; g[j * 3 + 1] += by * f; g[j * 3 + 2] += bz * f;
      g[pa * 3] -= bx * f; g[pa * 3 + 1] -= by * f; g[pa * 3 + 2] -= bz * f;
    }
  }
}

}  // namespace
}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) size_t vp3d_semi_loss_scratch_bytes(void) {
  return (size_t)1024 * vp3d::kPartStride * sizeof(float);
}

extern "C" __attribute__((visibility("default"))) int vp3d_semi_loss_fwd_bwd(
    const float* pos, const float* traj, const float* target_3d, const float* cam,
    const float* target_2d, const int32_t* parents, int64_t n_labeled, int64_t n_unlabeled,
    int32_t frames, int32_t joints, int32_t linear, int32_t terms, float* losses, float* dpos,
    float* dtraj, void* scratch, size_t scratch_bytes, void* stream) {
  using namespace vp3d;
  if (n_labeled < 0 || n_unlabeled < 0 || frames < 1 || joints < 1 || joints > kMaxJoints)
    return fail(VP3D_ERR_INVALID, "semi_loss: bad sizes (labeled %lld, unlabeled %lld, frames %d, "
                "joints %d; at most %d joints)", (long long)n_labeled, (long long)n_unlabeled, frames,
                joints, kMaxJoints);
  if (!losses || !scratch) return fail(VP3D_ERR_INVALID, "semi_loss: null losses / scratch pointer");
  if ((dpos == nullptr) != (dtraj == nullptr))
    return fail(VP3D_ERR_INVALID, "semi_loss: dpos and dtraj go together");
  if (terms < 0 || terms > 15) return fail(VP3D_ERR_INVALID, "semi_loss: terms must be a 4-bit mask");
  const bool t_pos = terms & VP3D_SEMI_POS, t_traj = terms & VP3D_SEMI_TRAJ;
  const bool t_proj = terms & VP3D_SEMI_PROJ, t_bone = terms & VP3D_SEMI_BONE;
  if (n_labeled + n_unlabeled > 0 && (!pos || !traj))
    return fail(VP3D_ERR_INVALID, "semi_loss: null prediction pointer");
  if (n_labeled > 0 && (t_pos || t_traj) && !target_3d)
    return fail(VP3D_ERR_INVALID, "semi_loss: the 3-D terms need target_3d");
  if (n_unlabeled > 0 && t_proj && (!cam || !target_2d))
    return fail(VP3D_ERR_INVALID, "semi_loss: the re-projection term needs cam and target_2d");
  // one joint has no bones: the penalty is the mean over none, 0 / 0 = NaN as in the reference,
  // and adds no gradient
  const bool bone = t_bone && n_labeled > 0 && n_unlabeled > 0;
  if (bone && !parents) return fail(VP3D_ERR_INVALID, "semi_loss: the bone-length term needs parents");
  const long long units = (n_labeled + n_unlabeled) * frames;
  if (units > 0x7fffffffll * 64) return fail(VP3D_ERR_UNSUPPORTED, "semi_loss: too large");
  int grid = (int)((units + kThreads - 1) / kThreads);
  const int sms = num_sms();
  if (grid > sms) grid = sms;                 // cooperative launch: one resident block per SM at most
  if (grid < 1) grid = 1;
  if ((size_t)grid * kPartStride * sizeof(float) > scratch_bytes)
    return fail(VP3D_ERR_WORKSPACE, "semi_loss: scratch too small (%zu bytes)", scratch_bytes);
  SemiArgs a;
  a.pos = pos; a.traj = traj; a.target_3d = target_3d; a.cam = cam; a.target_2d = target_2d;
  a.parents = parents; a.dpos = dpos; a.dtraj = dtraj; a.losses = losses;
  a.part = static_cast<float*>(scratch);
  a.n_lab = (int)n_labeled; a.n_unl = (int)n_unlabeled; a.F = frames; a.J = joints;
  a.linear = linear ? 1 : 0;
  a.use_pos = t_pos ? 1 : 0; a.use_traj = t_traj ? 1 : 0; a.use_proj = t_proj ? 1 : 0;
  a.use_bone = bone ? 1 : 0;
  void* params[] = {&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)semi_loss_kernel, dim3(grid), dim3(kThreads),
                                       params, 0, static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}
