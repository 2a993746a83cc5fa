// Training-step companions of the model (SURVEY §8 rows f2 and f4).
//
//  * vp3d_adam_step: AMSGrad/Adam over every parameter tensor in ONE launch.  Reference:
//    `optim.Adam(model.parameters(), lr=lr, amsgrad=True)` + `optimizer.step()` (run.py:252, 264,
//    396, 420), lr decay by mutating param_groups (run.py:583-586).  torch runs 8 multi-tensor
//    launches over 16.95 M parameters; this is one HBM-bound pass: 20 B read + 16 B written per
//    element.
//  * vp3d_mpjpe_fwd_bwd: mean per-joint position error (loss.py:11-17, run.py:413-418) and its
//    gradient w.r.t. the prediction in one launch.  The loss is summed in block order (no
//    floating-point atomics): the same input gives the same bits.
#include "internal.cuh"
#include "camera.cuh"

namespace vp3d {
namespace {

constexpr int kAdamThreads = 256;
constexpr int kAdamChunk = 8192;  // elements per block

struct AdamBatch {
  vp3d_adam_tensor t[VP3D_ADAM_MAX_TENSORS];
  int first_block[VP3D_ADAM_MAX_TENSORS + 1];
  int n;
};

struct AdamHyper {
  float one_minus_beta1, beta2, one_minus_beta2, eps, weight_decay, step_size, bc2_sqrt;
};

__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, float& vmax,
                                            bool amsgrad, const AdamHyper& h) {
  // explicit roundings: the plain and the re-packing kernel must produce bit-identical updates, so
  // nothing is left to the compiler's choice of FMA contraction
  if (h.weight_decay != 0.0f) g = __fmaf_rn(h.weight_decay, p, g);
  m = __fmaf_rn(h.one_minus_beta1, __fsub_rn(g, m), m);
  v = __fmaf_rn(__fmul_rn(h.one_minus_beta2, g), g, __fmul_rn(v, h.beta2));
  float second = v;
  if (amsgrad) {
    vmax = fmaxf(vmax, v);
    second = vmax;
  }
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(second), h.bc2_sqrt), h.eps);
  p = __fsub_rn(p, __fmul_rn(h.step_size, __fdiv_rn(m, denom)));
}

__global__ void __launch_bounds__(kAdamThreads)
adam_step_kernel(const __grid_constant__ AdamBatch batch, const AdamHyper h) {
  // which tensor owns this block (<= 64 entries: a short scan)
  int ti = 0;
  while (ti + 1 < batch.n && (int)blockIdx.x >= batch.first_block[ti + 1]) ++ti;
  const vp3d_adam_tensor& t = batch.t[ti];
  const long long begin = (long long)(blockIdx.x - batch.first_block[ti]) * kAdamChunk;
  const long long end = min(begin + (long long)kAdamChunk, (long long)t.numel);
  const bool amsgrad = t.max_exp_avg_sq != nullptr;
  const uintptr_t bits = (uintptr_t)t.param | (uintptr_t)t.grad | (uintptr_t)t.exp_avg |
                         (uintptr_t)t.exp_avg_sq | (uintptr_t)t.max_exp_avg_sq;
  long long i = begin;
  if ((bits & 15) == 0) {  // all five streams 16-byte aligned (chunks are multiples of 4 elements)
    const long long vec_end = begin + ((end - begin) & ~3ll);
    for (long long k = begin + 4ll * threadIdx.x; k < vec_end; k += 4ll * kAdamThreads) {
      float4 p = *reinterpret_cast<float4*>(t.param + k);
      const float4 g = *reinterpret_cast<const float4*>(t.grad + k);
      float4 m = *reinterpret_cast<float4*>(t.exp_avg + k);
      float4 v = *reinterpret_cast<float4*>(t.exp_avg_sq + k);
      float4 x = amsgrad ? *reinterpret_cast<float4*>(t.max_exp_avg_sq + k) : make_float4(0, 0, 0, 0);
      adam_update(p.x, g.x, m.x, v.x, x.x, amsgrad, h);
      adam_update(p.y, g.y, m.y, v.y, x.y, amsgrad, h);
      adam_update(p.z, g.z, m.z, v.z, x.z, amsgrad, h);
      adam_update(p.w, g.w, m.w, v.w, x.w, amsgrad, h);
      *reinterpret_cast<float4*>(t.param + k) = p;
      *reinterpret_cast<float4*>(t.exp_avg + k) = m;
      *reinterpret_cast<float4*>(t.exp_avg_sq + k) = v;
      if (amsgrad) *reinterpret_cast<float4*>(t.max_exp_avg_sq + k) = x;
    }
    i = vec_end;
  }
  for (long long k = i + threadIdx.x; k < end; k += kAdamThreads) {
    float p = t.param[k], m = t.exp_avg[k], v = t.exp_avg_sq[k];
    float x = amsgrad ? t.max_exp_avg_sq[k] : 0.0f;
    adam_update(p, t.grad[k], m, v, x, amsgrad, h);
    t.param[k] = p;
    t.exp_avg[k] = m;
    t.exp_avg_sq[k] = v;
    if (amsgrad) t.max_exp_avg_sq[k] = x;
  }
}

// ---- AMSGrad + bf16 re-pack of the conv weights in one pass (SURVEY §8 f4) ---------------------
// The forward GEMMs read bf16 [plane][tap][co][ci] packs of Conv1d.weight (co, ci, tap) and the
// data-gradient GEMMs the transposed [plane][tap][ci][co] packs.  Instead of re-reading the 68 MB of
// fp32 masters after every optimizer step to refresh them (pack_conv_weight_t_kernel, 9 launches),
// the optimizer update itself emits both packs: a block owns a 32 x 32 (co, ci) tile for every tap,
// updates p / m / v / vmax in place (36 B per element, as the plain kernel) and writes the fresh
// value through shared memory so that both packs receive coalesced 64-byte bf16 rows (+4 B per
// element instead of +8 B and a second sweep).
struct PackTensor {
  vp3d_adam_tensor t;
  __nv_bfloat16* fwd;      // [planes][taps][fwd_n_pad][fwd_k_pad]
  __nv_bfloat16* tr;       // [planes][taps][tr_n_pad][tr_k_pad]  (rows = ci, cols = co)
  int c_out, c_in, taps;
  int fwd_n_pad, fwd_k_pad, tr_n_pad, tr_k_pad;
  int first_block, tiles_ci;
};
constexpr int kMaxPackTensors = 16;
struct PackBatch {
  PackTensor t[kMaxPackTensors];
  int n, planes;
};

__global__ void __launch_bounds__(256)
adam_pack_kernel(const __grid_constant__ PackBatch batch, const AdamHyper h) {
  __shared__ float sm[32][33];
  int ti = 0;
  while (ti + 1 < batch.n && (int)blockIdx.x >= batch.t[ti + 1].first_block) ++ti;
  const PackTensor& q = batch.t[ti];
  const int tile = blockIdx.x - q.first_block;
  const int co0 = (tile / q.tiles_ci) * 32, ci0 = (tile % q.tiles_ci) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool amsgrad = q.t.max_exp_avg_sq != nullptr;
  const long long fwd_plane = (long long)q.taps * q.fwd_n_pad * q.fwd_k_pad;
  const long long tr_plane = (long long)q.taps * q.tr_n_pad * q.tr_k_pad;
  for (int tap = 0; tap < q.taps; ++tap) {
    // all five streams of this thread's four elements are loaded before the first update: the
    // stores of the update may alias the loads as far as the compiler knows, and one element at a
    // time (20 bytes in flight per thread) left the pass latency-bound at half the HBM rate
    float pv[4], gv[4], mv[4], vv[4], xv[4];
    bool live[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int co = co0 + ty + 8 * u, ci = ci0 + tx;
      live[u] = co < q.c_out && ci < q.c_in;
      const long long k = live[u] ? ((long long)co * q.c_in + ci) * q.taps + tap : 0;
      pv[u] = live[u] ? q.t.param[k] : 0.0f;
      gv[u] = live[u] ? q.t.grad[k] : 0.0f;
      mv[u] = live[u] ? q.t.exp_avg[k] : 0.0f;
      vv[u] = live[u] ? q.t.exp_avg_sq[k] : 0.0f;
      xv[u] = (live[u] && amsgrad) ? q.t.max_exp_avg_sq[k] : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = ty + 8 * u;
      const int co = co0 + j, ci = ci0 + tx;
      if (live[u]) {
        const long long k = ((long long)co * q.c_in + ci) * q.taps + tap;
        adam_update(pv[u], gv[u], mv[u], vv[u], xv[u], amsgrad, h);
        q.t.param[k] = pv[u];
        q.t.exp_avg[k] = mv[u];
        q.t.exp_avg_sq[k] = vv[u];
        if (amsgrad) q.t.max_exp_avg_sq[k] = xv[u];
        if (q.fwd)
          store_bits16(q.fwd, ((long long)tap * q.fwd_n_pad + co) * q.fwd_k_pad + ci, fwd_plane,
                       batch.planes, pv[u]);
      }
      sm[j][tx] = pv[u];
    }
    __syncthreads();
    if (q.tr) {
#pragma unroll
      for (int j = ty; j < 32; j += 8) {
        const int ci = ci0 + j, co = co0 + tx;
        if (ci < q.c_in && co < q.c_out)
          store_bits16(q.tr, ((long long)tap * q.tr_n_pad + ci) * q.tr_k_pad + co, tr_plane,
                       batch.planes, sm[tx][j]);
      }
    }
    __syncthreads();
  }
}

// ---- MPJPE ------------------------------------------------------------------------------------

constexpr int kLossThreads = 256;
constexpr long long kLossMaxBlocks = 4096;  // grid cap of the scratch-taking entry points

// Sum of v over the block in a fixed tree (lanes by xor shuffle, then warps 0..7); the total is
// valid in thread 0.
__device__ __forceinline__ float block_total(float v, float* s_part) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // s_part may still be read by the previous call
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < kLossThreads / 32 ? s_part[threadIdx.x] : 0.0f;
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

// loss = weight * (sum of the block totals in block order).  One block writes its total directly.
// Otherwise every block stores its total in part[blockIdx.x] and takes an integer ticket; the
// block that draws the last ticket adds the partials, each thread a fixed strided subset and then
// the fixed block tree, so the bits do not depend on which block finishes when.  *ticket must be
// 0 at launch.
__device__ void store_loss(float block_sum, float weight, float* loss, float* part,
                           unsigned* ticket, float* s_part) {
  __shared__ bool is_last;
  if (gridDim.x == 1) {
    if (threadIdx.x == 0) *loss = block_sum * weight;
    return;
  }
  if (threadIdx.x == 0) {
    part[blockIdx.x] = block_sum;
    __threadfence();
    is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float t = 0.0f;
  for (unsigned b = threadIdx.x; b < gridDim.x; b += kLossThreads) t += __ldcg(part + b);
  t = block_total(t, s_part);
  if (threadIdx.x == 0) *loss = t * weight;
}

// One thread per joint (grid-stride): d = ||pred - target||_2 over the last axis (dims = 3 for
// poses); loss = weight * sum w_j * d, dpred = weight * w_j * (pred - target) / d  (0 where d == 0,
// as autograd's norm backward yields for a zero vector).  weight = 1 / joints_total folds the mean
// (NaN for no joints: torch.mean of nothing); w_j = 1 without per-joint weights (mpjpe) or the
// caller's weight (weighted_mpjpe).
__global__ void __launch_bounds__(kLossThreads)
mpjpe_kernel(const float* __restrict__ pred, const float* __restrict__ target,
             const float* __restrict__ joint_w, float* __restrict__ dpred, float* __restrict__ loss,
             float* __restrict__ part, unsigned* __restrict__ ticket, long long joints_total,
             int dims, float weight) {
  __shared__ float s_part[kLossThreads / 32];
  float acc = 0.0f;
  for (long long j = (long long)blockIdx.x * kLossThreads + threadIdx.x; j < joints_total;
       j += (long long)gridDim.x * kLossThreads) {
    const float* p = pred + j * dims;
    const float* q = target + j * dims;
    float sq = 0.0f;
    for (int k = 0; k < dims; ++k) {
      const float e = p[k] - q[k];
      sq = fmaf(e, e, sq);
    }
    const float d = sqrtf(sq);
    const float wj = joint_w != nullptr ? joint_w[j] : 1.0f;
    if (dpred != nullptr) {
      const float s = d > 0.0f ? weight * wj / d : 0.0f;
      for (int k = 0; k < dims; ++k) dpred[j * dims + k] = (p[k] - q[k]) * s;
    }
    acc += d * wj;
  }
  store_loss(block_total(acc, s_part), weight, loss, part, ticket, s_part);
}

// ---- re-projection loss (semi-supervised branch) -------------------------------------------------

// One thread per frame (n, t): for each joint X = pos + traj, project with the camera of sample n
// (camera.cuh: camera.py:37-88, distortion-aware or linear), accumulate the 2-D
// distance to the target, and write d loss / d pos per joint and d loss / d traj per frame (the
// joint sum -- no atomics needed since the frame's joints live in one thread).  Frames are
// grid-strided; the loss is summed as in mpjpe_kernel.
__global__ void __launch_bounds__(kLossThreads)
projected_mpjpe_kernel(const float* __restrict__ pos, const float* __restrict__ traj,
                       const float* __restrict__ cam, const float* __restrict__ target,
                       float* __restrict__ dpos, float* __restrict__ dtraj, float* __restrict__ loss,
                       float* __restrict__ part, unsigned* __restrict__ ticket,
                       long long frames_total, int frames_per_sample, int joints, int linear,
                       float weight) {
  __shared__ float s_part[kLossThreads / 32];
  float acc = 0.0f;
  for (long long fr = (long long)blockIdx.x * kLossThreads + threadIdx.x; fr < frames_total;
       fr += (long long)gridDim.x * kLossThreads) {
    const Camera c = load_camera(cam + (fr / frames_per_sample) * 9);
    const float tx = traj[fr * 3 + 0], ty = traj[fr * 3 + 1], tz = traj[fr * 3 + 2];
    float gtx = 0.0f, gty = 0.0f, gtz = 0.0f;
    for (int j = 0; j < joints; ++j) {
      const long long e = fr * joints + j;
      const Projection P = project(c, pos[e * 3 + 0] + tx, pos[e * 3 + 1] + ty, pos[e * 3 + 2] + tz, linear);
      const float ex = P.x - target[e * 2 + 0];
      const float ey = P.y - target[e * 2 + 1];
      const float d = sqrtf(ex * ex + ey * ey);
      acc += d;
      if (dpos != nullptr) {
        const float3 g = project_backward(c, P, ex, ey, d > 0.0f ? weight / d : 0.0f, linear);
        dpos[e * 3 + 0] = g.x;
        dpos[e * 3 + 1] = g.y;
        dpos[e * 3 + 2] = g.z;
        gtx += g.x;
        gty += g.y;
        gtz += g.z;
      }
    }
    if (dtraj != nullptr) {
      dtraj[fr * 3 + 0] = gtx;
      dtraj[fr * 3 + 1] = gty;
      dtraj[fr * 3 + 2] = gtz;
    }
  }
  store_loss(block_total(acc, s_part), weight, loss, part, ticket, s_part);
}

// Grid of the loss kernels: one thread per item up to kLossMaxBlocks blocks with caller scratch,
// one block without.  Scratch = the ticket + one partial per block; none for a single block.
long long loss_blocks(long long items, bool scratch) {
  if (!scratch) return 1;
  const long long b = (items + kLossThreads - 1) / kLossThreads;
  return b < 1 ? 1 : (b > kLossMaxBlocks ? kLossMaxBlocks : b);
}
size_t loss_scratch_bytes(long long items) {
  const long long b = loss_blocks(items, true);
  return b > 1 ? (size_t)(b + 1) * sizeof(float) : 0;
}

}  // namespace
}  // namespace vp3d

#define VP3D_EXPORT extern "C" __attribute__((visibility("default")))

namespace vp3d {
static int adam_hyper(AdamHyper* h, const vp3d_adam_tensor* tensors, int32_t n_tensors, int64_t step,
                      double lr, double beta1, double beta2, double eps, double weight_decay) {
  if (n_tensors < 0 || (n_tensors > 0 && tensors == nullptr))
    return fail(VP3D_ERR_INVALID, "vp3d_adam_step: bad tensor list");
  if (step < 1) return fail(VP3D_ERR_INVALID, "vp3d_adam_step: step must be >= 1 (got %lld)",
                            (long long)step);
  if (!(lr >= 0.0) || !(eps >= 0.0) || !(beta1 >= 0.0 && beta1 < 1.0) ||
      !(beta2 >= 0.0 && beta2 < 1.0) || !(weight_decay >= 0.0))
    return fail(VP3D_ERR_INVALID, "vp3d_adam_step: invalid hyper-parameter (lr %g, betas %g %g, "
                "eps %g, weight_decay %g)", lr, beta1, beta2, eps, weight_decay);
  // bias corrections in double on the host, as torch.optim.Adam computes them from python floats
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  h->one_minus_beta1 = (float)(1.0 - beta1);
  h->beta2 = (float)beta2;
  h->one_minus_beta2 = (float)(1.0 - beta2);
  h->eps = (float)eps;
  h->weight_decay = (float)weight_decay;
  h->step_size = (float)(lr / bc1);
  h->bc2_sqrt = (float)sqrt(bc2);
  return VP3D_OK;
}

// One fused launch over the conv weights listed in `packs` (train_api.cu resolves the destinations).
int launch_adam_pack(const AdamPackItem* items, int n, int planes, int64_t step, double lr,
                     double beta1, double beta2, double eps, double weight_decay,
                     cudaStream_t stream) {
  if (n <= 0) return VP3D_OK;
  if (n > kMaxPackTensors) return fail(VP3D_ERR_UNSUPPORTED, "adam_pack: too many conv tensors");
  AdamHyper h;
  vp3d_adam_tensor dummy;
  VP3D_TRY(adam_hyper(&h, &dummy, 0, step, lr, beta1, beta2, eps, weight_decay));
  PackBatch b;
  b.n = 0;
  b.planes = planes;
  int blocks = 0;
  for (int i = 0; i < n; ++i) {
    const AdamPackItem& it = items[i];
    const PackedConv &fwd = *it.fwd, &tr = *it.tr;
    if (!it.t.param || !it.t.grad || !it.t.exp_avg || !it.t.exp_avg_sq)
      return fail(VP3D_ERR_INVALID, "adam_pack: tensor %d has a null pointer", i);
    if (it.t.numel != (int64_t)tr.c_out * tr.c_in * tr.taps)
      return fail(VP3D_ERR_INVALID, "adam_pack: tensor %d has %lld elements, expected %d x %d x %d", i,
                  (long long)it.t.numel, tr.c_out, tr.c_in, tr.taps);
    PackTensor& q = b.t[b.n++];
    q.t = it.t; q.fwd = fwd.w; q.tr = tr.w;
    q.c_out = tr.c_out; q.c_in = tr.c_in; q.taps = tr.taps;
    q.fwd_n_pad = fwd.n_pad; q.fwd_k_pad = fwd.k_pad;
    q.tr_n_pad = tr.n_pad; q.tr_k_pad = tr.k_pad;
    q.first_block = blocks;
    q.tiles_ci = (tr.c_in + 31) / 32;
    blocks += ((tr.c_out + 31) / 32) * q.tiles_ci;
  }
  adam_pack_kernel<<<blocks, 256, 0, stream>>>(b, h);
  CUDA_TRY(cudaGetLastError());
  return VP3D_OK;
}
}  // namespace vp3d

VP3D_EXPORT int vp3d_adam_step(const vp3d_adam_tensor* tensors, int32_t n_tensors, int64_t step,
                               double lr, double beta1, double beta2, double eps,
                               double weight_decay, void* stream) {
  using namespace vp3d;
  AdamHyper h;
  VP3D_TRY(adam_hyper(&h, tensors, n_tensors, step, lr, beta1, beta2, eps, weight_decay));
  for (int base = 0; base < n_tensors; base += VP3D_ADAM_MAX_TENSORS) {
    AdamBatch b;
    b.n = 0;
    int blocks = 0;
    const int stop = base + VP3D_ADAM_MAX_TENSORS < n_tensors ? base + VP3D_ADAM_MAX_TENSORS : n_tensors;
    for (int i = base; i < stop; ++i) {
      const vp3d_adam_tensor& t = tensors[i];
      if (t.numel < 0) return fail(VP3D_ERR_INVALID, "vp3d_adam_step: tensor %d has numel < 0", i);
      if (t.numel == 0) continue;
      if (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq)
        return fail(VP3D_ERR_INVALID, "vp3d_adam_step: tensor %d has a null pointer", i);
      const long long nb = (t.numel + kAdamChunk - 1) / kAdamChunk;
      if (blocks + nb > 0x3fffffff)
        return fail(VP3D_ERR_UNSUPPORTED, "vp3d_adam_step: too many elements in one launch");
      b.t[b.n] = t;
      b.first_block[b.n] = blocks;
      blocks += (int)nb;
      ++b.n;
    }
    b.first_block[b.n] = blocks;
    if (blocks == 0) continue;
    adam_step_kernel<<<blocks, kAdamThreads, 0, (cudaStream_t)stream>>>(b, h);
    CUDA_TRY(cudaGetLastError());
  }
  return VP3D_OK;
}

namespace vp3d {
// Scratch layout of the loss entry points: [0] the ticket (zeroed here, before the launch),
// [1 .. blocks] the block partials.
static int mpjpe_launch(const char* who, const float* pred, const float* target,
                        const float* joint_w, int64_t joints_total, int32_t dims, float* loss,
                        float* dpred, void* scratch, size_t scratch_bytes, bool ex, void* stream) {
  if (joints_total < 0 || dims < 1 || dims > 16)
    return fail(VP3D_ERR_INVALID, "%s: bad sizes (joints %lld, dims %d)", who,
                (long long)joints_total, dims);
  if (loss == nullptr) return fail(VP3D_ERR_INVALID, "%s: null loss pointer", who);
  if (joints_total > 0 && (pred == nullptr || target == nullptr))
    return fail(VP3D_ERR_INVALID, "%s: null pointer", who);
  const long long blocks = loss_blocks(joints_total, ex);
  const size_t need = ex ? loss_scratch_bytes(joints_total) : 0;
  if (need > 0 && (scratch == nullptr || scratch_bytes < need))
    return fail(VP3D_ERR_WORKSPACE, "%s: scratch too small (%zu bytes, need %zu)", who,
                scratch_bytes, need);
  unsigned* ticket = blocks > 1 ? static_cast<unsigned*>(scratch) : nullptr;
  float* part = blocks > 1 ? static_cast<float*>(scratch) + 1 : nullptr;
  if (ticket) CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned), (cudaStream_t)stream));
  // the mean over no joints is NaN, as torch.mean of an empty tensor
  const float weight = joints_total > 0 ? (float)(1.0 / (double)joints_total) : __builtin_nanf("");
  mpjpe_kernel<<<(unsigned)blocks, kLossThreads, 0, (cudaStream_t)stream>>>(
      pred, target, joint_w, dpred, loss, part, ticket, joints_total, dims, weight);
  CUDA_TRY(cudaGetLastError());
  return VP3D_OK;
}

static int projected_launch(const char* who, const float* pos, const float* traj, const float* cam,
                            const float* target, int64_t samples, int32_t frames_per_sample,
                            int32_t joints, int32_t linear, float* loss, float* dpos, float* dtraj,
                            void* scratch, size_t scratch_bytes, bool ex, void* stream) {
  if (samples < 0 || frames_per_sample < 1 || joints < 1)
    return fail(VP3D_ERR_INVALID, "%s: bad sizes (samples %lld, frames %d, joints %d)", who,
                (long long)samples, frames_per_sample, joints);
  if (loss == nullptr) return fail(VP3D_ERR_INVALID, "%s: null loss pointer", who);
  if ((dpos == nullptr) != (dtraj == nullptr))
    return fail(VP3D_ERR_INVALID, "%s: dpos and dtraj go together", who);
  if (samples > 0 && (!pos || !traj || !cam || !target))
    return fail(VP3D_ERR_INVALID, "%s: null pointer", who);
  const long long frames_total = samples * frames_per_sample;
  const long long blocks = loss_blocks(frames_total, ex);
  const size_t need = ex ? loss_scratch_bytes(frames_total) : 0;
  if (need > 0 && (scratch == nullptr || scratch_bytes < need))
    return fail(VP3D_ERR_WORKSPACE, "%s: scratch too small (%zu bytes, need %zu)", who,
                scratch_bytes, need);
  unsigned* ticket = blocks > 1 ? static_cast<unsigned*>(scratch) : nullptr;
  float* part = blocks > 1 ? static_cast<float*>(scratch) + 1 : nullptr;
  if (ticket) CUDA_TRY(cudaMemsetAsync(ticket, 0, sizeof(unsigned), (cudaStream_t)stream));
  const float weight = frames_total > 0 ? (float)(1.0 / ((double)frames_total * joints))
                                        : __builtin_nanf("");
  projected_mpjpe_kernel<<<(unsigned)blocks, kLossThreads, 0, (cudaStream_t)stream>>>(
      pos, traj, cam, target, dpos, dtraj, loss, part, ticket, frames_total, frames_per_sample,
      joints, linear, weight);
  CUDA_TRY(cudaGetLastError());
  return VP3D_OK;
}
}  // namespace vp3d

VP3D_EXPORT size_t vp3d_mpjpe_scratch_bytes(int64_t joints_total) {
  return vp3d::loss_scratch_bytes(joints_total);
}

VP3D_EXPORT int vp3d_mpjpe_fwd_bwd_ex(const float* pred, const float* target, const float* joint_w,
                                      int64_t joints_total, int32_t dims, float* loss, float* dpred,
                                      void* scratch, size_t scratch_bytes, void* stream) {
  return vp3d::mpjpe_launch("vp3d_mpjpe_fwd_bwd_ex", pred, target, joint_w, joints_total, dims,
                            loss, dpred, scratch, scratch_bytes, true, stream);
}

VP3D_EXPORT int vp3d_mpjpe_fwd_bwd(const float* pred, const float* target, const float* joint_w,
                                   int64_t joints_total, int32_t dims, float* loss, float* dpred,
                                   void* stream) {
  return vp3d::mpjpe_launch("vp3d_mpjpe_fwd_bwd", pred, target, joint_w, joints_total, dims, loss,
                            dpred, nullptr, 0, false, stream);
}

VP3D_EXPORT size_t vp3d_projected_mpjpe_scratch_bytes(int64_t samples, int32_t frames_per_sample) {
  if (samples < 0 || frames_per_sample < 1) return 0;
  return vp3d::loss_scratch_bytes(samples * frames_per_sample);
}

VP3D_EXPORT int vp3d_projected_mpjpe_fwd_bwd_ex(const float* pos, const float* traj,
                                                const float* cam, const float* target,
                                                int64_t samples, int32_t frames_per_sample,
                                                int32_t joints, int32_t linear, float* loss,
                                                float* dpos, float* dtraj, void* scratch,
                                                size_t scratch_bytes, void* stream) {
  return vp3d::projected_launch("vp3d_projected_mpjpe_fwd_bwd_ex", pos, traj, cam, target, samples,
                                frames_per_sample, joints, linear, loss, dpos, dtraj, scratch,
                                scratch_bytes, true, stream);
}

VP3D_EXPORT int vp3d_projected_mpjpe_fwd_bwd(const float* pos, const float* traj, const float* cam,
                                             const float* target, int64_t samples,
                                             int32_t frames_per_sample, int32_t joints,
                                             int32_t linear, float* loss, float* dpos, float* dtraj,
                                             void* stream) {
  return vp3d::projected_launch("vp3d_projected_mpjpe_fwd_bwd", pos, traj, cam, target, samples,
                                frames_per_sample, joints, linear, loss, dpos, dtraj, nullptr, 0,
                                false, stream);
}
