// Int8 calibration thresholds from the activation histograms of vp3d_calibrate_int8_hist: one
// clipping threshold t per quantised tensor (the int8 plan's s = t / 255), by maximum, percentile or
// least quantisation error.  Three launches: compact the non-empty bins of every layer, evaluate the
// error of every candidate (mse only), select.  Integer counts and fixed-order fp64 sums: the same
// histogram gives the same bits on every run.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "internal.cuh"

using namespace vp3d;

namespace {

constexpr int kCompactThreads = 1024;
constexpr int kBinsPerThread = (kHistBins + kCompactThreads - 1) / kCompactThreads;
// fp16 values in [amax / 256, amax]: 8 binades of 1024 patterns and amax itself (fewer below the
// normal range, where the patterns are evenly spaced)
constexpr int kMaxCands = 8 * 1024 + 1;
constexpr int kErrThreads = 256;

struct LayerStats {
  unsigned long long n;         // counted values, zeros included
  unsigned long long invalid;   // inf / NaN values
  int m;                        // non-empty bins
  int amax_bits;                // largest non-empty bin (0 when every value is 0)
  int lo_bits;                  // mse: the first candidate, the smallest fp16 >= amax / 256
  int cands;                    // mse: candidates lo_bits .. amax_bits (0 for an all-zero layer)
};

// Scratch of `layers` layers: stats, then per layer kHistBins compacted bins (fp32 value, count as
// fp64 -- exact below 2^53 -- and the cumulative count), then kMaxCands errors.
struct Scratch {
  LayerStats* stats;
  float* val;
  double* cnt;
  unsigned long long* cum;
  double* err;
};

// carves the scratch from address base (0: only its size is wanted); returns its size
size_t scratch_layout(int layers, uintptr_t base, Scratch* s) {
  Arena a{256};
  const size_t bins = (size_t)layers * kHistBins;
  s->stats = reinterpret_cast<LayerStats*>(base + a.take(layers * sizeof(LayerStats)));
  s->val = reinterpret_cast<float*>(base + a.take(bins * sizeof(float)));
  s->cnt = reinterpret_cast<double*>(base + a.take(bins * sizeof(double)));
  s->cum = reinterpret_cast<unsigned long long*>(base + a.take(bins * sizeof(unsigned long long)));
  s->err = reinterpret_cast<double*>(base + a.take((size_t)layers * kMaxCands * sizeof(double)));
  return a.total();
}

__device__ __forceinline__ float bin_value(int bits) {
  return __half2float(__ushort_as_half((unsigned short)bits));
}

// Block-wide exclusive scan of one value per thread (kCompactThreads threads); returns the total.
template <class V>
__device__ V block_exclusive_scan(V v, V* excl, V* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  V inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const V o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    V w = s_warp[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const V o = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += o;
    }
    s_warp[lane] = w;   // inclusive over warps
  }
  __syncthreads();
  const V before = warp ? s_warp[warp - 1] : V(0);
  *excl = before + inc - v;
  const V total = s_warp[31];
  __syncthreads();
  return total;
}

// One block per layer: every thread owns kBinsPerThread consecutive bins.
__global__ void __launch_bounds__(kCompactThreads)
compact_kernel(const unsigned long long* __restrict__ hist, Scratch s, int layers) {
  __shared__ unsigned s_wm[32];
  __shared__ unsigned long long s_wc[32];
  __shared__ int s_amax;
  const int l = blockIdx.x;
  const unsigned long long* h = hist + (size_t)l * kHistBins;
  const int b0 = threadIdx.x * kBinsPerThread;
  const int b1 = min(b0 + kBinsPerThread, kHistBins);
  unsigned m = 0;
  unsigned long long c = 0;
  int top = -1;
  for (int b = b0; b < b1; ++b) {
    const unsigned long long v = h[b];
    if (v) { ++m; c += v; top = b; }
  }
  if (threadIdx.x == 0) s_amax = 0;
  unsigned m_before;
  unsigned long long c_before;
  const unsigned m_total = block_exclusive_scan(m, &m_before, s_wm);
  const unsigned long long n = block_exclusive_scan(c, &c_before, s_wc);
  if (top > 0) atomicMax(&s_amax, top);
  const size_t base = (size_t)l * kHistBins;
  for (int b = b0, j = (int)m_before; b < b1; ++b) {
    const unsigned long long v = h[b];
    if (!v) continue;
    c_before += v;
    s.val[base + j] = bin_value(b);
    s.cnt[base + j] = (double)v;
    s.cum[base + j] = c_before;
    ++j;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    LayerStats st;
    st.n = n;
    st.invalid = hist[(size_t)layers * kHistBins + l];
    st.m = (int)m_total;
    st.amax_bits = s_amax;
    st.lo_bits = 0;
    st.cands = 0;
    if (s_amax > 0) {
      // amax / 256 is exact in fp32; rounding it up to fp16 gives the smallest candidate
      st.lo_bits = __half_as_ushort(__float2half_ru(bin_value(s_amax) * 0.00390625f));
      st.cands = s_amax - st.lo_bits + 1;
    }
    s.stats[l] = st;
  }
}

// One block per (candidate, layer): E(t) = sum_b n_b (x_b - s q_b)^2 in fp64 with s = fp32(t / 255),
// inv = fp32(1 / s) (vp3d_set_int8_scales) and q_b = min(255, rint(fp32(x_b inv))) (the kernels'
// cvt.rni.sat.u8.f32).  Thread i sums bins i, i + 256, ... in order, then a fixed tree.
__global__ void __launch_bounds__(kErrThreads) mse_kernel(Scratch s) {
  __shared__ double s_sum[kErrThreads];
  const int l = blockIdx.y, k = blockIdx.x;
  const LayerStats st = s.stats[l];
  if (k >= st.cands) return;
  const float t = bin_value(st.lo_bits + k);
  const float sc = __fdiv_rn(t, 255.0f);
  const float inv = __fdiv_rn(1.0f, sc);
  const size_t base = (size_t)l * kHistBins;
  double e = 0.0;
  for (int j = threadIdx.x; j < st.m; j += kErrThreads) {
    const float x = s.val[base + j];
    const float q = fminf(rintf(__fmul_rn(x, inv)), 255.0f);
    const double d = (double)x - (double)sc * (double)q;
    e = __fma_rn(s.cnt[base + j], d * d, e);
  }
  s_sum[threadIdx.x] = e;
  __syncthreads();
#pragma unroll
  for (int w = kErrThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) s_sum[threadIdx.x] += s_sum[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) s.err[(size_t)l * kMaxCands + k] = s_sum[0];
}

// One block per layer.  NaN for a layer with invalid values: the calibration is refused.
__global__ void __launch_bounds__(kErrThreads)
select_kernel(Scratch s, int method, double pct, float* __restrict__ out) {
  __shared__ double s_e[kErrThreads];
  __shared__ int s_k[kErrThreads];
  const int l = blockIdx.x;
  const LayerStats st = s.stats[l];
  if (st.invalid) {
    if (threadIdx.x == 0) out[l] = __int_as_float(0x7fc00000);
    return;
  }
  if (st.amax_bits == 0 || method == VP3D_INT8_CALIB_AMAX) {
    if (threadIdx.x == 0) out[l] = bin_value(st.amax_bits);
    return;
  }
  const size_t base = (size_t)l * kHistBins;
  if (method == VP3D_INT8_CALIB_PERCENTILE) {
    if (threadIdx.x == 0) {
      // the smallest bin whose cumulative count reaches c = ceil(p / 100 * n) (c <= n for p <= 100)
      const double c = ceil(pct / 100.0 * (double)st.n);
      int lo = 0, hi = st.m - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((double)s.cum[base + mid] >= c) hi = mid; else lo = mid + 1;
      }
      out[l] = s.val[base + lo];
    }
    return;
  }
  // mse: the smallest error, the larger candidate on an exact tie
  double best = INFINITY;
  int best_k = -1;
  for (int k = threadIdx.x; k < st.cands; k += kErrThreads) {
    const double e = s.err[(size_t)l * kMaxCands + k];
    if (e <= best) { best = e; best_k = k; }
  }
  s_e[threadIdx.x] = best;
  s_k[threadIdx.x] = best_k;
  __syncthreads();
  for (int w = kErrThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
      const double e = s_e[threadIdx.x + w];
      const int kk = s_k[threadIdx.x + w];
      if (e < s_e[threadIdx.x] || (e == s_e[threadIdx.x] && kk > s_k[threadIdx.x])) {
        s_e[threadIdx.x] = e;
        s_k[threadIdx.x] = kk;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[l] = bin_value(st.lo_bits + s_k[0]);
}

}  // namespace

extern "C" __attribute__((visibility("default"))) size_t vp3d_int8_thresholds_scratch_bytes(int layers) {
  if (layers < 1 || layers > VP3D_MAX_LAYERS) return 0;
  Scratch s;
  return scratch_layout(layers, 0, &s);
}

extern "C" __attribute__((visibility("default"))) int vp3d_int8_thresholds(
    const uint64_t* hist, int layers, int method, double param, float* amax_out, void* scratch,
    size_t scratch_bytes, void* stream_) {
  const char* what = "int8_thresholds";
  if (!hist || !amax_out) return fail(VP3D_ERR_INVALID, "%s: null hist or amax_out", what);
  if (layers < 1 || layers > VP3D_MAX_LAYERS)
    return fail(VP3D_ERR_INVALID, "%s: layers must be in [1, %d] (got %d)", what, VP3D_MAX_LAYERS,
                layers);
  if (method != VP3D_INT8_CALIB_AMAX && method != VP3D_INT8_CALIB_PERCENTILE &&
      method != VP3D_INT8_CALIB_MSE)
    return fail(VP3D_ERR_INVALID, "%s: unknown method %d", what, method);
  if (method == VP3D_INT8_CALIB_PERCENTILE && !(param > 0.0 && param <= 100.0))
    return fail(VP3D_ERR_INVALID, "%s: percentile must be in (0, 100] (got %g)", what, param);
  if (reinterpret_cast<uintptr_t>(hist) % 8 || reinterpret_cast<uintptr_t>(amax_out) % 4)
    return fail(VP3D_ERR_INVALID, "%s: hist or amax_out misaligned", what);
  Scratch s;
  const size_t need = scratch_layout(layers, 0, &s);
  if (!scratch || scratch_bytes < need)
    return fail(VP3D_ERR_WORKSPACE, "%s: scratch too small: %zu < %zu", what, scratch_bytes, need);
  scratch_layout(layers, reinterpret_cast<uintptr_t>(ws_base(scratch, 256)), &s);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const unsigned long long* h = reinterpret_cast<const unsigned long long*>(hist);
  compact_kernel<<<layers, kCompactThreads, 0, stream>>>(h, s, layers);
  CUDA_TRY(cudaGetLastError());
  if (method == VP3D_INT8_CALIB_MSE) {
    mse_kernel<<<dim3(kMaxCands, layers), kErrThreads, 0, stream>>>(s);
    CUDA_TRY(cudaGetLastError());
  }
  select_kernel<<<layers, kErrThreads, 0, stream>>>(s, method, param, amax_out);
  CUDA_TRY(cudaGetLastError());
  return VP3D_OK;
}
