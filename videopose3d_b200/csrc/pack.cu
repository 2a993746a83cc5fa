#include "pack.cuh"

#include "conv_gemm.cuh"   // kMaxDevices
#include "ptx.cuh"         // quant_u8

#include <string.h>

#include <stdint.h>

namespace vp3d {

// Rows are walked in SOURCE order (sample, then frame group) so that the fp32 read is one
// sequential stream; the scattered side (tap-major row order) is the 16-bit output, which stays in
// L2 for the expand GEMM.  A block owns a chunk of at most kPackRows consecutive rows of one sample:
// the row -> output-row map of the chunk (up to eight integer divisions per row) is computed once
// into shared memory, then every warp converts whole rows -- lanes stride over the element pairs
// with 8-byte loads and 4-byte stores, two rows in flight per warp.
constexpr int kPackRows = 96;

template <bool VEC2>
__device__ __forceinline__ void pack_load_pair(const float* src, int k, int k_valid, float& v0,
                                               float& v1) {
  v0 = 0.0f;
  v1 = 0.0f;
  if (VEC2) {   // c_raw even and x 8-byte aligned: k_valid is even too
    if (k < k_valid) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(src + k));
      v0 = v.x;
      v1 = v.y;
    }
  } else {
    if (k < k_valid) v0 = __ldg(src + k);
    if (k + 1 < k_valid) v1 = __ldg(src + k + 1);
  }
}

__device__ __forceinline__ void pack_store_pair(__nv_bfloat16* dst, long long plane_stride, int planes,
                                                int f16, float v0, float v1) {
  const Bits16 b0 = to_bits16(v0, f16), b1 = to_bits16(v1, f16);
  *reinterpret_cast<__nv_bfloat162*>(dst) = __halves2bfloat162(b0.hi, b1.hi);
  if (planes == 2) *reinterpret_cast<__nv_bfloat162*>(dst + plane_stride) = __halves2bfloat162(b0.lo, b1.lo);
}

template <bool VEC2>
__global__ void __launch_bounds__(256)
pack_input_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int planes, int N,
                  int T, int c_raw, int rows, int group, int frame_step, int k_pad,
                  long long plane_stride, const PackPerm perm, int f16) {
  __shared__ long long s_row[kPackRows];
  const int chunks = (rows + kPackRows - 1) / kPackRows;
  const long long items = (long long)N * chunks;
  const int k_valid = group * c_raw;
  const int pairs = k_pad >> 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long item = blockIdx.x; item < items; item += gridDim.x) {
    const long long n = item / chunks;
    const int r0 = (int)(item - n * chunks) * kPackRows;
    const int nr = min(kPackRows, rows - r0);
    __syncthreads();   // the previous chunk's map is no longer read
    if ((int)threadIdx.x < nr) {
      const int r = r0 + (int)threadIdx.x;
      // output row: natural order n*rows + r, or the tap-major position (pack.cuh): peel one tap
      // digit per block, innermost frame digit first
      long long row;
      if (perm.levels == 0) {
        row = n * rows + r;
      } else {
        unsigned t = (unsigned)r;
        row = 0;
        for (int lv = 0; lv < perm.levels; ++lv) {
          const unsigned w = (unsigned)perm.width[lv];
          const unsigned q = t / w;
          row += (long long)(t - q * w) * perm.region[lv];
          t = q;
        }
        row += n * perm.last_rows + t;
      }
      s_row[threadIdx.x] = row;
    }
    __syncthreads();
    const float* src0 = x + (n * T + (long long)r0 * frame_step) * c_raw;
    const long long src_step = (long long)frame_step * c_raw;
    for (int rl = warp * 2; rl < nr; rl += 16) {   // 8 warps x 2 rows
      const bool two = rl + 1 < nr;
      const float* sa = src0 + rl * src_step;
      const float* sb = sa + src_step;
      __nv_bfloat16* da = out + s_row[rl] * k_pad;
      __nv_bfloat16* db = out + s_row[two ? rl + 1 : rl] * k_pad;
      for (int c = lane; c < pairs; c += 64) {
        const int c2 = c + 32;
        float a0, a1, a2, a3, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
        pack_load_pair<VEC2>(sa, 2 * c, k_valid, a0, a1);
        pack_load_pair<VEC2>(sa, 2 * c2, c2 < pairs ? k_valid : 0, a2, a3);
        if (two) {
          pack_load_pair<VEC2>(sb, 2 * c, k_valid, b0, b1);
          pack_load_pair<VEC2>(sb, 2 * c2, c2 < pairs ? k_valid : 0, b2, b3);
        }
        pack_store_pair(da + 2 * c, plane_stride, planes, f16, a0, a1);
        if (c2 < pairs) pack_store_pair(da + 2 * c2, plane_stride, planes, f16, a2, a3);
        if (two) {
          pack_store_pair(db + 2 * c, plane_stride, planes, f16, b0, b1);
          if (c2 < pairs) pack_store_pair(db + 2 * c2, plane_stride, planes, f16, b2, b3);
        }
      }
    }
  }
}

cudaError_t launch_pack_input(const float* x, __nv_bfloat16* out, int planes, int N, int T,
                              int c_raw, int rows, int group, int frame_step, int k_pad,
                              long long plane_stride, cudaStream_t stream, const PackPerm* perm,
                              int f16) {
  PackPerm pp;
  memset(&pp, 0, sizeof(pp));
  if (perm) pp = *perm;
  if (k_pad % 8) return cudaErrorInvalidValue;
  if (N <= 0 || rows <= 0) return cudaSuccess;
  const long long items = (long long)N * ((rows + kPackRows - 1) / kPackRows);
  long long blocks = items;
  if (blocks > 132 * 8) blocks = 132 * 8;
  const bool vec2 = (c_raw % 2 == 0) && (reinterpret_cast<uintptr_t>(x) % 8 == 0);
  // (a plain launch: the input pack is the first kernel of a forward and usually follows a copy or
  // an event wait, where a programmatic edge buys nothing)
  if (vec2)
    pack_input_kernel<true><<<(int)blocks, 256, 0, stream>>>(
        x, out, planes, N, T, c_raw, rows, group, frame_step, k_pad, plane_stride, pp, f16);
  else
    pack_input_kernel<false><<<(int)blocks, 256, 0, stream>>>(
        x, out, planes, N, T, c_raw, rows, group, frame_step, k_pad, plane_stride, pp, f16);
  return cudaGetLastError();
}

// One thread per (co, k) position of the padded slab; the thread walks the taps, so the fp32 reads of
// a warp cover one contiguous span of Conv1d.weight and each tap slab receives a coalesced bf16 row.
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out,
                                        int planes, int c_out, int c_in, int taps, int n_pad,
                                        int k_pad, int merged, int f16) {
  const long long slab = (long long)n_pad * k_pad;
  const long long plane_elems = (merged ? 1 : taps) * slab;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < slab;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % k_pad);
    const int co = (int)(i / k_pad);
    if (merged) {
      float v = 0.0f;
      if (co < c_out && k < taps * c_in) {
        const int tap = k / c_in, ci = k - tap * c_in;
        v = __ldg(w + ((long long)co * c_in + ci) * taps + tap);
      }
      store_bits16(out, i, plane_elems, planes, v, f16);
    } else {
      const bool in = co < c_out && k < c_in;
      const float* src = w + ((long long)co * c_in + k) * taps;
      for (int tap = 0; tap < taps; ++tap)
        store_bits16(out, tap * slab + i, plane_elems, planes, in ? __ldg(src + tap) : 0.0f, f16);
    }
  }
}

cudaError_t launch_pack_conv_weight(const float* w, __nv_bfloat16* out, int planes, int c_out,
                                    int c_in, int taps, int n_pad, int k_pad, int merge_taps,
                                    cudaStream_t stream, int f16) {
  const long long total = (long long)n_pad * k_pad;
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  pack_conv_weight_kernel<<<(int)blocks, threads, 0, stream>>>(w, out, planes, c_out, c_in, taps,
                                                               n_pad, k_pad, merge_taps, f16);
  return cudaGetLastError();
}

// one block per output channel: the channel's |w| maximum, then its s8 row of every tap
__global__ void __launch_bounds__(256)
pack_conv_weight_s8_kernel(const float* __restrict__ w, int8_t* __restrict__ out,
                           float* __restrict__ w_scale, int c_out, int c_in, int taps, int n_pad,
                           int k_pad) {
  __shared__ float s_max[8];
  const int co = blockIdx.x;
  const float* src = w + (long long)co * c_in * taps;
  const int n = co < c_out ? c_in * taps : 0;
  float m = 0.0f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(__ldg(src + i)));
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0.0f;
  for (int i = 0; i < 8; ++i) m = fmaxf(m, s_max[i]);
  const float s = m > 0.0f ? __fdiv_rn(m, 127.0f) : 1.0f;
  if (threadIdx.x == 0) w_scale[co] = s;
  for (int tap = 0; tap < taps; ++tap) {
    int8_t* row = out + ((long long)tap * n_pad + co) * k_pad;
    for (int k = threadIdx.x; k < k_pad; k += blockDim.x) {
      float q = 0.0f;
      if (k < c_in && co < c_out)
        q = fminf(fmaxf(rintf(__fdiv_rn(__ldg(src + (long long)k * taps + tap), s)), -127.0f), 127.0f);
      row[k] = (int8_t)(int)q;
    }
  }
}

cudaError_t launch_pack_conv_weight_s8(const float* w, int8_t* out, float* w_scale, int c_out,
                                       int c_in, int taps, int n_pad, int k_pad,
                                       cudaStream_t stream) {
  pack_conv_weight_s8_kernel<<<n_pad, 256, 0, stream>>>(w, out, w_scale, c_out, c_in, taps, n_pad,
                                                        k_pad);
  return cudaGetLastError();
}

__global__ void int8_fold_kernel(const float* __restrict__ bn_scale, const float* __restrict__ w_scale,
                                 float s_in, float* __restrict__ q_scale, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) q_scale[i] = __fmul_rn(bn_scale[i], __fmul_rn(w_scale[i], s_in));
}

cudaError_t launch_int8_fold(const float* bn_scale, const float* w_scale, float s_in, float* q_scale,
                             int n, cudaStream_t stream) {
  int8_fold_kernel<<<(n + 255) / 256, 256, 0, stream>>>(bn_scale, w_scale, s_in, q_scale, n);
  return cudaGetLastError();
}

// fp16 bits of values >= 0 order like the values; -0 (0x8000) is mapped to 0
__global__ void __launch_bounds__(256)
amax_f16_kernel(const uint4* __restrict__ x, long long n8, unsigned* __restrict__ amax_bits) {
  __shared__ unsigned s_max[8];
  unsigned m = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(x + i);
    const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const unsigned lo = u[k] & 0xFFFFu, hi = u[k] >> 16;
      m = max(m, (lo & 0x8000u) ? 0u : lo);
      m = max(m, (hi & 0x8000u) ? 0u : hi);
    }
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) m = max(m, s_max[i]);
    const float f = __half2float(__ushort_as_half((unsigned short)m));
    atomicMax(amax_bits, __float_as_uint(f));
  }
}

cudaError_t launch_amax_f16(const void* x, long long n, unsigned* amax_bits, cudaStream_t stream) {
  if (n % 8 || reinterpret_cast<uintptr_t>(x) % 16) return cudaErrorInvalidValue;
  const long long n8 = n / 8;
  if (n8 == 0) return cudaSuccess;
  long long blocks = (n8 + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  amax_f16_kernel<<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), n8, amax_bits);
  return cudaGetLastError();
}

// Every block counts its share of the plane into a private u32 histogram in shared memory and adds
// the non-empty bins to the u64 one.  Zeros (half or more of post-ReLU activations) would serialise
// on one shared bin: they are counted in registers and added once per warp, like the invalid ones.
// Vector i holds channels 8 * (i mod c8) .. + 7 of its row; the column is stepped, not divided.
constexpr int kHistThreads = 1024;
constexpr int kHistMinVecs = 8 * kHistThreads;   // vectors per block below which fewer blocks run

__global__ void __launch_bounds__(kHistThreads)
hist_f16_kernel(const uint4* __restrict__ x, long long n8, int c8, int c_real,
                unsigned long long* __restrict__ hist, unsigned long long* __restrict__ invalid) {
  extern __shared__ unsigned s_hist[];
  for (int b = threadIdx.x; b < kHistBins; b += blockDim.x) s_hist[b] = 0;
  __syncthreads();
  unsigned zeros = 0, bad = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  int col = (int)(i % c8);
  const int col_step = (int)(stride % c8);
  for (; i < n8; i += stride) {
    const int valid = c_real - 8 * col;   // real channels in this vector (<= 0: all padding)
    if (valid > 0) {
      const uint4 v = __ldg(x + i);
      const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (k < valid) {
          const unsigned h = (u[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
          if (h == 0u || (h & 0x8000u)) ++zeros;   // what cvt.rni.sat.u8 makes 0
          else if (h >= (unsigned)kHistBins) ++bad;   // inf, NaN
          else atomicAdd(&s_hist[h], 1u);
        }
      }
    }
    col += col_step;
    if (col >= c8) col -= c8;
  }
  zeros = __reduce_add_sync(0xffffffffu, zeros);
  bad = __reduce_add_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    if (zeros) atomicAdd(&s_hist[0], zeros);
    if (bad) atomicAdd(invalid, (unsigned long long)bad);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kHistBins; b += blockDim.x)
    if (s_hist[b]) atomicAdd(hist + b, (unsigned long long)s_hist[b]);
}

cudaError_t launch_hist_f16(const void* x, long long rows, int ld, int c_real, unsigned long long* hist,
                            unsigned long long* invalid, int num_sms, cudaStream_t stream) {
  if (ld % 8 || c_real < 1 || c_real > ld || rows < 0 || reinterpret_cast<uintptr_t>(x) % 16)
    return cudaErrorInvalidValue;
  const long long n8 = rows * (ld / 8);
  if (n8 == 0) return cudaSuccess;
  // A block counts at most 8 * kHistThreads * ceil(n8 / (blocks * kHistThreads)) < 8 * n8 / blocks
  // + 8 * kHistThreads elements per launch; with blocks >= 8 * n8 / 2^31 that is below 2^31 + 2^13,
  // so no u32 shared bin (nor a thread's or a warp's register count) can wrap.
  long long blocks = (n8 + kHistMinVecs - 1) / kHistMinVecs;
  if (blocks > num_sms) blocks = num_sms;
  const long long floor_blocks = (8 * n8 + (1LL << 31) - 1) >> 31;
  if (blocks < floor_blocks) blocks = floor_blocks;
  if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
  const size_t smem = kHistBins * sizeof(unsigned);
  // the dynamic shared memory opt-in is a per-device attribute
  static bool attr_set[kMaxDevices] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  if (!attr_set[dev]) {
    e = cudaFuncSetAttribute(hist_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  hist_f16_kernel<<<(int)blocks, kHistThreads, smem, stream>>>(reinterpret_cast<const uint4*>(x), n8,
                                                               ld / 8, c_real, hist, invalid);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
count_nonfinite_kernel(const float* __restrict__ x, long long n, unsigned long long* __restrict__ count) {
  unsigned c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    c += (__float_as_uint(__ldg(x + i)) & 0x7f800000u) == 0x7f800000u;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

cudaError_t launch_count_nonfinite(const float* x, long long n, unsigned long long* count,
                                   int num_sms, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  long long blocks = (n + 255) / 256;
  if (blocks > 8LL * num_sms) blocks = 8LL * num_sms;
  count_nonfinite_kernel<<<(int)blocks, 256, 0, stream>>>(x, n, count);
  return cudaGetLastError();
}

// One 16-byte vector (8 fp16 values of one row) per thread and step; vector i holds channels
// 8 * (i mod c8) .. + 7, the column stepped as in hist_f16_kernel.
__global__ void __launch_bounds__(256)
quantize_u8_kernel(const uint4* __restrict__ x, uint2* __restrict__ q, long long n8, int c8,
                   int c_real, float inv_s) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  int col = (int)(i % c8);
  const int col_step = (int)(stride % c8);
  for (; i < n8; i += stride) {
    const int valid = c_real - 8 * col;   // real channels in this vector
    uint32_t b[2] = {0u, 0u};
    if (valid > 0) {
      const uint4 v = __ldg(x + i);
      const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float f = __half2float(__ushort_as_half((unsigned short)(u[k >> 1] >> (16 * (k & 1)))));
        if (k < valid) b[k >> 2] |= quant_u8(f, inv_s) << (8 * (k & 3));
      }
    }
    q[i] = make_uint2(b[0], b[1]);
    col += col_step;
    if (col >= c8) col -= c8;
  }
}

cudaError_t launch_quantize_u8(const void* x, uint8_t* q, long long rows, int ld, int c_real,
                               float inv_s, int num_sms, cudaStream_t stream) {
  if (ld % 8 || c_real < 1 || c_real > ld || rows < 0 || reinterpret_cast<uintptr_t>(x) % 16 ||
      reinterpret_cast<uintptr_t>(q) % 8)
    return cudaErrorInvalidValue;
  const long long n8 = rows * (ld / 8);
  if (n8 == 0) return cudaSuccess;
  long long blocks = (n8 + 255) / 256;
  if (blocks > 8LL * num_sms) blocks = 8LL * num_sms;
  quantize_u8_kernel<<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(x),
                                                      reinterpret_cast<uint2*>(q), n8, ld / 8,
                                                      c_real, inv_s);
  return cudaGetLastError();
}

__global__ void bn_fold_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ mean, const float* __restrict__ var,
                               float eps, float* __restrict__ scale, float* __restrict__ shift,
                               int c, int c_pad, float* __restrict__ mean_out,
                               float* __restrict__ invstd_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c_pad) return;
  float s = 0.0f, b = 0.0f;
  if (i < c) {
    s = gamma[i] / sqrtf(var[i] + eps);
    b = beta[i] - mean[i] * s;
  }
  scale[i] = s;
  shift[i] = b;
  if (mean_out) {
    mean_out[i] = i < c ? mean[i] : 0.0f;
    invstd_out[i] = i < c ? 1.0f / sqrtf(var[i] + eps) : 0.0f;
  }
}

cudaError_t launch_bn_fold(const float* gamma, const float* beta, const float* mean,
                           const float* var, float eps, float* scale, float* shift, int c,
                           int c_pad, cudaStream_t stream, float* mean_out, float* invstd_out) {
  bn_fold_kernel<<<(c_pad + 255) / 256, 256, 0, stream>>>(gamma, beta, mean, var, eps, scale, shift,
                                                          c, c_pad, mean_out, invstd_out);
  return cudaGetLastError();
}

__global__ void bias_affine_kernel(const float* __restrict__ bias, float* __restrict__ scale,
                                   float* __restrict__ shift, int c, int c_pad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c_pad) return;
  scale[i] = (i < c) ? 1.0f : 0.0f;
  shift[i] = (i < c) ? bias[i] : 0.0f;
}

cudaError_t launch_bias_affine(const float* bias, float* scale, float* shift, int c, int c_pad,
                               cudaStream_t stream) {
  bias_affine_kernel<<<(c_pad + 255) / 256, 256, 0, stream>>>(bias, scale, shift, c, c_pad);
  return cudaGetLastError();
}

}  // namespace vp3d
