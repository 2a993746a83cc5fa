// Offline inference on a list of clips as one GEMM chain (vp3d_forward_clips): the two kernels
// around the dilated chain.  The chain itself is the offline forward's (api.cu), run as a single
// sample over the concatenation of the clips, each edge-padded as UnchunkedGenerator pads it
// (common/generators.py:216-238, run.py:186-193).
//
// Layout of one chain.  Clip i of T_i frames takes copies * P_i packed rows, P_i = T_i + RF - 1:
// copy 0 is the clip padded with pad + shift copies of frame 0 in front and pad - shift copies of
// frame T_i - 1 behind; with augment, copy 1 is the mirrored clip padded the same way
// (common/generators.py:223-237).  Output row t of the chain depends on input rows [t, t + RF - 1]
// only, so the T_i outputs that start at a copy's first row are that copy's outputs; the RF - 1
// rows after them straddle two copies and are never read.
//
// Rows to clips.  Both kernels split the chain's rows evenly over their blocks.  A block walks the
// clip table 256 clips at a time, turning the lengths into a prefix table of first rows in shared
// memory (a block-wide scan), and maps each of its rows to its clip by binary search over that
// table.  Nothing is computed on the host from device lengths, so no copy back is ever needed.
#include "internal.cuh"
#include "launch.cuh"

namespace vp3d {

namespace {

constexpr int kClipThreads = 256;

struct ClipPackArgs {
  ClipChain t;
  const float* x;        // (rows of the store, c_raw) fp32
  int c_raw, feat;       // J_in * F, F
  __nv_bfloat16* a0;     // [planes][rows][ld]
  long long plane;
  int ld, planes, f16;
  int kps[kClipMaxJoints];   // mirror source of every input joint (copy 1, augment)
};

struct ClipOutArgs {
  ClipChain t;
  const float* ybuf;     // (out_rows, c_out) fp32, the shrink rows of the chain
  long long out_rows;
  float* y;              // (rows of the output, c_out) fp32
  int c_out;
  int swap;              // augment with an output joint map (else negate x only)
  int jsrc[kClipMaxJoints];
};

// packed rows of clip c: copies * (T + RF - 1), lengths below 1 read as 1
__device__ __forceinline__ long long clip_rows(const ClipChain& t, int c) {
  return (long long)t.copies * (max(__ldg(t.len + c), 1) + t.rf - 1);
}

// Block-wide: the prefix table of clips [c0, c0 + n), n = min(256, clips - c0), whose first clip
// starts at packed row `base`: s_row[k] = first row of clip c0 + k, s_row[n] = the end of the last.
// Returns n.  Every thread of the block must call it (it synchronises).
__device__ int scan_clips(const ClipChain& t, int c0, long long base, long long* s_row,
                          long long* s_warp) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __syncthreads();   // the previous chunk's table is no longer read
  long long v = c0 + tid < t.clips ? clip_rows(t, c0 + tid) : 0;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  long long pre = base;
  for (int w = 0; w < warp; ++w) pre += s_warp[w];
  s_row[tid + 1] = pre + v;
  if (tid == 0) s_row[0] = base;
  __syncthreads();
  return min(kClipThreads, t.clips - c0);
}

// the last k in [0, n) with s_row[k] <= row (s_row[0] <= row < s_row[n])
__device__ __forceinline__ int find_clip(const long long* s_row, int n, long long row) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (s_row[mid] <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// rows [r0, r1) of `total`, block b's even share
__device__ __forceinline__ void block_rows(long long total, long long* r0, long long* r1) {
  const long long per = (total + gridDim.x - 1) / gridDim.x;
  *r0 = min(total, (long long)blockIdx.x * per);
  *r1 = min(total, *r0 + per);
}

// The chain's input: every packed row [0, rows) that belongs to a clip, channel-last 16-bit with
// zeroed pad channels (the hi / lo planes for bf16x3), rounded by to_bits16 as the offline input
// pack rounds.  Frame f of a copy's row r is clamp(r - front, 0, T - 1): the generator's edge
// padding.  The mirrored copy negates feature 0 and reads input joint j from kps[j].
__global__ void __launch_bounds__(kClipThreads) clip_pack_kernel(const __grid_constant__ ClipPackArgs a) {
  __shared__ long long s_row[kClipThreads + 1];
  __shared__ long long s_warp[kClipThreads / 32];
  const ClipChain& t = a.t;
  long long r0, r1;
  block_rows(t.rows, &r0, &r1);
  const int pairs = a.ld >> 1;
  long long base = 0;
  for (int c0 = 0; c0 < t.clips && base < r1; c0 += kClipThreads) {
    const int n = scan_clips(t, c0, base, s_row, s_warp);
    const long long lo = max(r0, base), hi = min(r1, s_row[n]);
    base = s_row[n];
    const long long items = hi > lo ? (hi - lo) * pairs : 0;
    for (long long i = threadIdx.x; i < items; i += kClipThreads) {
      const long long row = lo + i / pairs;
      const int cp = (int)(i % pairs);
      const int k = find_clip(s_row, n, row);
      const int c = c0 + k;
      const long long P = (s_row[k + 1] - s_row[k]) / t.copies;
      const long long within = row - s_row[k];
      const bool mirrored = within >= P;
      const int T = (int)(P - t.rf + 1);
      const long long f = min(max(within - (mirrored ? P : 0) - t.front, 0ll), (long long)T - 1);
      const float* src = a.x + (__ldg(t.first + c) + f) * a.c_raw;
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ch = 2 * cp + h;
        v[h] = 0.0f;
        if (ch < a.c_raw) {
          if (mirrored) {
            const int j = ch / a.feat, e = ch - j * a.feat;
            const float s = __ldg(src + a.kps[j] * a.feat + e);
            v[h] = e == 0 ? -s : s;
          } else {
            v[h] = __ldg(src + ch);
          }
        }
      }
      const Bits16 b0 = to_bits16(v[0], a.f16), b1 = to_bits16(v[1], a.f16);
      __nv_bfloat16* dst = a.a0 + row * a.ld + 2 * cp;
      *reinterpret_cast<__nv_bfloat162*>(dst) = __halves2bfloat162(b0.hi, b1.hi);
      if (a.planes == 2)
        *reinterpret_cast<__nv_bfloat162*>(dst + a.plane) = __halves2bfloat162(b0.lo, b1.lo);
    }
  }
}

// Each clip's T valid output rows: chain row first + t (copy 0) to y row y_first + t; with augment
// the flip average (run.py:677-680) of rows first + t and first + P + t (copy 1), output joint j of
// the mirrored copy read from jsrc[j] (no map: the trajectory model, negate x only).
__global__ void __launch_bounds__(kClipThreads) clip_output_kernel(const __grid_constant__ ClipOutArgs a) {
  pdl_entry();
  __shared__ long long s_row[kClipThreads + 1];
  __shared__ long long s_warp[kClipThreads / 32];
  const ClipChain& t = a.t;
  long long r0, r1;
  block_rows(a.out_rows, &r0, &r1);
  long long base = 0;
  for (int c0 = 0; c0 < t.clips && base < r1; c0 += kClipThreads) {
    const int n = scan_clips(t, c0, base, s_row, s_warp);
    const long long lo = max(r0, base), hi = min(r1, s_row[n]);
    base = s_row[n];
    const long long items = hi > lo ? (hi - lo) * a.c_out : 0;
    for (long long i = threadIdx.x; i < items; i += kClipThreads) {
      const long long row = lo + i / a.c_out;
      const int ch = (int)(i % a.c_out);
      const int k = find_clip(s_row, n, row);
      const long long P = (s_row[k + 1] - s_row[k]) / t.copies;
      const long long tt = row - s_row[k];
      if (tt >= P - t.rf + 1) continue;   // padding rows, or the mirrored copy's
      const float* row0 = a.ybuf + row * a.c_out;
      float v = row0[ch];
      if (t.copies == 2) {
        if (row + P >= a.out_rows) continue;   // rows past a short `rows` (a caller error)
        const int j = ch / 3, e = ch - 3 * j;
        const int js = a.swap ? a.jsrc[j] : j;
        v = flip_average(v, row0[P * a.c_out + js * 3 + e], e);
      }
      a.y[(__ldg(t.y_first + c0 + k) + tt) * a.c_out + ch] = v;
    }
  }
}

int clip_grid(long long rows) {
  // at least 64 rows per block: every block scans the clip table up to its rows
  long long b = (rows + 63) / 64;
  const long long cap = 2LL * num_sms();
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

}  // namespace

cudaError_t launch_clip_pack(const ClipChain& t, const float* x, int c_raw, int feat, const int* kps,
                             __nv_bfloat16* a0, int ld, int planes, long long plane, int f16,
                             cudaStream_t stream) {
  ClipPackArgs a;
  memset(&a, 0, sizeof(a));
  a.t = t;
  a.x = x;
  a.c_raw = c_raw;
  a.feat = feat;
  a.a0 = a0;
  a.plane = plane;
  a.ld = ld;
  a.planes = planes;
  a.f16 = f16;
  if (kps) memcpy(a.kps, kps, (size_t)(c_raw / feat) * sizeof(int));
  // (a plain launch, as the offline input pack: the first kernel of the chain)
  clip_pack_kernel<<<clip_grid(t.rows), kClipThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_clip_output(const ClipChain& t, const float* ybuf, long long out_rows, int c_out,
                               const int* jsrc, float* y, cudaStream_t stream) {
  ClipOutArgs a;
  memset(&a, 0, sizeof(a));
  a.t = t;
  a.ybuf = ybuf;
  a.out_rows = out_rows;
  a.y = y;
  a.c_out = c_out;
  a.swap = jsrc != nullptr;
  if (jsrc) memcpy(a.jsrc, jsrc, (size_t)(c_out / 3) * sizeof(int));
  return launch_pdl(clip_output_kernel, dim3(clip_grid(out_rows)), dim3(kClipThreads), 0, stream, a);
}

}  // namespace vp3d
