#include "train_ops.cuh"

#include "launch.cuh"
#include "pack.cuh"

namespace vp3d {

namespace {

__device__ __forceinline__ float bf_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// 8 consecutive channels of one row, summed over the hi/lo planes.
__device__ __forceinline__ void load8(const __nv_bfloat16* p, long long plane, int planes,
                                      float (&v)[8]) {
  uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  v[0] = bf_lo(u.x); v[1] = bf_hi(u.x); v[2] = bf_lo(u.y); v[3] = bf_hi(u.y);
  v[4] = bf_lo(u.z); v[5] = bf_hi(u.z); v[6] = bf_lo(u.w); v[7] = bf_hi(u.w);
  if (planes == 2) {
    u = __ldg(reinterpret_cast<const uint4*>(p + plane));
    v[0] += bf_lo(u.x); v[1] += bf_hi(u.x); v[2] += bf_lo(u.y); v[3] += bf_hi(u.y);
    v[4] += bf_lo(u.z); v[5] += bf_hi(u.z); v[6] += bf_lo(u.w); v[7] += bf_hi(u.w);
  }
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
  v[0] = bf_lo(u.x); v[1] = bf_hi(u.x); v[2] = bf_lo(u.y); v[3] = bf_hi(u.y);
  v[4] = bf_lo(u.z); v[5] = bf_hi(u.z); v[6] = bf_lo(u.w); v[7] = bf_hi(u.w);
}

__device__ __forceinline__ void store8(__nv_bfloat16* p, long long plane, int planes,
                                       const float (&v)[8]) {
  uint32_t h[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = pack2(v[2 * j], v[2 * j + 1]);
  *reinterpret_cast<uint4*>(p) = make_uint4(h[0], h[1], h[2], h[3]);
  if (planes == 2) {
    uint32_t l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      l[j] = pack2(v[2 * j] - bf_lo(h[j]), v[2 * j + 1] - bf_hi(h[j]));
    *reinterpret_cast<uint4*>(p + plane) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// Counter-based dropout mask: one 32-bit mix per pair of elements, 16 random bits per element.
// keep <=> u16 >= p * 65536.  Forward and backward call this with the same (seed, layer, element).
__device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
__device__ __forceinline__ void dropout_keep8(const DropoutCfg& d, long long elem0, uint32_t thresh,
                                              float inv_keep, float (&m)[8]) {
  // one murmur3 finaliser per pair over a Weyl sequence of the pair index, keyed by
  // (seed, layer): ~9 integer ops per two elements keeps these passes bandwidth-bound
  const unsigned long long pair0 = (unsigned long long)elem0 >> 1;
  const uint32_t key = d.seed_lo ^ (d.seed_hi * 0x7F4A7C15u) ^ (d.layer * 0x632BE5ABu) ^
                       ((uint32_t)(pair0 >> 32) * 0x85EBCA77u);
  const uint32_t base = (uint32_t)pair0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t h = mix32((base + j) * 0x9E3779B1u + key);
    m[2 * j] = ((h & 0xFFFFu) >= thresh) ? inv_keep : 0.0f;
    m[2 * j + 1] = ((h >> 16) >= thresh) ? inv_keep : 0.0f;
  }
}

// ---------------------------------------------------------------------------------------------
// Ordered (run-to-run reproducible) per-channel reductions over slab partials.
// Grid = (channel groups of 32, S splits); 256 threads = 8 warps, lane = channel inside the group.
// Warp w of split y walks the partials p = y*8 + w, y*8 + w + 8S, ... in ascending order; the 8
// warps are then merged in warp order through shared memory; with S > 1 every block writes its
// result to `scratch` and the block that arrives last (ticket counter) merges the S results in
// split order and produces the output.  Nothing depends on timing, so a given shape always sums
// in the same order.
// ---------------------------------------------------------------------------------------------
struct SlabGeom {     // rows covered by slab s of a conv GEMM's row tiling (4 slabs per 128-row tile)
  int dilated;        // 1: per-sample tiles
  int out_rows;       // dilated: rows per sample; flat: total rows
  int tiles_per_sample;
};
__device__ __forceinline__ int slab_count(const SlabGeom& g, int s) {
  int tile = s >> 2;
  if (g.dilated) tile %= g.tiles_per_sample;
  const int row0 = tile * 128 + (s & 3) * 32;
  const int left = g.out_rows - row0;
  return left <= 0 ? 0 : (left < 32 ? left : 32);
}

struct Moments { float n, mean, m2; };
__device__ __forceinline__ void merge(Moments& a, const Moments& b) {  // Chan et al., ordered
  if (b.n <= 0.0f) return;
  if (a.n <= 0.0f) { a = b; return; }
  const float n = a.n + b.n;
  const float d = b.mean - a.mean;
  const float f = b.n / n;
  a.mean = fmaf(d, f, a.mean);
  a.m2 = a.m2 + b.m2 + d * d * a.n * f;
  a.n = n;
}

__device__ __forceinline__ bool last_block_of_group(unsigned* counter, int splits) {
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(counter + blockIdx.x, 1u);
    is_last = (t == (unsigned)splits - 1u);
    if (is_last) counter[blockIdx.x] = 0;   // self-resetting: ready for the next launch
  }
  __syncthreads();
  return is_last;
}

// Batch moments of channel ch -> scale, shift, mean, invstd and the running-statistics update
// (unbiased variance over acc.n rows).  The one epilogue of the local and the rank-merged finalize.
__device__ __forceinline__ void bn_finalize_channel(const Moments& acc, int ch, int c_real,
                                                    const float* gamma, const float* beta,
                                                    float* running_mean, float* running_var,
                                                    float momentum, float eps, float* scale,
                                                    float* shift, float* mean_out, float* invstd) {
  if (ch >= c_real) {   // padding channel (channels not a multiple of 64): identically zero
    scale[ch] = 0.0f; shift[ch] = 0.0f; mean_out[ch] = 0.0f; invstd[ch] = 0.0f;
    return;
  }
  const double n = (double)acc.n;
  const double m = (double)acc.mean;
  double var = n > 0.0 ? (double)acc.m2 / n : 0.0;
  if (var < 0.0) var = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = gamma[ch] * is;
  scale[ch] = sc;
  shift[ch] = beta[ch] - (float)m * sc;
  mean_out[ch] = (float)m;
  invstd[ch] = is;
  if (running_mean) {
    const double unbiased = n > 1.0 ? var * n / (n - 1.0) : var;
    running_mean[ch] = (float)((1.0 - momentum) * running_mean[ch] + momentum * m);
    running_var[ch] = (float)((1.0 - momentum) * running_var[ch] + momentum * unbiased);
  }
}

// moments != null (synchronized BatchNorm): instead of finalizing, store this rank's (n, mean, M2)
// into slot `rank` of moments [world][3][c] and zeros into every other slot.
__global__ void __launch_bounds__(256)
bn_stats_finalize_kernel(const float* __restrict__ part, int slabs, SlabGeom geom, int c,
                         int c_real, const float* __restrict__ gamma, const float* __restrict__ beta,
                         float* __restrict__ running_mean, float* __restrict__ running_var,
                         float momentum, float eps, float* __restrict__ scale,
                         float* __restrict__ shift, float* __restrict__ mean_out,
                         float* __restrict__ invstd, float* __restrict__ scratch,
                         unsigned* __restrict__ counter, float* __restrict__ moments, int world,
                         int rank) {
  pdl_entry();
  __shared__ float sm[8][3][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int ch = blockIdx.x * 32 + lane;
  const int S = gridDim.y;
  const bool live = ch < c;
  Moments acc = {0.0f, 0.0f, 0.0f};
  // warp w of split y owns the contiguous slab range [lo, hi): loads go out eight slabs at a time
  // (16 independent requests in flight), the merge stays in ascending slab order
  const int per = (slabs + 8 * S - 1) / (8 * S);
  const int lo = (blockIdx.y * 8 + w) * per;
  const int hi = min(slabs, lo + per);
  for (int s0 = lo; s0 < hi; s0 += 8) {
    float sum[8], sq[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int s = s0 + u;
      const bool ok = live && s < hi;
      sum[u] = ok ? __ldg(part + ((size_t)s * 2) * c + ch) : 0.0f;
      sq[u] = ok ? __ldg(part + ((size_t)s * 2 + 1) * c + ch) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int s = s0 + u;
      const int cnt = s < hi ? slab_count(geom, s) : 0;
      Moments b;
      b.n = (float)cnt;
      b.mean = cnt > 0 ? sum[u] / b.n : 0.0f;
      b.m2 = fmaxf(fmaf(-sum[u], b.mean, sq[u]), 0.0f);   // sum (x - mean)^2 inside the 32-row slab
      merge(acc, b);
    }
  }
  sm[w][0][lane] = acc.n; sm[w][1][lane] = acc.mean; sm[w][2][lane] = acc.m2;
  __syncthreads();
  if (w == 0) {
    acc = {sm[0][0][lane], sm[0][1][lane], sm[0][2][lane]};
    for (int k = 1; k < 8; ++k) merge(acc, Moments{sm[k][0][lane], sm[k][1][lane], sm[k][2][lane]});
    if (S > 1 && live) {
      float* o = scratch + ((size_t)blockIdx.y * 3) * c + ch;
      o[0] = acc.n; o[c] = acc.mean; o[2 * (size_t)c] = acc.m2;
    }
  }
  if (S > 1) {
    if (!last_block_of_group(counter, S)) return;
    // the last block merges the S results: warp w takes splits [w * S/8, ...) in order, then the
    // warps in order -- the same fixed tree every time
    acc = {0.0f, 0.0f, 0.0f};
    const int per2 = (S + 7) / 8;
    float n_[4], m_[4], q_[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int y = w * per2 + u;
      const bool ok = live && u < per2 && y < S;
      const float* o = scratch + ((size_t)(ok ? y : 0) * 3) * c + (live ? ch : 0);
      n_[u] = ok ? __ldcg(o) : 0.0f;
      m_[u] = ok ? __ldcg(o + c) : 0.0f;
      q_[u] = ok ? __ldcg(o + 2 * (size_t)c) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) merge(acc, Moments{n_[u], m_[u], q_[u]});
    __syncthreads();
    sm[w][0][lane] = acc.n; sm[w][1][lane] = acc.mean; sm[w][2][lane] = acc.m2;
    __syncthreads();
    if (w != 0) return;
    acc = {sm[0][0][lane], sm[0][1][lane], sm[0][2][lane]};
    for (int k = 1; k < 8; ++k) merge(acc, Moments{sm[k][0][lane], sm[k][1][lane], sm[k][2][lane]});
  } else if (w != 0) {
    return;
  }
  if (!live) return;
  if (moments) {
    for (int r = 0; r < world; ++r) {
      float* o = moments + (size_t)r * 3 * c + ch;
      const bool own = r == rank;
      o[0] = own ? acc.n : 0.0f;
      o[c] = own ? acc.mean : 0.0f;
      o[2 * (size_t)c] = own ? acc.m2 : 0.0f;
    }
    return;
  }
  bn_finalize_channel(acc, ch, c_real, gamma, beta, running_mean, running_var, momentum, eps, scale,
                      shift, mean_out, invstd);
}

// Synchronized BatchNorm, after the exchange: merge the world slots of moments [world][3][c] in
// rank order (Chan et al., as the slab stage) and finalize with the global moments; n_out[0] = the
// global row count (read by the backward's divisor).  One thread per channel.
__global__ void __launch_bounds__(256)
bn_sync_finalize_kernel(const float* __restrict__ moments, int world, int c, int c_real,
                        const float* __restrict__ gamma, const float* __restrict__ beta,
                        float* __restrict__ running_mean, float* __restrict__ running_var,
                        float momentum, float eps, float* __restrict__ scale,
                        float* __restrict__ shift, float* __restrict__ mean_out,
                        float* __restrict__ invstd, float* __restrict__ n_out) {
  pdl_entry();
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  Moments acc = {0.0f, 0.0f, 0.0f};
  for (int r = 0; r < world; ++r) {
    const float* o = moments + (size_t)r * 3 * c + ch;
    merge(acc, Moments{__ldcg(o), __ldcg(o + c), __ldcg(o + 2 * (size_t)c)});
  }
  if (ch == 0) n_out[0] = acc.n;
  bn_finalize_channel(acc, ch, c_real, gamma, beta, running_mean, running_var, momentum, eps, scale,
                      shift, mean_out, invstd);
}

// out[i] = sum_r slots[r][i] (i < n) in rank order, starting from slot 0 (one rank: a copy).
__global__ void __launch_bounds__(256)
rank_ordered_sum_kernel(const float* __restrict__ slots, int world, int n, float* __restrict__ out) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = __ldcg(slots + i);
  for (int r = 1; r < world; ++r) s += __ldcg(slots + (size_t)r * n + i);
  out[i] = s;
}

// out[st][ch] = mul_st[ch] * sum_p sum_f part[p][st][f * c + ch]   (st < nstat <= 2, f < folds):
// plain sums of slab partials in a fixed order; `folds` > 1 folds column blocks that belong to the
// same channel (the taps of a strided data-gradient GEMM).
__global__ void __launch_bounds__(256)
ordered_col_sums_kernel(const float* __restrict__ part, int n_part, int nstat, int ld, int c,
                        int folds, const float* __restrict__ mul0, const float* __restrict__ mul1,
                        float* __restrict__ out0, float* __restrict__ out1,
                        float* __restrict__ scratch, unsigned* __restrict__ counter) {
  pdl_entry();
  __shared__ float sm[8][2][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int ch = blockIdx.x * 32 + lane;
  const int S = gridDim.y;
  const bool live = ch < c;
  float a0 = 0.0f, a1 = 0.0f;
  const int per = (n_part + 8 * S - 1) / (8 * S);
  const int lo = (blockIdx.y * 8 + w) * per;
  const int hi = min(n_part, lo + per);
  for (int f = 0; f < folds; ++f) {
    for (int p0 = lo; p0 < hi; p0 += 8) {
      float x0[8], x1[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool ok = live && p0 + u < hi;
        const float* row = part + (size_t)(ok ? p0 + u : 0) * nstat * ld + (size_t)f * c + (live ? ch : 0);
        x0[u] = ok ? __ldg(row) : 0.0f;
        x1[u] = (ok && nstat == 2) ? __ldg(row + ld) : 0.0f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) { a0 += x0[u]; a1 += x1[u]; }
    }
  }
  sm[w][0][lane] = a0; sm[w][1][lane] = a1;
  __syncthreads();
  if (w == 0) {
    a0 = sm[0][0][lane]; a1 = sm[0][1][lane];
    for (int k = 1; k < 8; ++k) { a0 += sm[k][0][lane]; a1 += sm[k][1][lane]; }
    if (S > 1 && live) {
      scratch[((size_t)blockIdx.y * 2) * c + ch] = a0;
      scratch[((size_t)blockIdx.y * 2 + 1) * c + ch] = a1;
    }
  }
  if (S > 1) {
    if (!last_block_of_group(counter, S)) return;
    if (w != 0) return;
    float y0[32], y1[32];
#pragma unroll
    for (int y = 0; y < kReduceMaxSplits; ++y) {
      const bool ok = live && y < S;
      y0[y] = ok ? __ldcg(scratch + ((size_t)y * 2) * c + ch) : 0.0f;
      y1[y] = ok ? __ldcg(scratch + ((size_t)y * 2 + 1) * c + ch) : 0.0f;
    }
    a0 = a1 = 0.0f;
#pragma unroll
    for (int y = 0; y < kReduceMaxSplits; ++y) { a0 += y0[y]; a1 += y1[y]; }
  } else if (w != 0) {
    return;
  }
  if (!live) return;
  out0[ch] = mul0 ? a0 * mul0[ch] : a0;
  if (nstat == 2) out1[ch] = mul1 ? a1 * mul1[ch] : a1;
}

__device__ __forceinline__ long long map_row(const RowMap& m, long long r) {
  if (m.div > 0) {
    const long long s = r / m.div;
    const long long t = r - s * m.div;
    return s * m.rows_per_sample + t * m.step + m.off;
  }
  return r * m.step + m.off;
}

// Thread layout shared by the row-streaming kernels: 256 threads = 8 column groups (8 channels each,
// 64 channels per block) x 32 row lanes; a block walks kRowsPerBlock rows.  Per-channel vectors are
// loaded once into registers and reused for every row the thread touches; a warp's access is 4 rows
// x 128 contiguous bytes.
// G = column groups per block (power of two dividing c/8, <= 256), lanes = 256 / G row lanes.  For
// C = 1024 a block spans whole rows (G = 128): every warp reads 512 contiguous bytes.
struct RowTiling {
  int G;               // column groups (of 8 channels) handled by one block
  int rows_per_block;  // rows walked by one block
};

__device__ __forceinline__ void load_vec8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p + 4));
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__global__ void __launch_bounds__(256)
bn_apply_kernel(const __nv_bfloat16* __restrict__ z, long long z_plane,
                __nv_bfloat16* __restrict__ x, long long x_plane, int planes, long long rows, int c,
                const float* __restrict__ scale, const float* __restrict__ shift, DropoutCfg drop,
                const __nv_bfloat16* __restrict__ res, long long res_plane, RowMap map,
                RowTiling tl) {
  pdl_entry();
  const int cg = threadIdx.x % tl.G, rl = threadIdx.x / tl.G, lanes = 256 / tl.G;
  const int c0 = (blockIdx.x * tl.G + cg) * 8;
  const long long r_begin = (long long)blockIdx.y * tl.rows_per_block;
  const long long r_end = min(rows, r_begin + tl.rows_per_block);
  const bool do_drop = drop.p > 0.0f;
  const uint32_t thresh = (uint32_t)(drop.p * 65536.0f);
  const float inv_keep = do_drop ? 1.0f / (1.0f - drop.p) : 1.0f;
  float sc[8], sh[8];
  load_vec8(scale + c0, sc);
  load_vec8(shift + c0, sh);
  long long r = r_begin + rl;
  if (planes == 1) {
    // Single-plane fast path: the loads of four rows are issued before any of them is consumed
    // (the plain loop below keeps one row -- 32 bytes per thread -- in flight, which measured
    // 3.5 TB/s: latency-bound, not bandwidth-bound).
    for (; r + 3 * lanes < r_end; r += 4 * lanes) {
      uint4 zr[4], rr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        zr[u] = __ldg(reinterpret_cast<const uint4*>(z + (r + u * lanes) * c + c0));
      if (res) {
#pragma unroll
        for (int u = 0; u < 4; ++u)
          rr[u] = __ldg(reinterpret_cast<const uint4*>(res + map_row(map, r + u * lanes) * c + c0));
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float v[8];
        unpack8(zr[u], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.0f);
        if (do_drop) {
          float m[8];
          dropout_keep8(drop, (r + u * lanes) * c + c0, thresh, inv_keep, m);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] *= m[j];
        }
        if (res) {
          float rv[8];
          unpack8(rr[u], rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] += rv[j];
        }
        store8(x + (r + u * lanes) * c + c0, x_plane, 1, v);
      }
    }
  }
  for (; r < r_end; r += lanes) {
    float v[8];
    load8(z + r * c + c0, z_plane, planes, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.0f);
    if (do_drop) {
      float m[8];
      dropout_keep8(drop, r * c + c0, thresh, inv_keep, m);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= m[j];
    }
    if (res) {
      float rv[8];
      load8(res + map_row(map, r) * c + c0, res_plane, planes, rv);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += rv[j];
    }
    store8(x + r * c + c0, x_plane, planes, v);
  }
}

// dY for 8 channels of one row: dY = g * dropmask/(1-p) * [z*scale+shift > 0].
__device__ __forceinline__ void dy8(const __nv_bfloat16* g, long long g_plane,
                                    const __nv_bfloat16* z, long long z_plane, int planes,
                                    long long r, int c, int c0, const float (&sc)[8],
                                    const float (&sh)[8], const DropoutCfg& drop, bool do_drop,
                                    uint32_t thresh, float inv_keep, float (&dy)[8],
                                    float (&zv)[8]) {
  float gv[8];
  load8(g + r * c + c0, g_plane, planes, gv);
  load8(z + r * c + c0, z_plane, planes, zv);
  float m[8];
  if (do_drop) dropout_keep8(drop, r * c + c0, thresh, inv_keep, m);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float d = fmaf(zv[j], sc[j], sh[j]) > 0.0f ? gv[j] : 0.0f;
    if (do_drop) d *= m[j];
    dy[j] = d;
  }
}

__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ g, long long g_plane,
                     const __nv_bfloat16* __restrict__ z, long long z_plane, int planes,
                     long long rows, int c, const float* __restrict__ scale,
                     const float* __restrict__ shift, const float* __restrict__ mean,
                     const float* __restrict__ invstd, DropoutCfg drop, float* __restrict__ sums,
                     RowTiling tl) {
  pdl_entry();
  __shared__ float sm[2][2048];
  const int cg = threadIdx.x % tl.G, rl = threadIdx.x / tl.G, lanes = 256 / tl.G;
  const int c0 = (blockIdx.x * tl.G + cg) * 8;
  const long long r_begin = (long long)blockIdx.y * tl.rows_per_block;
  const long long r_end = min(rows, r_begin + tl.rows_per_block);
  const bool do_drop = drop.p > 0.0f;
  const uint32_t thresh = (uint32_t)(drop.p * 65536.0f);
  const float inv_keep = do_drop ? 1.0f / (1.0f - drop.p) : 1.0f;
  float s1[8], s2[8], mu[8], sc[8], sh[8];
  load_vec8(mean + c0, mu);
  load_vec8(scale + c0, sc);
  load_vec8(shift + c0, sh);
#pragma unroll
  for (int j = 0; j < 8; ++j) s1[j] = s2[j] = 0.0f;
#pragma unroll 4
  for (long long r = r_begin + rl; r < r_end; r += lanes) {
    float dy[8], zv[8];
    dy8(g, g_plane, z, z_plane, planes, r, c, c0, sc, sh, drop, do_drop, thresh, inv_keep, dy, zv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s1[j] += dy[j];
      s2[j] += dy[j] * (zv[j] - mu[j]);  // invstd factored out of the sum
    }
  }
  const int width = tl.G * 8;  // channels covered by this block
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sm[0][rl * width + cg * 8 + j] = s1[j];
    sm[1][rl * width + cg * 8 + j] = s2[j];  // x invstd after the ordered sum
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * width; i += 256) {
    const int which = i / width, ch = i - which * width;
    float t = 0.0f;
    for (int l = 0; l < lanes; ++l) t += sm[which][l * width + ch];
    // partials [blockIdx.y][2][c], reduced in a fixed order by launch_ordered_col_sums
    sums[((size_t)blockIdx.y * 2 + which) * c + blockIdx.x * width + ch] = t;
  }
}

// dz = scale*(dY - s1/n - xhat*s2/n) = scale*dY + B*z + D with per-channel
// B = -scale*invstd*s2/n,  D = -scale*s1/n - B*mean.  frozen (BatchNorm on running statistics):
// B = D = 0, dz = scale*dY; sums may then be null (no dgamma / dbeta wanted).
// Synchronized BatchNorm: B and D use the global sums `gsums` and the global row count *n_global;
// dgamma / dbeta come from this rank's `sums` (the gradient all-reduce averages them).  Otherwise
// gsums == sums and n_global is null (n = rows).
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ g, long long g_plane,
                    const __nv_bfloat16* __restrict__ z, long long z_plane,
                    __nv_bfloat16* __restrict__ dz, long long dz_plane, int planes, long long rows,
                    int c, const float* __restrict__ scale, const float* __restrict__ shift,
                    const float* __restrict__ mean, const float* __restrict__ invstd,
                    DropoutCfg drop, const float* sums, const float* gsums,
                    const float* __restrict__ n_global, float* __restrict__ dgamma,
                    float* __restrict__ dbeta, int c_real, int frozen, RowTiling tl) {
  pdl_entry();
  const int cg = threadIdx.x % tl.G, rl = threadIdx.x / tl.G, lanes = 256 / tl.G;
  const int c0 = (blockIdx.x * tl.G + cg) * 8;
  const long long r_begin = (long long)blockIdx.y * tl.rows_per_block;
  const long long r_end = min(rows, r_begin + tl.rows_per_block);
  const bool do_drop = drop.p > 0.0f;
  const uint32_t thresh = (uint32_t)(drop.p * 65536.0f);
  const float inv_keep = do_drop ? 1.0f / (1.0f - drop.p) : 1.0f;
  const float inv_n = 1.0f / (n_global ? __ldg(n_global) : (float)rows);
  float sc[8], sh[8], B[8], D[8];
  {
    float mu[8], is[8], s1[8], s2[8];
    load_vec8(scale + c0, sc);
    load_vec8(shift + c0, sh);
    if (sums) {
      load_vec8(gsums + c0, s1);
      load_vec8(gsums + c + c0, s2);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) s1[j] = s2[j] = 0.0f;
    }
    if (frozen) {
#pragma unroll
      for (int j = 0; j < 8; ++j) mu[j] = is[j] = 0.0f;
    } else {
      load_vec8(mean + c0, mu);
      load_vec8(invstd + c0, is);
    }
    if (sums && blockIdx.y == 0 && rl == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (c0 + j >= c_real) break;   // gradient tensors hold the model's real channel count
        if (dbeta) dbeta[c0 + j] = __ldg(sums + c0 + j);          // this rank's sums
        if (dgamma) dgamma[c0 + j] = __ldg(sums + c + c0 + j);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      B[j] = frozen ? 0.0f : -sc[j] * is[j] * s2[j] * inv_n;
      D[j] = frozen ? 0.0f : -sc[j] * s1[j] * inv_n - B[j] * mu[j];
    }
  }
  long long r = r_begin + rl;
  if (planes == 1) {
    // (loads of four rows in flight per thread, see bn_apply_kernel)
    for (; r + 3 * lanes < r_end; r += 4 * lanes) {
      uint4 gr[4], zr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        gr[u] = __ldg(reinterpret_cast<const uint4*>(g + (r + u * lanes) * c + c0));
        zr[u] = __ldg(reinterpret_cast<const uint4*>(z + (r + u * lanes) * c + c0));
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float gv[8], zv[8], m[8], o[8];
        unpack8(gr[u], gv);
        unpack8(zr[u], zv);
        if (do_drop) dropout_keep8(drop, (r + u * lanes) * c + c0, thresh, inv_keep, m);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float d = fmaf(zv[j], sc[j], sh[j]) > 0.0f ? gv[j] : 0.0f;
          if (do_drop) d *= m[j];
          o[j] = fmaf(sc[j], d, fmaf(B[j], zv[j], D[j]));
        }
        store8(dz + (r + u * lanes) * c + c0, dz_plane, 1, o);
      }
    }
  }
  for (; r < r_end; r += lanes) {
    float dy[8], zv[8], o[8];
    dy8(g, g_plane, z, z_plane, planes, r, c, c0, sc, sh, drop, do_drop, thresh, inv_keep, dy, zv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(sc[j], dy[j], fmaf(B[j], zv[j], D[j]));
    store8(dz + r * c + c0, dz_plane, planes, o);
  }
}

__global__ void col_sum_f32_kernel(const float* __restrict__ x, long long rows, int c,
                                   float* __restrict__ out) {
  pdl_entry();
  // one warp per 32-row chunk; lanes stride the channels
  const long long r0 = (long long)blockIdx.x * 64;
  for (int col = threadIdx.x; col < c; col += blockDim.x) {
    float s = 0.0f;
    for (long long r = r0; r < min(rows, r0 + 64); ++r) s += x[r * c + col];
    out[(size_t)blockIdx.x * c + col] = s;   // partials [chunk][c], reduced in a fixed order
  }
}

// w fp32 (c_out, c_in, taps) -> out_t[pl][tap][ci][co] (rows n_pad = padded c_in, cols k_pad = padded
// c_out).  32 x 32 (co, ci) tiles go through shared memory so that both the reads (ci fastest) and
// the writes (co fastest) are coalesced.  Padding entries are written as zeros.
// If `fwd` is non-null the same pass also writes the forward pack fwd[pl][tap][co][ci] (rows
// fwd_n_pad, cols fwd_k_pad), so one read of the fp32 master feeds both layouts.
// merged: one tap-merged slab out[pl][tap*c_in + ci][co] (rows n_pad >= taps*c_in; the last tap
// writes the padding rows) -- the data gradient of the strided expand conv.
__global__ void __launch_bounds__(256)
pack_conv_weight_t_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int planes,
                          int c_out, int c_in, int taps, int n_pad, int k_pad,
                          __nv_bfloat16* __restrict__ fwd, int fwd_n_pad, int fwd_k_pad,
                          int merged) {
  __shared__ float sm[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  const long long plane_elems = merged ? (long long)n_pad * k_pad : (long long)taps * n_pad * k_pad;
  const long long fwd_plane = (long long)taps * fwd_n_pad * fwd_k_pad;
  for (int tap = 0; tap < taps; ++tap) {
#pragma unroll
    for (int j = ty; j < 32; j += 8) {
      const int co = co0 + j, ci = ci0 + tx;
      const float v = (co < c_out && ci < c_in)
                          ? __ldg(w + ((long long)co * c_in + ci) * taps + tap) : 0.0f;
      sm[j][tx] = v;
      if (fwd && co < fwd_n_pad && ci < fwd_k_pad)
        store_bits16(fwd, ((long long)tap * fwd_n_pad + co) * fwd_k_pad + ci, fwd_plane, planes, v);
    }
    __syncthreads();
#pragma unroll
    for (int j = ty; j < 32; j += 8) {
      const int ci = ci0 + j, co = co0 + tx;
      const int row = merged ? tap * c_in + ci : ci;
      const bool own = !merged || ci < c_in || tap == taps - 1;
      if (own && row < n_pad && co < k_pad)
        store_bits16(out, ((long long)(merged ? 0 : tap) * n_pad + row) * k_pad + co, plane_elems,
                     planes, sm[tx][j]);
    }
    __syncthreads();
  }
}

RowTiling row_tiling(long long rows, int c, dim3& grid, int min_rows = 0) {
  RowTiling tl;
  const int groups = c / 8;
  tl.G = 8;
  while (tl.G * 2 <= 256 && groups % (tl.G * 2) == 0) tl.G *= 2;
  const int lanes = 256 / tl.G;
  const int col_blocks = groups / tl.G;
  // ~16 resident blocks per SM (the loads are latency-bound otherwise), at least 4 rows per thread,
  // at most 256 rows per block
  long long rpb = rows * col_blocks / (16 * 132);
  if (rpb > 256) rpb = 256;
  if (rpb < 4LL * lanes) rpb = 4LL * lanes;
  if (rpb < min_rows) rpb = min_rows;
  rpb = (rpb + lanes - 1) / lanes * lanes;
  tl.rows_per_block = (int)rpb;
  grid = dim3(col_blocks, (unsigned)((rows + rpb - 1) / rpb));
  return tl;
}

}  // namespace

static int pick_splits(int n_part) {
  int S = (n_part + 127) / 128;   // ~16 partials per warp
  if (S < 1) S = 1;
  if (S > kReduceMaxSplits) S = kReduceMaxSplits;
  return S;
}

cudaError_t launch_bn_stats_finalize(const float* part, int slabs, int dilated, int out_rows,
                                     int tiles_per_sample, const float* gamma, const float* beta,
                                     float* running_mean, float* running_var, float momentum,
                                     float eps, float* scale, float* shift, float* mean,
                                     float* invstd, int c, int c_real, float* scratch,
                                     unsigned* counter, cudaStream_t stream, float* moments,
                                     int world, int rank) {
  if (c > kReduceMaxChannels) return cudaErrorInvalidValue;
  if (moments && (world < 1 || rank < 0 || rank >= world)) return cudaErrorInvalidValue;
  SlabGeom g = {dilated, out_rows, tiles_per_sample};
  const dim3 grid((c + 31) / 32, pick_splits(slabs));
  const cudaError_t le = launch_pdl(bn_stats_finalize_kernel, grid, dim3(256), 0, stream, part, slabs, g, c, c_real, gamma, beta, running_mean,
                                                     running_var, momentum, eps, scale, shift, mean,
                                                     invstd, scratch, counter, moments, world, rank);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_bn_sync_finalize(const float* moments, int world, const float* gamma,
                                    const float* beta, float* running_mean, float* running_var,
                                    float momentum, float eps, float* scale, float* shift,
                                    float* mean, float* invstd, int c, int c_real, float* n_out,
                                    cudaStream_t stream) {
  if (world < 1 || c < 1) return cudaErrorInvalidValue;
  const cudaError_t le = launch_pdl(bn_sync_finalize_kernel, dim3((c + 255) / 256), dim3(256), 0,
                                    stream, moments, world, c, c_real, gamma, beta, running_mean,
                                    running_var, momentum, eps, scale, shift, mean, invstd, n_out);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_rank_ordered_sum(const float* slots, int world, int n, float* out,
                                    cudaStream_t stream) {
  if (world < 1 || n < 1) return cudaErrorInvalidValue;
  const cudaError_t le = launch_pdl(rank_ordered_sum_kernel, dim3((n + 255) / 256), dim3(256), 0,
                                    stream, slots, world, n, out);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_ordered_col_sums(const float* part, int n_part, int nstat, int ld, int c,
                                    int folds, const float* mul0, const float* mul1, float* out0,
                                    float* out1, float* scratch, unsigned* counter,
                                    cudaStream_t stream) {
  if (c > kReduceMaxChannels || nstat < 1 || nstat > 2) return cudaErrorInvalidValue;
  const dim3 grid((c + 31) / 32, pick_splits(n_part));
  const cudaError_t le = launch_pdl(ordered_col_sums_kernel, grid, dim3(256), 0, stream, part, n_part, nstat, ld, c, folds, mul0, mul1,
                                                    out0, out1, scratch, counter);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_bn_apply(const __nv_bfloat16* z, long long z_plane, __nv_bfloat16* x,
                            long long x_plane, int planes, long long rows, int c, const float* scale,
                            const float* shift, DropoutCfg drop, const __nv_bfloat16* res,
                            long long res_plane, RowMap map, cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  dim3 grid;
  const RowTiling tl = row_tiling(rows, c, grid);
  const cudaError_t le = launch_pdl(bn_apply_kernel, grid, dim3(256), 0, stream, z, z_plane, x, x_plane, planes, rows, c, scale, shift,
                                            drop, res, res_plane, map, tl);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_bn_bwd_reduce(const __nv_bfloat16* g, long long g_plane, const __nv_bfloat16* z,
                                 long long z_plane, int planes, long long rows, int c,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, DropoutCfg drop, float* partials,
                                 size_t partial_floats, float* sums, float* scratch,
                                 unsigned* counter, cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  dim3 grid;
  // >= 32 rows per block: the per-block partials then fit the slab-partial buffer (rows / 32 slabs)
  const RowTiling tl = row_tiling(rows, c, grid, 32);
  if ((size_t)grid.y * 2 * c > partial_floats) return cudaErrorInvalidValue;
  const cudaError_t le = launch_pdl(bn_bwd_reduce_kernel, grid, dim3(256), 0, stream, g, g_plane, z, z_plane, planes, rows, c, scale,
                                                 shift, mean, invstd, drop, partials, tl);
  cudaError_t e = le != cudaSuccess ? le : cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_ordered_col_sums(partials, (int)grid.y, 2, c, c, 1, nullptr, invstd, sums, sums + c,
                                 scratch, counter, stream);
}

cudaError_t launch_bn_bwd_apply(const __nv_bfloat16* g, long long g_plane, const __nv_bfloat16* z,
                                long long z_plane, __nv_bfloat16* dz, long long dz_plane, int planes,
                                long long rows, int c, const float* scale, const float* shift,
                                const float* mean, const float* invstd, DropoutCfg drop,
                                const float* sums, float* dgamma, float* dbeta, int c_real,
                                cudaStream_t stream, int frozen, const float* global_sums,
                                const float* n_global) {
  if (rows <= 0) return cudaSuccess;
  if (!sums && !frozen) return cudaErrorInvalidValue;
  if (!global_sums != !n_global) return cudaErrorInvalidValue;
  if (!global_sums) global_sums = sums;
  dim3 grid;
  const RowTiling tl = row_tiling(rows, c, grid);
  const cudaError_t le = launch_pdl(bn_bwd_apply_kernel, grid, dim3(256), 0, stream, g, g_plane, z, z_plane, dz, dz_plane, planes, rows,
                                                c, scale, shift, mean, invstd, drop, sums,
                                                global_sums, n_global, dgamma, dbeta, c_real,
                                                frozen, tl);
  return le != cudaSuccess ? le : cudaGetLastError();
}

cudaError_t launch_col_sum_f32(const float* x, long long rows, int c, float* partials,
                               size_t partial_floats, float* out, float* scratch, unsigned* counter,
                               cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  const unsigned chunks = (unsigned)((rows + 63) / 64);
  if ((size_t)chunks * c > partial_floats) return cudaErrorInvalidValue;
  const cudaError_t le = launch_pdl(col_sum_f32_kernel, dim3(chunks), dim3(64), 0, stream, x, rows, c, partials);
  cudaError_t e = le != cudaSuccess ? le : cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_ordered_col_sums(partials, (int)chunks, 1, c, c, 1, nullptr, nullptr, out, nullptr,
                                 scratch, counter, stream);
}

cudaError_t launch_pack_conv_weight_t(const float* w, __nv_bfloat16* out, int planes, int c_out,
                                      int c_in, int taps, int n_pad, int k_pad, cudaStream_t stream,
                                      __nv_bfloat16* fwd, int fwd_n_pad, int fwd_k_pad, int merged) {
  if (merged && (fwd || n_pad < taps * c_in)) return cudaErrorInvalidValue;
  int gx = (n_pad + 31) / 32, gy = (k_pad + 31) / 32;
  if (fwd) {  // the grid must also cover the forward pack's padding
    if ((fwd_k_pad + 31) / 32 > gx) gx = (fwd_k_pad + 31) / 32;
    if ((fwd_n_pad + 31) / 32 > gy) gy = (fwd_n_pad + 31) / 32;
  }
  pack_conv_weight_t_kernel<<<dim3(gx, gy), 256, 0, stream>>>(w, out, planes, c_out, c_in, taps,
                                                              n_pad, k_pad, fwd, fwd_n_pad, fwd_k_pad,
                                                              merged);
  return cudaGetLastError();
}

}  // namespace vp3d
