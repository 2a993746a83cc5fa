// wgmma implicit-GEMM kernel for the temporal convolutions.  See conv_gemm.cuh for the math.
//
// CTA = 384 threads (three warpgroups), persistent over output tiles (128 rows x BLOCK_N channels):
//   warp 0 lane 0 : TMA producer  (A tile 128x64 + W tile BLOCK_Nx64 16-bit per k-block)
//   warp 1 lane 0 : auxiliary producer (residual instances): TMA-loads the 128x64 residual tile(s) / the Z
//                   tile of every 64-column store block into shared memory ahead of the epilogue
//   warps 4..11   : two consumer warpgroups; warpgroup g owns rows [64 g, 64 g + 64) of every tile.
//                   Each issues the m64 x BLOCK_N x k16 wgmma stream of its rows (fp32 accumulators
//                   in registers) and then runs the epilogue on those registers:
//                   BN affine / ReLU / residual / batch sums -> 16-bit pack into a SWIZZLE_128B
//                   staging tile (two per warpgroup, alternating) -> TMA stores of its 64 x 64 slice
//                   (coalesced 128-byte rows, clipped at the tensor edge by the map)
// The operand pipeline keeps running across tiles: the producer fills the stages of the next tile
// while the consumers are in the epilogue of the current one.
// Lean inference launches with more tiles than CTAs use the ping-pong instances instead: each
// consumer warpgroup computes all 128 rows of every other tile, so that one warpgroup's epilogue
// runs under the other's MMAs.  At 128 wide, a last wave of at most half the grid runs as twice as
// many 128 x 64 half tiles (n64 MMAs, one 64-column store block), one per CTA.
// The int8 eval instances run the same pipeline on u8 A / s8 W tiles of 128 x 128 bytes per
// k-block (int32 accumulators, k32 MMAs), and may store a u8 copy of their output.
#include "conv_gemm.cuh"

#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "ptx.cuh"

namespace vp3d {

// What a kernel instance fixes at compile time.
// Epilogue: kTrain compiles in the training-only paths (BatchNorm batch statistics of the stored
// value, fused BatchNorm-backward reductions); kGeneral reads every option from ConvGemmArgs;
// kLean serves the inference layers, exactly affine + ReLU [+ a one-plane TMA residual over every
// column] into one 16-bit plane [+ its u8 copy], with every option resolved at compile time.
enum class Epi { kTrain, kGeneral, kLean };
// Operand / storage format: the lean instances fix it (so that each k-block is one branch-free
// group of wgmma), the others read p.f16.  kI8: u8 A times s8 W into int32 accumulators,
// 128-element k-blocks; the residual and the 16-bit output stay fp16.
enum class Fmt { kRuntime, kBf16, kF16, kI8 };
// kPingPong: each consumer warpgroup computes whole tiles (see the kernel's consumer branches).
enum class Sched { kCooperative, kPingPong };
// u8 quantisation of every stored value (ConvGemmArgs::out_u8): beside the 16-bit plane, with
// staging tiles of its own, or alone (no 16-bit output; staged in the unused 16-bit staging).
enum class U8Out { kNone, kBeside, kAlone };

struct InstKey {
  int block_n;
  Epi epi;
  Fmt fmt;
  Sched sched;
  bool res;    // auxiliary TMA tiles: the residual and / or the BatchNorm-backward Z
  bool out2;   // two output planes (hi, lo) -> two staging planes per buffer
  U8Out u8;
  constexpr bool operator==(const InstKey& o) const {
    return block_n == o.block_n && epi == o.epi && fmt == o.fmt && sched == o.sched &&
           res == o.res && out2 == o.out2 && u8 == o.u8;
  }
};

// One kernel instance: its compile-time options and its shared-memory layout.
template <int BLOCK_N, Epi EPI, Fmt FMT, Sched SCHED, bool RES, bool OUT2 = false,
          U8Out U8 = U8Out::kNone>
struct Inst {
  static_assert((BLOCK_N == 64 || BLOCK_N == 128) &&             // wgmma tiles are 64 or 128 wide
                    (EPI == Epi::kLean) == (FMT != Fmt::kRuntime) &&
                    !(EPI == Epi::kLean && OUT2) &&                 // lean: one output plane
                    (SCHED == Sched::kCooperative || EPI == Epi::kLean) &&
                    (U8 == U8Out::kNone || FMT == Fmt::kF16 || FMT == Fmt::kI8) &&
                    !(RES && U8 == U8Out::kAlone),                  // a residual stores 16 bits
                "not a conv GEMM instance");
  static constexpr InstKey kKey = {BLOCK_N, EPI, FMT, SCHED, RES, OUT2, U8};
  static constexpr int kBlockN = BLOCK_N;
  static constexpr Fmt kFmt = FMT;
  static constexpr bool kTrain = EPI == Epi::kTrain;
  static constexpr bool kLean = EPI == Epi::kLean;
  static constexpr bool kF16 = FMT == Fmt::kF16 || FMT == Fmt::kI8;
  static constexpr bool kI8 = FMT == Fmt::kI8;
  static constexpr bool kPP = SCHED == Sched::kPingPong;
  static constexpr bool kRes = RES;
  static constexpr bool kOut2 = OUT2;
  static constexpr bool kU8 = U8 != U8Out::kNone;
  static constexpr bool kU8Beside = U8 == U8Out::kBeside;
  static constexpr bool kU8Alone = U8 == U8Out::kAlone;
  static constexpr bool kStore16 = !kU8Alone;
  using Acc = std::conditional_t<kI8, int, float>;

  static constexpr uint32_t kABytes = kBlockM * kBlockK * 2;
  static constexpr uint32_t kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kTileBytes = kBlockM * 64 * 2;   // one 128 x 64 16-bit tile (16 KiB)
  static constexpr uint32_t kHalfBytes = 64 * 64 * 2;        // one warpgroup's 64 x 64 slice
  // staging: 2 warpgroups x 2 alternating buffers x (hi[, lo]).  Ping-pong: one 128 x 64 tile per
  // warpgroup; the residual instance stores in place from the residual's landing tile instead.
  static constexpr uint32_t kStagingBytes =
      kPP ? (RES ? 0 : 2 * kTileBytes) : 2 * 2 * (OUT2 ? 2 : 1) * kHalfBytes;
  // auxiliary (residual / Z) landing tiles: four, so that two-tile store blocks (hi+lo residual,
  // or residual + Z) still get two stages in flight.  Ping-pong: two per warpgroup.
  static constexpr int kResSlots = RES ? 4 : 0;
  // u8 staging (64 columns of 64 bytes per row): ping-pong one 128-row tile per warpgroup,
  // cooperative two alternating 64-row halves per warpgroup -- 16 KiB either way
  static constexpr uint32_t kU8Bytes = kU8Beside ? 2 * kBlockM * 64 : 0;
  static constexpr uint32_t kFixedBytes = kStagingBytes + kResSlots * kTileBytes + kU8Bytes;
  // per-channel affine (scale, shift) of the current N block: 2 x BLOCK_N floats.  Ping-pong reads
  // it through L1 instead: the two warpgroups may hold different N blocks, and a copy per
  // warpgroup would cost the 128-wide instance an operand stage.
  static constexpr uint32_t kAffineBytes = kPP ? 0 : 2 * BLOCK_N * 4;
  // training: per-column (sum, sumsq) of one warp of every 32-row slab pair, 4 slabs x 2 x 64
  static constexpr uint32_t kPairBytes = kTrain ? 4 * 2 * 64 * 4 : 0;
  static constexpr uint32_t kBarBytesMax = (2 * 8 + 8 + 1) * 8 + 32;
  // as many operand stages as fit into the 227 KiB a CTA may use (less 1 KiB of alignment slack),
  // at most 8
  static constexpr uint32_t kMaxSmem = 232448u;
  static constexpr int kStagesFit =
      (kMaxSmem - 1024 - kFixedBytes - kBarBytesMax - kAffineBytes - kPairBytes) / kStageBytes;
  static constexpr int kStages = kStagesFit > 8 ? 8 : kStagesFit;
  static_assert(kStages >= 2, "not enough shared memory for the operand pipeline");
  static constexpr uint32_t kBarBytes = (2 * kStages + 8 + 1) * 8 + 32;
  static constexpr uint32_t kSmemBytes =
      1024 + kStages * kStageBytes + kFixedBytes + kBarBytes + kAffineBytes + kPairBytes;
  static_assert(kSmemBytes <= kMaxSmem, "shared memory budget exceeded");
};

__device__ __forceinline__ void tile_coords(const ConvGemmArgs& p, int tile, int& n_blk,
                                            int& sample, int& row0) {
  n_blk = tile % p.n_tiles;
  int m_blk = tile / p.n_tiles;
  if (p.dilated) {
    sample = m_blk / p.tiles_per_sample;
    row0 = (m_blk - sample * p.tiles_per_sample) * kBlockM;
  } else {
    sample = 0;
    row0 = m_blk * kBlockM;
  }
}

// Work item w of a launch whose tiles [0, full_tiles) run whole and whose remaining tiles run as
// two 128 x 64 halves each (items full_tiles + 2 i + h: half h of tile full_tiles + i).  Returns
// whether the item is a half tile; c_off is its first column inside the N block (0 or 64).
__device__ __forceinline__ bool item_coords(const ConvGemmArgs& p, int full_tiles, int w,
                                            int& n_blk, int& sample, int& row0, int& c_off) {
  const bool half = w >= full_tiles;
  c_off = half ? 64 * ((w - full_tiles) & 1) : 0;
  tile_coords(p, half ? full_tiles + ((w - full_tiles) >> 1) : w, n_blk, sample, row0);
  return half;
}

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// byte offset of (row, column pair starting at even column c) in a 128-byte-row SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_off(int row, int c) {
  return (uint32_t)row * 128u + ((((uint32_t)c >> 3) ^ ((uint32_t)row & 7u)) << 4) + ((uint32_t)c & 7u) * 2u;
}
__device__ __forceinline__ void add_pair(float& a, float& b, uint32_t u, bool f16) {
  if (f16) { a += f16_lo_to_f(u); b += f16_hi_to_f(u); }
  else { a += bf16_lo_to_f(u); b += bf16_hi_to_f(u); }
}

// the u8 pair (columns c, c + 1) at byte `off` of a u8 staging tile (rows of 64 bytes, no swizzle)
__device__ __forceinline__ void st_u8_pair(uint32_t addr, float v0, float v1, float inv_s) {
  const uint32_t q = quant_u8(v0, inv_s) | (quant_u8(v1, inv_s) << 8);
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"((unsigned short)q) : "memory");
}

// Per-column sums over the 16 rows a warp holds of one 64-column store block (values v[jj][0..3]
// in the wgmma layout), then over the two warps of a 32-row slab (in a fixed order: the even warp's
// partial plus the odd warp's).  Lane l < 4 of the even warp ends up with the slab sums of columns
// 8 jj + 2 l (+1) in s[jj][0..1], q[jj][0..1].
__device__ __forceinline__ void slab_reduce(float (&s)[8][2], float (&q)[8][2], float* s_pair,
                                            int lane, int wq, uint32_t bar_id) {
#pragma unroll
  for (int off = 4; off <= 16; off <<= 1) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s[jj][e] += __shfl_xor_sync(0xffffffffu, s[jj][e], off);
        q[jj][e] += __shfl_xor_sync(0xffffffffu, q[jj][e], off);
      }
    }
  }
  // s_pair: [s | q][64 columns] of this slab
  if ((wq & 1) && lane < 4) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      *reinterpret_cast<float2*>(s_pair + 8 * jj + 2 * lane) = make_float2(s[jj][0], s[jj][1]);
      *reinterpret_cast<float2*>(s_pair + 64 + 8 * jj + 2 * lane) = make_float2(q[jj][0], q[jj][1]);
    }
  }
  named_bar_sync(bar_id, 64);
  if (!(wq & 1) && lane < 4) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 so = *reinterpret_cast<const float2*>(s_pair + 8 * jj + 2 * lane);
      const float2 qo = *reinterpret_cast<const float2*>(s_pair + 64 + 8 * jj + 2 * lane);
      s[jj][0] += so.x; s[jj][1] += so.y;
      q[jj][0] += qo.x; q[jj][1] += qo.y;
    }
  }
  named_bar_sync(bar_id, 64);   // the odd warp may overwrite s_pair for the next block from here on
}

#ifdef VP3D_TIMELINE
__device__ __forceinline__ void tl_stamp(const ConvGemmArgs& p, int ev) {
  if (!p.timeline) return;
  int slot;
  if (blockIdx.x == 0) slot = 0;
  else if (blockIdx.x == gridDim.x - 1) slot = 1;
  else return;
  unsigned long long g;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
  p.timeline[(slot * 32 + ev) * 2] = g;
  p.timeline[(slot * 32 + ev) * 2 + 1] = (unsigned long long)clock64();
}
#define TL(ev) tl_stamp(p, ev)
#else
#define TL(ev) ((void)0)
#endif

// One k-block (one 128-byte swizzle row of K) of m64 x N MMAs into each of the H accumulator
// halves in turn, half h reading the A rows of descriptor da[h]: four k16 steps of 16 elements, or
// for int8 (u8 x s8) four k32 steps of 32 elements -- 32 B each, +2 in the descriptors' address >> 4.
// An n64 MMA into a 128-wide accumulator (a half tile) uses its first 32 registers: columns 0-63.
template <int N, Fmt FMT, int H, int F, class Acc>
__device__ __forceinline__ void wgmma_kblock(Acc (&acc)[H][F], const uint64_t (&da)[H],
                                             uint64_t db, bool first) {
  static_assert((N == 64 || N == 128) && N / 2 <= F, "not a wgmma width of this accumulator");
#pragma unroll
  for (int h = 0; h < H; ++h) {
    auto& d = reinterpret_cast<Acc(&)[N / 2]>(acc[h]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t accumulate = (first && k == 0) ? 0u : 1u;
      if constexpr (FMT == Fmt::kI8) {
        if constexpr (N == 128) wgmma_m64n128k32_u8s8(d, da[h] + 2 * k, db + 2 * k, accumulate);
        else wgmma_m64n64k32_u8s8(d, da[h] + 2 * k, db + 2 * k, accumulate);
      } else if constexpr (N == 128) {
        if constexpr (FMT == Fmt::kF16) wgmma_m64n128_f16(d, da[h] + 2 * k, db + 2 * k, accumulate);
        else wgmma_m64n128_bf16(d, da[h] + 2 * k, db + 2 * k, accumulate);
      } else {
        if constexpr (FMT == Fmt::kF16) wgmma_m64n64_f16(d, da[h] + 2 * k, db + 2 * k, accumulate);
        else wgmma_m64n64_bf16(d, da[h] + 2 * k, db + 2 * k, accumulate);
      }
    }
  }
}

// The MMA main loop of one tile, over H 64-row halves of every A stage from byte a_off on (the
// cooperative schedule: H = 1, this warpgroup's rows; ping-pong: H = 2, the whole tile).  The tile's
// first k-block sits in pipeline stage `stage` of parity `phase`; both are left at the next fill.
// Each k-block is one wgmma group; a stage is released once wait_group 1 shows the group reading it
// has retired.  `issued()` runs after the last group is issued, before the wait for it.
// The runtime format test of the general instances stays outside the k16 steps: a branch inside a
// group makes ptxas close it with an extra null HGMMA (DESIGN.md section 4).  N: the MMA width,
// I::kBlockN, or 64 for a half tile of a 128-wide instance (its W stage holds the first 64 rows).
template <class I, int N = I::kBlockN, int H, class Issued>
__device__ __forceinline__ void mma_tile(typename I::Acc (&acc)[H][I::kBlockN / 2],
                                         const ConvGemmArgs& p, bool f16, uint32_t smem_a,
                                         uint32_t a_off, uint32_t smem_b, uint32_t full_bar,
                                         uint32_t empty_bar, uint32_t& stage_io, uint32_t& phase_io,
                                         int k_iters, int lane, bool tl_first, Issued issued) {
  uint32_t stage = stage_io, phase = phase_io;
  uint32_t prev_stage = 0;
  for (int it = 0; it < k_iters; ++it) {
    mbar_wait(full_bar + stage * 8, phase);
#ifdef VP3D_TIMELINE
    if (tl_first && it == 0) TL(4);
#endif
    const uint32_t a_st = smem_a + stage * I::kABytes + a_off;
    uint64_t da[H];
#pragma unroll
    for (int h = 0; h < H; ++h) da[h] = make_gmma_desc_sw128(a_st + h * 64 * 128, 16, 1024);
    const uint64_t db = make_gmma_desc_sw128(smem_b + stage * I::kBBytes, 16, 1024);
#pragma unroll
    for (int h = 0; h < H; ++h) wgmma_fence_operands(acc[h]);
    wgmma_fence();
    if constexpr (I::kFmt != Fmt::kRuntime) wgmma_kblock<N, I::kFmt>(acc, da, db, it == 0);
    else if (f16) wgmma_kblock<N, Fmt::kF16>(acc, da, db, it == 0);
    else wgmma_kblock<N, Fmt::kBf16>(acc, da, db, it == 0);
    wgmma_commit();
#pragma unroll
    for (int h = 0; h < H; ++h) wgmma_fence_operands(acc[h]);
    if (it > 0) {
      // the previous k-block's MMAs have retired: its stage may be refilled
      wgmma_wait<1>();
#pragma unroll
      for (int h = 0; h < H; ++h) wgmma_fence_operands(acc[h]);
      if (lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
    }
    prev_stage = stage;
    if (++stage == I::kStages) { stage = 0; phase ^= 1; }
  }
  stage_io = stage; phase_io = phase;
  issued();
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < H; ++h) wgmma_fence_operands(acc[h]);
  if (k_iters > 0 && lane == 0) mbar_arrive(empty_bar + prev_stage * 8);
}

template <class I>
__global__ void __launch_bounds__(384, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a,
                 const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ CUtensorMap tmap_w64,
                 const __grid_constant__ CUtensorMap tmap_out,
                 const __grid_constant__ CUtensorMap tmap_res,
                 const __grid_constant__ CUtensorMap tmap_z, const ConvGemmArgs p) {
  using Acc = typename I::Acc;
  constexpr int kBlocksPerTile = I::kBlockN / 64;
  constexpr int kFrag = I::kBlockN / 2;   // accumulator registers per consumer thread
  constexpr int kBK = I::kI8 ? kBlockK8 : kBlockK;   // elements per k-block (128 bytes either way)

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024 B alignment
  uint8_t* smem = smem_raw + (base - raw_addr);

  const uint32_t smem_a = base;
  const uint32_t smem_b = base + I::kStages * I::kABytes;
  const uint32_t smem_store = base + I::kStages * I::kStageBytes;
  const uint32_t smem_res = smem_store + I::kStagingBytes;
  const uint32_t smem_u8 = smem_res + I::kResSlots * I::kTileBytes;   // (u8 beside the 16-bit plane)
  const uint32_t bar_base = smem_u8 + I::kU8Bytes;
  const uint32_t full_bar = bar_base;
  const uint32_t empty_bar = bar_base + I::kStages * 8;
  const uint32_t rfull_bar = bar_base + 2 * I::kStages * 8;   // up to 4 auxiliary stages
  const uint32_t rempty_bar = rfull_bar + 32;
  const uint32_t dep_bar = rempty_bar + 32;     // "the dependency wait has returned" (see the producer)
  const uint32_t affine_off = (dep_bar + 8 - base + 15u) & ~15u;   // [scale | shift][kBlockN]
  float* s_affine = reinterpret_cast<float*>(smem + affine_off);
  float* s_pairs = reinterpret_cast<float*>(smem + affine_off + I::kAffineBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) TL(0);

  const int m_tiles = p.dilated ? p.samples * p.tiles_per_sample : p.tiles_per_sample;
  const int total_tiles = m_tiles * p.n_tiles;
  // work items: whole tiles, then (128-wide ping-pong instances, planned by launch_impl) the last
  // half_items / 2 tiles as half_items 128 x 64 halves, at most one per CTA
  constexpr bool kHalves = I::kPP && I::kBlockN == 128;
  const int half_items = kHalves ? p.half_items : 0;
  const int full_tiles = total_tiles - half_items / 2;
  const int n_items = full_tiles + half_items;
  const int k_iters = p.pairs * p.taps * p.kblocks_per_tap;
  // auxiliary tiles per 64-column store block: the residual plane(s) and, for the fused
  // BatchNorm-backward reductions, the Z tile.  kResSlots / tiles stages are in flight.
  const bool has_res = (p.flags & kEpiResidual) != 0;
  const bool bnb = I::kTrain && p.bnb != 0;
  const int aux_tiles = (has_res ? p.res_planes : 0) + (bnb ? 1 : 0);
  const int res_stages =
      (aux_tiles > 0 && I::kResSlots >= aux_tiles) ? I::kResSlots / aux_tiles : 1;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    if (kHalves && half_items > 0) tma_prefetch_desc(&tmap_w64);
    tma_prefetch_desc(&tmap_out);
    if (I::kRes) tma_prefetch_desc(&tmap_res);
    if (I::kRes && bnb) tma_prefetch_desc(&tmap_z);
    if (I::kU8) tma_prefetch_desc(&tmap_z);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < I::kStages; ++s) {
      mbar_init(full_bar + s * 8, 1);
      // lane 0 of each consumer warp that reads the stage: all 8, or the 4 of one ping-pong warpgroup
      mbar_init(empty_bar + s * 8, I::kPP ? 4 : 8);
    }
    for (int s = 0; s < 4; ++s) {
      mbar_init(rfull_bar + s * 8, 1);
      // every consumer thread reads its rows of the stage; ping-pong: the thread that issued the
      // stores from the tile, once they have read it
      mbar_init(rempty_bar + s * 8, I::kPP ? 1 : 256);
    }
    mbar_init(dep_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) TL(1);
  // Everything above touched only this CTA's shared memory.  From here on global memory written by
  // the previous kernel of the stream is read: wait for it (no-op without PDL), then let the next
  // kernel start its own prologue on SMs this grid leaves.  The TMA producer thread waits inside its
  // own loop (below): in inference kernels it first streams the W tiles of the first pipeline
  // stages, which no kernel of the forward writes.  No lane of the producer's warp executes
  // griddepcontrol.wait (the instruction stalls the whole warp, diverged lanes included); warp 1
  // tells the producer through an mbarrier that the wait has returned -- the prerequisite grids'
  // writes are visible to the whole grid from then on.
  if (warp != 0) {
    griddep_wait();
    griddep_launch_dependents();
  }
  if (threadIdx.x == 32) {
    mbar_arrive(dep_bar);
    TL(2);
  }

  if (warp == 0) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      // Weights ahead of the dependency wait: the packed weights are written at plan build / by the
      // optimiser step, always at least one full kernel boundary (the input pack) before any conv
      // kernel of a forward, so they are safe to read while the previous layer is still running.
      // Training kernels keep the plain order (their weight packs change every step).
      constexpr bool kEarlyW = !I::kTrain;
      if (!kEarlyW) mbar_wait(dep_bar, 0);
      // mode 0: W only (before the wait), 1: the A tiles of those same stages, 2: steady state
      const int n_pre = kEarlyW ? (k_iters < I::kStages ? k_iters : I::kStages) : 0;
      int mode = n_pre > 0 ? 0 : 2;
      if (kEarlyW && mode == 2) mbar_wait(dep_bar, 0);
      // whole tiles first: w < full_tiles (a CTA's first item is always a whole tile)
      int w = blockIdx.x;
      if (w < full_tiles) {
        int n_blk, sample, row0;
        tile_coords(p, w, n_blk, sample, row0);
        uint32_t stage = 0, phase = 0;
        int it = 0, pair = 0, tap = 0, kb = 0;
        for (;;) {
          const int a_plane = (pair == 1) ? 1 : 0;
          const int w_plane = (pair == 2) ? 1 : 0;
          const uint32_t fb = full_bar + stage * 8;
          if (mode != 1) {
            mbar_wait(empty_bar + stage * 8, phase ^ 1);
            mbar_expect_tx(fb, I::kStageBytes);
            const int w_row = (w_plane * p.taps + tap) * p.n_pad + n_blk * I::kBlockN;
            tma_load_2d(&tmap_w, fb, smem_b + stage * I::kBBytes, kb * kBK, w_row);
          }
          if (mode != 0) {
            const int a_row = row0 + tap * p.tap_row_step;
            const int a_col = tap * p.tap_col_step + kb * kBK;
            tma_load_4d(&tmap_a, fb, smem_a + stage * I::kABytes, a_col, a_row, sample, a_plane);
#ifdef VP3D_TIMELINE
            if (w == (int)blockIdx.x && it == 0) TL(3);
#endif
          }
          if (++stage == I::kStages) { stage = 0; phase ^= 1; }
          ++it;
          if (++kb == p.kblocks_per_tap) {
            kb = 0;
            if (++tap == p.taps) { tap = 0; ++pair; }
          }
          if (mode == 0 && it == n_pre) {
            mbar_wait(dep_bar, 0);
            mode = 1;   // rewind: the A tiles of the stages just primed
            it = 0; pair = 0; tap = 0; kb = 0;
            stage = 0; phase = 0;
          } else if (mode == 1 && it == n_pre) {
            mode = 2;
          }
          if (it == k_iters) {
            w += gridDim.x;
            if (w >= full_tiles) break;
            tile_coords(p, w, n_blk, sample, row0);
            it = 0; pair = 0; tap = 0; kb = 0;
          }
        }
        if constexpr (kHalves) {
          // then the CTA's half tile, if it has one (its last item, see item_coords): the whole A
          // tile and the 64 W rows of its columns (box of tmap_w64) into the first half of the
          // stage's W slot.  (Kept out of the loop above, which stays the whole-tile loop.)
          if (w < n_items) {
            int c_off;
            item_coords(p, full_tiles, w, n_blk, sample, row0, c_off);
            for (int h_it = 0, h_pair = 0, h_tap = 0, h_kb = 0; h_it < k_iters; ++h_it) {
              const uint32_t fb = full_bar + stage * 8;
              mbar_wait(empty_bar + stage * 8, phase ^ 1);
              mbar_expect_tx(fb, I::kABytes + I::kBBytes / 2);
              const int w_row = ((h_pair == 2 ? 1 : 0) * p.taps + h_tap) * p.n_pad +
                                n_blk * I::kBlockN + c_off;
              tma_load_2d(&tmap_w64, fb, smem_b + stage * I::kBBytes, h_kb * kBK, w_row);
              tma_load_4d(&tmap_a, fb, smem_a + stage * I::kABytes,
                          h_tap * p.tap_col_step + h_kb * kBK, row0 + h_tap * p.tap_row_step,
                          sample, h_pair == 1 ? 1 : 0);
              if (++stage == I::kStages) { stage = 0; phase ^= 1; }
              if (++h_kb == p.kblocks_per_tap) {
                h_kb = 0;
                if (++h_tap == p.taps) { h_tap = 0; ++h_pair; }
              }
            }
          }
        }
      }
    }
  } else if (warp == 1) {
    // ------------------------------------------------------------ auxiliary-tile producer
    if (I::kPP && I::kRes && lane == 0) {
      // ping-pong: the residual tiles in tile order; tile j goes to warpgroup j & 1, whose two
      // landing slots (2 g, 2 g + 1) form a ring of their own
      uint32_t filled[2] = {0u, 0u};   // residual tiles sent to warpgroup 0 / 1 so far
      for (int j = 0, w = blockIdx.x; w < n_items; ++j, w += gridDim.x) {
        int n_blk, sample, row0, c_off;
        const bool half = item_coords(p, full_tiles, w, n_blk, sample, row0, c_off);
        const int g = j & 1;
        for (int sb = 0; sb < (half ? 1 : kBlocksPerTile); ++sb) {
          const uint32_t n = g ? filled[1] : filled[0];
          const uint32_t slot = 2u * g + (n & 1u);
          mbar_wait(rempty_bar + slot * 8, ((n >> 1) & 1u) ^ 1u);
          mbar_expect_tx(rfull_bar + slot * 8, I::kTileBytes);
          tma_load_4d(&tmap_res, rfull_bar + slot * 8, smem_res + slot * I::kTileBytes,
                      n_blk * I::kBlockN + c_off + sb * 64 + p.res_tma_col_off,
                      row0 + p.res_tma_row_off,
                      sample, 0);
          if (g) ++filled[1];
          else ++filled[0];
        }
      }
    } else if (!I::kPP && I::kRes && lane == 0) {
      uint32_t rs = 0, rphase = 0;
      for (int w = blockIdx.x; w < total_tiles; w += gridDim.x) {
        int n_blk, sample, row0;
        tile_coords(p, w, n_blk, sample, row0);
        for (int sb = 0; sb < kBlocksPerTile; ++sb) {
          const int col = n_blk * I::kBlockN + sb * 64;
          const bool res_here = has_res && col >= p.res_col_begin && col < p.res_col_begin + p.res_cols;
          if (!res_here && !bnb) continue;
          const int n_res = res_here ? p.res_planes : 0;
          mbar_wait(rempty_bar + rs * 8, rphase ^ 1);
          mbar_expect_tx(rfull_bar + rs * 8, (n_res + (bnb ? 1 : 0)) * I::kTileBytes);
          const uint32_t slot0 = smem_res + rs * aux_tiles * I::kTileBytes;
          for (int pl = 0; pl < n_res; ++pl)
            tma_load_4d(&tmap_res, rfull_bar + rs * 8, slot0 + pl * I::kTileBytes,
                        col - p.res_col_begin + p.res_tma_col_off, row0 + p.res_tma_row_off, sample,
                        pl);
          if (bnb)  // the Z tile always sits in the last slot of the stage
            tma_load_4d(&tmap_z, rfull_bar + rs * 8, slot0 + (aux_tiles - 1) * I::kTileBytes, col,
                        row0, sample, 0);
          if (++rs == (uint32_t)res_stages) { rs = 0; rphase ^= 1; }
        }
      }
    }
  } else if (I::kPP && warp >= 4) {
    // ------------------------------------------------------------ ping-pong MMA + lean epilogue
    // Warpgroup g computes all 128 rows of the CTA's tiles j = g, g + 2, ... (w = blockIdx.x +
    // j gridDim.x): per k16 step one m64 wgmma per 64-row half of the A stage, into acc[0] and
    // acc[1].  The warpgroups issue their k-loops in tile order, taking turns through two named
    // barriers (8 + g: "warpgroup g may issue"), so that one warpgroup's epilogue runs under the
    // other's MMAs.  Because the k-loops are ordered, every earlier fill of a stage has been
    // consumed before a warpgroup waits on it, and the parity wait is exact.
    const int wg = (warp - 4) >> 2;
    const int wq = warp & 3;
    const int tid = (int)threadIdx.x - 128 - 128 * wg;
    const int rl0 = 16 * wq + (lane >> 2);   // this thread's rows in each 64-row half: rl0, rl0 + 8
    const int cq = 2 * (lane & 3);
    const uint32_t bar_wg = 2u + (uint32_t)wg;
    const uint32_t bar_mine = 8u + (uint32_t)wg, bar_other = 9u - (uint32_t)wg;
    const uint32_t staging = smem_store + wg * I::kTileBytes;   // (no-residual instance)
    uint32_t res_seen = 0;            // residual tiles this warpgroup has received
    Acc acc[2][kFrag];
#pragma unroll
    for (int i = 0; i < kFrag; ++i) acc[0][i] = acc[1][i] = 0.0f;

    // Item j = w's k-loop and epilogue; kHalf: a half tile (one 64-column store block, n64 MMAs
    // into the first 64 columns of acc).  The loop below runs the whole tiles; a half tile is
    // always a CTA's last item (launch_impl gives at most one to a CTA), so it runs after the loop
    // from a copy of its own, and the loop keeps the registers of the whole-tile path alone.
    const auto run_item = [&](int j, int w, auto half_tag) {
      constexpr bool kHalf = decltype(half_tag)::value;
      constexpr int kSb = kHalf ? 1 : kBlocksPerTile;   // 64-column store blocks
      int n_blk, sample, row0, c_off = 0;
      if constexpr (kHalf) item_coords(p, full_tiles, w, n_blk, sample, row0, c_off);
      else tile_coords(p, w, n_blk, sample, row0);

      // ---- main loop: k-block it of item j sits in the producer's (j k_iters + it)-th fill
      const uint32_t fill = (uint32_t)j * (uint32_t)k_iters;
      uint32_t stage = fill % I::kStages, phase = (fill / I::kStages) & 1u;
      if (j > 0) named_bar_sync(bar_mine, 256);   // item j - 1's k-loop has been issued
      mma_tile<I, kHalf ? 64 : I::kBlockN>(
          acc, p, I::kF16, smem_a, 0u, smem_b, full_bar, empty_bar, stage, phase, k_iters, lane,
          warp == 4 && lane == 0 && w == (int)blockIdx.x, [&] {
            // item j + 1 may issue
            if (w + (int)gridDim.x < n_items) named_bar_arrive(bar_other, 256);
          });
#ifdef VP3D_TIMELINE
      if (warp == 4 && lane == 0) { if (w == (int)blockIdx.x) TL(7); TL(8); }
#endif

      const float* scale = p.scale + n_blk * I::kBlockN + c_off;
      const float* shift = p.shift + n_blk * I::kBlockN + c_off;
#pragma unroll
      for (int sb = 0; sb < kSb; ++sb) {
        const int cb = n_blk * I::kBlockN + c_off + sb * 64;   // first column of the store block
        uint32_t tile_smem;
        if constexpr (I::kRes) {
          // in place: every thread overwrites the residual elements it adds with its results
          const uint32_t slot = 2u * wg + (res_seen & 1u);
          mbar_wait(rfull_bar + slot * 8, (res_seen >> 1) & 1u);
          ++res_seen;
          tile_smem = smem_res + slot * I::kTileBytes;
          if constexpr (I::kU8) {
            // the u8 tile must have been read out by the bulk stores issued from it last
            if (tid == 0) tma_store_wait_read<0>();
            named_bar_sync(bar_wg, 128);
          }
        } else {
          // the staging tile must have been read out by the bulk stores issued from it last
          if (tid == 0) tma_store_wait_read<0>();
          named_bar_sync(bar_wg, 128);
          tile_smem = staging;
        }
        // u8 tile of this warpgroup: 128 rows of 64 bytes (u8 alone: inside the 16-bit staging)
        const uint32_t u8_tile = I::kU8Alone ? staging : smem_u8 + (uint32_t)wg * (kBlockM * 64);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j4 = 4 * (sb * 8 + jj);
          const int cl = sb * 64 + jj * 8 + cq;   // column inside the N block
          const float2 sc = __ldg(reinterpret_cast<const float2*>(scale + cl));
          const float2 sh = __ldg(reinterpret_cast<const float2*>(shift + cl));
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = fmaxf(fmaf(static_cast<float>(acc[h2][j4 + 2 * h]), sc.x, sh.x), 0.0f);
              float v1 = fmaxf(fmaf(static_cast<float>(acc[h2][j4 + 2 * h + 1]), sc.y, sh.y), 0.0f);
              const uint32_t off = sw128_off(64 * h2 + rl0 + 8 * h, jj * 8 + cq);
              if (I::kRes) add_pair(v0, v1, ld_shared_u32(tile_smem + off), I::kF16);
              if constexpr (I::kStore16)
                st_shared_u32(tile_smem + off, I::kF16 ? pack_f16x2(v0, v1) : pack_bf16x2(v0, v1));
              if constexpr (I::kU8)
                st_u8_pair(u8_tile + (uint32_t)(64 * h2 + rl0 + 8 * h) * 64u + jj * 8 + cq, v0, v1,
                           p.u8_inv_s);
            }
          }
        }
        fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA engine
        named_bar_sync(bar_wg, 128);
        if (tid == 0) {
          // four 32-row boxes: 4 KiB-aligned quarters of the tile, same swizzle phase as written
#pragma unroll
          for (int hb = 0; hb < 4; ++hb) {
            if constexpr (I::kStore16)
              tma_store_4d(&tmap_out, tile_smem + hb * 4096u, cb, row0 + 32 * hb, sample, 0);
            // (u8 instances are lean, never BatchNorm-backward: tmap_z maps the u8 plane)
            if constexpr (I::kU8)
              tma_store_4d(&tmap_z, u8_tile + hb * 2048u, cb, row0 + 32 * hb, sample, 0);
          }
          tma_store_commit();
        }
      }
      if (I::kRes && tid == 0) {
        // the landing tiles go back to the auxiliary producer once the stores have read them
        tma_store_wait_read<0>();
#pragma unroll
        for (int sb = 0; sb < kSb; ++sb)
          mbar_arrive(rempty_bar + (2u * wg + ((res_seen - kSb + sb) & 1u)) * 8);
      }
#ifdef VP3D_TIMELINE
      if (warp == 4 && lane == 0) { if (w == (int)blockIdx.x) TL(9); TL(10); }
#endif
    };
    int j = wg, w = blockIdx.x + wg * gridDim.x;
    for (; w < full_tiles; j += 2, w += 2 * gridDim.x) run_item(j, w, std::false_type{});
    if constexpr (kHalves) {
      if (w < n_items) run_item(j, w, std::true_type{});
    }
    // the staging tiles must outlive every bulk store that reads them
    if (tid == 0) tma_store_wait_all<0>();
#ifdef VP3D_TIMELINE
    if (warp == 4 && lane == 0) TL(11);
#endif
  } else if (!I::kPP && warp >= 4) {
    // ------------------------------------------------------------ MMA + epilogue (two warpgroups)
    const int wg = (warp - 4) >> 2;   // rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp & 3;          // warp inside the warpgroup: 16 rows each
    const int tid = (int)threadIdx.x - 128 - 128 * wg;
    const int rl0 = 16 * wq + (lane >> 2);   // this thread's rows inside the warpgroup's 64: rl0, rl0+8
    const int cq = 2 * (lane & 3);           // first of this thread's two columns in every 8
    const uint32_t bar_wg = 2u + (uint32_t)wg;               // named barrier: this warpgroup
    const uint32_t bar_slab = 4u + (uint32_t)(wg * 2 + (wq >> 1));   // the two warps of a slab
    float* s_pair = s_pairs + (wg * 2 + (wq >> 1)) * 128;
    // IEEE fp16 operands / storage instead of bf16 (eval fp16 mode)
    const bool f16 = I::kLean ? I::kF16 : p.f16 != 0;
    const bool do_relu = I::kLean || (p.flags & kEpiRelu);
    const bool do_res = I::kLean ? I::kRes : (p.flags & kEpiResidual) != 0;
    const bool do_stats = I::kTrain && (p.flags & kEpiStats);
    const bool do_f32 = !I::kLean && (p.flags & kEpiOutF32);
    const bool do_affine = I::kLean || (p.flags & kEpiAffine);
    const bool two_planes = I::kOut2 && p.out_planes == 2;
    uint32_t stage = 0, phase = 0;
    uint32_t ablock = 0;              // auxiliary stages seen so far
    uint32_t sbuf = 0;                // staging buffer of the next store block
    int aff_n_blk = -1;               // N block whose scale / shift sit in shared memory
    Acc acc[1][kFrag];
#pragma unroll
    for (int i = 0; i < kFrag; ++i) acc[0][i] = 0.0f;

    for (int w = blockIdx.x; w < total_tiles; w += gridDim.x) {
      int n_blk, sample, row0;
      tile_coords(p, w, n_blk, sample, row0);
      const int m_blk = w / p.n_tiles;  // row-tile index: 4 slabs of 32 rows each

      // ---- main loop: wgmma over this warpgroup's 64 rows, one k-block per pipeline stage; its
      // rows of the A tile start 8 KiB in (a whole number of swizzle atoms)
      mma_tile<I>(acc, p, f16, smem_a, wg * 64 * 128, smem_b, full_bar, empty_bar, stage, phase,
                  k_iters, lane, warp == 4 && lane == 0 && w == (int)blockIdx.x, [] {});
#ifdef VP3D_TIMELINE
      if (warp == 4 && lane == 0) { if (w == (int)blockIdx.x) TL(7); TL(8); }
#endif

      // Per-channel affine of this N block: staged once in shared memory (the 256 consumer threads,
      // two barriers per change of N block, none while it stays the same -- the usual case).
      if (do_affine && n_blk != aff_n_blk) {
        named_bar_sync(1, 256);
        const int e = (int)threadIdx.x - 128;
        if (e < I::kBlockN) {
          s_affine[e] = __ldg(p.scale + n_blk * I::kBlockN + e);
          s_affine[I::kBlockN + e] = __ldg(p.shift + n_blk * I::kBlockN + e);
        }
        named_bar_sync(1, 256);
        aff_n_blk = n_blk;
      }

      // rows of this thread: tile rows rt[0] = 64 wg + rl0 and rt[1] = rt[0] + 8
      int t_in[2];
      bool valid[2];
      long long out_row[2], res_row[2];
      bool res_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rt = 64 * wg + rl0 + 8 * h;
        t_in[h] = row0 + rt;
        valid[h] = t_in[h] < p.out_rows;
        out_row[h] = (long long)sample * p.out_rows + t_in[h];
        res_row[h] = 0;
        res_ok[h] = valid[h];
        if (!I::kRes) {
          int rsmp = sample, rtt = t_in[h];
          if (!p.dilated && p.res_sample_div > 0) {
            rsmp = t_in[h] / p.res_sample_div;
            rtt = t_in[h] - rsmp * p.res_sample_div;
          }
          const long long in_sample = (long long)rtt * p.res_row_step + p.res_row_off;
          if (p.res_check_rows && (in_sample < 0 || in_sample >= p.res_rows_per_sample)) res_ok[h] = false;
          res_row[h] = (long long)rsmp * p.res_rows_per_sample + in_sample;
        }
      }
      // lo plane only where somebody reads it (tile-uniform)
      const bool two_planes_t =
          two_planes && (p.dilated || (row0 < p.lo_row_end && row0 + kBlockM > p.lo_row_begin));

#pragma unroll
      for (int sb = 0; sb < kBlocksPerTile; ++sb) {
        const int cb = n_blk * I::kBlockN + sb * 64;  // first column of the store block
        const bool res_here = do_res && cb >= p.res_col_begin && cb < p.res_col_begin + p.res_cols;
        const bool aux_here = I::kRes && (res_here || bnb);
        const uint32_t rs = aux_here ? ablock % (uint32_t)res_stages : 0u;
        const uint32_t rphase = aux_here ? (ablock / (uint32_t)res_stages) & 1u : 0u;
        if (aux_here) {
          ++ablock;
          mbar_wait(rfull_bar + rs * 8, rphase);  // tiles have landed
        }
        const uint32_t aux0 = smem_res + (rs * aux_tiles) * I::kTileBytes;
        // this warpgroup's staging slice(s): [hi] or [hi, lo], 64 rows x 128 B each
        const uint32_t my_store = smem_store + (wg * 2 + sbuf) * (I::kOut2 ? 2 : 1) * I::kHalfBytes;
        // its u8 slice: 64 rows of 64 bytes (u8 alone: inside the 16-bit slice)
        const uint32_t my_u8 = I::kU8Alone ? my_store : smem_u8 + (uint32_t)(wg * 2 + sbuf) * (64 * 64);
        if (!do_f32) {
          // The slice must have been read out by the bulk store issued from it two blocks ago.
          if (tid == 0) tma_store_wait_read<1>();
          named_bar_sync(bar_wg, 128);
        }
        float ss[8][2], sq[8][2];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = sb * 8 + jj;
          const int cl = sb * 64 + jj * 8 + cq;   // column inside the N block
          const int c = cb + jj * 8 + cq;         // output column
          float v[2][2] = {{static_cast<float>(acc[0][4 * j]), static_cast<float>(acc[0][4 * j + 1])},
                           {static_cast<float>(acc[0][4 * j + 2]), static_cast<float>(acc[0][4 * j + 3])}};
          if (do_affine) {
            const float2 sc = *reinterpret_cast<const float2*>(s_affine + cl);
            const float2 sh = *reinterpret_cast<const float2*>(s_affine + I::kBlockN + cl);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              v[h][0] = fmaf(v[h][0], sc.x, sh.x);
              v[h][1] = fmaf(v[h][1], sc.y, sh.y);
            }
          }
          if (do_relu) {
#pragma unroll
            for (int h = 0; h < 2; ++h) { v[h][0] = fmaxf(v[h][0], 0.0f); v[h][1] = fmaxf(v[h][1], 0.0f); }
          }
          if (I::kRes) {
            if (res_here) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t off = sw128_off(64 * wg + rl0 + 8 * h, jj * 8 + cq);
                add_pair(v[h][0], v[h][1], ld_shared_u32(aux0 + off), f16);
                for (int pl = 1; pl < p.res_planes; ++pl)   // lo plane of a split-bf16 residual
                  add_pair(v[h][0], v[h][1], ld_shared_u32(aux0 + pl * I::kTileBytes + off), false);
              }
            }
          } else if (res_here) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (!res_ok[h]) continue;
              const __nv_bfloat16* rp = p.res + res_row[h] * p.res_ld + (c - p.res_col_begin);
#pragma unroll
              for (int pl = 0; pl < 2; ++pl) {
                if (pl < p.res_planes) {
                  const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(rp + pl * p.res_plane_stride));
                  add_pair(v[h][0], v[h][1], u, f16 && pl == 0);
                }
              }
            }
          }
          if (do_f32) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (!valid[h]) continue;
              float* op = p.out_f32 + out_row[h] * p.out_f32_ld + c;
              if (c < p.n_valid) op[0] = v[h][0];
              if (c + 1 < p.n_valid) op[1] = v[h][1];
            }
          } else {
            if constexpr (I::kU8) {
#pragma unroll
              for (int h = 0; h < 2; ++h)
                st_u8_pair(my_u8 + (uint32_t)(rl0 + 8 * h) * 64u + jj * 8 + cq, v[h][0], v[h][1],
                           p.u8_inv_s);
            }
#pragma unroll
            for (int h = 0; h < 2 && I::kStore16; ++h) {
              const uint32_t hi = f16 ? pack_f16x2(v[h][0], v[h][1]) : pack_bf16x2(v[h][0], v[h][1]);
              const uint32_t off = sw128_off(rl0 + 8 * h, jj * 8 + cq);
              st_shared_u32(my_store + off, hi);
              if (two_planes_t) {
                const uint32_t lo = pack_bf16x2(v[h][0] - bf16_lo_to_f(hi), v[h][1] - bf16_hi_to_f(hi));
                st_shared_u32(my_store + I::kHalfBytes + off, lo);
              }
            }
          }
          if (I::kRes && bnb) {
            // dY = G(as stored) * dropmask/(1-p) * [Z*scale+shift > 0]; sums over the slab's rows
            const int ch = c % p.bnb_c;   // channel of the layer below (columns repeat per tap)
            const bool drop = p.bnb_p > 0.0f;
            const uint32_t thresh = (uint32_t)(p.bnb_p * 65536.0f);
            const float inv_keep = drop ? 1.0f / (1.0f - p.bnb_p) : 1.0f;
            ss[jj][0] = ss[jj][1] = sq[jj][0] = sq[jj][1] = 0.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t zu =
                  ld_shared_u32(aux0 + (aux_tiles - 1) * I::kTileBytes + sw128_off(64 * wg + rl0 + 8 * h, jj * 8 + cq));
              const float z2[2] = {bf16_lo_to_f(zu), bf16_hi_to_f(zu)};
              // mask hash of the element pair (c, c + 1), keyed by the 32-column chunk it lies in
              const int c0 = c & ~31;
              const unsigned long long elem0 = (unsigned long long)out_row[h] * p.out_ld + c0;
              const uint32_t key = p.bnb_seed_lo ^ (p.bnb_seed_hi * 0x7F4A7C15u) ^
                                   (p.bnb_layer * 0x632BE5ABu) ^
                                   ((uint32_t)((elem0 >> 1) >> 32) * 0x85EBCA77u);
              float m[2] = {1.0f, 1.0f};
              if (drop) {
                uint32_t hh = ((uint32_t)(elem0 >> 1) + (uint32_t)((c - c0) >> 1)) * 0x9E3779B1u + key;
                hh ^= hh >> 16; hh *= 0x85EBCA6Bu; hh ^= hh >> 13; hh *= 0xC2B2AE35u; hh ^= hh >> 16;
                m[0] = ((hh & 0xFFFFu) >= thresh) ? inv_keep : 0.0f;
                m[1] = ((hh >> 16) >= thresh) ? inv_keep : 0.0f;
              }
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                // gradient exactly as the next pass will read it back (bf16-rounded)
                const float g = __bfloat162float(__float2bfloat16_rn(v[h][e]));
                const float y = fmaf(z2[e], __ldg(p.bnb_scale + ch + e), __ldg(p.bnb_shift + ch + e));
                float dy = (valid[h] && y > 0.0f) ? g : 0.0f;
                dy *= m[e];
                ss[jj][e] += dy;
                sq[jj][e] += dy * (z2[e] - __ldg(p.bnb_mean + ch + e));
              }
            }
          } else if (do_stats) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x0 = valid[0] ? v[0][e] : 0.0f;
              const float x1 = valid[1] ? v[1][e] : 0.0f;
              ss[jj][e] = x0 + x1;
              sq[jj][e] = x0 * x0 + x1 * x1;
            }
          }
        }
        if (I::kRes && aux_here) mbar_arrive(rempty_bar + rs * 8);  // this thread is done with the stage
        if (I::kTrain && ((I::kRes && bnb) || do_stats)) {
          // per-slab (32 rows) partials, summed in a fixed order afterwards (bn_stats_finalize /
          // launch_ordered_col_sums): run-to-run reproducible, unlike atomics
          slab_reduce(ss, sq, s_pair, lane, wq, bar_slab);
          if (!(wq & 1) && lane < 4) {
            float* sp = ((I::kRes && bnb) ? p.bnb_sums : p.stats) +
                        ((size_t)(m_blk * 4 + 2 * wg + (wq >> 1)) * 2) * p.n_pad + cb + 2 * lane;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              sp[8 * jj] = ss[jj][0];
              sp[8 * jj + 1] = ss[jj][1];
              sp[p.n_pad + 8 * jj] = sq[jj][0];   // (bnb: x invstd is applied after the ordered sum)
              sp[p.n_pad + 8 * jj + 1] = sq[jj][1];
            }
          }
        }
        if (!do_f32) {
          fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA engine
          named_bar_sync(bar_wg, 128);
          if (tid == 0) {
            // two 32-row boxes: 4 KiB-aligned halves of the slice, same swizzle phase as written
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
              const int r = row0 + 64 * wg + 32 * hb;
              if constexpr (I::kStore16) tma_store_4d(&tmap_out, my_store + hb * 4096u, cb, r, sample, 0);
              // (u8 instances are lean, never BatchNorm-backward: tmap_z maps the u8 plane)
              if constexpr (I::kU8) tma_store_4d(&tmap_z, my_u8 + hb * 2048u, cb, r, sample, 0);
              if (two_planes_t) tma_store_4d(&tmap_out, my_store + I::kHalfBytes + hb * 4096u, cb, r, sample, 1);
            }
            tma_store_commit();
          }
          sbuf ^= 1u;
        }
      }
#ifdef VP3D_TIMELINE
      if (warp == 4 && lane == 0) { if (w == (int)blockIdx.x) TL(9); TL(10); }
#endif
    }
    // the staging tiles must outlive every bulk store that reads them
    if (tid == 0) tma_store_wait_all<0>();
#ifdef VP3D_TIMELINE
    if (warp == 4 && lane == 0) TL(11);
#endif
  }
}

// Programmatic dependent launch (on by default, VP3D_PDL=0 turns it off): the next kernel of the
// stream may start its prologue (barrier init, descriptor prefetch) on SMs this grid has already
// left; its griddepcontrol.wait still orders every global access behind the completion of this grid.
static int g_pdl = -1;   // -1: not decided yet (VP3D_PDL, default on); conv_gemm_set_pdl overrides
static bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("VP3D_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl != 0;
}
void conv_gemm_set_pdl(int on) { g_pdl = on ? 1 : 0; }
bool conv_gemm_pdl_enabled() { return pdl_enabled(); }

static int conv_tiles(const ConvGemmArgs& a) {
  const int m_tiles = a.dilated ? a.samples * a.tiles_per_sample : a.tiles_per_sample;
  return m_tiles * a.n_tiles;
}

template <class I>
static cudaError_t launch_impl(const CUtensorMap& tmap_a, const CUtensorMap& tmap_w,
                               const CUtensorMap& tmap_w64, const CUtensorMap& tmap_out,
                               const CUtensorMap& tmap_res, const CUtensorMap& tmap_z,
                               const ConvGemmArgs& args_in, int num_sms, cudaStream_t stream) {
  auto kernel = conv_gemm_kernel<I>;
  // the dynamic shared memory opt-in is a per-device attribute
  static bool attr_set[kMaxDevices] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
  if (!attr_set[dev]) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, I::kSmemBytes);
    if (e != cudaSuccess) return e;
    attr_set[dev] = true;
  }
  const int total = conv_tiles(args_in);
  if (total <= 0) return cudaSuccess;
  const int workers = total < num_sms ? total : num_sms;
  // The last wave of a 128-wide ping-pong launch: its `left` tiles would keep `left` SMs busy for
  // a whole tile while the other workers - left wait.  Where they fit twice into the grid they run
  // as 2 left half tiles of 128 x 64 instead, one per CTA, each about half as long.  The plan
  // follows from the tile count and the grid alone, and a half tile stores the bits of the whole
  // one (the same k order and n64 instruction path as the 64-wide instances).
  ConvGemmArgs args = args_in;
  args.half_items = 0;
  if constexpr (I::kPP && I::kBlockN == 128) {
    const int left = total % workers;
    if (left > 0 && 2 * left <= workers) args.half_items = 2 * left;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(workers, 1, 1);
  cfg.blockDim = dim3(384, 1, 1);
  cfg.dynamicSmemBytes = I::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int n_attr = 0;
  if (pdl_enabled()) {
    attr[n_attr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n_attr].val.programmaticStreamSerializationAllowed = 1;
    ++n_attr;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n_attr;
  return cudaLaunchKernelEx(&cfg, kernel, tmap_a, tmap_w, tmap_w64, tmap_out, tmap_res, tmap_z,
                            args);
}

// Lean inference epilogue (VP3D_LEAN=0 falls back to the general one): exactly affine + ReLU
// [+ a one-plane TMA residual over every column] into one 16-bit plane.
static bool lean_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VP3D_LEAN");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}
static bool lean_ok(const ConvGemmArgs& a, bool res) {
  if (!lean_enabled() || a.bnb || a.out_planes != 1 || !a.out) return false;
  if (!res) return a.flags == (kEpiAffine | kEpiRelu) && !a.res_tma;
  return a.flags == (kEpiAffine | kEpiRelu | kEpiResidual) && a.res_tma && a.res_planes == 1 &&
         a.res_col_begin == 0 && a.res_cols >= a.n_pad;
}

// The instance a launch runs.  run_conv has checked the int8 / u8 combinations already.
static InstKey select_instance(const ConvGemmArgs& a, int block_n, bool multi_tile) {
  InstKey k = {block_n, Epi::kGeneral, Fmt::kRuntime, Sched::kCooperative, a.res_tma || a.bnb,
               a.out_planes == 2 && !(a.flags & kEpiOutF32), U8Out::kNone};
  if ((a.flags & kEpiStats) || a.bnb) {
    k.epi = Epi::kTrain;
    return k;
  }
  // the int8 and u8-output launches have no general counterpart: always lean
  const bool quant = a.i8 || a.out_u8;
  if (!quant && (k.out2 || !lean_ok(a, k.res))) return k;
  k.epi = Epi::kLean;
  k.fmt = a.i8 ? Fmt::kI8 : a.f16 ? Fmt::kF16 : Fmt::kBf16;
  if (a.out_u8) k.u8 = a.out ? U8Out::kBeside : U8Out::kAlone;
  // Ping-pong pays only where a CTA gets a second tile whose MMAs can run under the first tile's
  // epilogue; with one tile per CTA both warpgroups share it (cooperative).
  if (multi_tile) k.sched = Sched::kPingPong;
  return k;
}

template <class... Is>
struct InstList {};

// Every compiled instance, for BN = 128 and 64.
template <int BN>
using Instances = InstList<
    // training forward and data-gradient GEMMs: [residual / BatchNorm-backward Z] x [two planes]
    Inst<BN, Epi::kTrain, Fmt::kRuntime, Sched::kCooperative, false, false>,
    Inst<BN, Epi::kTrain, Fmt::kRuntime, Sched::kCooperative, false, true>,
    Inst<BN, Epi::kTrain, Fmt::kRuntime, Sched::kCooperative, true, false>,
    Inst<BN, Epi::kTrain, Fmt::kRuntime, Sched::kCooperative, true, true>,
    // every other eval launch: the shrink (fp32), split-bf16, register-path residuals, VP3D_LEAN=0
    Inst<BN, Epi::kGeneral, Fmt::kRuntime, Sched::kCooperative, false, false>,
    Inst<BN, Epi::kGeneral, Fmt::kRuntime, Sched::kCooperative, false, true>,
    Inst<BN, Epi::kGeneral, Fmt::kRuntime, Sched::kCooperative, true, false>,
    Inst<BN, Epi::kGeneral, Fmt::kRuntime, Sched::kCooperative, true, true>,
    // lean 16-bit inference layers: format x schedule x [residual]
    Inst<BN, Epi::kLean, Fmt::kBf16, Sched::kCooperative, false>,
    Inst<BN, Epi::kLean, Fmt::kBf16, Sched::kCooperative, true>,
    Inst<BN, Epi::kLean, Fmt::kBf16, Sched::kPingPong, false>,
    Inst<BN, Epi::kLean, Fmt::kBf16, Sched::kPingPong, true>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kCooperative, false>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kCooperative, true>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kPingPong, false>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kPingPong, true>,
    // the int8 chain, per schedule: H (u8 alone), X_i (fp16 [+ u8]), the fp16 expand with Q_0
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kCooperative, false, false, U8Out::kAlone>,
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kCooperative, true, false, U8Out::kNone>,
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kCooperative, true, false, U8Out::kBeside>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kCooperative, false, false, U8Out::kBeside>,
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kPingPong, false, false, U8Out::kAlone>,
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kPingPong, true, false, U8Out::kNone>,
    Inst<BN, Epi::kLean, Fmt::kI8, Sched::kPingPong, true, false, U8Out::kBeside>,
    Inst<BN, Epi::kLean, Fmt::kF16, Sched::kPingPong, false, false, U8Out::kBeside>>;

// launch_impl of the listed instance whose key is k (cudaErrorInvalidValue if none is)
template <class... Is>
static cudaError_t launch_listed(InstList<Is...>, const InstKey& k, const CUtensorMap& a,
                                 const CUtensorMap& w, const CUtensorMap& w64,
                                 const CUtensorMap& o, const CUtensorMap& r,
                                 const CUtensorMap& z, const ConvGemmArgs& args, int num_sms,
                                 cudaStream_t stream) {
  cudaError_t e = cudaErrorInvalidValue;
  (void)((k == Is::kKey &&
          ((e = launch_impl<Is>(a, w, w64, o, r, z, args, num_sms, stream)), true)) ||
         ...);
  return e;
}

#ifdef VP3D_TIMELINE
static unsigned long long* g_timeline = nullptr;
static int g_timeline_max = 0, g_timeline_next = 0;
void conv_gemm_debug_set_timeline(unsigned long long* buf, int max_launches) {
  g_timeline = buf;
  g_timeline_max = max_launches;
  g_timeline_next = 0;
}
#endif

// The instance a launch of `args` at tile width block_n on num_sms SMs runs (launch_conv_gemm and
// conv_gemm_instance both ask here)
static InstKey launch_key(const ConvGemmArgs& args, int block_n, int num_sms) {
  return select_instance(args, block_n, conv_tiles(args) > num_sms);
}

template <class... Is>
static bool listed(InstList<Is...>, const InstKey& k) {
  return ((k == Is::kKey) || ...);
}

static void key_ints(const InstKey& k, int* out) {
  out[0] = k.block_n;
  out[1] = (int)k.epi;
  out[2] = (int)k.fmt;
  out[3] = (int)k.sched;
  out[4] = k.res ? 1 : 0;
  out[5] = k.out2 ? 1 : 0;
  out[6] = (int)k.u8;
}

bool conv_gemm_instance(const ConvGemmArgs& args, int block_n, int num_sms, int key[7]) {
  const InstKey k = launch_key(args, block_n, num_sms);
  key_ints(k, key);
  return block_n == 128 ? listed(Instances<128>{}, k) : listed(Instances<64>{}, k);
}

// the keys of a list's instances into keys[7 i], at most max of them; returns the list's length
template <class... Is>
static int list_keys(InstList<Is...>, int* keys, int max) {
  const InstKey all[] = {Is::kKey...};
  const int n = (int)sizeof...(Is);
  for (int i = 0; i < n && i < max; ++i) key_ints(all[i], keys + 7 * i);
  return n;
}

int conv_gemm_instances(int* keys, int max) {
  const int n128 = list_keys(Instances<128>{}, keys, max);
  const int done = n128 < max ? n128 : max;
  return n128 + list_keys(Instances<64>{}, keys + 7 * done, max - done);
}

cudaError_t launch_conv_gemm(const CUtensorMap& tmap_a, const CUtensorMap& tmap_w,
                             const CUtensorMap& tmap_w64, const CUtensorMap& tmap_out,
                             const CUtensorMap& tmap_res, const CUtensorMap& tmap_z,
                             const ConvGemmArgs& args_in, int block_n, int num_sms,
                             cudaStream_t stream) {
#ifdef VP3D_TIMELINE
  ConvGemmArgs args = args_in;
  args.timeline = (g_timeline && g_timeline_next < g_timeline_max)
                      ? g_timeline + (size_t)(g_timeline_next++) * 128 : nullptr;
#else
  const ConvGemmArgs& args = args_in;
#endif
  const InstKey k = launch_key(args, block_n, num_sms);
  if (block_n == 128)
    return launch_listed(Instances<128>{}, k, tmap_a, tmap_w, tmap_w64, tmap_out, tmap_res, tmap_z,
                         args, num_sms, stream);
  return launch_listed(Instances<64>{}, k, tmap_a, tmap_w, tmap_w64, tmap_out, tmap_res, tmap_z,
                       args, num_sms, stream);
}

}  // namespace vp3d
