// Temporal-convolution implicit GEMM for sm_90a (wgmma + TMA).
//
// One kernel covers every Conv1d on the VideoPose3D hot path (reference: common/model.py:102,
// 113-118, 167, 178-180 and the shrink conv at :33) on channel-last activations:
//
//   D[row, co] = sum_{tap} sum_{ci} A[rowmap(row, tap), ci] * W[tap][co][ci]
//
//   * "flat" geometry: the conv's stride equals its width (TemporalModelOptimized1f, and the
//     eval-mode dependency cone of TemporalModel when T == receptive field), so the w taps of one
//     output row are w consecutive input rows == one contiguous K = w*C_in row of a 2-D matrix.
//   * "dilated" geometry: tile = 128 consecutive output frames of one sample, tap k reads the
//     same tile shifted by k*dilation frames (TMA zero-fills past the end of the sample).
//
// The fused epilogue applies the BatchNorm affine (eval: folded running stats), ReLU, the sliced
// residual add (model.py:130-135 / :191-194) and writes bf16 planes (hi, optional lo for the
// bf16x3 fp32-faithful mode) or fp32 (+bias) for the shrink layer; in training mode it instead
// stores the raw conv output and accumulates per-channel sum / sum-of-squares for the batch
// statistics with a warp-shuffle transpose-reduce.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vp3d {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 bf16 = one 128-byte swizzle row
constexpr int kBlockK8 = 128; // the same row holds 128 one-byte (int8) elements
constexpr int kUmmaK = 16;
constexpr int kMaxDevices = 64;  // per-device caches (function attributes, SM counts)

enum ConvGemmFlags : int {
  kEpiRelu = 1,        // y = max(y, 0)
  kEpiResidual = 2,    // y += res[rowmap]
  kEpiStats = 4,       // accumulate per-channel sum / sumsq of the stored value (training BN)
  kEpiOutF32 = 8,      // write fp32 (shrink) instead of bf16 planes
  kEpiAffine = 16,     // y = acc*scale[c] + shift[c]  (else y = acc)
};

struct ConvGemmArgs {
  // ---- geometry
  int dilated;        // 0 = flat, 1 = per-sample dilated tiles
  int samples;        // dilated: batch size; flat: 1
  int out_rows;       // dilated: valid output frames per sample; flat: total output rows
  int tiles_per_sample;  // dilated: ceil(out_rows/128); flat: ceil(out_rows/128) as well
  int taps;           // filter taps
  int kblocks_per_tap;   // padded C_in per tap / 64
  int tap_row_step;   // dilated: dilation; flat: 0
  int tap_col_step;   // flat: padded C_in per tap (elements); dilated: 0
  int n_tiles;        // padded C_out / BLOCK_N
  int n_pad;          // padded C_out (rows per (plane, tap) slab of W)
  int pairs;          // 1 = bf16, 3 = bf16x3 (a_hi*w_hi + a_lo*w_hi + a_hi*w_lo)
  int f16;            // 1: operands, residual and 16-bit outputs are IEEE fp16 instead of bf16
  int flags;
  // ---- epilogue
  const float* scale;   // [n_pad] or null
  const float* shift;   // [n_pad] or null (bias for the shrink layer)
  const __nv_bfloat16* res;    // residual source (plane 0), channel-last, ld = res_ld
  long long res_plane_stride;  // elements between hi and lo planes (0 if single plane)
  int res_planes;
  int res_ld;
  int res_rows_per_sample;     // dilated: rows per sample in the residual tensor
  int res_row_step;            // residual row = sample*res_rows_per_sample + t*res_row_step + res_row_off
  int res_row_off;
  int res_sample_div;           // flat tiling: split row -> (row / div, row % div) for the residual map; 0 = off
  int res_col_begin;            // residual is added only to output columns [res_col_begin, +res_cols)
  int res_cols;                 //   reading residual column (col - res_col_begin)   (dgrad skip path)
  int res_check_rows;           // 1: skip rows whose mapped in-sample row falls outside [0, res_rows_per_sample)
  int res_tma;                  // 1: residual tiles are TMA-loaded by warp 3 through tmap_res (RES variant)
  int res_tma_col_off;          //   column offset inside the residual map's row view
  int res_tma_row_off;          //   row offset (added to the tile's first row)
  // ---- fused BatchNorm-backward reductions (training data-gradient GEMMs, single-plane bf16):
  // the GEMM output G is the gradient w.r.t. the activation of the layer below, whose pre-BN
  // output Z has the same [rows][ld] view.  With the Z tile TMA-loaded next to the residual tile the
  // epilogue forms dY = G * dropmask/(1-p) * [Z*scale+shift > 0] and accumulates sum(dY) and
  // invstd * sum(dY * (Z - mean)) per channel (channel = column % bnb_c), replacing a separate
  // pass over G and Z.
  int bnb;                      // 1: enabled (requires the RES kernel variant and tmap_z)
  int bnb_c;
  const float* bnb_scale;
  const float* bnb_shift;
  const float* bnb_mean;
  const float* bnb_invstd;
  float* bnb_sums;              // partials [4 * row tiles][2][n_pad], see `stats`
  float bnb_p;                  // dropout probability of that layer (0 = none)
  unsigned bnb_seed_lo, bnb_seed_hi, bnb_layer;
  __nv_bfloat16* out;          // bf16 output plane 0, [samples*out_rows, out_ld]
  long long out_plane_stride;
  int out_planes;              // 1 or 2
  int out_ld;
  float* out_f32;              // fp32 output [rows, out_f32_ld], only first n_valid columns
  int out_f32_ld;
  int n_valid;                 // number of real output channels (<= n_pad)
  float* stats;                // partials [4 * row tiles][2][n_pad]: per 32-row slab of every row
                               // tile the per-channel sum and sum of squares (plain stores, every
                               // entry written; reduced in a fixed order afterwards)
  // two output planes: the lo plane is only produced for tiles that intersect rows
  // [lo_row_begin, lo_row_end) (flat tiling; the rows a later residual add / split-bf16 GEMM reads)
  int lo_row_begin, lo_row_end;
  // ---- int8 inference (lean instances only)
  int i8;                      // 1: A is u8 and W s8, k-blocks of 128 one-byte elements, int32 acc
  // u8 copy of the stored value, q = cvt.rni.sat.u8(v * u8_inv_s), rows as in `out`: staged in
  // shared memory and TMA-stored through tmap_z (64 x 32 byte boxes, no swizzle); next to the
  // 16-bit plane, or alone when `out` is null.  out_u8 (non-null) selects the u8 instances.
  uint8_t* out_u8;
  float u8_inv_s;
  // ---- work items (set by the launcher, not the caller): the last half_items / 2 tiles run as
  // half_items 128 x 64 half tiles (128-wide ping-pong instances; 0 = whole tiles only)
  int half_items;
#ifdef VP3D_TIMELINE
  // debug build (`make dbg`): per-launch time stamps of the first and the last CTA
  unsigned long long* timeline;   // [2 CTAs][32 events][globaltimer ns, clock64] or null
#endif
};
#ifdef VP3D_TIMELINE
void conv_gemm_debug_set_timeline(unsigned long long* buf, int max_launches);
#endif

// Host-side launcher (conv_gemm.cu). tmap_a: 4-D (k, row, sample, plane); tmap_w: 2-D (k, slab row);
// tmap_out: 4-D (channel, row, sample, plane) over the bf16 output, box (64, 32, 1, 1) (ignored —
// pass any valid map — when the launch writes fp32).
// tmap_res: 4-D (channel, row, sample, plane) over the residual's row view, box (64, 128, 1, 1); used
// only when args.res_tma is set.
// tmap_z: same geometry as tmap_out over the Z tensor of the layer below; used only when args.bnb.
// With args.out_u8 it maps the u8 output instead: 4-D (channel, row, sample, 1) bytes, box
// (64, 32, 1, 1), no swizzle.
// tmap_w: box rows = block_n.  block_n is 128 or 64.  tmap_w64: the same weights with box rows 64
// (the half tiles of a 128-wide launch; at block_n 64 pass tmap_w again).
void conv_gemm_set_pdl(int on);   // programmatic dependent launch of the GEMM kernels (default on)
bool conv_gemm_pdl_enabled();     // (also honoured by the small kernels between the GEMMs, launch.cuh)
// The instance launch_conv_gemm runs for these arguments, as the 7 ints of vp3d_conv_gemm_instance
// (include/vp3d_b200.h); false if it is not compiled (launch_conv_gemm then returns
// cudaErrorInvalidValue).
bool conv_gemm_instance(const ConvGemmArgs& args, int block_n, int num_sms, int key[7]);
// The keys of every compiled instance (block_n 128, then 64) into keys[7 i], at most max of them;
// returns how many are compiled.
int conv_gemm_instances(int* keys, int max);
cudaError_t launch_conv_gemm(const CUtensorMap& tmap_a, const CUtensorMap& tmap_w,
                             const CUtensorMap& tmap_w64, const CUtensorMap& tmap_out,
                             const CUtensorMap& tmap_res, const CUtensorMap& tmap_z,
                             const ConvGemmArgs& args, int block_n, int num_sms,
                             cudaStream_t stream);

}  // namespace vp3d
