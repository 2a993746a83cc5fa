// Bandwidth-bound helper kernels around the conv GEMMs: fp32 -> bf16 (hi/lo plane) packing of the
// network input and of the Conv1d weights, and folding of BatchNorm1d eval statistics into a
// per-channel affine.  Kernel definitions in pack.cu; the 16-bit rounding every pack shares is here.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vp3d {

// The one rounding of an fp32 value into the 16-bit operand slots every pack writes (input, forward
// and transposed weight packs, the fused optimizer, the streaming rings): bf16 hi (round to nearest)
// and the bf16 residual lo of the split (bf16x3), or with f16 IEEE half bits in a bf16-typed slot,
// saturated at +-65504 like the GEMM epilogue (single plane: lo is not stored).
struct Bits16 {
  __nv_bfloat16 hi, lo;
};
__device__ __forceinline__ Bits16 to_bits16(float v, int f16 = 0) {
  Bits16 b;
  if (f16) {
    b.hi = __ushort_as_bfloat16(__half_as_ushort(__float2half_rn(fminf(fmaxf(v, -65504.0f), 65504.0f))));
    b.lo = b.hi;
  } else {
    b.hi = __float2bfloat16_rn(v);
    b.lo = __float2bfloat16_rn(v - __bfloat162float(b.hi));
  }
  return b;
}
// element o of a [planes][...] pack: hi into plane 0, lo into plane 1 when there are two
__device__ __forceinline__ void store_bits16(__nv_bfloat16* pack, long long o, long long plane_elems,
                                             int planes, float v, int f16 = 0) {
  const Bits16 b = to_bits16(v, f16);
  pack[o] = b.hi;
  if (planes == 2) pack[plane_elems + o] = b.lo;
}

// x: fp32 (N, T, c_raw) contiguous (model.py:68 view of (N,T,J,F)).
// out: bf16 [planes][N][rows][k_pad]; row r of sample n gathers `group` consecutive frames starting
// at frame r*frame_step, i.e. columns [0, group*c_raw) = x[n, r*frame_step : r*frame_step+group, :]
// flattened, zero padded to k_pad.  (group = 1, frame_step = 1 for the dilated layout; group =
// frame_step = w0 for the strided layout where expand_conv becomes a plain GEMM.)
//
// Row order.  Default (perm == nullptr or perm->levels == 0): row index = n*rows + r.  Tap-major
// order (eval strided schedule): the rows of every activation are ordered so that the `w` taps of
// the next strided conv are `w` contiguous row regions.  With block widths w_1..w_B and
// R_i = N * rows_out(block i):  pos_0(n, t0) = (t0 mod w_1)*R_1 + pos_1(n, t0 / w_1), ...,
// pos_B(n, t) = n*rows_out(B) + t.  `perm` carries (R_i, w_i) for i = 1..levels and rows_out(B).
// f16 != 0 (both pack launchers): planes must be 1 and the 16-bit slots receive IEEE fp16 bits
// (saturated at +-65504) instead of bf16 -- the operand format of the fp16 eval mode.
struct PackPerm {
  int levels;        // number of residual blocks B (0 = natural order)
  int last_rows;     // rows per sample after the last block
  unsigned region[8];   // R_1 .. R_B  (row counts < 2^31)
  int width[8];         // w_1 .. w_B
};
cudaError_t launch_pack_input(const float* x, __nv_bfloat16* out, int planes, int N, int T,
                              int c_raw, int rows, int group, int frame_step, int k_pad,
                              long long plane_stride, cudaStream_t stream,
                              const PackPerm* perm = nullptr, int f16 = 0);

// w: fp32 Conv1d weight (c_out, c_in, taps) (tap index innermost, model.py:102,113-118).
// out: bf16 [planes][taps_out][n_pad][k_pad], zero padded.
//   merge_taps = 0: taps_out = taps, out[pl][tap][co][ci] = w[co][ci][tap]
//   merge_taps = 1: taps_out = 1,    out[pl][0][co][tap*c_in + ci] = w[co][ci][tap]
cudaError_t launch_pack_conv_weight(const float* w, __nv_bfloat16* out, int planes, int c_out,
                                    int c_in, int taps, int n_pad, int k_pad, int merge_taps,
                                    cudaStream_t stream, int f16 = 0);

// int8 eval weights, per output channel co (fp32 throughout, IEEE division and rint):
//   w_scale[co] = max_{ci, tap} |w[co][ci][tap]| / 127   (1 for an all-zero or padding channel)
//   out[tap][co][ci] = clamp(rint(w[co][ci][tap] / w_scale[co]), -127, 127)   (s8, zero padded)
// out: s8 [taps][n_pad][k_pad]; w_scale: [n_pad].
cudaError_t launch_pack_conv_weight_s8(const float* w, int8_t* out, float* w_scale, int c_out,
                                       int c_in, int taps, int n_pad, int k_pad,
                                       cudaStream_t stream);
// The int8 dequantisation folded into the eval affine: q_scale[c] = bn_scale[c] * (w_scale[c] * s_in)
// (two fp32 roundings in this order), c < n.
cudaError_t launch_int8_fold(const float* bn_scale, const float* w_scale, float s_in, float* q_scale,
                             int n, cudaStream_t stream);
// amax_bits = max(amax_bits, fp32 bits of max(x)) over n fp16 values >= 0 (n % 8 == 0, x 16-byte
// aligned; -0 counts as 0), one integer atomicMax per block.
cudaError_t launch_amax_f16(const void* x, long long n, unsigned* amax_bits, cudaStream_t stream);
// Calibration histogram of one stored fp16 plane [rows][ld] (x 16-byte aligned, ld % 8 == 0): of
// every row's first c_real channels, bit patterns with the sign bit set add to hist[0], patterns
// 0x0001 .. 0x7BFF to hist[pattern], inf and NaN to *invalid.  u64 counts, so calls accumulate.
constexpr int kHistBins = 0x7C00;   // 31 744: every finite fp16 value >= 0
cudaError_t launch_hist_f16(const void* x, long long rows, int ld, int c_real, unsigned long long* hist,
                            unsigned long long* invalid, int num_sms, cudaStream_t stream);
// u8 codes of one stored fp16 plane [rows][ld] (x 16-byte, q 8-byte aligned, ld % 8 == 0) into q
// [rows][ld]: q = cvt.rni.sat.u8.f32(fp32(x) * inv_s) on every row's first c_real channels, 0 on
// the rest.  Makes Q_i of an int8 block whose input an fp16 block wrote.
cudaError_t launch_quantize_u8(const void* x, uint8_t* q, long long rows, int ld, int c_real,
                               float inv_s, int num_sms, cudaStream_t stream);
// *count += the number of inf / NaN values among x[0, n)
cudaError_t launch_count_nonfinite(const float* x, long long n, unsigned long long* count,
                                   int num_sms, cudaStream_t stream);

// Eval-mode BatchNorm1d (model.py:32,117,119; eps = 1e-5) as y = x*scale + shift.
// gamma/beta/mean/var: [c]; scale/shift: [c_pad] (padding: scale 0, shift 0).  mean_out /
// invstd_out (both or neither, [c_pad]) also receive running_mean and 1/sqrt(var + eps), padding 0:
// the frozen-BatchNorm training forward needs them for its backward.
cudaError_t launch_bn_fold(const float* gamma, const float* beta, const float* mean,
                           const float* var, float eps, float* scale, float* shift, int c,
                           int c_pad, cudaStream_t stream, float* mean_out = nullptr,
                           float* invstd_out = nullptr);

// shrink bias (model.py:33): scale = 1, shift = bias, padded with zeros.
cudaError_t launch_bias_affine(const float* bias, float* scale, float* shift, int c, int c_pad,
                               cudaStream_t stream);

}  // namespace vp3d
