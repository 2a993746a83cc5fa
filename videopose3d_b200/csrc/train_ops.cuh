// Bandwidth-bound training-mode kernels around the GEMMs: BatchNorm1d batch statistics ->
// affine (+ running-stat update), BN-apply + ReLU + Dropout + residual, and the BatchNorm / ReLU /
// Dropout backward (two-pass: per-channel reductions, then dZ).  Reference semantics:
// nn.BatchNorm1d(momentum) train mode (model.py:32,117,119), nn.ReLU, nn.Dropout(p) (model.py:28-29)
// and the residual slice-add (model.py:130-135, 191-194).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace vp3d {

struct RowMap {          // residual row of output row r: (r / div)*rows_per_sample + (r % div)*step + off
  int div;               // 0: no split (row = r*step + off)
  int rows_per_sample;
  int step;
  int off;
};

struct DropoutCfg {
  float p;               // drop probability (0 = identity)
  uint32_t seed_lo, seed_hi;
  uint32_t layer;        // decorrelates layers sharing a seed
};

// Ordered reductions (run-to-run reproducible; no floating-point atomics anywhere in training).
constexpr int kReduceMaxSplits = 32;      // (the finalize kernel's last-block stage assumes <= 32)      // second-level splits of an ordered reduction
constexpr int kReduceMaxChannels = 8192;  // scratch: kReduceMaxSplits x 3 x channels floats
constexpr size_t kReduceScratchFloats = (size_t)kReduceMaxSplits * 3 * kReduceMaxChannels;
constexpr int kReduceCounters = kReduceMaxChannels / 32;  // zero-initialised once, self-resetting

// part: [slabs][2][c] per-slab sum / sum of squares written by the conv GEMM epilogue (slab s =
// rows (s%4)*32.. of row tile s/4; geometry as in the GEMM: dilated = per-sample tiles).  Every
// slab becomes (count, mean, M2) and the slabs are merged in a fixed order (Chan et al.), so the
// batch variance never forms E[x^2] - E[x]^2 over the whole batch.  gamma / beta / running_* hold
// c_real <= c channels; channels [c_real, c) are layout padding and get a zero affine.  Writes scale = gamma*invstd,
// shift = beta - mean*scale, mean, invstd and updates running_mean / running_var in place
// (running = (1-m)*running + m*batch, unbiased variance for running_var).
cudaError_t launch_bn_stats_finalize(const float* part, int slabs, int dilated, int out_rows,
                                     int tiles_per_sample, const float* gamma, const float* beta,
                                     float* running_mean, float* running_var, float momentum,
                                     float eps, float* scale, float* shift, float* mean,
                                     float* invstd, int c, int c_real, float* scratch,
                                     unsigned* counter, cudaStream_t stream,
                                     float* moments = nullptr, int world = 0, int rank = 0);
// With `moments` (synchronized BatchNorm) the launch above stops after the slab merge: it writes
// this rank's (n, mean, M2) into slot `rank` of moments [world][3][c], zeros into the other slots,
// and nothing else.  After the slots have been exchanged, launch_bn_sync_finalize merges them in
// rank order 0..world-1 and runs the same finalize (running statistics over the global n);
// n_out[0] = the global row count.
cudaError_t launch_bn_sync_finalize(const float* moments, int world, const float* gamma,
                                    const float* beta, float* running_mean, float* running_var,
                                    float momentum, float eps, float* scale, float* shift,
                                    float* mean, float* invstd, int c, int c_real, float* n_out,
                                    cudaStream_t stream);

// out[i] = sum_r slots[r][i] for slots [world][n], in rank order (world = 1: a copy).
cudaError_t launch_rank_ordered_sum(const float* slots, int world, int n, float* out,
                                    cudaStream_t stream);

// out_st[ch] = mul_st[ch] * sum_p sum_f part[p][st][f*c + ch], st < nstat (1 or 2), f < folds, in
// a fixed order.  part: [n_part][nstat][ld].  mul_st may be null (= 1).
cudaError_t launch_ordered_col_sums(const float* part, int n_part, int nstat, int ld, int c,
                                    int folds, const float* mul0, const float* mul1, float* out0,
                                    float* out1, float* scratch, unsigned* counter,
                                    cudaStream_t stream);

// x = dropout(relu(z*scale + shift)) [+ res[map(row)]]; z, x, res: bf16 [planes][rows][c].
cudaError_t launch_bn_apply(const __nv_bfloat16* z, long long z_plane, __nv_bfloat16* x,
                            long long x_plane, int planes, long long rows, int c, const float* scale,
                            const float* shift, DropoutCfg drop, const __nv_bfloat16* res,
                            long long res_plane, RowMap map, cudaStream_t stream);

// sums[0][c] = sum_rows dY, sums[1][c] = sum_rows dY * xhat, with
// dY = g * dropmask/(1-p) * [z*scale+shift > 0], xhat = (z - mean) * invstd.  Per-block partials
// go to `partials` (>= 2*c floats per row block) and are summed in a fixed order into sums[2][c].
cudaError_t launch_bn_bwd_reduce(const __nv_bfloat16* g, long long g_plane, const __nv_bfloat16* z,
                                 long long z_plane, int planes, long long rows, int c,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, DropoutCfg drop, float* partials,
                                 size_t partial_floats, float* sums, float* scratch,
                                 unsigned* counter, cudaStream_t stream);

// dz = scale * (dY - sums[0]/n - xhat * sums[1]/n); also writes dgamma = sums[1], dbeta = sums[0]
// (done by block 0).  dz: bf16 [planes][rows][c].  frozen != 0 (BatchNorm on running statistics,
// eval-mode backward): dz = scale * dY, mean / invstd are not read, and sums may be null (then no
// dgamma / dbeta are written).  Synchronized BatchNorm: global_sums [2][c] (summed over ranks) and
// the device scalar n_global (global row count) replace sums and rows in dz, while dgamma / dbeta
// still come from this rank's `sums`; both null otherwise.
cudaError_t launch_bn_bwd_apply(const __nv_bfloat16* g, long long g_plane, const __nv_bfloat16* z,
                                long long z_plane, __nv_bfloat16* dz, long long dz_plane, int planes,
                                long long rows, int c, const float* scale, const float* shift,
                                const float* mean, const float* invstd, DropoutCfg drop,
                                const float* sums, float* dgamma, float* dbeta, int c_real,
                                cudaStream_t stream, int frozen = 0,
                                const float* global_sums = nullptr, const float* n_global = nullptr);

// out[c] = sum_rows x[row][c] for fp32 x [rows][c] (shrink.bias gradient), via per-64-row partials
// summed in a fixed order.
cudaError_t launch_col_sum_f32(const float* x, long long rows, int c, float* partials,
                               size_t partial_floats, float* out, float* scratch, unsigned* counter,
                               cudaStream_t stream);

// Transposed weight pack for dgrad: w fp32 (c_out, c_in, taps) -> bf16 [planes][taps][n_pad][k_pad]
// with out[pl][tap][ci][co] = w[co][ci][tap]  (rows = input channels, K = output channels).
// If fwd != nullptr the same pass also writes the forward pack fwd[pl][tap][co][ci] (rows fwd_n_pad,
// cols fwd_k_pad): one read of the fp32 master feeds both layouts.
// merged != 0 (fwd must be null): one slab out[pl][0][tap*c_in + ci][co], rows padded to n_pad >=
// taps*c_in -- the tap-merged layout of the strided expand conv's data gradient.
cudaError_t launch_pack_conv_weight_t(const float* w, __nv_bfloat16* out, int planes, int c_out,
                                      int c_in, int taps, int n_pad, int k_pad, cudaStream_t stream,
                                      __nv_bfloat16* fwd = nullptr, int fwd_n_pad = 0,
                                      int fwd_k_pad = 0, int merged = 0);

}  // namespace vp3d
