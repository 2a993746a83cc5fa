/*
 * vp3d_b200 — C ABI of the H100-native temporal-convolution engine that replaces the
 * PyTorch/cuDNN execution of VideoPose3D's model hot path.
 *
 * The reference (facebookresearch/VideoPose3D) has no FFI: its "operator interface" for this path
 * is the nn.Module contract of common/model.py (TemporalModelBase :10-77, TemporalModel :79-138,
 * TemporalModelOptimized1f :140-197) as exercised by run.py.  Each entry point below names the
 * reference call site it replaces.  All pointers are plain host/device addresses, sizes are plain
 * integers, streams are cudaStream_t passed as void*; nothing here depends on torch.
 *
 * Conventions: every function returns 0 on success or a negative vp3d_status; the message for the
 * last failure on the calling thread is available from vp3d_last_error().  The library never
 * aborts the process and never falls back to a CPU path.
 */
#ifndef VP3D_B200_H_
#define VP3D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VP3D_VERSION 200
#define VP3D_MAX_WIDTHS 8                       /* len(filter_widths) <= 8 (RF up to 3^8) */
#define VP3D_MAX_LAYERS (2 * (VP3D_MAX_WIDTHS - 1)) /* layers_conv / layers_bn entries */

typedef enum {
  VP3D_OK = 0,
  VP3D_ERR_INVALID = -1,     /* bad argument (mirrors the AssertionErrors of model.py:20-21, 64-66) */
  VP3D_ERR_UNSUPPORTED = -2, /* configuration the kernels do not cover; never a silent fallback */
  VP3D_ERR_CUDA = -3,        /* CUDA runtime / driver error, text in vp3d_last_error() */
  VP3D_ERR_WORKSPACE = -4,   /* workspace too small / misaligned */
  VP3D_ERR_STATE = -5        /* call order violated (e.g. forward before weights were loaded) */
} vp3d_status;

typedef enum {
  VP3D_VARIANT_DILATED = 0,  /* TemporalModel            (model.py:79-138)  */
  VP3D_VARIANT_STRIDED = 1   /* TemporalModelOptimized1f (model.py:140-197) */
} vp3d_variant;

typedef enum {
  VP3D_PRECISION_BF16 = 0,   /* bf16 operands, fp32 accumulate (fast path; BASELINE cfg 2) */
  VP3D_PRECISION_BF16X3 = 1, /* split-bf16 (hi+lo) operands, 3 MMAs per product: fp32-faithful */
  VP3D_PRECISION_MIXED = 2,  /* bf16 residual blocks, split-bf16 expand and shrink (and blocks below
                                0.5% of the FLOPs), residual stream kept in hi+lo planes; ~1e-3 of
                                fp32 (<= 2e-3) close to bf16 cost */
  VP3D_PRECISION_FP16 = 3,   /* eval default: IEEE fp16 operands and activations (11-bit significand,
                                single plane), fp32 accumulate -- the tensor rate of bf16 at 1/8 of
                                its rounding error: ~4e-4 of fp32 on cfg2, inside north_star's 1e-3.
                                Stores saturate at +-65504.  Inference only (training runs bf16 /
                                bf16x3: gradients need the bf16 exponent range) */
  VP3D_PRECISION_INT8 = 4    /* eval only: the two convs of every residual block (or of those
                                vp3d_set_int8_blocks selects; the rest run as in FP16) multiply u8
                                activations by s8 weights into exact int32 sums (one activation scale
                                s = amax / 255 per quantised tensor from vp3d_calibrate_int8, weight
                                scale max|W| / 127 per output channel, folded into the BatchNorm
                                affine); expand, shrink and the residual stream are fp16 as in FP16.
                                Needs vp3d_set_int8_scales before its vp3d_set_weights.  Not for
                                streaming or training.  Op level: u8 A, s8 W, k_per_tap % 128 == 0 */
} vp3d_precision;

/* Constructor arguments of TemporalModel / TemporalModelOptimized1f (model.py:85-86, :151-152). */
typedef struct {
  int num_joints_in;
  int in_features;
  int num_joints_out;
  int num_widths;
  int filter_widths[VP3D_MAX_WIDTHS];
  int causal;
  int channels;
  int dense;      /* TemporalModel(dense=True) ablation, model.py:113-116 */
  int variant;    /* vp3d_variant */
  int precision;  /* vp3d_precision */
} vp3d_config;

/* Device pointers to the fp32 tensors of the module's state_dict (same names / shapes as the
 * reference: expand_conv.weight (C, J*F, w0); expand_bn.{weight,bias,running_mean,running_var};
 * layers_conv.{i}.weight; layers_bn.{i}.*; shrink.weight (3*J_out, C, 1); shrink.bias). */
typedef struct {
  const float* expand_conv_weight;
  const float* expand_bn[4]; /* weight, bias, running_mean, running_var */
  const float* layers_conv_weight[VP3D_MAX_LAYERS];
  const float* layers_bn[VP3D_MAX_LAYERS][4];
  const float* shrink_weight;
  const float* shrink_bias;
} vp3d_weights;

typedef struct vp3d_plan vp3d_plan;

int vp3d_version(void);
const char* vp3d_last_error(void);
/* Cap the persistent grids of the GEMM kernels at n SMs (0 = all): a data-parallel host leaves the
 * remaining SMs to the NCCL kernels of an overlapped gradient all-reduce, which otherwise cannot be
 * scheduled next to one-CTA-per-SM grids (no reference counterpart: the reference is single-GPU). */
int vp3d_set_sm_limit(int n);
/* Programmatic dependent launch of the GEMM kernels (on by default: the next kernel's prologue
 * overlaps the tail of the current one).  A host that overlaps NCCL collectives with the backward
 * turns it off: gap-free hand-over between one-CTA-per-SM grids starves the NCCL kernels of SMs
 * (measured: 2-GPU step 2.76 ms with it off, tens of ms per synchronised step with it on). */
int vp3d_set_pdl(int on);

/* Replaces TemporalModel.__init__ / TemporalModelOptimized1f.__init__ (model.py:85-124, 151-185):
 * validates odd filter widths, derives pad / causal_shift / dilation per block, allocates the packed
 * bf16 weight store on the current CUDA device. */
int vp3d_plan_create(const vp3d_config* cfg, vp3d_plan** out_plan);
void vp3d_plan_destroy(vp3d_plan* plan);

/* Replaces TemporalModelBase.receptive_field (model.py:41-48). */
int vp3d_receptive_field(const vp3d_plan* plan);
/* Replaces TemporalModelBase.total_causal_shift (model.py:50-61). */
int vp3d_total_causal_shift(const vp3d_plan* plan);

/* Re-pack parameters after load_state_dict / optimizer.step (state_dict contract, run.py:209-210,
 * 426).  what: bit 0 = conv weights -> bf16 planes, bit 1 = BatchNorm eval affine
 * (scale = w / sqrt(running_var + 1e-5), shift = b - running_mean * scale) and shrink bias. */
#define VP3D_PACK_CONV 1
#define VP3D_PACK_BN_EVAL 2
#define VP3D_PACK_CONV_T 4 /* transposed conv weights for the data-gradient GEMMs (training only) */
/* transposed expand-conv weights for the input gradient of vp3d_backward_ex (training plans only;
 * not refreshed by vp3d_adam_step_packed: re-pack after every change of expand_conv.weight) */
#define VP3D_PACK_EXPAND_T 8
int vp3d_set_weights(vp3d_plan* plan, const vp3d_weights* w, int what, void* stream);

/* Output frames for an input of T frames: T - receptive_field + 1 for the dilated variant
 * (model.py:130-135 valid convolutions), floor-division chain for the strided one (:167, :178). */
int vp3d_output_frames(const vp3d_plan* plan, int T);

/* Bytes of device scratch needed by vp3d_forward_eval for a batch of N sequences of T frames. */
size_t vp3d_workspace_bytes(const vp3d_plan* plan, int N, int T);

/* Replaces TemporalModelBase.forward in eval() mode (model.py:63-77 + _forward_blocks :126-138 /
 * :187-197): x is (N, T, J_in, F) fp32 contiguous, y is (N, T_out, J_out, 3) fp32 contiguous, both
 * DEVICE pointers.  workspace is device memory of at least vp3d_workspace_bytes(), 1024-B aligned.
 * Asynchronous on `stream`. */
int vp3d_forward_eval(vp3d_plan* plan, const float* x, float* y, int N, int T, void* workspace,
                      size_t workspace_bytes, void* stream);

/* Activation calibration of the int8 eval mode: runs the fp16 eval chain of `fp16_plan` (a
 * VP3D_PRECISION_FP16 plan with its weights set; no shrink) on x (N, T, J_in, F), and after each GEMM
 * whose output an int8 plan quantises reads the stored fp16 plane and folds its maximum into
 * amax[2B] (device fp32, B residual blocks): amax[2(i-1)] = max X_{i-1} (the input of block i's
 * first conv; X_0 is the expand output), amax[2(i-1)+1] = max H_i (the input of its 1x1 conv).  The
 * fold is an integer atomicMax on the fp32 bits (every value is >= 0): order-independent and
 * reproducible.  Calls accumulate (zero amax before the first batch). */
int vp3d_calibrate_int8(vp3d_plan* fp16_plan, const float* x, int N, int T, void* workspace,
                        size_t workspace_bytes, float* amax, void* stream);
/* Activation histograms for the int8 calibration, so that a threshold below the maximum can be
 * chosen (vp3d_int8_thresholds; not in the reference).  hist is a DEVICE array of
 * vp3d_int8_hist_bytes(plan) bytes (0 for a plan without residual blocks): u64 counts hist[l][b],
 * l < 2B as amax above and b < 31744 one bin per fp16 bit pattern 0x0000 .. 0x7BFF (values with the
 * sign bit count as 0, which they quantise to), then 2B counts of invalid values (inf / NaN; a
 * non-finite value of x counts for layer 0).  Only the model's `channels` real channels count.
 * vp3d_calibrate_int8_hist has vp3d_calibrate_int8's preconditions and ADDS one batch to hist:
 * calls accumulate (zero hist once), and integer counts make the result independent of order. */
size_t vp3d_int8_hist_bytes(const vp3d_plan* fp16_plan);
int vp3d_calibrate_int8_hist(vp3d_plan* fp16_plan, const float* x, int N, int T, void* workspace,
                             size_t workspace_bytes, uint64_t* hist, void* stream);
/* Clipping thresholds from such histograms, one per layer (not in the reference): amax_out[l]
 * (DEVICE fp32) is the value of one fp16 bin, ready for vp3d_set_int8_scales.
 *   AMAX:       the largest non-empty bin; equals what vp3d_calibrate_int8 gives, bit for bit.
 *   PERCENTILE: param = p in (0, 100]: the smallest bin whose cumulative count reaches
 *               c = ceil(p / 100 * n) (fp64, n the layer's count, zeros included); p = 100 is AMAX.
 *   MSE:        the fp16 value t in [amax / 256, amax] with the smallest quantisation error
 *               E(t) = sum_b n_b (x_b - s q_b)^2 (fp64; s = fp32(t / 255), q_b = min(255,
 *               rint(fp32(x_b * fp32(1 / s)))) as the int8 forward quantises); the larger t on a tie.
 * An all-zero layer gives 0; a layer with invalid values gives NaN, which vp3d_set_int8_scales
 * refuses.  Integer counts and fixed-order fp64 sums: the same histogram gives the same bits on every
 * run.  scratch: DEVICE memory of vp3d_int8_thresholds_scratch_bytes(layers) bytes. */
#define VP3D_INT8_CALIB_AMAX 0
#define VP3D_INT8_CALIB_PERCENTILE 1
#define VP3D_INT8_CALIB_MSE 2
size_t vp3d_int8_thresholds_scratch_bytes(int layers);
int vp3d_int8_thresholds(const uint64_t* hist, int layers, int method, double param,
                         float* amax_out, void* scratch, size_t scratch_bytes, void* stream);
/* Stores the activation scales of an int8 plan from n = 2B HOST amax values (as above): s = amax /
 * 255 in fp32 (1 when amax is 0), 1 / s in fp32.  The next vp3d_set_weights that leaves both the
 * conv and the BatchNorm packs current folds them into the int8 affine; until then vp3d_forward_eval
 * returns VP3D_ERR_STATE. */
int vp3d_set_int8_scales(vp3d_plan* int8_plan, const float* amax_host, int n);
/* Chooses which residual blocks of an int8 plan run u8 x s8 (not in the reference): bit i - 1 of
 * mask selects block i (1..B); the default is every block.  The other blocks run exactly as in
 * VP3D_PRECISION_FP16 (fp16 operands and packs, K per tap = channels rounded up to 64); expand and
 * shrink stay fp16.  Where an fp16 block i feeds an int8 block, one extra launch quantises the
 * stored fp16 X_i to Q_i.  The calibration is the same for every mask.  A changed mask marks the
 * conv packs stale: vp3d_forward_eval returns VP3D_ERR_STATE until the next vp3d_set_weights
 * (VP3D_PACK_CONV) re-packs and re-folds.  VP3D_ERR_INVALID for a null plan, a plan that is not
 * int8 or bits at or above B. */
int vp3d_set_int8_blocks(vp3d_plan* int8_plan, uint32_t mask);
/* Copies the int8 packs of layers_conv[layer] of an int8 plan (as its last vp3d_set_weights left
 * them) to DEVICE buffers, each may be NULL: w_s8 [taps][n_pad][k_pad] s8 with n_pad = channels
 * rounded up to 64 and k_pad = n_pad rounded up to 128; w_scale and q_scale [n_pad] fp32 (q_scale
 * as last folded; VP3D_ERR_STATE before the first fold).  VP3D_ERR_INVALID for a layer of a block
 * that vp3d_set_int8_blocks left in fp16.  For checking the packs. */
int vp3d_int8_packs(const vp3d_plan* int8_plan, int layer, void* w_s8, float* w_scale,
                    float* q_scale, void* stream);

/* Same computation with HOST buffers (the call run.py makes: numpy batch -> .cuda() -> model ->
 * .cpu(), run.py:663-672): copies x host->device, runs the forward, copies y device->host and
 * synchronises.  Device staging buffers are owned by the plan.  x_host / y_host should be pinned
 * for full PCIe bandwidth but pageable memory is accepted. */
int vp3d_forward_eval_host(vp3d_plan* plan, const float* x_host, float* y_host, int N, int T);

/* Pipelined form of vp3d_forward_eval_host for streams of batches (the evaluation loop of
 * run.py:663-721 visits one batch after another): submit() enqueues copy-in -> forward -> copy-out
 * for one batch on slot 0 or 1 and returns; wait() blocks until that slot's y_host is complete.
 * Alternating the two slots overlaps the PCIe copy of batch i+1 with the kernels of batch i.
 * x_host / y_host must stay valid (and should be pinned) until wait() returns. */
int vp3d_forward_eval_host_submit(vp3d_plan* plan, const float* x_host, float* y_host, int N, int T,
                                  int slot);
int vp3d_forward_eval_host_wait(vp3d_plan* plan, int slot);

/* ---- training (TemporalModelOptimized1f; run.py:318-420) ------------------------------------
 * Gradient buffers, one per learnable tensor of the state_dict (same shapes, fp32, device).  They
 * are OVERWRITTEN by vp3d_backward (autograd accumulates them into .grad on the Python side). */
typedef struct {
  float* expand_conv_weight;
  float* expand_bn[2]; /* weight, bias */
  float* layers_conv_weight[VP3D_MAX_LAYERS];
  float* layers_bn[VP3D_MAX_LAYERS][2];
  float* shrink_weight;
  float* shrink_bias;
} vp3d_grads;

/* Device scratch for one training step: saved activations for backward + gradient scratch. */
size_t vp3d_train_workspace_bytes(const vp3d_plan* plan, int N, int T);

/* Replaces TemporalModelOptimized1f.forward in train() mode (model.py:187-197 with BatchNorm batch
 * statistics and Dropout active).  w: gamma / beta are read, running_mean / running_var are UPDATED
 * in place with bn_momentum[l] (l = 0 expand_bn, 1.. = layers_bn[l-1]; host array of 1 + 2B floats,
 * read at call time, model.py:36-39).  Conv weights must have been packed with
 * VP3D_PACK_CONV | VP3D_PACK_CONV_T since their last update.  Dropout masks come from a counter-based
 * generator keyed by `seed` (statistically, not bitwise, equal to torch's).  `workspace` must stay
 * untouched until the matching vp3d_backward. */
int vp3d_forward_train(vp3d_plan* plan, const float* x, float* y, int N, int T, const vp3d_weights* w,
                       const float* bn_momentum, float dropout_p, unsigned long long seed,
                       void* workspace, size_t workspace_bytes, void* stream);

/* vp3d_forward_train with flags.  VP3D_TRAIN_FROZEN_BN: every BatchNorm is the fixed affine of its
 * running statistics (the eval-mode fold of VP3D_PACK_BN_EVAL: scale = w / sqrt(running_var + 1e-5),
 * shift = b - running_mean * scale), as model.eval() computes it; running statistics are neither
 * read for an update nor written, bn_momentum may be NULL and dropout_p must be 0.  The matching
 * vp3d_backward_ex then differentiates that forward: dZ = scale * dY without batch-statistics terms,
 * d weight = sum dY * (z - running_mean) / sqrt(running_var + 1e-5), d bias = sum dY -- autograd
 * through the reference's module in eval() mode.  flags == 0 is vp3d_forward_train. */
#define VP3D_TRAIN_FROZEN_BN 1
int vp3d_forward_train_ex(vp3d_plan* plan, const float* x, float* y, int N, int T,
                          const vp3d_weights* w, const float* bn_momentum, float dropout_p,
                          unsigned long long seed, int flags, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Replaces autograd's backward through the model (run.py:394, 418): dy is (N, T_out, J_out, 3) fp32;
 * writes every parameter gradient.  Uses the activations saved by the last vp3d_forward_train. */
int vp3d_backward(vp3d_plan* plan, const float* dy, const vp3d_grads* grads, void* workspace,
                  size_t workspace_bytes, void* stream);

/* Same as vp3d_backward, calling stage_done(stage, user) on the host right after the kernels that
 * produce one group of gradients have been enqueued on `stream`: stage 0 = shrink.{weight,bias};
 * stage s = 1..B = residual block B - s + 1 (its two convs and two BatchNorms); stage B + 1 =
 * expand_conv / expand_bn.  A data-parallel host uses it to start the all-reduce of a finished
 * group on a side stream while the rest of the backward is still running (run.py has no
 * counterpart: the reference is single-GPU). */
typedef void (*vp3d_stage_fn)(int stage, void* user);
int vp3d_backward_staged(vp3d_plan* plan, const float* dy, const vp3d_grads* grads, void* workspace,
                         size_t workspace_bytes, void* stream, vp3d_stage_fn stage_done, void* user);

/* vp3d_backward_staged with optional outputs (stage_done may be NULL):
 *   grads == NULL: no parameter gradients -- no weight-gradient GEMMs, no shrink-bias sum, and after
 *     a VP3D_TRAIN_FROZEN_BN forward no BatchNorm-backward reductions: only the data-gradient chain
 *     runs (test-time refinement of the input through a frozen model).
 *   dx != NULL: the input gradient dL/dx, an fp32 DEVICE buffer shaped like the forward's x
 *     (N, T, J_in, F); it is overwritten entirely, with zeros for frames no output depends on.
 *     Needs the transposed expand pack (vp3d_set_weights with VP3D_PACK_EXPAND_T) of the current
 *     expand_conv.weight.
 * At least one of grads / dx must be given.  vp3d_backward_staged is _ex with dx = NULL. */
int vp3d_backward_ex(vp3d_plan* plan, const float* dy, const vp3d_grads* grads, float* dx,
                     void* workspace, size_t workspace_bytes, void* stream, vp3d_stage_fn stage_done,
                     void* user);

/* Synchronized BatchNorm for data-parallel training over `world` ranks (replaces
 * nn.SyncBatchNorm / convert_sync_batchnorm for this model; no reference counterpart: the reference
 * is single-GPU).  Every following vp3d_forward_train_ex without VP3D_TRAIN_FROZEN_BN, and the
 * vp3d_backward_ex that matches it (the forward's setting is kept for it), then take each training
 * BatchNorm's statistics over the rows of all ranks:
 *   forward: per BatchNorm l = 0 (expand_bn), 1.. 2B (layers_bn[l-1]) this rank writes its
 *     per-channel (n, mean, M2) into slot `rank` of slots [world][3][C] (C = channels, the other
 *     slots zero) and calls exchange(l, VP3D_BN_SYNC_FORWARD, slots, 3 * C, user); the slots are
 *     merged in rank order 0..world-1 and batch mean, variance and the running-statistics update
 *     (unbiased over the global row count) follow from the merged moments.
 *   backward: the same with [world][2][C] slots holding this rank's sum dY and invstd * sum dY (z -
 *     mean), VP3D_BN_SYNC_BACKWARD; dZ uses the rank-ordered sum over ranks and the global row
 *     count, d weight / d bias this rank's own sums (averaging them over ranks, as the gradient
 *     all-reduce does, gives the global-batch gradient, as nn.SyncBatchNorm computes it).
 * exchange runs on the host once the kernel writing this rank's slot is enqueued on the call's
 * stream; before it returns it must enqueue on that stream an operation that fills every rank's
 * slot (an element-wise sum of the ranks' zero-padded buffers is exact).  It cannot fail the call:
 * a host records its own errors, as with vp3d_stage_fn.  The slot buffers belong to the plan; the
 * workspace sizes do not change.  world = 0 switches synchronisation off (exchange may be NULL);
 * world = 1 runs the synchronized kernels with one slot and gives the unsynchronized results bit
 * for bit. */
#define VP3D_BN_SYNC_FORWARD 0
#define VP3D_BN_SYNC_BACKWARD 1
typedef void (*vp3d_bn_exchange_fn)(int layer, int phase, float* slots, int floats_per_rank,
                                    void* user);
int vp3d_set_bn_sync(vp3d_plan* plan, int world, int rank, vp3d_bn_exchange_fn exchange, void* user);

/* Number of kernels the last forward on this plan launched (for bench.py's gpu_launches). */
int vp3d_last_launch_count(const vp3d_plan* plan);

/* Measurement hook (bench.py roofline): bracket launch number `launch_index` (0-based position in
 * the forward's launch sequence, -1 = off) of every following forward with CUDA events recorded on
 * the forward's own stream.  vp3d_profile_read synchronises those events, returns the summed
 * duration in milliseconds and the number of bracketed launches, and resets the accumulator. */
int vp3d_profile_launch(vp3d_plan* plan, int launch_index);
int vp3d_profile_read(vp3d_plan* plan, float* total_ms, int* count);

/* ---- operator-level entry (used by the parity tests; the model-level calls are built on it) ----
 * One temporal convolution on channel-last bf16 activations with the fused epilogue.
 * Replaces nn.Conv1d (+ BatchNorm1d eval affine + ReLU + residual slice-add), model.py:127, 134-135. */
typedef struct {
  /* A operand: bf16, [a_planes][samples][a_rows][a_ld] (a_ld = elements per row, multiple of 64) */
  const void* a;
  int a_planes;
  int samples;
  int a_rows;
  int a_ld;
  /* W operand: bf16, [w_planes][taps][n_pad][k_per_tap] */
  const void* w;
  int taps;
  int k_per_tap; /* multiple of 64 */
  int n_pad;     /* multiple of 64 */
  /* geometry */
  int per_sample_tiles; /* 1: tile = 128 output rows of one sample; 0: rows flattened over samples */
  int tap_row_step;     /* input-row offset between taps (dilation), 0 when taps are column blocks */
  int tap_col_step;     /* input-column offset between taps (strided conv: k_per_tap), else 0 */
  int out_rows;         /* output rows per sample (per_sample_tiles) or in total (flat) */
  int precision;        /* vp3d_precision (FP16: a, w, res and out hold IEEE fp16, one plane) */
  /* epilogue */
  const float* scale;   /* per channel, may be NULL (-> no affine) */
  const float* shift;
  int relu;
  const void* res;      /* bf16 residual [res_planes][*][res_ld] or NULL */
  int res_planes;
  long long res_plane_stride; /* elements */
  int res_ld;
  int res_rows_per_sample;
  int res_row_step;
  int res_row_off;
  int res_sample_div;   /* flat tiling only: rows per sample used to split row -> (sample, t); 0 = none */
  int res_col_begin;    /* residual only for output columns [res_col_begin, res_col_begin + res_cols) */
  int res_cols;         /*   (0 = all columns); used by the dgrad skip-connection path */
  int res_check_rows;   /* 1: ignore residual rows mapping outside [0, res_rows_per_sample) */
  void* out;            /* bf16 [out_planes][rows][out_ld] or NULL */
  int out_planes;
  long long out_plane_stride; /* elements */
  int out_ld;
  float* out_f32;       /* fp32 [rows][out_f32_ld] (first n_valid channels) or NULL */
  int out_f32_ld;
  int n_valid;
  float* stats;         /* NULL, or per-slab partials [4 * row tiles][2][n_pad]: for every 32-row slab of
                         * every 128-row tile the per-channel sum and sum of squares of the stored
                         * value (plain stores, every entry written, no atomics: reproducible) */
  /* fused BatchNorm-backward reductions (training data-gradient GEMMs, single-plane bf16 only):
   * bnb_z = pre-BN output Z of the layer whose activation gradient this GEMM produces, same
   * [rows][out_ld] view as `out`; writes slab partials of sum(dY) and sum(dY*(Z-mean)) to bnb_sums. */
  const void* bnb_z;    /* NULL = off */
  const float* bnb_scale;
  const float* bnb_shift;
  const float* bnb_mean;
  const float* bnb_invstd;
  float* bnb_sums;      /* per-slab partials [4 * row tiles][2][n_pad] of sum(dY) and sum(dY*(Z-mean))
                         * (summed in a fixed order, folded modulo bnb_c and scaled by invstd by the
                         * caller; bnb_invstd is not read by the kernel) */
  int bnb_c;            /* channels of that layer (column index modulo bnb_c) */
  float bnb_p;          /* its dropout probability */
  unsigned long long bnb_seed;
  int bnb_layer;
  /* out_planes == 2, flat tiling: rows [lo_row_begin, lo_row_end) are the only ones whose lo plane
   * a later stage reads (residual sources in the tap-major row order); tiles outside skip it.
   * lo_row_end == 0 means every row. */
  int lo_row_begin;
  int lo_row_end;
  /* elements between the A planes; 0 = samples * a_rows * a_ld (A is exactly its planes).  Set when
   * the A rows are a window into a larger buffer, such as a streaming history ring. */
  long long a_plane_stride;
  /* u8 copy of the output (precision FP16 or INT8, affine + ReLU [+ residual] launches only):
   * out_u8[row][c] = cvt.rni.sat.u8.f32(v * out_u8_inv_scale) of the fp32 value v that the fp16 store
   * rounds, rows as in `out`.  With INT8 and no residual `out` must be NULL (u8 only); NULL = off. */
  void* out_u8;
  int out_u8_ld;        /* >= n_pad, a multiple of 16 (out_u8 16-byte aligned) */
  float out_u8_inv_scale;
} vp3d_conv_desc;

int vp3d_conv_gemm(const vp3d_conv_desc* d, void* stream);
/* The kernel instance vp3d_conv_gemm(d) would run on the current device, under the SM limit of
 * vp3d_set_sm_limit: validates d and builds the launch exactly as vp3d_conv_gemm does, then writes
 * key[0..6] instead of launching:
 *   block_n (64 | 128), epilogue (0 training, 1 general, 2 lean),
 *   operand format (0 bf16 / fp16 read from the launch, 1 bf16, 2 fp16, 3 int8),
 *   schedule (0 cooperative, 1 ping-pong), auxiliary TMA tiles (0 | 1), two output planes (0 | 1),
 *   u8 output (0 none, 1 beside the 16-bit plane, 2 alone).
 * VP3D_ERR_UNSUPPORTED if that instance is not compiled (vp3d_conv_gemm then fails too);
 * VP3D_ERR_INVALID for out_rows == 0 (nothing is launched). */
int vp3d_conv_gemm_instance(const vp3d_conv_desc* d, int* key);
/* The keys of every compiled conv GEMM instance, 7 ints each as above, into keys[0 .. 7 * max);
 * returns how many instances are compiled (possibly more than max). */
int vp3d_conv_gemm_instances(int* keys, int max);

/* Weight gradient of one temporal convolution, the call vp3d_backward makes for every conv layer
 * (autograd's conv backward-filter):
 *   grad[(co * c_in + ci) * taps_out + tap] = sum_row dz[row][co] * x[xrow(row, tap)][xcol(tap, ci)]
 * flat (per_sample = 0): row < rows, xrow = row + tap * tap_row_step,
 *   xcol = tap * tap_col_step + ci, or tap * c_in + ci when merged (one GEMM over the taps_out * c_in
 *   columns of the strided expand conv's packed input; taps must then be 1);
 * per_sample = 1: the sum also runs over the samples, dz row t of sample n pairs with x row
 *   t + tap * tap_row_step of the same sample.
 * Operands are bf16 planes (planes 2: hi + lo, the three products hi*hi + lo*hi + hi*lo), fp32
 * accumulation.  The reduction is split over row ranges into `partial` and the splits are summed in
 * a fixed order (bit-reproducible); the tile width and the split count follow from the shape and the
 * SM count as in the training step, fewer splits when `partial` is small, VP3D_ERR_WORKSPACE (and
 * nothing launched) when it cannot hold one: taps * round_up(c_out, 128) * round_up(c_in_cols, 128)
 * floats always suffice for one split. */
typedef struct {
  const void* dz;     /* bf16 [planes][samples][rows][dz_ld] */
  int dz_ld;          /* multiple of 64, >= c_out rounded up to 64 */
  const void* x;      /* bf16 [planes][samples][x_rows][x_ld] (flat: [planes][rows][x_ld]) */
  int x_ld;           /* multiple of 64 */
  int planes;         /* 1 or 2 */
  long long rows;     /* dz rows: per sample when per_sample, else in total */
  int per_sample;
  int samples;        /* per_sample only */
  long long x_rows;   /* x rows per sample (per_sample only) */
  int taps;           /* GEMM taps (merged: 1) */
  int tap_row_step;   /* x row offset per tap (dilation), 0 for column taps */
  int tap_col_step;   /* x column offset per tap (strided layout), else 0 */
  int c_out;
  int c_in_cols;      /* x columns one tap's GEMM spans (merged: taps_out * c_in) */
  int c_in;
  int taps_out;       /* taps of the gradient tensor (= taps unless merged) */
  int merged;
  float* grad;        /* fp32 (c_out, c_in, taps_out), every entry overwritten */
  float* partial;     /* fp32 scratch */
  size_t partial_bytes;
} vp3d_wgrad_desc;

int vp3d_wgrad_gemm(const vp3d_wgrad_desc* d, void* stream);

/* The BatchNorm training passes around the GEMMs (each the launch the training step makes), with
 * DropoutCfg / RowMap flattened into plain arguments.  Channels c <= 8192.  The ordered reductions
 * take a caller-owned scratch of 96 * c floats (bn_stats_finalize) or 64 * c floats (the others) and
 * ceil(c / 32) ticket counters that the caller zeroes once; every launch leaves them zero again.
 *
 * vp3d_bn_stats_finalize: part = [slabs][2][c] per-slab sum / sum of squares as the conv GEMM
 *   epilogue writes them (slab s = rows (s % 4) * 32 .. + 32 of row tile s / 4; dilated: tiles per
 *   sample, out_rows rows each; flat: out_rows rows in total) -> batch mean, invstd =
 *   1 / sqrt(var + eps), scale = gamma * invstd, shift = beta - mean * scale; channels [c_real, c)
 *   get zeros.  running_mean / running_var (both or neither) are updated in place with `momentum`
 *   and the unbiased variance.
 * vp3d_ordered_col_sums: out_st[ch] = mul_st[ch] * sum_p sum_f part[p][st][f * c + ch] for
 *   st < nstat (1 or 2), f < folds; mul_st may be NULL (= 1).
 * vp3d_bn_apply: x = dropout(relu(z * scale + shift)) [+ res[map(row)]] on bf16 [planes][rows][c]
 *   (c a multiple of 64), map(r) = (r / res_div) * res_rows_per_sample + (r % res_div) * res_step +
 *   res_off, or r * res_step + res_off when res_div = 0.  Dropout keyed by (seed, layer, element).
 * vp3d_bn_bwd_reduce: sums[0][c] = sum dY, sums[1][c] = invstd * sum dY * (z - mean) with
 *   dY = g * mask * [z * scale + shift > 0]; `partials` holds the per-block partials
 *   (VP3D_ERR_WORKSPACE when too small).
 * vp3d_bn_bwd_apply: dz = scale * (dY - sums[0] / rows - (z - mean) * invstd * sums[1] / rows), and
 *   dbeta = sums[0], dgamma = sums[1] for the first c_real channels (each may be NULL).  frozen:
 *   dz = scale * dY; mean / invstd are not read and sums may be NULL (then nothing else written). */
int vp3d_bn_stats_finalize(const float* part, int slabs, int dilated, int out_rows,
                           int tiles_per_sample, const float* gamma, const float* beta,
                           float* running_mean, float* running_var, float momentum, float eps,
                           float* scale, float* shift, float* mean, float* invstd, int c, int c_real,
                           float* scratch, size_t scratch_floats, unsigned* counter, int counters,
                           void* stream);
int vp3d_ordered_col_sums(const float* part, int n_part, int nstat, int ld, int c, int folds,
                          const float* mul0, const float* mul1, float* out0, float* out1,
                          float* scratch, size_t scratch_floats, unsigned* counter, int counters,
                          void* stream);
int vp3d_bn_apply(const void* z, long long z_plane, void* x, long long x_plane, int planes,
                  long long rows, int c, const float* scale, const float* shift, float dropout_p,
                  unsigned long long seed, int layer, const void* res, long long res_plane,
                  int res_div, int res_rows_per_sample, int res_step, int res_off, void* stream);
int vp3d_bn_bwd_reduce(const void* g, long long g_plane, const void* z, long long z_plane, int planes,
                       long long rows, int c, const float* scale, const float* shift,
                       const float* mean, const float* invstd, float dropout_p,
                       unsigned long long seed, int layer, float* partials, size_t partial_floats,
                       float* sums, float* scratch, size_t scratch_floats, unsigned* counter,
                       int counters, void* stream);
int vp3d_bn_bwd_apply(const void* g, long long g_plane, const void* z, long long z_plane, void* dz,
                      long long dz_plane, int planes, long long rows, int c, const float* scale,
                      const float* shift, const float* mean, const float* invstd, float dropout_p,
                      unsigned long long seed, int layer, const float* sums, float* dgamma,
                      float* dbeta, int c_real, int frozen, void* stream);

/* ---- device-resident batch gather (SURVEY §8 row f1) --------------------------------------------
 * Replaces the per-chunk Python loops of the reference generators:
 *   common/generators.py:99-160  ChunkedGenerator.next_epoch   (training windows)
 *   common/generators.py:213-240 UnchunkedGenerator.next_epoch (whole padded sequences)
 * All sequences are stored once in device memory, back to back; one launch produces a batch from a
 * row table.  A row is 4 x int32 (sequence, first frame, end frame, flip) -- the reference's
 * `pairs` tuple (generators.py:39-48); `first_offset` is added to the first frame (2-D input:
 * -(pad + causal_shift), generators.py:103-104; 3-D target: 0).  Frames outside the sequence
 * replicate the nearest edge frame (np.pad 'edge', :108-118); flip negates feature 0 and reads
 * joint j from src_joint[j] (:120-123, :137-143).  Results are exact copies (bit-exact). */
typedef struct vp3d_gather_desc {
  const float* src;         /* [total_frames][joints][features] fp32 */
  const int64_t* seq_first; /* [n_seq] index of each sequence's first frame in src */
  const int32_t* seq_len;   /* [n_seq] frames per sequence (>= 1) */
  const int32_t* rows;      /* [n_windows][4] */
  const int32_t* src_joint; /* [joints] mirror source of each joint, or NULL (no joint swap) */
  float* out;               /* [n_windows][frames][joints][features] fp32 */
  int32_t n_windows;
  int32_t frames;           /* frames per window */
  int32_t joints;
  int32_t features;
  int32_t first_offset;
} vp3d_gather_desc;

int vp3d_gather_windows(const vp3d_gather_desc* d, void* stream);

/* Camera intrinsics rows for a batch: out[w] = cams[rows[w].sequence], entries 2 and 7 negated for
 * flipped rows (generators.py:146-152).  cams: [n_seq][cam_dim] fp32. */
int vp3d_gather_cameras(const float* cams, int32_t cam_dim, const int32_t* rows, int32_t n_windows,
                        float* out, void* stream);

/* ---- training-step companions (SURVEY §8 rows f4, f2) -------------------------------------------
 * vp3d_adam_step: one launch of Adam / AMSGrad over a list of fp32 tensors -- what
 * `optim.Adam(model.parameters(), lr=lr, amsgrad=True).step()` does per step (run.py:252, 264, 396,
 * 420) with torch's update rule: g += weight_decay*p; m += (1-b1)(g-m); v = b2 v + (1-b2) g^2;
 * vmax = max(vmax, v); p -= lr/(1-b1^t) * m / (sqrt(vmax)/sqrt(1-b2^t) + eps).  All pointers are
 * device pointers; `tensors` itself is a host array.  max_exp_avg_sq == NULL selects plain Adam for
 * that tensor.  `step` is the 1-based step count AFTER this update (torch's state['step']). */
#define VP3D_ADAM_MAX_TENSORS 64 /* per launch; longer lists are split */
typedef struct vp3d_adam_tensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  float* max_exp_avg_sq; /* NULL = no AMSGrad */
  int64_t numel;
} vp3d_adam_tensor;

int vp3d_adam_step(const vp3d_adam_tensor* tensors, int32_t n_tensors, int64_t step, double lr,
                   double beta1, double beta2, double eps, double weight_decay, void* stream);

/* vp3d_adam_step for the parameters of a model with a training plan, fused with the bf16 re-pack
 * of the conv weights (SURVEY §8 f4): tensors whose `param` is one of w->layers_conv_weight[] /
 * w->shrink_weight are updated by a kernel that writes the fresh value into the plan's forward
 * [tap][co][ci] and transposed [tap][ci][co] bf16 packs in the same pass; all others (BatchNorm,
 * bias, expand conv) go through the plain kernel.  After the call the plan's packs match the
 * updated parameters: the next vp3d_forward_train needs no vp3d_set_weights(VP3D_PACK_CONV |
 * VP3D_PACK_CONV_T).  Requires that the plan has run (or packed for) a training forward. */
int vp3d_adam_step_packed(vp3d_plan* plan, const vp3d_weights* w, const vp3d_adam_tensor* tensors,
                          int32_t n_tensors, int64_t step, double lr, double beta1, double beta2,
                          double eps, double weight_decay, void* stream);

/* Mean per-joint position error and its gradient in one launch (common/loss.py:11-17 mpjpe, :19-25
 * weighted_mpjpe; used at run.py:359, 413): loss = mean_j w_j * ||pred_j - target_j||_2 over
 * `joints_total` vectors of `dims` components; dpred (same shape as pred, may be NULL) receives
 * d loss / d pred.  joint_w: per-vector weights or NULL (= 1).  loss: one device float; NaN when
 * joints_total = 0, as torch.mean of an empty tensor.  The block sums are added in block order (no
 * floating-point atomics), so the same input gives the same bits.  `_ex` spreads the work over up
 * to 4096 blocks and needs `scratch`: device memory of at least
 * vp3d_mpjpe_scratch_bytes(joints_total) bytes (0 for a single block; then scratch may be NULL),
 * used by one call at a time.  The plain entry point runs one block: same results up to the order
 * of the fp32 sum, but slow on large inputs (0.49 ms instead of 9 us for 64 x 243 x 17 joints on
 * an H100 80GB HBM3 at 700 W). */
size_t vp3d_mpjpe_scratch_bytes(int64_t joints_total);
int vp3d_mpjpe_fwd_bwd_ex(const float* pred, const float* target, const float* joint_w,
                          int64_t joints_total, int32_t dims, float* loss, float* dpred,
                          void* scratch, size_t scratch_bytes, void* stream);
int vp3d_mpjpe_fwd_bwd(const float* pred, const float* target, const float* joint_w,
                       int64_t joints_total, int32_t dims, float* loss, float* dpred, void* stream);

/* Re-projection loss of the semi-supervised branch and its gradients in one launch (run.py:374-379:
 * `mpjpe(project_to_2d(predicted_pos + predicted_traj, cam), target_2d)`, projection per
 * common/camera.py:37-67, or :69-88 when `linear` != 0).  pos: [samples][frames][joints][3],
 * traj: [samples][frames][1][3], cam: [samples][9] = f(2) c(2) k(3) p(2), target:
 * [samples][frames][joints][2]; dpos / dtraj (same shapes as pos / traj) are both NULL or both set.
 * loss: NaN for samples = 0.  Block-ordered sum and `_ex` / scratch as for vp3d_mpjpe_fwd_bwd_ex,
 * with vp3d_projected_mpjpe_scratch_bytes(samples, frames_per_sample) bytes. */
size_t vp3d_projected_mpjpe_scratch_bytes(int64_t samples, int32_t frames_per_sample);
int vp3d_projected_mpjpe_fwd_bwd_ex(const float* pos, const float* traj, const float* cam,
                                    const float* target, int64_t samples, int32_t frames_per_sample,
                                    int32_t joints, int32_t linear, float* loss, float* dpos,
                                    float* dtraj, void* scratch, size_t scratch_bytes, void* stream);
int vp3d_projected_mpjpe_fwd_bwd(const float* pos, const float* traj, const float* cam,
                                 const float* target, int64_t samples, int32_t frames_per_sample,
                                 int32_t joints, int32_t linear, float* loss, float* dpos,
                                 float* dtraj, void* stream);

/* The whole loss head of the semi-supervised step (run.py:350-390, BASELINE configs[4]) and its
 * gradients in ONE cooperative launch:
 *   losses[0] = mpjpe(pos[:n_labeled], target_3d with joint 0 zeroed)                 run.py:336, 352
 *   losses[1] = weighted_mpjpe(traj[:n_labeled], target_3d[:, :, 0:1], 1 / z_root)    run.py:335, 358-360
 *   losses[2] = mpjpe(project_to_2d(pos[n_labeled:] + traj[n_labeled:], cam), target_2d)
 *               (common/camera.py:37-67, or :69-88 when `linear`)                     run.py:374-379
 *   losses[3] = mean_bone |mean_labeled(len) - mean_unlabeled(len)|, len = mean over frames of
 *               ||joint - parents[joint]||_2 (parents = dataset.skeleton().parents()) run.py:383-387
 *   losses[4] = sum of the terms selected by `terms` (run.py:354, 361, 380, 388; --no-proj and
 *               --no-bone-length clear VP3D_SEMI_PROJ / VP3D_SEMI_BONE); unselected terms are still
 *               reported in losses[0..3] when their inputs are given but carry no gradient
 * pos: [n_labeled + n_unlabeled][frames][joints][3]; traj: [...][frames][1][3]; target_3d:
 * [n_labeled][frames][joints][3] as the generator yields it (joint 0 = global trajectory);
 * cam: [n_unlabeled][9]; target_2d: [n_unlabeled][frames][joints][2]; parents: [joints] int32
 * (device; entries 1.. must lie in [0, joints): the library cannot check device memory, the Python
 * wrapper checks them on the host).  dpos / dtraj (shapes of pos / traj; both NULL or both set)
 * receive d losses[4] / d pos, / d traj.  n_unlabeled = 0 drops the penalty; with joints = 1 there
 * are no bones and the penalty is NaN, as the reference's mean over none.  target_3d / cam / target_2d may be NULL when the
 * terms that read them are not selected.  `scratch`: device memory of
 * vp3d_semi_loss_scratch_bytes() bytes.  joints <= 32. */
#define VP3D_SEMI_POS 1
#define VP3D_SEMI_TRAJ 2
#define VP3D_SEMI_PROJ 4
#define VP3D_SEMI_BONE 8
size_t vp3d_semi_loss_scratch_bytes(void);
int vp3d_semi_loss_fwd_bwd(const float* pos, const float* traj, const float* target_3d,
                           const float* cam, const float* target_2d, const int32_t* parents,
                           int64_t n_labeled, int64_t n_unlabeled, int32_t frames, int32_t joints,
                           int32_t linear, int32_t terms, float* losses, float* dpos, float* dtraj,
                           void* scratch, size_t scratch_bytes, void* stream);

/* ---- evaluation metrics (run.py:674-704, common/loss.py:11-17, :27-89) ------------------------
 * The four per-sequence means run.py's evaluate() computes, in one launch.  pred:
 * [copies][frames][joints][3] (copies 1 or 2); target: [frames][joints][3]; both fp32, device.
 * With copies == 2 the prediction is first flip-averaged as run.py:677-680 does:
 * avg = (pred[0] + mirror(pred[1])) * 0.5, mirror = negate x and read joint j from mirror_src[j]
 * (the map generators.mirror_source() builds; NULL = no joint swap, the trajectory model's case
 * at run.py:678).  `averaged` ([frames][joints][3] or NULL) receives avg, bit-identical to the
 * torch expression (return_predictions, run.py:682-683).  means[k] (device doubles) receives:
 *   [0] VP3D_EVAL_MPJPE     mean ||avg - target||                              loss.py:11-17
 *   [1] VP3D_EVAL_P_MPJPE   the same after per-frame similarity Procrustes     loss.py:27-66
 *   [2] VP3D_EVAL_N_MPJPE   the same after per-frame least-squares scale       loss.py:68-78
 *   [3] VP3D_EVAL_VELOCITY  mean ||diff(avg) - diff(target)|| along frames     loss.py:80-89
 * for the metrics selected in `which` (others are written as 0).  Per-frame algebra and every sum
 * are fp64 and in a fixed order: reproducible.  which == 0 only writes `averaged` (target, means and
 * scratch may then be NULL).  joints <= 32; frames == 0 is a no-op.  `scratch`: device memory of
 * vp3d_pose_errors_scratch_bytes(frames) bytes. */
#define VP3D_EVAL_MPJPE 1
#define VP3D_EVAL_P_MPJPE 2
#define VP3D_EVAL_N_MPJPE 4
#define VP3D_EVAL_VELOCITY 8
size_t vp3d_pose_errors_scratch_bytes(int64_t frames);
int vp3d_pose_errors(const float* pred, int32_t copies, const int32_t* mirror_src, const float* target,
                     int64_t frames, int32_t joints, int32_t which, float* averaged, double* means,
                     void* scratch, size_t scratch_bytes, void* stream);

/* ---- differentiable pose losses (common/loss.py:11-17, :27-89) ------------------------------
 * Any weighted subset of four terms and the gradient of their weighted sum with respect to `pred`,
 * in one cooperative launch.  pred, target: [seqs][frames_per_seq][joints][3] fp32, device; a pose
 * is one (seq, frame) slice.  Term k (flag bit 1 << k) is evaluated when term_weights[k] != 0:
 *   [0] VP3D_POSE_LOSS_MPJPE     mean ||p - t||                                  loss.py:11-17
 *   [1] VP3D_POSE_LOSS_N_MPJPE   mean ||s p - t||, s = mean <t, p> / mean <p, p> per pose
 *                                (ds/dp included in the gradient)                loss.py:68-78
 *   [2] VP3D_POSE_LOSS_P_MPJPE   mean distance after per-pose similarity Procrustes (centre,
 *                                normalise, rotation, scale, translation; the gradient flows through
 *                                all of them)                                    loss.py:27-66
 *   [3] VP3D_POSE_LOSS_VELOCITY  mean ||diff(p) - diff(t)||, first differences along the frame axis
 *                                within each sequence; NaN for frames_per_seq == 1 (np.mean of
 *                                nothing)                                        loss.py:80-89
 * term_weights: 4 host doubles.  terms_out[k] (device, 4 floats) receives term k, 0 when it is not
 * evaluated; loss_out (device float) receives sum_k term_weights[k] * terms_out[k] over the
 * evaluated terms.  dpred (shape of pred, or NULL: no backward) receives d loss / d pred.
 * Rotations: the top eigenpair of Horn's 4x4 matrix (fp64 Jacobi); a pose whose two largest
 * eigenvalues satisfy lambda_0 - lambda_1 <= 1e-12 max(|lambda_0|, 1) has no differentiable rotation
 * and gets the gradient with its rotation held fixed; degenerate_out (device int32, or NULL)
 * receives the number of such poses.  All-zero predictions give NaN, as the reference does.
 * fp64 inside, one rounding to fp32 per output; sums in a fixed order: the same input gives the same
 * bits.  joints <= 32; seqs == 0 is a no-op.  `scratch`: device memory of
 * vp3d_pose_loss_scratch_bytes(frames_per_seq, seqs) bytes. */
#define VP3D_POSE_LOSS_MPJPE 1
#define VP3D_POSE_LOSS_N_MPJPE 2
#define VP3D_POSE_LOSS_P_MPJPE 4
#define VP3D_POSE_LOSS_VELOCITY 8
size_t vp3d_pose_loss_scratch_bytes(int32_t frames_per_seq, int64_t seqs);
int vp3d_pose_loss_fwd_bwd(const float* pred, const float* target, int32_t frames_per_seq, int64_t seqs,
                           int32_t joints, const double* term_weights, float* terms_out, float* loss_out,
                           float* dpred, int32_t* degenerate_out, void* scratch, size_t scratch_bytes,
                           void* stream);

/* ---- streaming inference (common/model.py:63-77, 126-138 applied incrementally) ---------------
 * A session of S stream slots pushes k <= K new frames per slot at a time and gets back the output
 * frames they complete.  Per slot the concatenated outputs equal vp3d_forward_eval on the sequence
 * edge-padded as UnchunkedGenerator pads it (common/generators.py:216-238, run.py:186-193): pad +
 * causal_shift copies of the first frame in front, pad - causal_shift copies of the last behind.
 * Every conv layer keeps its input history in a time-major device ring inside the caller's state
 * buffer; a push costs the new frames' share of the FLOPs.  TemporalModel (VP3D_VARIANT_DILATED,
 * dense or not) in any precision but MIXED (INT8 with VP3D_STREAM_INT8, below); the plan's packed
 * eval weights are read at every push.
 *
 * vp3d_stream_lookahead: output frame t of a slot is returned by the push that delivers its input
 * frame t + lookahead (lookahead = pad - causal_shift: 0 for a causal model).
 * vp3d_stream_state_bytes: device bytes of a session's state (0 for an invalid or too large size).
 * vp3d_stream_init: registers `state` (device memory of at least state_bytes) with the plan and
 * clears it: every slot idle, all history dropped (also the way to reset a session).
 * vp3d_stream_push: x is (S, k, J_in, F) fp32; start_mask (S bytes, device, or NULL = none): slot
 * s begins a new sequence whose first frame is x[s, 0] (its history becomes the edge padding of
 * that frame, the other slots continue undisturbed); y receives (S, k, J_out, 3) fp32 and frame
 * (S, k) int64 the frame number within each slot's current sequence of every y row, -1 for rows
 * that are no frame (look-ahead warm-up, idle slot).  Asynchronous, no host synchronisation.
 * vp3d_stream_push_ex: vp3d_stream_push with three optional DEVICE arrays (vp3d_stream_push is
 * push_ex with all three NULL: the same bits and launches as before them):
 *   end (S int32, or NULL): end[s] = n in [0, k] ends slot s's sequence after frame n - 1 of this
 *     push (length = frames pushed before + n); -1 = it continues.  From then on the slot is fed the
 *     generator's end padding, its last real frame repeated (common/generators.py:216-238,
 *     run.py:186-193: pad - causal_shift copies behind), x[s, f >= n] is never read, and frame
 *     length - 1 comes out `lookahead` frames later (in the same push for a causal model); the push
 *     that returns it leaves the slot idle.  Rows past the end get frame -1.  end is ignored for an
 *     idle slot and for a sequence that has already ended; start_mask on a slot that is still
 *     draining begins the new sequence and drops the undelivered tail; start with end = 0 leaves the
 *     slot idle.  Values outside [-1, k] are read as -1 (a device array is not checked on the host).
 *     No extra launch.
 *   x_rows (S int64, or NULL): x is a flat (rows, J_in, F) fp32 store; frame f of slot s is row
 *     x_rows[s] + f, read only for f < n of an active slot whose sequence has not ended.
 *   y_rows (S int64, or NULL): y is a flat (rows, J_out, 3) fp32 buffer; the returned frame t of
 *     slot s (frame >= 0) is written to row y_rows[s] + t, rows of frame -1 are not written.  frame
 *     (S, k) is still written and is required.  The output kernel then always runs (one launch
 *     more where a push would shrink straight into y).
 * vp3d_stream_push_counts: vp3d_stream_push_ex plus one optional DEVICE array (push_ex is
 * push_counts with count = NULL: the same bits and launches):
 *   count (S int32, or NULL = k for every slot): slot s has count[s] real frames in this push, 0 to
 *     k, so streams that skip or drop frames share one session.  They are x[s, :count[s]] (rows
 *     x_rows[s] + f in row-addressed mode); x[s, f >= count[s]] is never read.  count is read only
 *     for a slot that holds an open sequence (active, or starting in this push) and does not end in
 *     this push: an ending slot's real frames are its first end[s], draining and idle slots advance
 *     as without counts.  Output row f of a counted slot is frame (frames pushed before) + f -
 *     lookahead for f < count[s] (under the warm-up rule), -1 for f >= count[s]; the slot's frame
 *     counter advances by count[s], and its later outputs stay those of the offline forward on its
 *     own padded sequence.  Values outside [0, k], and 0 on a slot that starts in this push (a start
 *     needs its first frame), are read as k.  With count != NULL two realign launches follow the
 *     last GEMM (the host cannot see the values): they move the history of every slot with
 *     count[s] < k forward by k - count[s] frames, 4 * sum_l H_l * ld_l * planes * 2 bytes per
 *     physical row moved (about 2 MB at arc 3,3,3,3,3, C = 1024, fp16), nothing for the others.
 * vp3d_stream_finish: emits the last `lookahead` frames of every slot by repeating each slot's
 * newest frame (the generator's end padding) into y (S, lookahead, J_out, 3) / frame (S,
 * lookahead), then marks every slot idle.  A slot whose sequence ended in an earlier push returns
 * what is left of its tail, and -1 after that.
 * vp3d_stream_release: forgets `state` (the caller frees the memory).
 *
 * Test-time flip augmentation (VP3D_STREAM_AUGMENT, the default of run.py, common/arguments.py:43):
 * vp3d_stream_state_bytes_ex / vp3d_stream_init_ex with flags = VP3D_STREAM_AUGMENT give every slot
 * a second, mirrored copy, as UnchunkedGenerator(augment=True) appends it (common/generators.py:
 * 223-237: x negated, input joint j read from kps_src[j]), run in the same launches (rows [S, 2S) of
 * every ring; the state is about twice as large).  Push and finish then return, per slot, the flip
 * average of run.py:674-680, bit-identical to it: (plain + mirror(mirrored)) * 0.5 with mirror =
 * negate x and read output joint j from joints_src[j].  kps_src: HOST int32 array of J_in entries
 * (the map generators.mirror_source(J_in, kps_left, kps_right) builds), required with AUGMENT;
 * joints_src: HOST int32 array of J_out entries, or NULL = negate x only (the trajectory model,
 * run.py:678).  init_ex checks every entry is in [0, J) and copies the maps into the state, so a push
 * still makes no host-to-device copy.  Unknown flag bits, and maps without AUGMENT, are errors.
 * vp3d_stream_state_bytes / vp3d_stream_init are the _ex calls with flags = 0 and no maps; push,
 * finish and release take either kind of session, with x, start_mask, y and frame shaped by S.
 *
 * Provisional outputs (VP3D_STREAM_PROVISIONAL, flags of the _ex calls, combinable with AUGMENT):
 * the session may also be pushed with vp3d_stream_push_provisional, which is
 * vp3d_stream_push_counts with dense x / y (x_rows = y_rows = NULL) that in addition writes what
 * vp3d_stream_finish would return if it were called right after this push, without ending anything:
 *   y_prov (S, lookahead, J_out, 3) fp32, frame_prov (S, lookahead) int64 (both DEVICE, required):
 *     per slot the frames [c - lookahead, c) of its sequence that are not final yet (c = frames
 *     pushed so far), computed with the generator's end padding as if the sequence ended now; -1
 *     below frame 0, past an ended sequence's length and for idle slots; flip-averaged with AUGMENT.
 *     The same bits as that finish, and the push's own y / frame and every later push are what
 *     they would be without the request.  The push's GEMMs run over k + lookahead frame rows
 *     (the look-ahead tail rides in the same launches); the output kernel always runs.
 * The flag sizes every ring for K + lookahead new rows (vp3d_stream_state_bytes_ex grows) and is
 * VP3D_ERR_INVALID on a causal plan (lookahead 0; state_bytes_ex returns 0).  A push_provisional on a
 * session initialised without it is VP3D_ERR_STATE.  Plain pushes and finish of a flagged session
 * keep their bits and launches.
 *
 * int8 sessions (VP3D_STREAM_INT8, flags of the _ex calls, combinable with AUGMENT and
 * PROVISIONAL): an INT8 plan streams only with this flag (init / init_ex without it stay
 * VP3D_ERR_UNSUPPORTED, and state_bytes_ex without it keeps its size), and the flag needs an INT8
 * plan (state_bytes_ex returns 0, init_ex VP3D_ERR_INVALID).  Every push and finish returns, per
 * slot, the bits of the offline int8 forward (vp3d_forward_eval) on the padded sequence: the blocks
 * of the plan's int8 mask run u8 x s8, the rest fp16, in the push's own launches.  Each ring of a
 * residual block keeps a u8 copy of its history next to the 16-bit one (sized for every block,
 * whatever the mask: about 1.5x the 16-bit ring bytes in all).  Launches: those of the same fp16
 * session when every block runs int8, plus one quantise launch per fp16 -> int8 block transition in
 * the push and one in the start pass where it contains that transition.  A push or finish needs
 * folded scales (vp3d_set_int8_scales, then vp3d_set_weights), VP3D_ERR_STATE otherwise.  The
 * history depends on the block mask and the activation scales: the session records both at its
 * first push (or finish) after init, and a later push or finish that finds either changed
 * (vp3d_set_int8_blocks, vp3d_set_int8_scales) is VP3D_ERR_STATE until the session is initialised
 * again, so old and new quantisations never mix.
 *
 * Held provisional outputs (VP3D_STREAM_HELD, flags of the _ex calls, combinable with AUGMENT and
 * INT8, valid on causal plans; together with PROVISIONAL it is VP3D_ERR_INVALID and state_bytes_ex
 * returns 0, because push_held with max_held = 0 already is the provisional push): the provisional
 * outputs of a detector-fed session (streaming.StreamingSession.push_detections), whose slots may
 * hold pending frames after their last detection that vp3d_stream_finish would first receive as
 * that detection repeated.  The flag sizes every ring for K + RF - 1 new rows (RF =
 * vp3d_receptive_field): past RF - 1 end-padding rows every tail row is a bit copy of the last one
 * computed, so no push computes more.  Flag bits 2, 8 and 32 stay unknown.
 * vp3d_stream_push_held is vp3d_stream_push_provisional with, per slot, the pending frames of its
 * open sequence:
 *   held: DEVICE (S,) int32, read for open sequences only; values outside [0, max_held] read as 0.
 *   max_held >= 0 and rows >= lookahead + max_held: y_prov (S, rows, J_out, 3) fp32 and frame_prov
 *     (S, rows) int64 (DEVICE, required).  frame_prov[s, j] = c - lookahead + j for j < lookahead +
 *     held[s] under the rules of `frame` (c = frames pushed so far), -1 otherwise; y_prov row j with
 *     a frame >= 0 is, bit for bit, the row vp3d_stream_finish would return for that frame right
 *     after pushing the held frames as the slot's last frame repeated.  Other rows are unspecified.
 *   The chain runs over k + T frame rows, T = min(lookahead + max_held, RF - 1); T = 0 (a causal
 *     plan, max_held = 0) computes no tail and leaves y_prov unwritten.  Launches: those of
 *     vp3d_stream_push_counts, plus the output kernel where that shrinks straight into y.  Nothing
 *     of the request persists.  VP3D_ERR_STATE on a session initialised without the flag. */
#define VP3D_STREAM_AUGMENT 1
#define VP3D_STREAM_PROVISIONAL 4
#define VP3D_STREAM_INT8 16
#define VP3D_STREAM_HELD 64
int vp3d_stream_lookahead(const vp3d_plan* plan);
size_t vp3d_stream_state_bytes(const vp3d_plan* plan, int S, int K);
int vp3d_stream_init(vp3d_plan* plan, void* state, size_t state_bytes, int S, int K, void* stream);
size_t vp3d_stream_state_bytes_ex(const vp3d_plan* plan, int S, int K, int flags);
int vp3d_stream_init_ex(vp3d_plan* plan, void* state, size_t state_bytes, int S, int K, int flags,
                        const int32_t* kps_src, const int32_t* joints_src, void* stream);
int vp3d_stream_push(vp3d_plan* plan, void* state, const float* x, int k, const uint8_t* start_mask,
                     float* y, int64_t* frame, void* stream);
int vp3d_stream_push_ex(vp3d_plan* plan, void* state, const float* x, int k,
                        const uint8_t* start_mask, const int32_t* end, const int64_t* x_rows,
                        const int64_t* y_rows, float* y, int64_t* frame, void* stream);
int vp3d_stream_push_counts(vp3d_plan* plan, void* state, const float* x, int k,
                            const uint8_t* start_mask, const int32_t* end, const int64_t* x_rows,
                            const int64_t* y_rows, float* y, int64_t* frame, const int32_t* count,
                            void* stream);
int vp3d_stream_push_provisional(vp3d_plan* plan, void* state, const float* x, int k,
                                 const uint8_t* start_mask, const int32_t* end,
                                 const int32_t* count, float* y, int64_t* frame, float* y_prov,
                                 int64_t* frame_prov, void* stream);
int vp3d_stream_push_held(vp3d_plan* plan, void* state, const float* x, int k,
                          const uint8_t* start_mask, const int32_t* end, const int32_t* count,
                          const int32_t* held, int max_held, int rows, float* y, int64_t* frame,
                          float* y_prov, int64_t* frame_prov, void* stream);
int vp3d_stream_finish(vp3d_plan* plan, void* state, float* y, int64_t* frame, void* stream);

/* Moving slots between sessions (streaming.StreamSlots).  A slot's sequence is the reference's
 * padded forward (run.py:186-193, common/generators.py:216-238) wherever its pushes run: export
 * copies what a later push reads of the listed slots into a DEVICE blob, import puts it into slots of
 * another compatible session, and each imported slot then continues its sequence -- frame numbers,
 * `end`, draining tail and outputs -- bit for bit as if every push had gone to the session it came
 * from (the offline forward on its padded sequence).  What a slot carries: per physical row (two
 * with AUGMENT) and ring l, the H_l newest history positions of every plane (and of the u8 plane of
 * rings 1..nb with INT8), by rank, plus its frame bookkeeping; nothing else persists between pushes.
 * The blob stores frame ranks, not ring positions, so S, K, the PROVISIONAL / HELD sizing and the
 * device of the two sessions may differ.
 *
 * vp3d_stream_slot_bytes: bytes of one slot's record for a session of `flags` (AUGMENT and INT8
 *   shape it; 0 for a null plan, unknown flags or INT8 on a plan that is not int8).  At arc
 *   3,3,3,3,3, C = 1024, fp16: 32 + 2 * 64 * 2 + 240 * 1024 * 2 bytes, about 0.49 MB.
 * vp3d_stream_export: copies slots[0..n) (HOST int32, each in [0, S), repeats allowed) of `state`
 *   into `blob` (DEVICE, 16-byte aligned, blob_bytes >= n * slot_bytes) record after record, and
 *   fills the HOST `header` with what import checks without reading the device: the configuration,
 *   ring geometry, the AUGMENT / INT8 flags and the session's int8 snapshot (block mask and
 *   activation scales of its history).  The session is not changed; idle, open and draining slots
 *   export alike.
 * vp3d_stream_import: replaces slots[0..n) (HOST int32, distinct, in [0, S)) of `state` with the n
 *   records of a blob exported with `header`, as a start replaces a sequence; the other slots are
 *   not disturbed.  The header must match this session: n, configuration (precision included),
 *   geometry and flags, and with an int8 snapshot the plan's current block mask and scales and the
 *   session's own snapshot, if it has one (it records the blob's otherwise); VP3D_ERR_STATE
 *   otherwise.  The weights and the AUGMENT mirror maps live on the device and are the caller's to
 *   match (streaming.StreamSlots fingerprints them).
 * Both return argument errors (null pointers, n < 1, a misaligned or too small blob, a slot out of
 * range, a repeated import slot) and header mismatches before any device work, under their own
 * names.  Each runs one launch per 1024 listed slots on `stream`, in order with the pushes, and no
 * host synchronisation. */
#define VP3D_STREAM_SLOTS_VERSION 1
typedef struct {
  int32_t version;          /* VP3D_STREAM_SLOTS_VERSION */
  int32_t n;                /* slot records in the blob */
  vp3d_config cfg;          /* the exporting plan's configuration */
  int32_t flags;            /* the exporting session's AUGMENT | INT8 bits */
  int32_t rings, planes, f16, lookahead;
  int32_t H[VP3D_MAX_WIDTHS], ld[VP3D_MAX_WIDTHS];   /* per ring: history positions, row values */
  int32_t int8_snap;        /* 1: the history holds the quantisation below */
  uint32_t int8_mask;
  float act_scale[VP3D_MAX_LAYERS];
  int64_t slot_bytes;       /* bytes of one record */
} vp3d_stream_slots_header;
size_t vp3d_stream_slot_bytes(const vp3d_plan* plan, int flags);
int vp3d_stream_export(vp3d_plan* plan, void* state, const int32_t* slots, int n, void* blob,
                       size_t blob_bytes, vp3d_stream_slots_header* header, void* stream);
int vp3d_stream_import(vp3d_plan* plan, void* state, const int32_t* slots, int n, const void* blob,
                       size_t blob_bytes, const vp3d_stream_slots_header* header, void* stream);

/* Detector input (streaming.StreamingSession.push_detections): the input rows of the pushes one
 * call makes, from a 2-D detector's pixel keypoints, as the reference's in-the-wild pipeline
 * prepares them.  It replaces, per released frame, joint and coordinate:
 *   data/prepare_data_2d_custom.py:39-49  np.interp(indices, indices[mask], kp[mask, i, j]) over
 *     the frames without a detection (float64, stored as float32): slope = (r - l) / (ib - ia),
 *     then slope * (t - ia) + l; a detected frame is its own value;
 *   run.py:93-97, common/camera.py:14-18  X / w * 2 - [1, h / w]: float32 X / w and * 2, a float64
 *     subtraction of 1 (x) or h / w (y), stored as float32.
 * Each operation is rounded on its own (no FMA contraction), so the rows are numpy's bits.
 * kps_px: DEVICE (S, k, J, 2) fp32 pixel keypoints of this call.  last: DEVICE (2, S, J, 2) fp32,
 * the last detection of every slot, double-buffered: half `parity` is read, half 1 - parity
 * written.  table: DEVICE int32, S triples (w, h, keep) then `rows` records (slot, left, right,
 * num, den); keep = the row of kps_px[s] with the slot's newest detection (written to the new
 * half), -1 = copy the old half.  Record r makes out row r (J x 2 fp32): left = row of kps_px[slot]
 * with the left value, -1 = the slot's stored last detection, -2 = no frame (zeros); right = row of
 * the right value of an interpolation with num = t - ia and den = ib - ia, -1 = a copy of the left
 * value.  Records whose indices fall outside kps_px, or a slot with w or h <= 0, give zeros.  out:
 * DEVICE (rows, J, 2) fp32.  One launch; argument errors (sizes, parity, null or not 8-byte aligned
 * pointers) are returned before any device work. */
int vp3d_stream_pack_detections(const float* kps_px, int S, int k, int J, const int32_t* table,
                                int64_t rows, float* last, int parity, float* out, void* stream);
int vp3d_stream_release(vp3d_plan* plan, void* state);

/* ---- offline inference on a list of clips (run.py:186-193, 663-721 over a known set of clips) ----
 * Replaces the per-clip loop of run.py's evaluate() -- UnchunkedGenerator(common/generators.py:
 * 213-240) padding each clip, model(batch) (common/model.py:63-77, 126-138), the flip average of
 * run.py:674-680 -- with ONE GEMM chain over many clips.  Each clip is edge-padded as the generator
 * pads it (pad + causal_shift copies of its first frame in front, pad - causal_shift of its last
 * behind, pad = (RF - 1) / 2), the padded clips are concatenated, and the dilated eval chain of
 * vp3d_forward_eval runs over them as one sample of `rows` frames.  Output row t of the chain
 * depends on rows [t, t + RF - 1] only, so a clip's T outputs are exactly its own forward: per clip
 * bit-identical to vp3d_forward_eval on the padded clip whenever that takes the dilated schedule
 * (T >= 2 or a dense model; a 1-frame clip pads to RF frames, where vp3d_forward_eval takes the
 * strided schedule and sums in another order -- the chain then gives a streaming session's bits).
 *
 * Clip i of T_i frames takes copies * (T_i + RF - 1) packed rows (copies = 2 with
 * VP3D_CLIPS_AUGMENT: the plain copy, then the mirrored one of common/generators.py:223-237).
 * vp3d_clips_workspace_bytes: device bytes of one chain's workspace (0 for a plan or size the chain
 * does not cover).
 * vp3d_forward_clips: one chain.  x: the flat fp32 store (rows, J_in, F) the clips are read from;
 * clip_first (int64), clip_len (int32) and y_first (int64): DEVICE arrays of `clips` entries, frame f
 * of clip i is store row clip_first[i] + f, its output frame t goes to row y_first[i] + t of the flat
 * fp32 output y (rows, J_out, 3).  rows must equal copies * sum_i (clip_len[i] + RF - 1); the host
 * checks what it can see without reading the device table (at least copies * RF rows per clip, a
 * multiple of copies), and the kernels touch no chain row outside [0, rows) whatever the table holds
 * (lengths below 1 read as 1).  kps_src / joints_src: HOST int32 mirror maps of J_in / J_out entries
 * as for vp3d_stream_init_ex (kps_src required with VP3D_CLIPS_AUGMENT, joints_src NULL = negate x
 * only, the trajectory model; up to 256 joints), checked and passed to the kernels by value: the
 * call makes no copy.  With augment y receives the flip average, (plain + mirror(mirrored)) * 0.5.
 * TemporalModel (VP3D_VARIANT_DILATED, dense or not) in bf16, bf16x3, fp16 and int8 (folded scales);
 * `mixed` is refused (its per-layer split depends on the geometry).  Launches 1 + (2B + 2) + 1
 * kernels (vp3d_last_launch_count), asynchronous on `stream`, no host synchronisation. */
#define VP3D_CLIPS_AUGMENT 1
size_t vp3d_clips_workspace_bytes(const vp3d_plan* plan, int64_t rows, int flags);
int vp3d_forward_clips(vp3d_plan* plan, const float* x, const int64_t* clip_first,
                       const int32_t* clip_len, int clips, int64_t rows, int flags,
                       const int32_t* kps_src, const int32_t* joints_src, float* y,
                       const int64_t* y_first, void* workspace, size_t workspace_bytes,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VP3D_B200_H_ */
