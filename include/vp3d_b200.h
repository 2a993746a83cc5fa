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
  VP3D_PRECISION_FP16 = 3    /* eval default: IEEE fp16 operands and activations (11-bit significand,
                                single plane), fp32 accumulate -- the tensor rate of bf16 at 1/8 of
                                its rounding error: ~4e-4 of fp32 on cfg2, inside north_star's 1e-3.
                                Stores saturate at +-65504.  Inference only (training runs bf16 /
                                bf16x3: gradients need the bf16 exponent range) */
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
} vp3d_conv_desc;

int vp3d_conv_gemm(const vp3d_conv_desc* d, void* stream);

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
 * d loss / d pred.  joint_w: per-vector weights or NULL (= 1).  loss: one device float. */
int vp3d_mpjpe_fwd_bwd(const float* pred, const float* target, const float* joint_w,
                       int64_t joints_total, int32_t dims, float* loss, float* dpred, void* stream);

/* Re-projection loss of the semi-supervised branch and its gradients in one launch (run.py:374-379:
 * `mpjpe(project_to_2d(predicted_pos + predicted_traj, cam), target_2d)`, projection per
 * common/camera.py:37-67, or :69-88 when `linear` != 0).  pos: [samples][frames][joints][3],
 * traj: [samples][frames][1][3], cam: [samples][9] = f(2) c(2) k(3) p(2), target:
 * [samples][frames][joints][2]; dpos / dtraj (same shapes as pos / traj) are both NULL or both set. */
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
 * (device).  dpos / dtraj (shapes of pos / traj; both NULL or both set) receive d losses[4] / d pos,
 * / d traj.  n_unlabeled = 0 drops the penalty.  target_3d / cam / target_2d may be NULL when the
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

#ifdef __cplusplus
}
#endif
#endif /* VP3D_B200_H_ */
