// Internals shared by the C-ABI translation units (api.cu: plan + eval; train_api.cu: training).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <map>
#include <vector>

#include "../../include/vp3d_b200.h"
#include "conv_gemm.cuh"
#include "pack.cuh"

namespace vp3d {

int fail(int code, const char* fmt, ...);

#define CUDA_TRY(expr)                                                                       \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return ::vp3d::fail(VP3D_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                     \
                          cudaGetErrorString(_e), __FILE__, __LINE__);                       \
  } while (0)
#define VP3D_TRY(expr)            \
  do {                            \
    int _s = (expr);              \
    if (_s != VP3D_OK) return _s; \
  } while (0)

// 4-D bf16 map (k, row, sample, plane), box (64, box_rows, 1, 1), 128-byte swizzle; with
// elem_bytes = 1 a byte map (u8 / s8 operands) whose box is 128 elements wide (the same 128 bytes).
// box_bytes and swizzle set another box width (in bytes) and swizzle.
int make_map_4d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t row_stride,
                uint64_t samples, uint64_t sample_stride, uint64_t planes, uint64_t plane_stride,
                uint32_t box_rows, int elem_bytes = 2, uint32_t box_bytes = 128,
                CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);
// 2-D bf16 map (k, row), box (64, box_rows), 128-byte swizzle; elem_bytes as above.
int make_map_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint32_t box_rows,
                int elem_bytes = 2);

int pick_block_n(int n_pad);
inline int round_up(int v, int m) { return (v + m - 1) / m * m; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
// Carves a caller-sized device buffer (workspace, streaming state, scratch) into buffers that each
// start on an `align` boundary.  total() adds `align` bytes of slack so that any pointer the caller
// passes can be rounded up by ws_base: the two halves of one contract.
struct Arena {
  size_t align, off = 0;
  // the offset of the next buffer of `bytes` bytes
  size_t take(size_t bytes) {
    const size_t o = off;
    off = align_up(off + bytes, align);
    return o;
  }
  size_t total() const { return off + align; }
};
// the aligned base of a caller's buffer sized by Arena::total with the same alignment
inline uint8_t* ws_base(void* ws, size_t align = 1024) {
  return reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(ws), align));
}
int num_sms();
int run_conv(const vp3d_conv_desc* d, cudaStream_t stream);


// One 16-bit pack of a Conv1d weight (c_out, c_in, taps) (model.py:102,113-118), stored as
// [planes][stored_taps][n_pad][k_pad], zero padded:
//   forward:    [tap][co][ci]; merged: one slab [co][tap*c_in + ci] (expand conv as a plain GEMM)
//   transposed: [tap][ci][co] for the data-gradient GEMMs; merged: one slab [tap*c_in + ci][co]
// Every pack of a plan is one entry of its pack table (vp3d_plan::packs), whose geometry
// vp3d_plan_create fixes once; allocation, packing, the fused optimizer and the GEMM descriptors
// all read it from there.
enum { kSrcExpand = -1, kSrcShrink = -2 };
struct PackedConv {
  int src = 0;  // vp3d_weights tensor: kSrcExpand, kSrcShrink or l for layers_conv[l]
  int c_out = 0, c_in = 0, taps = 0;
  bool transposed = false, merged = false;
  int stored_taps = 0, n_pad = 0, k_pad = 0;
  __nv_bfloat16* w = nullptr;  // transposed packs: allocated with the training state
  float* scale = nullptr;      // forward packs: eval affine of the conv's output [n_pad]
  float* shift = nullptr;
  // int8 plans, the convs of the blocks in int8_mask: w holds s8 [taps][n_pad][k_pad] (k_pad a
  // multiple of 128), w_scale its per-channel weight scales and q_scale the affine scale with both
  // dequantisation factors folded in (launch_int8_fold), both [n_pad]; the other blocks' convs
  // hold the fp16 pack of an FP16 plan (k_pad = C)
  float* w_scale = nullptr;
  float* q_scale = nullptr;
};
constexpr int kMaxPacks = 2 * VP3D_MAX_LAYERS + 5;

inline const float* conv_weight(const vp3d_weights* w, int src) {
  return src == kSrcExpand ? w->expand_conv_weight
         : src == kSrcShrink ? w->shrink_weight : w->layers_conv_weight[src];
}

// One coordinate of the test-time flip average (run.py:677-680): p0 from the plain copy, p1 from the
// mirrored copy (its joints already swapped back), axis 0 negated back.  Rounded as torch rounds
// `torch.mean(stack(p0, mirror(p1)), dim=0)`: one fp32 add, then the exact * 0.5.  The one
// definition of run.py's averaging, shared by the metrics of pose_loss.cu and stream.cu.
__device__ __forceinline__ float flip_average(float p0, float p1, int axis) {
  return __fmul_rn(__fadd_rn(p0, axis == 0 ? -p1 : p1), 0.5f);
}

struct TrainState;  // train_api.cu

// stream.cu: host side of one streaming session (vp3d_stream_init); the rings live in the
// caller's device state buffer
struct StreamHost {
  int S = 0, K = 0;       // logical stream slots, max frames per push
  int flags = 0;          // VP3D_STREAM_* of vp3d_stream_init_ex
  bool joint_src = false; // AUGMENT: an output joint map is stored in the state (else negate x only)
  long long q = 0;        // frames pushed since vp3d_stream_init (all slots advance together)
  long long prev_q = 0;   // q before the last push
  int prev_k = 0;         // frames of the last push (their ring rows still need their mirror copy)
  int parity = 0;         // bookkeeping buffer the next push reads (the pushes alternate the two)
  // VP3D_STREAM_INT8: the plan's block mask and activation scales at the first push or finish after
  // init; the history holds their quantisation, so a later push with other values is an error
  bool int8_snap = false;
  uint32_t int8_mask = 0;
  float act_scale[VP3D_MAX_LAYERS] = {};
};

// step_ops.cu: Adam / AMSGrad update of conv weights that also refreshes their bf16 packs
struct AdamPackItem {
  vp3d_adam_tensor t;
  const PackedConv* fwd;  // the conv's forward pack
  const PackedConv* tr;   // and its transposed pack (neither merged)
};
int launch_adam_pack(const AdamPackItem* items, int n, int planes, int64_t step, double lr,
                     double beta1, double beta2, double eps, double weight_decay,
                     cudaStream_t stream);

// A device allocation that grows to the largest size asked of it and is freed with its owner.
template <class T>
struct DeviceBuffer {
  T* ptr = nullptr;
  size_t bytes = 0;
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  ~DeviceBuffer() { if (ptr) cudaFree(ptr); }
  int grow(size_t n) {
    if (n <= bytes) return VP3D_OK;
    if (ptr) cudaFree(ptr);
    ptr = nullptr; bytes = 0;
    CUDA_TRY(cudaMalloc(&ptr, n));
    bytes = n;
    return VP3D_OK;
  }
};

constexpr int kMaxHostChunks = 16;   // H2D chunks of one vp3d_forward_eval_host call

// What the host-buffer entries (vp3d_forward_eval_host, _submit / _wait) create on first use and
// keep for the plan's lifetime.
struct HostStaging {
  DeviceBuffer<float> x, y;
  DeviceBuffer<void> ws;                     // shared by every host entry and both slots
  cudaStream_t stream = nullptr;             // compute
  cudaStream_t copy_stream = nullptr;        // H2D chunks overlap the compute stream
  cudaEvent_t copy_events[kMaxHostChunks] = {};
  // pipelined host API: two independent staging slots
  struct Slot {
    DeviceBuffer<float> x, y;
    cudaEvent_t copied = nullptr, done = nullptr;
    bool busy = false;
  };
  Slot slots[2];
  ~HostStaging();
};

}  // namespace vp3d

struct vp3d_plan {
  vp3d_config cfg;
  int nb = 0;  // residual blocks
  int C = 0;        // channels of the residual stream as laid out in memory: padded to 64
  int c_real = 0;   // the model's `channels` argument (any positive value, model.py:85-86)
  int c_in_raw = 0, c_out_raw = 0, c_in_pad = 0, k0_pad = 0, c_out_pad = 0;
  int planes = 1;
  int f16 = 0;  // VP3D_PRECISION_FP16 (and INT8): 16-bit stores hold IEEE fp16
  int int8 = 0; // VP3D_PRECISION_INT8: the residual blocks' convs run u8 x s8
  // int8: bit i - 1 set = block i runs u8 x s8, the others as in FP16 (vp3d_set_int8_blocks)
  uint32_t int8_mask = 0;
  // int8: activation scale s and 1 / s of every block conv's input (vp3d_set_int8_scales), and
  // whether the packs' q_scale vectors have been folded from the current scales
  bool int8_scales = false, int8_folded = false;
  float act_scale[VP3D_MAX_LAYERS] = {}, act_inv[VP3D_MAX_LAYERS] = {};
  int pad[VP3D_MAX_WIDTHS];
  int shift_dil[VP3D_MAX_WIDTHS];  // causal shift in frames (TemporalModel, model.py:111)
  int shift_str[VP3D_MAX_WIDTHS];  // causal shift in strided units (Optimized1f, model.py:176)
  int dilation[VP3D_MAX_WIDTHS];
  int taps[VP3D_MAX_WIDTHS];       // taps of block i's first conv (dense: 2*pad+1)
  // the pack table: forward packs (expand dilated and tap-merged, layers_conv, shrink), then the
  // transposed ones of training (layers_conv, shrink, expand in the variant's layout)
  vp3d::PackedConv packs[vp3d::kMaxPacks];
  int n_packs = 0;
  // views into it
  vp3d::PackedConv *expand_dil = nullptr, *expand_flat = nullptr, *shrink = nullptr;
  vp3d::PackedConv* conv[VP3D_MAX_LAYERS] = {};
  vp3d::PackedConv *expand_t = nullptr, *shrink_t = nullptr;
  vp3d::PackedConv* conv_t[VP3D_MAX_LAYERS] = {};
  std::vector<void*> allocs;
  bool conv_packed = false, bn_packed = false;
  vp3d::HostStaging host;
  int last_launches = 0;
  // measurement hook: event pairs around one chosen launch of each forward
  int prof_launch = -1;
  std::vector<cudaEvent_t> prof_events;  // start/stop pairs
  size_t prof_used = 0;                  // events consumed since the last read
  // training-mode state (transposed weight packs, per-layer BN vectors, dropout config)
  vp3d::TrainState* train = nullptr;
  // streaming sessions of this plan, keyed by their device state buffer
  std::map<const void*, vp3d::StreamHost> streams;
};

namespace vp3d {
int plan_alloc(vp3d_plan* p, void** out, size_t bytes);
bool use_strided(const vp3d_plan* p, int T);
// rows per sample after each stage: L[0] = rows out of expand, L[i] = rows out of block i
int layer_rows(const vp3d_plan* p, int T, bool strided, int* L);
int strided_trim(const vp3d_plan* p, int* L);
// whether residual block i (1..nb) runs u8 x s8
inline bool block_is_int8(const vp3d_plan* p, int i) {
  return p->int8 && ((p->int8_mask >> (i - 1)) & 1u);
}
// operands of chain layer i (0 = expand, 1..nb = residual blocks, nb + 1 = shrink) in every
// precision but `mixed` (whose split depends on the rows, eval_chain): int8 runs the blocks of
// int8_mask u8 x s8 and expand, shrink and the other blocks fp16
inline int layer_precision(const vp3d_plan* p, int i) {
  if (!p->int8) return p->cfg.precision;
  return i >= 1 && i <= p->nb && block_is_int8(p, i) ? VP3D_PRECISION_INT8 : VP3D_PRECISION_FP16;
}
// int8 plans keep the forward packs of their int8 blocks' convs in s8
inline bool pack_is_s8(const vp3d_plan* p, const PackedConv& k) {
  return !k.transposed && k.src >= 0 && block_is_int8(p, k.src / 2 + 1);
}
inline size_t pack_bytes(const vp3d_plan* p, const PackedConv& k) {
  return (size_t)p->planes * k.stored_taps * k.n_pad * k.k_pad *
         (pack_is_s8(p, k) ? 1 : sizeof(__nv_bfloat16));
}
// packs k from its fp32 weight in w; a transposed pack given `fwd` writes that forward pack of the
// same conv in the same pass
int pack_weight(const vp3d_plan* p, const PackedConv& k, const vp3d_weights* w, cudaStream_t stream,
                const PackedConv* fwd = nullptr);
// the forward packs of the expand conv (dilated and tap-merged) from w->expand_conv_weight
int pack_expand_forward(const vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream);
// GEMM weight operand of a conv descriptor: pointer, taps, K per tap and N as stored in k
void use_pack(vp3d_conv_desc* d, const PackedConv& k);
// a conv GEMM descriptor over one flat sample with the plan's planes and operands in `precision`,
// every other field cleared
inline vp3d_conv_desc conv_desc(const vp3d_plan* p, int precision) {
  vp3d_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.a_planes = d.out_planes = d.res_planes = p->planes;
  d.precision = precision;
  d.samples = 1;
  return d;
}

// One stage of the eval-mode GEMM chain: the expand conv (stage 0) or residual block i, whose k-tap
// conv writes H and whose 1x1 conv reads H, adds the block input as residual and writes X_i.
struct ChainStage {
  // input [plane][samples][in_rows][pitch], pitch the expand pack's K (stage 0) or C, planes as the
  // stage before wrote them: A of the k-tap conv and, res_row_off rows into a sample, the residual
  const __nv_bfloat16* in;
  int in_rows;
  __nv_bfloat16* out;        // X_i, [plane][rows][C]
  long long out_plane, h_plane;   // elements between the planes of X_i, and of H in this block
  int out_rows;              // per sample (per-sample tiles) or in all (flat)
  int tap_row_step, res_row_off;
  int lo_row_begin, lo_row_end;   // as in vp3d_conv_desc, of the GEMM that writes X_i
  // int8 block i: its u8 A operand Q_{i-1}, [samples][in_rows][C] (the rows of `in`), and the bytes
  // of the buffer it lies in; the offline chains read what stage i - 1's q_out wrote, a streaming
  // push a window of ring i's u8 plane
  const uint8_t* q_in;
  long long q_in_bytes;
  uint8_t* q_out;            // int8 chain: the u8 copy Q_i of X_i that block i + 1 reads, or null
};
// The geometry of one run of the chain: what the offline forward (strided, dilated), the streaming
// push and its start pass differ in.  run_infer_chain makes every GEMM descriptor from it.
struct InferChain {
  ChainStage st[VP3D_MAX_WIDTHS];
  int stages;                  // stages 0 .. stages-1 run
  int samples;                 // of every stage's input
  long long in_plane;          // elements between the planes of stage 0's input
  int per_sample_tiles;        // of every GEMM but shrink (else: flat rows)
  const PackedConv* expand;    // the plan's expand_flat or expand_dil
  __nv_bfloat16* h;
  float* y;                    // fp32 rows shrink writes from the last stage's output; null: no shrink
  int precision[VP3D_MAX_WIDTHS + 1];   // operands of expand, of block i, of shrink (nb + 1)
  bool profile;                // honour vp3d_profile_launch
  uint8_t* hq;                 // int8 blocks: H as u8 [rows][C]
  // calibration (vp3d_calibrate_int8): fp32 bits of amax[2B], folded after every GEMM whose output
  // an int8 plan quantises; null otherwise
  unsigned* amax;
  // calibration (vp3d_calibrate_int8_hist): the histograms of the same planes, [2B][kHistBins]
  // counts followed by the 2B invalid counts; null otherwise
  unsigned long long* hist;
};
// runs the chain on `stream` and adds its launches to *launches
int run_infer_chain(vp3d_plan* p, const InferChain& c, cudaStream_t stream, int* launches);

// clips.cu: the clip table of one vp3d_forward_clips chain (device arrays) and its geometry
constexpr int kClipMaxJoints = 256;   // joints a mirror map (kernel parameter) can hold
struct ClipChain {
  const long long* first;    // [clips] store row of each clip's frame 0
  const int* len;            // [clips] frames (values below 1 read as 1)
  const long long* y_first;  // [clips] output row of each clip's frame 0
  int clips, copies, rf, front;   // front = pad + causal shift: edge copies ahead of frame 0
  long long rows;            // packed rows of the chain
};
// the chain's 16-bit input [planes][rows][ld] from the fp32 store x; kps: the host mirror map of
// the J_in = c_raw / feat input joints (augment, copies == 2) or null
cudaError_t launch_clip_pack(const ClipChain& t, const float* x, int c_raw, int feat, const int* kps,
                             __nv_bfloat16* a0, int ld, int planes, long long plane, int f16,
                             cudaStream_t stream);
// each clip's valid rows of the shrink output ybuf [out_rows][c_out] into y (flip-averaged with two
// copies; jsrc: host map of the c_out / 3 output joints, or null)
cudaError_t launch_clip_output(const ClipChain& t, const float* ybuf, long long out_rows, int c_out,
                               const int* jsrc, float* y, cudaStream_t stream);
// stream.cu: every entry of a host mirror map lies in [0, n)
int check_mirror_map(const int32_t* map, int n, const char* what, const char* name);
void train_state_destroy(TrainState* t);
int train_pack_transposed(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream,
                          bool also_forward);
int train_pack_expand_t(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream);
}  // namespace vp3d
