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

// 4-D bf16 map (k, row, sample, plane), box (64, box_rows, 1, 1), 128-byte swizzle.
int make_map_4d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t row_stride,
                uint64_t samples, uint64_t sample_stride, uint64_t planes, uint64_t plane_stride,
                uint32_t box_rows);
// 2-D bf16 map (k, row), box (64, box_rows), 128-byte swizzle.
int make_map_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint32_t box_rows);

int pick_block_n(int n_pad);
inline int round_up(int v, int m) { return (v + m - 1) / m * m; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
// the 1 KiB-aligned base of a caller's workspace or state buffer (their sizes include the slack)
inline uint8_t* ws_base(void* ws) {
  return reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(ws), 1024));
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

}  // namespace vp3d

struct vp3d_plan {
  vp3d_config cfg;
  int nb = 0;  // residual blocks
  int C = 0;        // channels of the residual stream as laid out in memory: padded to 64
  int c_real = 0;   // the model's `channels` argument (any positive value, model.py:85-86)
  int c_in_raw = 0, c_out_raw = 0, c_in_pad = 0, k0_pad = 0, c_out_pad = 0;
  int planes = 1;
  int f16 = 0;  // VP3D_PRECISION_FP16: 16-bit stores hold IEEE fp16
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
  // host-API staging (owned)
  float* d_x = nullptr;
  float* d_y = nullptr;
  void* d_ws = nullptr;
  size_t d_x_bytes = 0, d_y_bytes = 0, d_ws_bytes = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;     // host API: H2D chunks overlap the compute stream
  std::vector<cudaEvent_t> copy_events;
  int last_launches = 0;
  // pipelined host API (vp3d_forward_eval_host_submit / _wait): two independent staging slots
  struct HostSlot {
    float* d_x = nullptr;
    float* d_y = nullptr;
    size_t x_bytes = 0, y_bytes = 0;
    cudaEvent_t copied = nullptr, done = nullptr;
    bool busy = false;
  };
  HostSlot slots[2];
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
inline size_t pack_bytes(const vp3d_plan* p, const PackedConv& k) {
  return (size_t)p->planes * k.stored_taps * k.n_pad * k.k_pad * sizeof(__nv_bfloat16);
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
};
// runs the chain on `stream` and adds its launches to *launches
int run_infer_chain(vp3d_plan* p, const InferChain& c, cudaStream_t stream, int* launches);
void train_state_destroy(TrainState* t);
int train_pack_transposed(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream,
                          bool also_forward);
int train_pack_expand_t(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream);
}  // namespace vp3d
