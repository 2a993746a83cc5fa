// Training-mode forward and backward (C ABI): vp3d_forward_train / vp3d_backward.
//
// Forward, per conv layer (model.py:127,134-135 / :188,193-194 in train() mode):
//   Z  = conv(X_prev)                 wgmma GEMM, raw bf16 store + per-channel sum / sumsq epilogue
//   (scale, shift, mean, invstd)      bn_finalize (+ running_mean / running_var update, momentum
//                                     read from the caller at call time, model.py:36-39)
//   X  = dropout(relu(Z*scale+shift)) [+ residual slice]   bn_apply (bandwidth pass)
// Saved for backward: the packed input, every Z and every X/H (bf16 planes) + the BN vectors.
//
// Backward, per layer top-down: BN/ReLU/Dropout backward (bn_bwd_reduce + bn_bwd_apply -> dZ,
// dgamma, dbeta), weight gradient dW = dZ^T * X (MN-major wgmma GEMM, split over rows),
// data gradient G_prev = dZ * W^T through the same conv GEMM kernel on transposed weight packs,
// with the skip-connection gradient added in the epilogue.  On request (vp3d_backward_ex with dx)
// the chain ends with the expand conv's data gradient dX = dZ0 * W0^T, written as fp32 in x's layout.
//
// Frozen BatchNorm (vp3d_forward_train_ex with VP3D_TRAIN_FROZEN_BN, the eval-mode backward):
// every BatchNorm is the fixed affine of its running statistics (the eval fold, bn_fold), running
// statistics are left alone and no batch-statistics slabs are written; the backward then applies
// dZ = scale * dY without the batch-statistics terms, and dgamma / dbeta come from the same sums
// with the running mean / invstd.
//
// Both layouts are covered: strided (TemporalModelOptimized1f, the model run.py trains with by
// default, run.py:172-175) and dilated (TemporalModel, run.py:176-180: per-sample tiles, transposed
// convolution for the data gradient, per-sample reduction for the weight gradient).
#include <stdio.h>

#include "internal.cuh"
#include "pack.cuh"
#include "train_ops.cuh"
#include "wgrad_gemm.cuh"

namespace vp3d {

// Everything a training plan adds, built whole by ensure_train_state; it owns every buffer in
// `allocs`, among them the plan's transposed packs (vp3d_plan::conv_t, shrink_t, expand_t).
struct TrainState {
  bool packed_t = false;         // transposed layer and shrink packs are current
  bool packed_expand_t = false;  // transposed expand pack (VP3D_PACK_EXPAND_T) is current
  float* vec = nullptr;       // per BN layer l: scale, shift, mean, invstd, stats[2C], sums[2C]
  size_t vec_floats = 0;
  float* shrink_affine = nullptr;  // scale / shift of the shrink bias [2 * c_out_pad]
  float* red_scratch = nullptr;    // second-level scratch of the ordered reductions
  unsigned* red_counter = nullptr; // their ticket counters (zeroed once, self-resetting)
  // configuration of the last forward (needed by backward)
  int N = 0, T = 0;
  int L[VP3D_MAX_WIDTHS] = {};
  float dropout_p = 0.0f;
  uint64_t seed = 0;
  bool frozen_bn = false;
  bool have_forward = false;
  // synchronized BatchNorm (vp3d_set_bn_sync): the current setting and the one the last forward ran
  // with, which its backward keeps (world 0 = off)
  struct BnSync {
    int world = 0, rank = 0;
    vp3d_bn_exchange_fn exchange = nullptr;
    void* user = nullptr;
  } sync, fwd_sync;
  // exchange slots, per BN layer l: forward moments at l * cap * 3C ([world][3][C]), backward sums
  // at (layers * 3 + l * 2) * cap * C ([world][2][C]); cap = ranks the buffer holds (grows only)
  float* sync_slots = nullptr;
  int sync_cap = 0;
  float* sync_n = nullptr;    // per BN layer: global row count of the last synchronized forward
  std::vector<void*> allocs;
};

void train_state_destroy(TrainState* t) {
  if (!t) return;
  for (void* q : t->allocs) cudaFree(q);
  delete t;
}

namespace {

template <typename T>
int t_alloc(TrainState* t, T** out, size_t bytes) {
  void* q = nullptr;
  CUDA_TRY(cudaMalloc(&q, bytes));
  t->allocs.push_back(q);
  *out = static_cast<T*>(q);
  return VP3D_OK;
}

void t_free(TrainState* t, void* q) {
  for (size_t i = 0; i < t->allocs.size(); ++i)
    if (t->allocs[i] == q) {
      t->allocs.erase(t->allocs.begin() + i);
      break;
    }
  cudaFree(q);
}

// every buffer of the training state, the transposed packs into tr[] (indexed like p->packs)
int train_state_alloc(const vp3d_plan* p, TrainState* t, __nv_bfloat16** tr) {
  for (int i = 0; i < p->n_packs; ++i)
    if (p->packs[i].transposed) VP3D_TRY(t_alloc(t, &tr[i], pack_bytes(p, p->packs[i])));
  t->vec_floats = (size_t)(2 * p->nb + 1) * 8 * p->C;
  VP3D_TRY(t_alloc(t, &t->vec, t->vec_floats * sizeof(float)));
  VP3D_TRY(t_alloc(t, &t->shrink_affine, 2 * p->c_out_pad * sizeof(float)));
  VP3D_TRY(t_alloc(t, &t->red_scratch, kReduceScratchFloats * sizeof(float)));
  VP3D_TRY(t_alloc(t, &t->red_counter, kReduceCounters * sizeof(unsigned)));
  CUDA_TRY(cudaMemset(t->red_counter, 0, kReduceCounters * sizeof(unsigned)));
  return VP3D_OK;
}

// Attaches the training state to the plan once every buffer of it exists; on a failure nothing is
// attached, so the next call fails the same way.
int ensure_train_state(vp3d_plan* p) {
  if (p->train) return VP3D_OK;
  if (p->C > kReduceMaxChannels)
    return fail(VP3D_ERR_UNSUPPORTED, "training supports at most %d channels", kReduceMaxChannels);
  TrainState* t = new TrainState();
  __nv_bfloat16* tr[kMaxPacks] = {};
  const int st = train_state_alloc(p, t, tr);
  if (st) {
    train_state_destroy(t);
    return st;
  }
  for (int i = 0; i < p->n_packs; ++i)
    if (p->packs[i].transposed) p->packs[i].w = tr[i];
  p->train = t;
  return VP3D_OK;
}

struct LayerVec {
  float *scale, *shift, *mean, *invstd, *stats, *sums;
};
LayerVec layer_vec(const vp3d_plan* p, int l) {
  float* b = p->train->vec + (size_t)l * 8 * p->C;
  return {b, b + p->C, b + 2 * p->C, b + 3 * p->C, b + 4 * p->C, b + 6 * p->C};
}

// exchange slots of BN layer l (layout in TrainState::sync_slots)
float* sync_fwd_slots(const vp3d_plan* p, int l) {
  const TrainState* t = p->train;
  return t->sync_slots + (size_t)l * t->sync_cap * 3 * p->C;
}
float* sync_bwd_slots(const vp3d_plan* p, int l) {
  const TrainState* t = p->train;
  return t->sync_slots + ((size_t)(2 * p->nb + 1) * 3 + (size_t)l * 2) * t->sync_cap * p->C;
}

// ---------------------------------------------------------------- workspace layout (strided)
struct TrainLayout {
  size_t a0 = 0;
  size_t z[VP3D_MAX_LAYERS + 1] = {};   // pre-BN conv outputs, layer 0 = expand
  size_t x[VP3D_MAX_WIDTHS] = {};       // x[0] = expand output, x[i] = output of block i
  size_t h[VP3D_MAX_WIDTHS] = {};       // h[i] = output of the first conv (post act) of block i
  size_t g0 = 0, g1 = 0, dz = 0, dyp = 0, partial = 0;
  size_t partial_bytes = 0;
  size_t slab = 0;         // per-slab statistics partials of the GEMM epilogues (fp32)
  size_t slab_floats = 0;
  size_t dx_stage = 0;     // strided model with T % w0 != 0: fp32 [N * L0][w0 * c_in] input gradient
                           // before the copy that opens each sample's tail (else unused)
  size_t total = 0;
  long long rows[VP3D_MAX_WIDTHS] = {};  // rows[i] = N * L[i]
};

TrainLayout train_layout(const vp3d_plan* p, int N, int T, const int* L) {
  const bool strided = p->cfg.variant == VP3D_VARIANT_STRIDED;
  TrainLayout w;
  const size_t C = p->C, pl = p->planes;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off = align_up(off + bytes, 1024);
    return o;
  };
  for (int i = 0; i <= p->nb; ++i) w.rows[i] = (long long)N * L[i];
  w.a0 = take(strided ? pl * w.rows[0] * p->k0_pad * 2 : pl * (size_t)N * T * p->c_in_pad * 2);
  w.z[0] = take(pl * w.rows[0] * C * 2);
  w.x[0] = take(pl * w.rows[0] * C * 2);
  for (int i = 1; i <= p->nb; ++i) {
    const size_t b = pl * w.rows[i] * C * 2;
    w.z[2 * i - 1] = take(b);
    w.h[i] = take(b);
    w.z[2 * i] = take(b);
    w.x[i] = take(b);
  }
  const size_t big = pl * w.rows[0] * C * 2;
  w.g0 = take(big);
  w.g1 = take(big);
  w.dz = take(big);
  w.dyp = take(pl * w.rows[p->nb] * p->shrink_t->k_pad * 2);   // dY in K layout of shrink_t
  // wgrad partials: up to 8 splits x taps x C x max(C, k0_pad) fp32
  int max_taps = 1;
  for (int i = 1; i <= p->nb; ++i) max_taps = p->taps[i] > max_taps ? p->taps[i] : max_taps;
  size_t n_max = p->C > p->k0_pad ? p->C : p->k0_pad;
  if ((size_t)p->c_in_pad > n_max) n_max = p->c_in_pad;
  if (!strided && p->cfg.filter_widths[0] > max_taps) max_taps = p->cfg.filter_widths[0];
  w.partial_bytes = (size_t)8 * max_taps * round_up(p->C, 128) * round_up((int)n_max, 64) * 4;
  w.partial = take(w.partial_bytes);
  // slab partials [4 * row tiles][2][columns]: the widest producer is a GEMM over rows[i] rows with
  // taps*C columns (strided data gradient) or N * tiles(L) row tiles with C columns (dilated)
  {
    size_t need = 0;
    for (int i = 0; i <= p->nb; ++i) {
      const size_t tiles = strided ? (size_t)(w.rows[i] + 127) / 128
                                   : (size_t)N * ((L[i] + 127) / 128);
      const size_t cols = (strided && i >= 1) ? (size_t)p->taps[i] * C : C;
      const size_t f = tiles * 4 * 2 * cols;
      need = f > need ? f : need;
    }
    const size_t bias_part = (size_t)((w.rows[p->nb] + 63) / 64) * (p->c_out_raw > 64 ? p->c_out_raw : 64);
    need = bias_part > need ? bias_part : need;
    w.slab_floats = need + 1024;
    w.slab = take(w.slab_floats * sizeof(float));
  }
  if (strided && T != p->cfg.filter_widths[0] * L[0])
    w.dx_stage = take((size_t)w.rows[0] * p->cfg.filter_widths[0] * p->c_in_raw * sizeof(float));
  w.total = off + 1024;
  return w;
}

// dW = dZ^T X for one conv layer.  dz: [planes][samples][rows][dz_ld]; x: [planes][samples][x_rows][x_ld]
// (flat layers: samples = 1).
struct WgradCall {
  const __nv_bfloat16* dz = nullptr;
  int dz_ld = 0;
  const __nv_bfloat16* x = nullptr;
  int x_ld = 0;
  long long rows = 0;     // dZ rows (per sample when per_sample)
  int per_sample = 0;
  int samples = 1;
  long long x_rows = 0;   // X rows per sample (per_sample only)
  int taps = 1;
  int tap_col_step = 0;
  int tap_row_step = 0;
  int c_out = 0;
  int c_in_cols = 0;      // columns of X spanned by one tap (merged: taps*c_in)
  int c_in = 0;
  int taps_out = 1;
  int merged = 0;
  float* grad = nullptr;
};

// planes: 1 (bf16) or 2 (hi + lo, three products per pair of planes).  The tile width and the
// split count follow from the shape alone; vp3d_wgrad_gemm reaches the same code.
int run_wgrad(int planes, const WgradCall& c, float* partial, size_t partial_bytes,
              cudaStream_t stream) {
  const int block_n = pick_block_n(round_up(c.c_in_cols, 64));
  WgradArgs a;
  memset(&a, 0, sizeof(a));
  a.per_sample = c.per_sample;
  a.samples = c.per_sample ? c.samples : 1;
  a.rows = (int)c.rows;
  a.kchunks = (int)((c.rows + 63) / 64);
  a.taps = c.taps;
  a.tap_row_step = c.tap_row_step;
  a.tap_col_step = c.tap_col_step;
  a.m_pad = round_up(c.c_out, 128);
  a.n_pad = round_up(c.c_in_cols, block_n);
  a.m_tiles = a.m_pad / 128;
  a.n_tiles = a.n_pad / block_n;
  a.pairs = planes == 2 ? 3 : 1;
  const int items = c.taps * a.m_tiles * a.n_tiles;
  const long long total_kb = (long long)a.kchunks * a.samples;
  int splits = (2 * num_sms() + items - 1) / items;
  // (up to 16 row ranges: the expand conv's gradient has only C_out / 128 tiles to spread)
  if (splits > 16) splits = 16;
  if (splits > total_kb) splits = (int)total_kb;
  if (splits < 1) splits = 1;
  while ((size_t)splits * c.taps * a.m_pad * a.n_pad * 4 > partial_bytes && splits > 1) --splits;
  if ((size_t)splits * c.taps * a.m_pad * a.n_pad * 4 > partial_bytes)
    return fail(VP3D_ERR_WORKSPACE, "wgrad partial buffer too small");
  a.splits = splits;
  a.partial = partial;
  CUtensorMap mdz, mx;
  const uint64_t x_rows = c.per_sample ? (uint64_t)c.x_rows : (uint64_t)c.rows;
  VP3D_TRY(make_map_4d(&mdz, c.dz, c.dz_ld, c.rows, c.dz_ld, a.samples, (uint64_t)c.rows * c.dz_ld,
                       planes, (uint64_t)a.samples * c.rows * c.dz_ld, 64));
  VP3D_TRY(make_map_4d(&mx, c.x, c.x_ld, x_rows, c.x_ld, a.samples, x_rows * c.x_ld, planes,
                       (uint64_t)a.samples * x_rows * c.x_ld, 64));
  CUDA_TRY(launch_wgrad_gemm(mdz, mx, a, block_n, num_sms(), stream));
  CUDA_TRY(launch_wgrad_reduce(partial, c.grad, splits, c.taps, a.m_pad, a.n_pad, c.c_out, c.c_in,
                               c.taps_out, c.merged, stream));
  return VP3D_OK;
}

DropoutCfg drop_cfg(const TrainState* t, int layer) {
  DropoutCfg d;
  d.p = t->dropout_p;
  d.seed_lo = (uint32_t)(t->seed & 0xFFFFFFFFu);
  d.seed_hi = (uint32_t)(t->seed >> 32);
  d.layer = (uint32_t)layer;
  return d;
}

}  // namespace

// the forward pack a transposed layer / shrink pack is written with
static const PackedConv* forward_of(const vp3d_plan* p, const PackedConv& k) {
  return k.src == kSrcShrink ? p->shrink : p->conv[k.src];
}

// also_forward: the same kernels write the forward packs of the block convs and of shrink (one read
// of the fp32 weights per optimizer step instead of two).
int train_pack_transposed(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream,
                          bool also_forward) {
  VP3D_TRY(ensure_train_state(p));
  for (int i = 0; i < p->n_packs; ++i) {
    const PackedConv& k = p->packs[i];
    if (k.transposed && k.src != kSrcExpand)
      VP3D_TRY(pack_weight(p, k, w, stream, also_forward ? forward_of(p, k) : nullptr));
  }
  p->train->packed_t = true;
  return VP3D_OK;
}

int train_pack_expand_t(vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream) {
  VP3D_TRY(ensure_train_state(p));
  VP3D_TRY(pack_weight(p, *p->expand_t, w, stream));
  p->train->packed_expand_t = true;
  return VP3D_OK;
}

}  // namespace vp3d

using namespace vp3d;

#define VP3D_API extern "C" __attribute__((visibility("default")))

VP3D_API size_t vp3d_train_workspace_bytes(const vp3d_plan* p, int N, int T) {
  if (!p || N < 1) return 0;
  int L[VP3D_MAX_WIDTHS];
  const bool strided = p->cfg.variant == VP3D_VARIANT_STRIDED;
  if (!layer_rows(p, T, strided, L)) return 0;
  return train_layout(p, N, T, L).total;
}

VP3D_API int vp3d_set_bn_sync(vp3d_plan* p, int world, int rank, vp3d_bn_exchange_fn exchange,
                              void* user) {
  if (!p) return fail(VP3D_ERR_INVALID, "set_bn_sync: null plan");
  if (world < 0 || (world > 0 && (rank < 0 || rank >= world || !exchange)))
    return fail(VP3D_ERR_INVALID, "set_bn_sync: need 0 <= rank < world and an exchange function "
                "(world %d, rank %d)", world, rank);
  if (p->f16) return fail(VP3D_ERR_UNSUPPORTED, "set_bn_sync: fp16 plans are inference-only");
  VP3D_TRY(ensure_train_state(p));
  TrainState* t = p->train;
  if (world == 0) {
    t->sync = TrainState::BnSync();
    return VP3D_OK;
  }
  if (!t->sync_n) VP3D_TRY(t_alloc(t, &t->sync_n, (VP3D_MAX_LAYERS + 1) * sizeof(float)));
  if (world > t->sync_cap) {
    // grows only; a backward still pending across the reallocation stays valid: it zeroes its
    // slots itself and the forward's global counts live in sync_n
    float* q = nullptr;
    VP3D_TRY(t_alloc(t, &q, (size_t)(2 * p->nb + 1) * 5 * world * p->C * sizeof(float)));
    if (t->sync_slots) t_free(t, t->sync_slots);
    t->sync_slots = q;
    t->sync_cap = world;
  }
  t->sync.world = world;
  t->sync.rank = rank;
  t->sync.exchange = exchange;
  t->sync.user = user;
  return VP3D_OK;
}

VP3D_API int vp3d_forward_train_ex(vp3d_plan* p, const float* x, float* y, int N, int T,
                                   const vp3d_weights* w, const float* bn_momentum, float dropout_p,
                                   unsigned long long seed, int flags, void* ws, size_t ws_bytes,
                                   void* stream_);

VP3D_API int vp3d_forward_train(vp3d_plan* p, const float* x, float* y, int N, int T,
                                const vp3d_weights* w, const float* bn_momentum, float dropout_p,
                                unsigned long long seed, void* ws, size_t ws_bytes, void* stream_) {
  if (!bn_momentum) return fail(VP3D_ERR_INVALID, "forward_train: null argument");
  return vp3d_forward_train_ex(p, x, y, N, T, w, bn_momentum, dropout_p, seed, 0, ws, ws_bytes,
                               stream_);
}

VP3D_API int vp3d_forward_train_ex(vp3d_plan* p, const float* x, float* y, int N, int T,
                                   const vp3d_weights* w, const float* bn_momentum, float dropout_p,
                                   unsigned long long seed, int flags, void* ws, size_t ws_bytes,
                                   void* stream_) {
  if (flags & ~VP3D_TRAIN_FROZEN_BN)
    return fail(VP3D_ERR_INVALID, "forward_train: unknown flags 0x%x", flags);
  const bool frozen = (flags & VP3D_TRAIN_FROZEN_BN) != 0;
  if (!p || !x || !y || !w || (!bn_momentum && !frozen))
    return fail(VP3D_ERR_INVALID, "forward_train: null argument");
  if (frozen && dropout_p != 0.0f)
    return fail(VP3D_ERR_INVALID, "forward_train: VP3D_TRAIN_FROZEN_BN (the eval-mode forward) "
                "runs without dropout; dropout p must be 0");
  const bool strided = p->cfg.variant == VP3D_VARIANT_STRIDED;
  if (N < 1) return fail(VP3D_ERR_INVALID, "forward_train: batch must be >= 1");
  if (dropout_p < 0.0f || dropout_p >= 1.0f)
    return fail(VP3D_ERR_INVALID, "forward_train: dropout p must be in [0, 1)");
  if (p->f16)
    return fail(VP3D_ERR_UNSUPPORTED, "forward_train: fp16 plans are inference-only");
  if (!p->conv_packed) return fail(VP3D_ERR_STATE, "forward_train: conv weights not packed");
  VP3D_TRY(ensure_train_state(p));
  TrainState* t = p->train;
  if (!t->packed_t) return fail(VP3D_ERR_STATE, "forward_train: transposed weights not packed");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int L[VP3D_MAX_WIDTHS];
  if (!layer_rows(p, T, strided, L))
    return fail(VP3D_ERR_INVALID, "forward_train: sequence of %d frames is too short", T);
  const int* fw = p->cfg.filter_widths;
  for (int i = 1; strided && i <= p->nb; ++i)
    if (L[i - 1] != fw[i] * L[i])
      return fail(VP3D_ERR_UNSUPPORTED, "strided training needs layer lengths divisible by the "
                  "filter width (block %d: %d frames, width %d): the BatchNorm batch statistics of "
                  "a layer include the trailing frames its consumer ignores, which the flat row "
                  "layout cannot express; run.py always trains on exactly one receptive field",
                  i, L[i - 1], fw[i]);
  const TrainLayout wl = train_layout(p, N, T, L);
  if (!ws || ws_bytes < wl.total)
    return fail(VP3D_ERR_WORKSPACE, "train workspace too small: %zu < %zu", ws_bytes, wl.total);
  uint8_t* base = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(ws), 1024));
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(base + off); };
  const int C = p->C, pl = p->planes;
  t->N = N; t->T = T; t->dropout_p = dropout_p; t->seed = seed; t->frozen_bn = frozen;
  t->have_forward = false;
  // frozen BatchNorm has no batch statistics: nothing to exchange, in this forward or its backward
  t->fwd_sync = frozen ? TrainState::BnSync() : t->sync;
  const TrainState::BnSync sync = t->fwd_sync;
  for (int i = 0; i <= p->nb; ++i) t->L[i] = L[i];
  int launches = 0;

  float* slab_part = reinterpret_cast<float*>(base + wl.slab);
  CUDA_TRY(launch_bias_affine(w->shrink_bias, t->shrink_affine, t->shrink_affine + p->c_out_pad,
                              p->c_out_raw, p->c_out_pad, stream));
  ++launches;

  vp3d_conv_desc d;
  auto common = [&](vp3d_conv_desc& q) {
    memset(&q, 0, sizeof(q));
    q.a_planes = pl;
    q.precision = p->cfg.precision;
    q.out_planes = pl;
    q.samples = 1;
    q.per_sample_tiles = 0;
  };
  int stats_per_sample_rows = 0;  // rows per sample of the last stats-producing GEMM if it ran on
                                  // per-sample tiles (dilated layout), else 0
  auto bn = [&](int layer, const float* const* bnp, long long rows, const __nv_bfloat16* z,
                __nv_bfloat16* out, const __nv_bfloat16* res, long long res_plane, RowMap map) -> int {
    const LayerVec v = layer_vec(p, layer);
    // the GEMM that produced z left per-slab sums in slab_part; its row tiling: flat over all rows
    // (strided model and every 1x1 conv) or per-sample tiles (dilated model's k-tap convs)
    const int per_sample_rows = stats_per_sample_rows;
    const int tps = per_sample_rows ? (per_sample_rows + 127) / 128 : 0;
    const int slabs = per_sample_rows ? N * tps * 4 : (int)((rows + 127) / 128) * 4;
    if (frozen) {  // the eval fold of the running statistics, plus the mean / invstd backward reads
      CUDA_TRY(launch_bn_fold(bnp[0], bnp[1], bnp[2], bnp[3], 1e-5f, v.scale, v.shift, p->c_real, C,
                              stream, v.mean, v.invstd));
    } else if (sync.world > 0) {
      // this rank's moments into its slot, the exchange fills the others, then the rank-ordered
      // merge and the finalize over the global batch
      float* slots = sync_fwd_slots(p, layer);
      CUDA_TRY(launch_bn_stats_finalize(slab_part, slabs, per_sample_rows ? 1 : 0,
                                        per_sample_rows ? per_sample_rows : (int)rows, tps, bnp[0],
                                        bnp[1], nullptr, nullptr, 0.0f, 1e-5f, v.scale, v.shift,
                                        v.mean, v.invstd, C, p->c_real, t->red_scratch,
                                        t->red_counter, stream, slots, sync.world, sync.rank));
      sync.exchange(layer, VP3D_BN_SYNC_FORWARD, slots, 3 * C, sync.user);
      CUDA_TRY(launch_bn_sync_finalize(slots, sync.world, bnp[0], bnp[1], const_cast<float*>(bnp[2]),
                                       const_cast<float*>(bnp[3]), bn_momentum[layer], 1e-5f,
                                       v.scale, v.shift, v.mean, v.invstd, C, p->c_real,
                                       t->sync_n + layer, stream));
      ++launches;
    } else {
      CUDA_TRY(launch_bn_stats_finalize(slab_part, slabs, per_sample_rows ? 1 : 0,
                                        per_sample_rows ? per_sample_rows : (int)rows, tps, bnp[0],
                                        bnp[1], const_cast<float*>(bnp[2]), const_cast<float*>(bnp[3]),
                                        bn_momentum[layer], 1e-5f, v.scale, v.shift, v.mean, v.invstd,
                                        C, p->c_real, t->red_scratch, t->red_counter, stream));
    }
    CUDA_TRY(launch_bn_apply(z, rows * C, out, rows * C, pl, rows, C, v.scale, v.shift,
                             drop_cfg(t, layer), res, res_plane, map, stream));
    launches += 2;
    return VP3D_OK;
  };
  const RowMap no_map = {0, 0, 1, 0};

  // ---- expand (model.py:188 strided / :127 dilated)
  common(d);
  if (strided) {
    CUDA_TRY(launch_pack_input(x, bf(wl.a0), pl, N, T, p->c_in_raw, L[0], fw[0], fw[0], p->k0_pad,
                               wl.rows[0] * p->k0_pad, stream));
    d.a = bf(wl.a0); d.a_rows = (int)wl.rows[0]; d.a_ld = p->k0_pad;
    use_pack(&d, *p->expand_flat);
    d.out_rows = (int)wl.rows[0];
  } else {
    CUDA_TRY(launch_pack_input(x, bf(wl.a0), pl, N, T, p->c_in_raw, T, 1, 1, p->c_in_pad,
                               (long long)N * T * p->c_in_pad, stream));
    d.a = bf(wl.a0); d.samples = N; d.a_rows = T; d.a_ld = p->c_in_pad;
    use_pack(&d, *p->expand_dil);
    d.per_sample_tiles = 1; d.tap_row_step = 1; d.out_rows = L[0];
  }
  ++launches;
  d.out = bf(wl.z[0]); d.out_plane_stride = wl.rows[0] * C; d.out_ld = C;
  d.stats = frozen ? nullptr : slab_part;
  stats_per_sample_rows = d.per_sample_tiles ? d.out_rows : 0;
  VP3D_TRY(run_conv(&d, stream));
  ++launches;
  VP3D_TRY(bn(0, w->expand_bn, wl.rows[0], bf(wl.z[0]), bf(wl.x[0]), nullptr, 0, no_map));

  // ---- residual blocks (model.py:190-194)
  for (int i = 1; i <= p->nb; ++i) {
    const long long rows = wl.rows[i];
    const int l1 = 2 * i - 1, l2 = 2 * i;
    common(d);
    use_pack(&d, *p->conv[2 * (i - 1)]);
    if (strided) {
      d.a = bf(wl.x[i - 1]); d.a_rows = (int)rows; d.a_ld = fw[i] * C;
      d.tap_col_step = C; d.out_rows = (int)rows;
    } else {
      d.a = bf(wl.x[i - 1]); d.samples = N; d.a_rows = L[i - 1]; d.a_ld = C;
      d.per_sample_tiles = 1; d.tap_row_step = p->dilation[i]; d.out_rows = L[i];
    }
    d.out = bf(wl.z[l1]); d.out_plane_stride = rows * C; d.out_ld = C;
    d.stats = frozen ? nullptr : slab_part;
    stats_per_sample_rows = d.per_sample_tiles ? d.out_rows : 0;
    VP3D_TRY(run_conv(&d, stream));
    ++launches;
    VP3D_TRY(bn(l1, w->layers_bn[2 * (i - 1)], rows, bf(wl.z[l1]), bf(wl.h[i]), nullptr, 0, no_map));

    common(d);
    d.a = bf(wl.h[i]); d.a_rows = (int)rows; d.a_ld = C;
    use_pack(&d, *p->conv[2 * (i - 1) + 1]);
    d.out_rows = (int)rows;
    d.out = bf(wl.z[l2]); d.out_plane_stride = rows * C; d.out_ld = C;
    d.stats = frozen ? nullptr : slab_part;
    stats_per_sample_rows = 0;
    VP3D_TRY(run_conv(&d, stream));
    ++launches;
    const RowMap rm = strided ? RowMap{0, 0, fw[i], fw[i] / 2 + p->shift_str[i]}
                              : RowMap{L[i], L[i - 1], 1, p->pad[i] + p->shift_dil[i]};
    VP3D_TRY(bn(l2, w->layers_bn[2 * (i - 1) + 1], rows, bf(wl.z[l2]), bf(wl.x[i]), bf(wl.x[i - 1]),
                wl.rows[i - 1] * C, rm));
  }

  // ---- shrink (model.py:196)
  common(d);
  d.a = bf(wl.x[p->nb]); d.a_rows = (int)wl.rows[p->nb]; d.a_ld = C;
  use_pack(&d, *p->shrink);
  d.out_rows = (int)wl.rows[p->nb];
  d.scale = t->shrink_affine; d.shift = t->shrink_affine + p->c_out_pad;
  d.out_f32 = y; d.out_f32_ld = p->c_out_raw; d.n_valid = p->c_out_raw;
  VP3D_TRY(run_conv(&d, stream));
  ++launches;
  p->last_launches = launches;
  t->have_forward = true;
  return VP3D_OK;
}

static int backward_impl(vp3d_plan* p, const float* dy, const vp3d_grads* g, float* dx, void* ws,
                         size_t ws_bytes, void* stream_, vp3d_stage_fn stage_done, void* user);

VP3D_API int vp3d_backward(vp3d_plan* p, const float* dy, const vp3d_grads* g, void* ws,
                           size_t ws_bytes, void* stream_) {
  if (!g) return fail(VP3D_ERR_INVALID, "backward: null argument");
  return backward_impl(p, dy, g, nullptr, ws, ws_bytes, stream_, nullptr, nullptr);
}

VP3D_API int vp3d_backward_staged(vp3d_plan* p, const float* dy, const vp3d_grads* g, void* ws,
                                  size_t ws_bytes, void* stream_, vp3d_stage_fn stage_done,
                                  void* user) {
  if (!g) return fail(VP3D_ERR_INVALID, "backward: null argument");
  return backward_impl(p, dy, g, nullptr, ws, ws_bytes, stream_, stage_done, user);
}

VP3D_API int vp3d_backward_ex(vp3d_plan* p, const float* dy, const vp3d_grads* g, float* dx, void* ws,
                              size_t ws_bytes, void* stream_, vp3d_stage_fn stage_done, void* user) {
  if (!g && !dx) return fail(VP3D_ERR_INVALID, "backward: neither parameter nor input gradients asked for");
  return backward_impl(p, dy, g, dx, ws, ws_bytes, stream_, stage_done, user);
}

// g == nullptr: no parameter gradients (no weight-gradient GEMMs, no shrink-bias sum, and under
// frozen BatchNorm no BatchNorm-backward reductions either); dx == nullptr: no input gradient.
static int backward_impl(vp3d_plan* p, const float* dy, const vp3d_grads* g, float* dx, void* ws,
                         size_t ws_bytes, void* stream_, vp3d_stage_fn stage_done, void* user) {
  if (!p || !dy) return fail(VP3D_ERR_INVALID, "backward: null argument");
  TrainState* t = p->train;
  if (!t || !t->have_forward) return fail(VP3D_ERR_STATE, "backward: no training forward to match");
  if (dx && !t->packed_expand_t)
    return fail(VP3D_ERR_STATE, "backward: the input gradient needs the transposed expand pack "
                "(vp3d_set_weights with VP3D_PACK_EXPAND_T)");
  const bool want_w = g != nullptr;
  const bool frozen = t->frozen_bn;
  const bool need_sums = want_w || !frozen;   // BatchNorm-backward reductions
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int N = t->N, C = p->C, Cr = p->c_real, pl = p->planes;   // padded / real channels
  const int* L = t->L;
  const int* fw = p->cfg.filter_widths;
  const bool strided = p->cfg.variant == VP3D_VARIANT_STRIDED;
  const TrainLayout wl = train_layout(p, N, t->T, L);
  if (!ws || ws_bytes < wl.total) return fail(VP3D_ERR_WORKSPACE, "backward: workspace too small");
  uint8_t* base = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(ws), 1024));
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(base + off); };
  float* partial = reinterpret_cast<float*>(base + wl.partial);
  float* slab_part = reinterpret_cast<float*>(base + wl.slab);
  if (want_w) {
    if (!g->expand_conv_weight || !g->shrink_weight || !g->shrink_bias || !g->expand_bn[0] ||
        !g->expand_bn[1])
      return fail(VP3D_ERR_INVALID, "backward: missing gradient buffer");
    for (int l = 0; l < 2 * p->nb; ++l)
      if (!g->layers_conv_weight[l] || !g->layers_bn[l][0] || !g->layers_bn[l][1])
        return fail(VP3D_ERR_INVALID, "backward: missing gradient buffer for layer %d", l);
  }
  int launches = 0;
  const int dy_ld = p->shrink_t->k_pad;   // padded dY, the K operand of the shrink data gradient
  const long long rows_top = wl.rows[p->nb];
  // the forward's synchronized-BatchNorm setting (never set after a frozen-BatchNorm forward)
  const TrainState::BnSync sync = t->fwd_sync;
  const bool synced = sync.world > 0;
  if (synced) {
    if (!t->sync_slots || sync.world > t->sync_cap)
      return fail(VP3D_ERR_STATE, "backward: no exchange slots for %d ranks", sync.world);
    // every rank's slot starts at zero, so that summing the ranks' buffers is an exact gather
    CUDA_TRY(cudaMemsetAsync(sync_bwd_slots(p, 0), 0,
                             (size_t)(2 * p->nb + 1) * 2 * t->sync_cap * C * sizeof(float), stream));
    ++launches;
  }

  vp3d_conv_desc d;
  auto common = [&](vp3d_conv_desc& q) {
    memset(&q, 0, sizeof(q));
    q.a_planes = pl;
    q.precision = p->cfg.precision;
    q.out_planes = pl;
    q.samples = 1;
    q.per_sample_tiles = 0;
  };
  // In single-plane bf16 mode the per-channel reductions of the BatchNorm backward are fused into
  // the epilogue of the GEMM that produces the incoming gradient (fuse_bnb); otherwise a separate
  // pass over (G, Z) computes them.
  const bool fuse = (pl == 1);
  // geometry of the slab partials the last fused GEMM left behind (consumed by the next bn_bwd)
  int bnb_slabs = 0, bnb_ld = 0;
  auto fuse_bnb = [&](vp3d_conv_desc& q, int layer) {
    if (!fuse || !need_sums) return;
    const LayerVec v = layer_vec(p, layer);
    q.bnb_z = bf(wl.z[layer]);
    q.bnb_scale = v.scale; q.bnb_shift = v.shift; q.bnb_mean = v.mean; q.bnb_invstd = v.invstd;
    q.bnb_sums = slab_part; q.bnb_c = C; q.bnb_p = t->dropout_p; q.bnb_seed = t->seed;
    q.bnb_layer = layer;
    const int tiles = (q.out_rows + 127) / 128;
    bnb_slabs = (q.per_sample_tiles ? q.samples * tiles : tiles) * 4;
    bnb_ld = q.n_pad;
  };
  // BN + ReLU + dropout backward of `layer`: (gin, z) -> dz (+ dgamma, dbeta)
  auto bn_bwd = [&](int layer, long long rows, const __nv_bfloat16* gin, const __nv_bfloat16* z,
                    float* dgamma, float* dbeta) -> int {
    const LayerVec v = layer_vec(p, layer);
    const DropoutCfg dc = drop_cfg(t, layer);
    // synchronized BatchNorm: this rank's sums go to its exchange slot, v.sums receives the
    // rank-ordered global sums
    float* slots = synced ? sync_bwd_slots(p, layer) : nullptr;
    float* local = synced ? slots + (size_t)sync.rank * 2 * C : v.sums;
    if (!need_sums) {
      // frozen BatchNorm without parameter gradients: dZ = scale * dY needs no reduction
    } else if (!fuse) {
      CUDA_TRY(launch_bn_bwd_reduce(gin, rows * C, z, rows * C, pl, rows, C, v.scale, v.shift,
                                    v.mean, v.invstd, dc, slab_part, wl.slab_floats, local,
                                    t->red_scratch, t->red_counter, stream));
      launches += 2;
    } else {
      // ordered sum of the slab partials the producing GEMM's epilogue wrote; column blocks of a
      // strided data gradient (one per tap) fold onto the same channel
      if ((size_t)bnb_slabs * 2 * bnb_ld > wl.slab_floats)
        return fail(VP3D_ERR_WORKSPACE, "backward: slab partial buffer too small");
      CUDA_TRY(launch_ordered_col_sums(slab_part, bnb_slabs, 2, bnb_ld, C, bnb_ld / C, nullptr,
                                       v.invstd, local, local + C, t->red_scratch, t->red_counter,
                                       stream));
      ++launches;
    }
    if (synced) {
      sync.exchange(layer, VP3D_BN_SYNC_BACKWARD, slots, 2 * C, sync.user);
      CUDA_TRY(launch_rank_ordered_sum(slots, sync.world, 2 * C, v.sums, stream));
      ++launches;
    }
    CUDA_TRY(launch_bn_bwd_apply(gin, rows * C, z, rows * C, bf(wl.dz), rows * C, pl, rows, C,
                                 v.scale, v.shift, v.mean, v.invstd, dc,
                                 need_sums ? local : nullptr, want_w ? dgamma : nullptr,
                                 want_w ? dbeta : nullptr, p->c_real, stream, frozen ? 1 : 0,
                                 synced ? v.sums : nullptr, synced ? t->sync_n + layer : nullptr));
    ++launches;
    return VP3D_OK;
  };

  // ---- shrink backward: y = X_nb * Wsh^T + b
  CUDA_TRY(launch_pack_input(dy, bf(wl.dyp), pl, 1, (int)rows_top, p->c_out_raw, (int)rows_top, 1, 1,
                             dy_ld, rows_top * dy_ld, stream));
  ++launches;
  if (want_w) {
    CUDA_TRY(launch_col_sum_f32(dy, rows_top, p->c_out_raw, slab_part, wl.slab_floats, g->shrink_bias,
                                t->red_scratch, t->red_counter, stream));
    launches += 2;
    WgradCall c;
    c.dz = bf(wl.dyp); c.dz_ld = dy_ld; c.x = bf(wl.x[p->nb]); c.x_ld = C; c.rows = rows_top;
    c.c_out = p->c_out_raw; c.c_in_cols = Cr; c.c_in = Cr; c.grad = g->shrink_weight;
    VP3D_TRY(run_wgrad(pl, c, partial, wl.partial_bytes, stream));
    launches += 2;
  }
  __nv_bfloat16* gb[2] = {bf(wl.g0), bf(wl.g1)};
  int cur = 0;
  common(d);
  d.a = bf(wl.dyp); d.a_rows = (int)rows_top; d.a_ld = dy_ld;
  use_pack(&d, *p->shrink_t);
  d.out_rows = (int)rows_top;
  d.out = gb[cur]; d.out_plane_stride = rows_top * C; d.out_ld = C;
  fuse_bnb(d, 2 * p->nb);  // G_nb feeds the BN backward of the top block's second conv (or expand)
  VP3D_TRY(run_conv(&d, stream));
  ++launches;
  if (stage_done) stage_done(0, user);  // shrink.weight / shrink.bias gradients are enqueued

  // ---- residual blocks, top-down
  for (int i = p->nb; i >= 1; --i) {
    const long long rows = wl.rows[i];
    const int l1 = 2 * i - 1, l2 = 2 * i;
    const int c1 = 2 * (i - 1), c2 = c1 + 1;
    // second conv (1x1): X_i = res + act(bn(conv2(H_i)))
    VP3D_TRY(bn_bwd(l2, rows, gb[cur], bf(wl.z[l2]), want_w ? g->layers_bn[c2][0] : nullptr,
                    want_w ? g->layers_bn[c2][1] : nullptr));
    if (want_w) {
      WgradCall c;
      c.dz = bf(wl.dz); c.dz_ld = C; c.x = bf(wl.h[i]); c.x_ld = C; c.rows = rows;
      c.c_out = Cr; c.c_in_cols = Cr; c.c_in = Cr; c.grad = g->layers_conv_weight[c2];
      VP3D_TRY(run_wgrad(pl, c, partial, wl.partial_bytes, stream));
      launches += 2;
    }
    common(d);
    d.a = bf(wl.dz); d.a_rows = (int)rows; d.a_ld = C;
    use_pack(&d, *p->conv_t[c2]);
    d.out_rows = (int)rows;
    d.out = gb[cur ^ 1]; d.out_plane_stride = rows * C; d.out_ld = C;
    fuse_bnb(d, l1);
    VP3D_TRY(run_conv(&d, stream));
    ++launches;
    // first conv (w taps, stride w): H_i = act(bn(conv1(X_{i-1})))
    VP3D_TRY(bn_bwd(l1, rows, gb[cur ^ 1], bf(wl.z[l1]), want_w ? g->layers_bn[c1][0] : nullptr,
                    want_w ? g->layers_bn[c1][1] : nullptr));
    if (want_w) {
      WgradCall c;
      c.dz = bf(wl.dz); c.dz_ld = C; c.x = bf(wl.x[i - 1]); c.taps = p->taps[i];
      c.c_out = Cr; c.c_in_cols = Cr; c.c_in = Cr; c.taps_out = p->taps[i];
      c.grad = g->layers_conv_weight[c1];
      if (strided) {
        c.x_ld = fw[i] * C; c.rows = rows; c.tap_col_step = C;
      } else {
        c.x_ld = C; c.per_sample = 1; c.samples = N; c.rows = L[i]; c.x_rows = L[i - 1];
        c.tap_row_step = p->dilation[i];
      }
      VP3D_TRY(run_wgrad(pl, c, partial, wl.partial_bytes, stream));
      launches += 2;
    }
    common(d);
    use_pack(&d, *p->conv_t[c1]);
    d.res = gb[cur]; d.res_planes = pl; d.res_plane_stride = rows * C; d.res_ld = C;
    d.out = gb[cur ^ 1];
    if (strided) {
      // G_{i-1}[rows, w*C] = dZ1 * W1^T  (+ G_i in the columns of the residual tap): the pack's
      // taps slabs [ci][co] read as one [taps*ci][co] slab
      d.a = bf(wl.dz); d.a_rows = (int)rows; d.a_ld = C;
      d.n_pad = d.taps * d.n_pad; d.taps = 1;
      d.out_rows = (int)rows;
      d.out_plane_stride = rows * fw[i] * C; d.out_ld = fw[i] * C;
      d.res_rows_per_sample = 0; d.res_row_step = 1; d.res_row_off = 0;
      d.res_col_begin = (fw[i] / 2 + p->shift_str[i]) * C; d.res_cols = C;
    } else {
      // transposed convolution: G_{i-1}[n, t] = sum_k dZ1[n, t - k*d] * W1_k^T  (+ G_i[n, t - off]);
      // rows outside [0, L_i) are zero-filled by the A / residual tensor maps
      d.a = bf(wl.dz); d.samples = N; d.a_rows = L[i]; d.a_ld = C;
      d.per_sample_tiles = 1;
      d.tap_row_step = -p->dilation[i];
      d.out_rows = L[i - 1];
      d.out_plane_stride = wl.rows[i - 1] * C; d.out_ld = C;
      d.res_rows_per_sample = L[i]; d.res_row_step = 1;
      d.res_row_off = -(p->pad[i] + p->shift_dil[i]); d.res_check_rows = 1;
    }
    fuse_bnb(d, 2 * (i - 1));  // G_{i-1}: BN backward of block i-1's second conv (expand for i = 1)
    VP3D_TRY(run_conv(&d, stream));
    ++launches;
    cur ^= 1;
    if (stage_done) stage_done(p->nb - i + 1, user);  // all four parameter groups of block i
  }

  // ---- expand backward (the data gradient only on request: run.py's 2-D input needs none,
  // run.py:402-412; a differentiable front end or test-time refinement of x does)
  VP3D_TRY(bn_bwd(0, wl.rows[0], gb[cur], bf(wl.z[0]), want_w ? g->expand_bn[0] : nullptr,
                  want_w ? g->expand_bn[1] : nullptr));
  if (want_w) {
    WgradCall c;
    c.dz = bf(wl.dz); c.dz_ld = C; c.x = bf(wl.a0); c.c_out = Cr; c.c_in = p->c_in_raw;
    c.taps_out = fw[0]; c.grad = g->expand_conv_weight;
    if (strided) {
      c.x_ld = p->k0_pad; c.rows = wl.rows[0]; c.c_in_cols = fw[0] * p->c_in_raw; c.merged = 1;
    } else {
      c.x_ld = p->c_in_pad; c.per_sample = 1; c.samples = N; c.rows = L[0]; c.x_rows = t->T;
      c.taps = fw[0]; c.tap_row_step = 1; c.c_in_cols = p->c_in_raw;
    }
    VP3D_TRY(run_wgrad(pl, c, partial, wl.partial_bytes, stream));
    launches += 2;
  }
  if (dx) {
    // dX = dZ0 * W0^T through the conv GEMM, fp32 epilogue straight into x's (N, T, J*F) layout
    const int cin = p->c_in_raw, T = t->T;
    common(d);
    d.a = bf(wl.dz); d.a_ld = C;
    use_pack(&d, *p->expand_t);   // tap-merged (strided) or per tap (dilated)
    d.out_f32 = dx;
    if (strided) {
      // G_x[rows0, w0*cin] = dZ0 * W0^T with the tap-merged pack: column tap*cin + ci of row
      // (n, r) is x[n, r*w0 + tap, ci], i.e. x's own memory order when T = w0 * L0
      d.a_rows = (int)wl.rows[0]; d.out_rows = (int)wl.rows[0];
      d.out_f32_ld = fw[0] * cin; d.n_valid = fw[0] * cin;
      const size_t used = (size_t)fw[0] * L[0] * cin;   // floats per sample the output depends on
      const bool tail = T != fw[0] * L[0];
      // trailing frames no output depends on: the GEMM writes a staging buffer, one strided copy
      // moves each sample's rows into place and one strided memset zeroes the tails
      if (tail) d.out_f32 = reinterpret_cast<float*>(base + wl.dx_stage);
      VP3D_TRY(run_conv(&d, stream));
      ++launches;
      if (tail) {
        const size_t pitch = (size_t)T * cin * sizeof(float);
        CUDA_TRY(cudaMemcpy2DAsync(dx, pitch, d.out_f32, used * sizeof(float), used * sizeof(float),
                                   N, cudaMemcpyDeviceToDevice, stream));
        CUDA_TRY(cudaMemset2DAsync(dx + used, pitch, 0, pitch - used * sizeof(float), N, stream));
        launches += 2;
      }
    } else {
      // transposed convolution: dX[n, t] = sum_k dZ0[n, t - k] * W0_k^T; rows outside [0, L0) are
      // zero-filled by the A tensor map, so every one of the T rows is written
      d.samples = N; d.a_rows = L[0]; d.per_sample_tiles = 1;
      d.tap_row_step = -1;
      d.out_rows = T; d.out_f32_ld = cin; d.n_valid = cin;
      VP3D_TRY(run_conv(&d, stream));
      ++launches;
    }
  }
  if (stage_done) stage_done(p->nb + 1, user);  // expand_conv / expand_bn
  p->last_launches = launches;
  return VP3D_OK;
}

// Optimizer step that keeps the packed bf16 weights of a training plan current (SURVEY §8 f4):
// conv weights named in `w` are updated by the fused update + re-pack kernel, everything else by the
// plain single-launch kernel; afterwards the plan's forward and transposed packs are fresh, so the
// next vp3d_forward_train needs no vp3d_set_weights.  Replaces `optimizer.step()` (run.py:396, 420)
// AND the re-pack that used to follow it.
VP3D_API int vp3d_adam_step_packed(vp3d_plan* p, const vp3d_weights* w,
                                   const vp3d_adam_tensor* tensors, int32_t n_tensors, int64_t step,
                                   double lr, double beta1, double beta2, double eps,
                                   double weight_decay, void* stream_) {
  if (!p || !w || (n_tensors > 0 && !tensors))
    return fail(VP3D_ERR_INVALID, "adam_step_packed: null argument");
  if (p->f16) return fail(VP3D_ERR_UNSUPPORTED, "adam_step_packed: fp16 plans are inference-only");
  TrainState* t = p->train;
  if (!t || !t->packed_t || !p->conv_packed)
    return fail(VP3D_ERR_STATE, "adam_step_packed: the plan has no packed training weights yet "
                "(run a training forward first)");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  std::vector<vp3d_adam_tensor> plain;
  std::vector<AdamPackItem> packed;
  bool expand_seen = false;
  for (int i = 0; i < n_tensors; ++i) {
    const vp3d_adam_tensor& a = tensors[i];
    // a layer or shrink weight: the fused update writes its forward and transposed packs
    const PackedConv* tr = nullptr;
    for (int j = 0; j < p->n_packs && a.param && !tr; ++j) {
      const PackedConv& k = p->packs[j];
      if (k.transposed && k.src != kSrcExpand && conv_weight(w, k.src) == a.param) tr = &k;
    }
    if (tr) packed.push_back({a, forward_of(p, *tr), tr});
    else plain.push_back(a);
    if (a.param && a.param == w->expand_conv_weight) expand_seen = true;
  }
  VP3D_TRY(vp3d_adam_step(plain.data(), (int32_t)plain.size(), step, lr, beta1, beta2, eps,
                          weight_decay, stream_));
  VP3D_TRY(launch_adam_pack(packed.data(), (int)packed.size(), p->planes, step, lr, beta1, beta2, eps,
                            weight_decay, stream));
  // 104 k elements: the two expand packs (dilated / tap-merged) the usual way
  if (expand_seen) VP3D_TRY(pack_expand_forward(p, w, stream));
  p->last_launches = (plain.empty() ? 0 : 1) + (packed.empty() ? 0 : 1) + (expand_seen ? 2 : 0);
  return VP3D_OK;
}

// ---- operator-level entries (include/vp3d_b200.h): the launch functions the training step uses,
// with the step's own shape rules, for tests that compare one operator with a reference.
VP3D_API int vp3d_wgrad_gemm(const vp3d_wgrad_desc* d, void* stream) {
  if (!d || !d->dz || !d->x || !d->grad || !d->partial)
    return fail(VP3D_ERR_INVALID, "wgrad_gemm: null argument");
  if (d->planes != 1 && d->planes != 2) return fail(VP3D_ERR_INVALID, "wgrad_gemm: planes must be 1 or 2");
  if (d->rows < 1 || d->taps < 1 || d->c_out < 1 || d->c_in < 1 || d->c_in_cols < 1 ||
      d->taps_out < 1 || (d->per_sample && (d->samples < 1 || d->x_rows < 1)))
    return fail(VP3D_ERR_INVALID, "wgrad_gemm: empty shape");
  if (d->merged ? (d->taps != 1 || d->c_in_cols < d->taps_out * d->c_in)
                : (d->taps != d->taps_out || d->c_in_cols < d->c_in))
    return fail(VP3D_ERR_INVALID, "wgrad_gemm: taps / columns inconsistent with merged = %d", d->merged);
  if (d->dz_ld < round_up(d->c_out, 64) || d->dz_ld % 64 || d->x_ld % 64)
    return fail(VP3D_ERR_INVALID, "wgrad_gemm: row pitches must be multiples of 64 covering the channels");
  WgradCall c;
  c.dz = static_cast<const __nv_bfloat16*>(d->dz); c.dz_ld = d->dz_ld;
  c.x = static_cast<const __nv_bfloat16*>(d->x); c.x_ld = d->x_ld;
  c.rows = d->rows; c.per_sample = d->per_sample ? 1 : 0; c.samples = d->samples;
  c.x_rows = d->x_rows; c.taps = d->taps; c.tap_col_step = d->tap_col_step;
  c.tap_row_step = d->tap_row_step; c.c_out = d->c_out; c.c_in_cols = d->c_in_cols; c.c_in = d->c_in;
  c.taps_out = d->taps_out; c.merged = d->merged ? 1 : 0; c.grad = d->grad;
  return run_wgrad(d->planes, c, d->partial, d->partial_bytes, static_cast<cudaStream_t>(stream));
}

namespace {
int check_reduce_scratch(const char* what, int c, int per_split, size_t scratch_floats, int counters) {
  if (c < 1) return fail(VP3D_ERR_INVALID, "%s: channels must be positive", what);
  if (c > kReduceMaxChannels)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: %d channels, at most %d", what, c, kReduceMaxChannels);
  if (scratch_floats < (size_t)kReduceMaxSplits * per_split * c || counters < (c + 31) / 32)
    return fail(VP3D_ERR_WORKSPACE, "%s: scratch of %zu floats / %d counters, %zu / %d needed", what,
                scratch_floats, counters, (size_t)kReduceMaxSplits * per_split * c, (c + 31) / 32);
  return VP3D_OK;
}

int check_rows_c(const char* what, long long rows, int c, int planes) {
  if (rows < 1 || c < 64 || c % 64) return fail(VP3D_ERR_INVALID, "%s: rows >= 1 and channels a multiple of 64", what);
  if (planes != 1 && planes != 2) return fail(VP3D_ERR_INVALID, "%s: planes must be 1 or 2", what);
  return VP3D_OK;
}

DropoutCfg flat_drop(float p, unsigned long long seed, int layer) {
  DropoutCfg d;
  d.p = p;
  d.seed_lo = (uint32_t)(seed & 0xFFFFFFFFu);
  d.seed_hi = (uint32_t)(seed >> 32);
  d.layer = (uint32_t)layer;
  return d;
}
}  // namespace

VP3D_API int vp3d_bn_stats_finalize(const float* part, int slabs, int dilated, int out_rows,
                                    int tiles_per_sample, const float* gamma, const float* beta,
                                    float* running_mean, float* running_var, float momentum,
                                    float eps, float* scale, float* shift, float* mean,
                                    float* invstd, int c, int c_real, float* scratch,
                                    size_t scratch_floats, unsigned* counter, int counters,
                                    void* stream) {
  if (!part || !gamma || !beta || !scale || !shift || !mean || !invstd || !scratch || !counter ||
      (!running_mean != !running_var))
    return fail(VP3D_ERR_INVALID, "bn_stats_finalize: null argument");
  if (slabs < 1 || out_rows < 1 || c_real < 1 || c_real > c || (dilated && tiles_per_sample < 1))
    return fail(VP3D_ERR_INVALID, "bn_stats_finalize: bad geometry");
  VP3D_TRY(check_reduce_scratch("bn_stats_finalize", c, 3, scratch_floats, counters));
  CUDA_TRY(launch_bn_stats_finalize(part, slabs, dilated ? 1 : 0, out_rows, tiles_per_sample, gamma,
                                    beta, running_mean, running_var, momentum, eps, scale, shift,
                                    mean, invstd, c, c_real, scratch, counter,
                                    static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}

VP3D_API int vp3d_ordered_col_sums(const float* part, int n_part, int nstat, int ld, int c, int folds,
                                   const float* mul0, const float* mul1, float* out0, float* out1,
                                   float* scratch, size_t scratch_floats, unsigned* counter,
                                   int counters, void* stream) {
  if (!part || !out0 || (nstat == 2 && !out1) || !scratch || !counter)
    return fail(VP3D_ERR_INVALID, "ordered_col_sums: null argument");
  if (nstat < 1 || nstat > 2 || n_part < 1 || folds < 1 || ld < folds * c)
    return fail(VP3D_ERR_INVALID, "ordered_col_sums: bad geometry");
  VP3D_TRY(check_reduce_scratch("ordered_col_sums", c, 2, scratch_floats, counters));
  CUDA_TRY(launch_ordered_col_sums(part, n_part, nstat, ld, c, folds, mul0, mul1, out0, out1, scratch,
                                   counter, static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}

VP3D_API int vp3d_bn_apply(const void* z, long long z_plane, void* x, long long x_plane, int planes,
                           long long rows, int c, const float* scale, const float* shift,
                           float dropout_p, unsigned long long seed, int layer, const void* res,
                           long long res_plane, int res_div, int res_rows_per_sample, int res_step,
                           int res_off, void* stream) {
  if (!z || !x || !scale || !shift) return fail(VP3D_ERR_INVALID, "bn_apply: null argument");
  VP3D_TRY(check_rows_c("bn_apply", rows, c, planes));
  if (dropout_p < 0.0f || dropout_p >= 1.0f)
    return fail(VP3D_ERR_INVALID, "bn_apply: dropout p must be in [0, 1)");
  const RowMap map = {res_div, res_rows_per_sample, res_step, res_off};
  CUDA_TRY(launch_bn_apply(static_cast<const __nv_bfloat16*>(z), z_plane,
                           static_cast<__nv_bfloat16*>(x), x_plane, planes, rows, c, scale, shift,
                           flat_drop(dropout_p, seed, layer), static_cast<const __nv_bfloat16*>(res),
                           res_plane, map, static_cast<cudaStream_t>(stream)));
  return VP3D_OK;
}

VP3D_API int vp3d_bn_bwd_reduce(const void* g, long long g_plane, const void* z, long long z_plane,
                                int planes, long long rows, int c, const float* scale,
                                const float* shift, const float* mean, const float* invstd,
                                float dropout_p, unsigned long long seed, int layer, float* partials,
                                size_t partial_floats, float* sums, float* scratch,
                                size_t scratch_floats, unsigned* counter, int counters,
                                void* stream) {
  if (!g || !z || !scale || !shift || !mean || !invstd || !partials || !sums || !scratch || !counter)
    return fail(VP3D_ERR_INVALID, "bn_bwd_reduce: null argument");
  VP3D_TRY(check_rows_c("bn_bwd_reduce", rows, c, planes));
  if (dropout_p < 0.0f || dropout_p >= 1.0f)
    return fail(VP3D_ERR_INVALID, "bn_bwd_reduce: dropout p must be in [0, 1)");
  VP3D_TRY(check_reduce_scratch("bn_bwd_reduce", c, 2, scratch_floats, counters));
  const cudaError_t e = launch_bn_bwd_reduce(
      static_cast<const __nv_bfloat16*>(g), g_plane, static_cast<const __nv_bfloat16*>(z), z_plane,
      planes, rows, c, scale, shift, mean, invstd, flat_drop(dropout_p, seed, layer), partials,
      partial_floats, sums, scratch, counter, static_cast<cudaStream_t>(stream));
  // the one argument error of the launch: per-block partials larger than `partials` (nothing ran)
  if (e == cudaErrorInvalidValue)
    return fail(VP3D_ERR_WORKSPACE, "bn_bwd_reduce: %zu partial floats are too few", partial_floats);
  CUDA_TRY(e);
  return VP3D_OK;
}

VP3D_API int vp3d_bn_bwd_apply(const void* g, long long g_plane, const void* z, long long z_plane,
                               void* dz, long long dz_plane, int planes, long long rows, int c,
                               const float* scale, const float* shift, const float* mean,
                               const float* invstd, float dropout_p, unsigned long long seed,
                               int layer, const float* sums, float* dgamma, float* dbeta,
                               int c_real, int frozen, void* stream) {
  if (!g || !z || !dz || !scale || !shift || (!frozen && (!mean || !invstd || !sums)))
    return fail(VP3D_ERR_INVALID, "bn_bwd_apply: null argument");
  VP3D_TRY(check_rows_c("bn_bwd_apply", rows, c, planes));
  if (dropout_p < 0.0f || dropout_p >= 1.0f)
    return fail(VP3D_ERR_INVALID, "bn_bwd_apply: dropout p must be in [0, 1)");
  if (c_real < 1 || c_real > c) return fail(VP3D_ERR_INVALID, "bn_bwd_apply: c_real out of range");
  CUDA_TRY(launch_bn_bwd_apply(static_cast<const __nv_bfloat16*>(g), g_plane,
                               static_cast<const __nv_bfloat16*>(z), z_plane,
                               static_cast<__nv_bfloat16*>(dz), dz_plane, planes, rows, c, scale,
                               shift, mean, invstd, flat_drop(dropout_p, seed, layer), sums, dgamma,
                               dbeta, c_real, static_cast<cudaStream_t>(stream), frozen ? 1 : 0));
  return VP3D_OK;
}
