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
  Arena a{1024};
  for (int i = 0; i <= p->nb; ++i) w.rows[i] = (long long)N * L[i];
  w.a0 = a.take(strided ? pl * w.rows[0] * p->k0_pad * 2 : pl * (size_t)N * T * p->c_in_pad * 2);
  w.z[0] = a.take(pl * w.rows[0] * C * 2);
  w.x[0] = a.take(pl * w.rows[0] * C * 2);
  for (int i = 1; i <= p->nb; ++i) {
    const size_t b = pl * w.rows[i] * C * 2;
    w.z[2 * i - 1] = a.take(b);
    w.h[i] = a.take(b);
    w.z[2 * i] = a.take(b);
    w.x[i] = a.take(b);
  }
  const size_t big = pl * w.rows[0] * C * 2;
  w.g0 = a.take(big);
  w.g1 = a.take(big);
  w.dz = a.take(big);
  w.dyp = a.take(pl * w.rows[p->nb] * p->shrink_t->k_pad * 2);   // dY in K layout of shrink_t
  // wgrad partials: up to 8 splits x taps x C x max(C, k0_pad) fp32
  int max_taps = 1;
  for (int i = 1; i <= p->nb; ++i) max_taps = p->taps[i] > max_taps ? p->taps[i] : max_taps;
  size_t n_max = p->C > p->k0_pad ? p->C : p->k0_pad;
  if ((size_t)p->c_in_pad > n_max) n_max = p->c_in_pad;
  if (!strided && p->cfg.filter_widths[0] > max_taps) max_taps = p->cfg.filter_widths[0];
  w.partial_bytes = (size_t)8 * max_taps * round_up(p->C, 128) * round_up((int)n_max, 64) * 4;
  w.partial = a.take(w.partial_bytes);
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
    w.slab = a.take(w.slab_floats * sizeof(float));
  }
  if (strided && T != p->cfg.filter_widths[0] * L[0])
    w.dx_stage = a.take((size_t)w.rows[0] * p->cfg.filter_widths[0] * p->c_in_raw * sizeof(float));
  w.total = a.total();
  return w;
}

// dW = dZ^T X for one conv layer (the descriptor of vp3d_wgrad_gemm).  The tile width and the
// split count follow from the shape alone.
int run_wgrad(const vp3d_wgrad_desc& c, cudaStream_t stream) {
  const int planes = c.planes;
  const int block_n = pick_block_n(round_up(c.c_in_cols, 64));
  WgradArgs a;
  memset(&a, 0, sizeof(a));
  a.per_sample = c.per_sample ? 1 : 0;
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
  while ((size_t)splits * c.taps * a.m_pad * a.n_pad * 4 > c.partial_bytes && splits > 1) --splits;
  if ((size_t)splits * c.taps * a.m_pad * a.n_pad * 4 > c.partial_bytes)
    return fail(VP3D_ERR_WORKSPACE, "wgrad partial buffer too small");
  a.splits = splits;
  a.partial = c.partial;
  CUtensorMap mdz, mx;
  const uint64_t x_rows = c.per_sample ? (uint64_t)c.x_rows : (uint64_t)c.rows;
  VP3D_TRY(make_map_4d(&mdz, c.dz, c.dz_ld, c.rows, c.dz_ld, a.samples, (uint64_t)c.rows * c.dz_ld,
                       planes, (uint64_t)a.samples * c.rows * c.dz_ld, 64));
  VP3D_TRY(make_map_4d(&mx, c.x, c.x_ld, x_rows, c.x_ld, a.samples, x_rows * c.x_ld, planes,
                       (uint64_t)a.samples * x_rows * c.x_ld, 64));
  CUDA_TRY(launch_wgrad_gemm(mdz, mx, a, block_n, num_sms(), stream));
  CUDA_TRY(launch_wgrad_reduce(c.partial, c.grad, splits, c.taps, a.m_pad, a.n_pad, c.c_out, c.c_in,
                               c.taps_out, c.merged ? 1 : 0, stream));
  return VP3D_OK;
}

DropoutCfg dropout_cfg(float p, unsigned long long seed, int layer) {
  DropoutCfg d;
  d.p = p;
  d.seed_lo = (uint32_t)(seed & 0xFFFFFFFFu);
  d.seed_hi = (uint32_t)(seed >> 32);
  d.layer = (uint32_t)layer;
  return d;
}

// elements of one plane of a GEMM's A operand, the conv's input
long long in_plane(const vp3d_conv_desc& d) { return (long long)d.samples * d.a_rows * d.a_ld; }

// 32-row slabs of the per-channel partials a GEMM epilogue writes (statistics or fused BatchNorm
// backward): four per 128-row tile, the tiles per sample (per-sample tiling) or over all rows
int stat_slabs(const vp3d_conv_desc& d) {
  return (d.per_sample_tiles ? d.samples : 1) * ((d.out_rows + 127) / 128) * 4;
}

// columns of the input one tap of conv k spans: all taps' when they are merged into one GEMM
int in_cols(const PackedConv& k) { return k.merged ? k.taps * k.c_in : k.c_in; }

// One conv of the training step.  `fwd` is its forward GEMM: the A view of its input (samples,
// rows, ld, per-sample tiles, tap step), the output rows and the forward pack, writing Z.  The
// backward derives its weight and data gradients from it (wgrad_desc, dgrad_desc), so that they
// read and write the views the forward used.
struct TrainConv {
  vp3d_conv_desc fwd;        // shrink: no output set (the forward adds its fp32 epilogue)
  const PackedConv* pack;    // forward pack: the gradient's c_out, c_in, taps, merged
  const PackedConv* t;       // transposed pack of the data gradient
  __nv_bfloat16 *in, *z, *act;   // input (= fwd.a), Z (= fwd.out), the BatchNorm's output
  RowMap res;                // block second conv: the block input rows its skip connection adds
                             // (res.off: the frame of the input row, or the row offset, it takes)
};

// The convs of the training step indexed by BatchNorm layer (0 expand, 2i-1 / 2i block i's first
// and second conv) and shrink at 2B + 1.  Besides train_layout the only code that tells the two
// layouts apart: strided (flat rows; the expand conv's taps merged into one GEMM over w0 frames per
// input row, a first conv's taps column blocks of a w*C-wide view of the rows) and dilated
// (per-sample tiles, the taps rows `dilation` apart).
void train_convs(const vp3d_plan* p, const TrainLayout& wl, uint8_t* base, int N, int T,
                 const int* L, TrainConv* cv) {
  const bool strided = p->cfg.variant == VP3D_VARIANT_STRIDED;
  const int C = p->C, nb = p->nb;
  const int* fw = p->cfg.filter_widths;
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(base + off); };
  auto conv = [&](int l, const PackedConv* k, const PackedConv* kt, size_t in, long long a_rows,
                  int a_ld, long long out_rows) -> vp3d_conv_desc& {
    TrainConv& c = cv[l];
    c.pack = k; c.t = kt; c.in = bf(in); c.z = c.act = nullptr; c.res = RowMap{0, 0, 1, 0};
    vp3d_conv_desc& d = c.fwd = conv_desc(p, p->cfg.precision);
    use_pack(&d, *k);
    d.a = c.in; d.a_rows = (int)a_rows; d.a_ld = a_ld; d.out_rows = (int)out_rows;
    return d;
  };
  auto per_sample = [&](vp3d_conv_desc& d, int step) {
    d.samples = N; d.per_sample_tiles = 1; d.tap_row_step = step;
  };
  if (strided) {
    conv(0, p->expand_flat, p->expand_t, wl.a0, wl.rows[0], p->k0_pad, wl.rows[0]);
  } else {
    per_sample(conv(0, p->expand_dil, p->expand_t, wl.a0, T, p->c_in_pad, L[0]), 1);
  }
  for (int i = 1; i <= nb; ++i) {
    const int l1 = 2 * i - 1, l2 = 2 * i;
    if (strided) {
      conv(l1, p->conv[l1 - 1], p->conv_t[l1 - 1], wl.x[i - 1], wl.rows[i], fw[i] * C, wl.rows[i])
          .tap_col_step = C;
    } else {
      per_sample(conv(l1, p->conv[l1 - 1], p->conv_t[l1 - 1], wl.x[i - 1], L[i - 1], C, L[i]),
                 p->dilation[i]);
    }
    conv(l2, p->conv[l2 - 1], p->conv_t[l2 - 1], wl.h[i], wl.rows[i], C, wl.rows[i]);
    cv[l2].res = strided ? RowMap{0, 0, fw[i], fw[i] / 2 + p->shift_str[i]}
                         : RowMap{L[i], L[i - 1], 1, p->pad[i] + p->shift_dil[i]};
  }
  conv(2 * nb + 1, p->shrink, p->shrink_t, wl.x[nb], wl.rows[nb], C, wl.rows[nb]);
  for (int l = 0; l <= 2 * nb; ++l) {
    const int i = (l + 1) / 2;   // the block whose rows layer l has (0: expand)
    TrainConv& c = cv[l];
    c.z = bf(wl.z[l]);
    c.act = bf(l % 2 ? wl.h[i] : wl.x[i]);
    c.fwd.out = c.z; c.fwd.out_plane_stride = wl.rows[i] * C; c.fwd.out_ld = C;
  }
}

// The weight gradient of conv c from its forward GEMM: dZ (rows as the forward's output, pitch the
// transposed pack's K) against the forward's A view with the forward's taps.
vp3d_wgrad_desc wgrad_desc(const TrainConv& c, const __nv_bfloat16* dz, float* grad, float* partial,
                           size_t partial_bytes) {
  const vp3d_conv_desc& f = c.fwd;
  vp3d_wgrad_desc w;
  memset(&w, 0, sizeof(w));
  w.dz = dz; w.dz_ld = c.t->k_pad;
  w.x = f.a; w.x_ld = f.a_ld; w.x_rows = f.a_rows;
  w.planes = f.a_planes;
  w.rows = f.out_rows; w.per_sample = f.per_sample_tiles; w.samples = f.samples;
  w.taps = f.taps; w.tap_row_step = f.tap_row_step; w.tap_col_step = f.tap_col_step;
  w.c_out = c.pack->c_out; w.c_in = c.pack->c_in; w.taps_out = c.pack->taps;
  w.merged = c.pack->merged; w.c_in_cols = in_cols(*c.pack);
  w.grad = grad; w.partial = partial; w.partial_bytes = partial_bytes;
  return w;
}

// The data gradient of conv c from its forward GEMM: dZ, read in the view the forward wrote Z in
// (pitch the transposed pack's K: C, or the padded dY of shrink), times the transposed pack, into
// `out` in the view the forward read its input from.  With `res`: plus the skip gradient (dZ's
// shape) at the input rows the forward's skip connection took, res_off as in TrainConv::res.
vp3d_conv_desc dgrad_desc(const vp3d_plan* p, const TrainConv& c, const __nv_bfloat16* dz,
                          __nv_bfloat16* out, const __nv_bfloat16* res = nullptr, int res_off = 0) {
  const vp3d_conv_desc& f = c.fwd;
  vp3d_conv_desc d = conv_desc(p, p->cfg.precision);
  use_pack(&d, *c.t);
  d.a = dz; d.a_rows = f.out_rows; d.a_ld = c.t->k_pad;
  d.out = out; d.out_rows = f.a_rows; d.out_plane_stride = in_plane(f); d.out_ld = f.a_ld;
  if (f.per_sample_tiles) {
    // row taps: the transposed convolution G[n, t] = sum_k dZ[n, t - k*step] * W_k^T; rows outside
    // the sample are zero-filled by the A / residual tensor maps
    d.samples = f.samples; d.per_sample_tiles = 1; d.tap_row_step = -f.tap_row_step;
  } else {
    // column or merged taps: one flat GEMM, the pack's tap slabs [ci][co] read as one [taps*ci][co]
    d.n_pad *= d.taps; d.taps = 1;
  }
  if (res) {
    d.res = res; d.res_planes = f.out_planes; d.res_plane_stride = f.out_plane_stride;
    d.res_ld = f.out_ld; d.res_row_step = 1;
    if (f.per_sample_tiles) {   // G_in[n, t] += res[n, t - off]
      d.res_rows_per_sample = f.out_rows; d.res_row_off = -res_off; d.res_check_rows = 1;
    } else {                    // frame `off` of each input row
      d.res_col_begin = res_off * f.out_ld; d.res_cols = f.out_ld;
    }
  }
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
  uint8_t* base = ws_base(ws);
  const int C = p->C, pl = p->planes;
  t->N = N; t->T = T; t->dropout_p = dropout_p; t->seed = seed; t->frozen_bn = frozen;
  t->have_forward = false;
  // frozen BatchNorm has no batch statistics: nothing to exchange, in this forward or its backward
  t->fwd_sync = frozen ? TrainState::BnSync() : t->sync;
  const TrainState::BnSync sync = t->fwd_sync;
  const bool synced = sync.world > 0;
  for (int i = 0; i <= p->nb; ++i) t->L[i] = L[i];
  TrainConv cv[VP3D_MAX_LAYERS + 2];
  train_convs(p, wl, base, N, T, L, cv);
  int launches = 0;

  float* slab_part = reinterpret_cast<float*>(base + wl.slab);
  CUDA_TRY(launch_bias_affine(w->shrink_bias, t->shrink_affine, t->shrink_affine + p->c_out_pad,
                              p->c_out_raw, p->c_out_pad, stream));
  ++launches;

  // BatchNorm (+ ReLU, dropout, skip connection) of `layer` over the Z that GEMM d wrote, whose
  // epilogue left the per-slab statistics partials in slab_part with its own row tiling
  auto bn = [&](int layer, const vp3d_conv_desc& d, const float* const* bnp, __nv_bfloat16* out,
                const __nv_bfloat16* res, long long res_plane, RowMap map) -> int {
    const LayerVec v = layer_vec(p, layer);
    const long long rows = (long long)d.samples * d.out_rows;
    if (frozen) {  // the eval fold of the running statistics, plus the mean / invstd backward reads
      CUDA_TRY(launch_bn_fold(bnp[0], bnp[1], bnp[2], bnp[3], 1e-5f, v.scale, v.shift, p->c_real, C,
                              stream, v.mean, v.invstd));
    } else {
      // synchronized: this rank's moments into its slot, the exchange fills the others, then the
      // rank-ordered merge and the finalize over the global batch update the running statistics
      float* slots = synced ? sync_fwd_slots(p, layer) : nullptr;
      CUDA_TRY(launch_bn_stats_finalize(
          slab_part, stat_slabs(d), d.per_sample_tiles, d.out_rows,
          d.per_sample_tiles ? (d.out_rows + 127) / 128 : 0, bnp[0], bnp[1],
          synced ? nullptr : const_cast<float*>(bnp[2]), synced ? nullptr : const_cast<float*>(bnp[3]),
          synced ? 0.0f : bn_momentum[layer], 1e-5f, v.scale, v.shift, v.mean, v.invstd, C,
          p->c_real, t->red_scratch, t->red_counter, stream, slots, sync.world, sync.rank));
      if (synced) {
        sync.exchange(layer, VP3D_BN_SYNC_FORWARD, slots, 3 * C, sync.user);
        CUDA_TRY(launch_bn_sync_finalize(slots, sync.world, bnp[0], bnp[1], const_cast<float*>(bnp[2]),
                                         const_cast<float*>(bnp[3]), bn_momentum[layer], 1e-5f,
                                         v.scale, v.shift, v.mean, v.invstd, C, p->c_real,
                                         t->sync_n + layer, stream));
        ++launches;
      }
    }
    CUDA_TRY(launch_bn_apply(static_cast<const __nv_bfloat16*>(d.out), rows * C, out, rows * C, pl,
                             rows, C, v.scale, v.shift, dropout_cfg(dropout_p, seed, layer), res,
                             res_plane, map, stream));
    launches += 2;
    return VP3D_OK;
  };

  // the input rows the expand GEMM reads, w0 frames per row when its taps are merged (model.py:188
  // strided / :127 dilated)
  const vp3d_conv_desc& e = cv[0].fwd;
  const int group = cv[0].pack->merged ? cv[0].pack->taps : 1;
  CUDA_TRY(launch_pack_input(x, cv[0].in, pl, N, T, p->c_in_raw, e.samples * e.a_rows / N, group,
                             group, e.a_ld, in_plane(e), stream));
  ++launches;
  // expand, then the residual blocks (model.py:190-194)
  for (int l = 0; l <= 2 * p->nb; ++l) {
    vp3d_conv_desc d = cv[l].fwd;
    d.stats = frozen ? nullptr : slab_part;
    VP3D_TRY(run_conv(&d, stream));
    ++launches;
    // a block's second conv adds the block's input back (the skip connection)
    const TrainConv* skip = l > 0 && l % 2 == 0 ? &cv[l - 1] : nullptr;
    VP3D_TRY(bn(l, d, l ? w->layers_bn[l - 1] : w->expand_bn, cv[l].act, skip ? skip->in : nullptr,
                skip ? in_plane(skip->fwd) : 0, cv[l].res));
  }

  // ---- shrink (model.py:196)
  vp3d_conv_desc d = cv[2 * p->nb + 1].fwd;
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
  const int N = t->N, C = p->C, pl = p->planes;
  const int* L = t->L;
  const TrainLayout wl = train_layout(p, N, t->T, L);
  if (!ws || ws_bytes < wl.total) return fail(VP3D_ERR_WORKSPACE, "backward: workspace too small");
  uint8_t* base = ws_base(ws);
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
  TrainConv cv[VP3D_MAX_LAYERS + 2];
  train_convs(p, wl, base, N, t->T, L, cv);
  const int top = 2 * p->nb;   // the BatchNorm under shrink

  // In single-plane bf16 mode the per-channel reductions of the BatchNorm backward are fused into
  // the epilogue of the GEMM that produces the incoming gradient (fuse_bnb); otherwise a separate
  // pass over (G, Z) computes them.
  const bool fuse = (pl == 1);
  // geometry of the slab partials the last fused GEMM left behind (consumed by the next bn_bwd)
  int bnb_slabs = 0, bnb_ld = 0;
  auto fuse_bnb = [&](vp3d_conv_desc& q, int layer) {
    if (!fuse || !need_sums) return;
    const LayerVec v = layer_vec(p, layer);
    q.bnb_z = cv[layer].z;
    q.bnb_scale = v.scale; q.bnb_shift = v.shift; q.bnb_mean = v.mean; q.bnb_invstd = v.invstd;
    q.bnb_sums = slab_part; q.bnb_c = C; q.bnb_p = t->dropout_p; q.bnb_seed = t->seed;
    q.bnb_layer = layer;
    bnb_slabs = stat_slabs(q);
    bnb_ld = q.n_pad;
  };
  // BN + ReLU + dropout backward of `layer`: (gin, z) -> dz (+ dgamma, dbeta)
  auto bn_bwd = [&](int layer, const __nv_bfloat16* gin) -> int {
    const LayerVec v = layer_vec(p, layer);
    const DropoutCfg dc = dropout_cfg(t->dropout_p, t->seed, layer);
    const long long rows = (long long)cv[layer].fwd.samples * cv[layer].fwd.out_rows;
    const __nv_bfloat16* z = cv[layer].z;
    float* const* dbn = !want_w ? nullptr : layer ? g->layers_bn[layer - 1] : g->expand_bn;
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
                                 need_sums ? local : nullptr, dbn ? dbn[0] : nullptr,
                                 dbn ? dbn[1] : nullptr, p->c_real, stream, frozen ? 1 : 0,
                                 synced ? v.sums : nullptr, synced ? t->sync_n + layer : nullptr));
    ++launches;
    return VP3D_OK;
  };

  auto wgrad = [&](const TrainConv& c, const __nv_bfloat16* dz, float* grad) -> int {
    VP3D_TRY(run_wgrad(wgrad_desc(c, dz, grad, partial, wl.partial_bytes), stream));
    launches += 2;
    return VP3D_OK;
  };

  // ---- shrink backward: y = X_nb * Wsh^T + b
  const TrainConv& sh = cv[top + 1];
  CUDA_TRY(launch_pack_input(dy, bf(wl.dyp), pl, 1, (int)rows_top, p->c_out_raw, (int)rows_top, 1, 1,
                             dy_ld, rows_top * dy_ld, stream));
  ++launches;
  if (want_w) {
    CUDA_TRY(launch_col_sum_f32(dy, rows_top, p->c_out_raw, slab_part, wl.slab_floats, g->shrink_bias,
                                t->red_scratch, t->red_counter, stream));
    launches += 2;
    VP3D_TRY(wgrad(sh, bf(wl.dyp), g->shrink_weight));
  }
  __nv_bfloat16* gb[2] = {bf(wl.g0), bf(wl.g1)};
  int cur = 0;
  vp3d_conv_desc d = dgrad_desc(p, sh, bf(wl.dyp), gb[cur]);
  fuse_bnb(d, top);  // G_nb feeds the BN backward of the top block's second conv (or expand)
  VP3D_TRY(run_conv(&d, stream));
  ++launches;
  if (stage_done) stage_done(0, user);  // shrink.weight / shrink.bias gradients are enqueued

  // ---- the BatchNorm layers top-down, each with its conv's weight and data gradient.  Block i's
  // output gradient G_i stays in gb[cur] while its second conv's data gradient goes to gb[cur ^ 1];
  // its first conv's data gradient G_{i-1} overwrites that, plus G_i through the skip connection.
  for (int l = top; l >= 0; --l) {
    const TrainConv& c = cv[l];
    VP3D_TRY(bn_bwd(l, gb[l % 2 ? cur ^ 1 : cur]));
    if (want_w)
      VP3D_TRY(wgrad(c, bf(wl.dz), l ? g->layers_conv_weight[l - 1] : g->expand_conv_weight));
    if (l > 0) {
      d = l % 2 ? dgrad_desc(p, c, bf(wl.dz), gb[cur ^ 1], gb[cur], cv[l + 1].res.off)
                : dgrad_desc(p, c, bf(wl.dz), gb[cur ^ 1]);
      fuse_bnb(d, l - 1);  // BN backward of the layer below: block i-1's second conv, or expand
      VP3D_TRY(run_conv(&d, stream));
      ++launches;
    } else if (dx) {
      // the expand conv's data gradient only on request (run.py's 2-D input needs none,
      // run.py:402-412; a differentiable front end or test-time refinement of x does): fp32
      // epilogue straight into x's (N, T, J*F) layout.  The strided model's tap-merged row (n, r)
      // holds x[n, r*w0 + tap, ci] at column tap*cin + ci, x's own memory order when T = w0 * L0;
      // the dilated model's transposed convolution writes every one of the T rows.
      d = dgrad_desc(p, c, bf(wl.dz), nullptr);
      d.out_f32 = dx; d.out_f32_ld = d.n_valid = in_cols(*c.pack);
      const int cin = p->c_in_raw, T = t->T, w0 = p->cfg.filter_widths[0];
      // trailing frames no output depends on: the GEMM writes a staging buffer, one strided copy
      // moves each sample's rows into place and one strided memset zeroes the tails
      const bool tail = p->cfg.variant == VP3D_VARIANT_STRIDED && T != w0 * L[0];
      if (tail) d.out_f32 = reinterpret_cast<float*>(base + wl.dx_stage);
      VP3D_TRY(run_conv(&d, stream));
      ++launches;
      if (tail) {
        const size_t used = (size_t)w0 * L[0] * cin;   // floats per sample the output depends on
        const size_t pitch = (size_t)T * cin * sizeof(float);
        CUDA_TRY(cudaMemcpy2DAsync(dx, pitch, d.out_f32, used * sizeof(float), used * sizeof(float),
                                   N, cudaMemcpyDeviceToDevice, stream));
        CUDA_TRY(cudaMemset2DAsync(dx + used, pitch, 0, pitch - used * sizeof(float), N, stream));
        launches += 2;
      }
    }
    if (l % 2) {
      cur ^= 1;
      const int i = (l + 1) / 2;
      if (stage_done) stage_done(p->nb - i + 1, user);  // all four parameter groups of block i
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
  return run_wgrad(*d, static_cast<cudaStream_t>(stream));
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
                           dropout_cfg(dropout_p, seed, layer), static_cast<const __nv_bfloat16*>(res),
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
      planes, rows, c, scale, shift, mean, invstd, dropout_cfg(dropout_p, seed, layer), partials,
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
                               shift, mean, invstd, dropout_cfg(dropout_p, seed, layer), sums, dgamma,
                               dbeta, c_real, static_cast<cudaStream_t>(stream), frozen ? 1 : 0));
  return VP3D_OK;
}
