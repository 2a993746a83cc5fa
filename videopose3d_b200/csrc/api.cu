// C-ABI implementation: plan construction, parameter packing, eval-mode forward schedules
// (strided / dependency-cone and dilated) built from the conv GEMM kernel.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "internal.cuh"
#include "pack.cuh"
#include "train_ops.cuh"

using namespace vp3d;

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
namespace vp3d {
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace vp3d

// ------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

namespace vp3d {
int make_map_4d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows,
                       uint64_t row_stride, uint64_t samples, uint64_t sample_stride,
                       uint64_t planes, uint64_t plane_stride, uint32_t box_rows, int elem_bytes,
                       uint32_t box_bytes, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(VP3D_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  const uint64_t eb = (uint64_t)elem_bytes;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (row_stride * eb) % 16 || (sample_stride * eb) % 16 ||
      (plane_stride * eb) % 16)
    return fail(VP3D_ERR_INVALID, "tensor map operand not 16-byte aligned");
  cuuint64_t dims[4] = {inner, rows, samples, planes};
  cuuint64_t strides[3] = {row_stride * eb, sample_stride * eb, plane_stride * eb};
  cuuint32_t box[4] = {box_bytes / (cuuint32_t)elem_bytes, box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(VP3D_ERR_CUDA,
                "cuTensorMapEncodeTiled(4d) failed: %d (inner=%llu rows=%llu rs=%llu samples=%llu "
                "ss=%llu planes=%llu ps=%llu)",
                (int)r, (unsigned long long)inner, (unsigned long long)rows,
                (unsigned long long)row_stride, (unsigned long long)samples,
                (unsigned long long)sample_stride, (unsigned long long)planes,
                (unsigned long long)plane_stride);
  return VP3D_OK;
}

// 2-D bf16 map (k, row), box (64, box_rows), 128-byte swizzle.
int make_map_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows,
                       uint32_t box_rows, int elem_bytes) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(VP3D_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {inner * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)(elem_bytes == 1 ? kBlockK8 : kBlockK), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(VP3D_ERR_CUDA, "cuTensorMapEncodeTiled(2d) failed: %d (inner=%llu rows=%llu)",
                (int)r, (unsigned long long)inner, (unsigned long long)rows);
  return VP3D_OK;
}

int pick_block_n(int n_pad) {
  if (n_pad % 128 == 0) return 128;
  return 64;
}

// SM count of the CURRENT device (cached per device ordinal: one process may drive several GPUs)
static int g_sm_limit = 0;   // vp3d_set_sm_limit: persistent grids leave the other SMs to NCCL
int num_sms() {
  static int cache[kMaxDevices] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 132;
  if (!cache[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = n > 0 ? n : 132;
    if (const char* e = getenv("VP3D_SM_LIMIT")) {
      const int lim = atoi(e);
      if (lim >= 2 && !g_sm_limit) g_sm_limit = lim;
    }
  }
  int n = cache[dev];
  if (g_sm_limit >= 2 && g_sm_limit < n) n = g_sm_limit;
  return n;
}

// ------------------------------------------------------------------ operator level
// Everything one conv GEMM launch passes to launch_conv_gemm, validated and built from its
// descriptor by prepare_conv.  run_conv launches it; vp3d_conv_gemm_instance asks which kernel
// instance that launch would run -- the same preparation either way.
struct ConvLaunch {
  CUtensorMap ma, mw, mw64, mo, mr, mz;   // (mw64: W in 64-row boxes, for the half tiles)
  ConvGemmArgs g;
  int block_n = 64;
  int sms = 0;
  bool empty = false;   // no output rows: nothing to launch
};

static int prepare_conv(const vp3d_conv_desc* d, ConvLaunch* L) {
  if (!d || !d->a || !d->w) return fail(VP3D_ERR_INVALID, "conv_gemm: null operand");
  if (d->a_ld % 64 || d->k_per_tap % 64 || d->n_pad % 64)
    return fail(VP3D_ERR_INVALID, "conv_gemm: a_ld, k_per_tap and n_pad must be multiples of 64");
  if (d->taps < 1 || d->out_rows < 0 || d->samples < 1)
    return fail(VP3D_ERR_INVALID, "conv_gemm: bad geometry");
  L->empty = d->out_rows == 0;
  if (L->empty) return VP3D_OK;
  const int a_planes = d->a_planes > 0 ? d->a_planes : 1;
  const int pairs = d->precision == VP3D_PRECISION_BF16X3 ? 3 : 1;
  const int i8 = d->precision == VP3D_PRECISION_INT8 ? 1 : 0;
  const int f16 = (d->precision == VP3D_PRECISION_FP16 || i8) ? 1 : 0;   // (int8: fp16 res / out)
  if (f16 && (a_planes != 1 || d->out_planes > 1 || d->stats || d->bnb_z))
    return fail(VP3D_ERR_INVALID, "conv_gemm: fp16 is a single-plane, inference-only format");
  if (i8 && (d->k_per_tap % kBlockK8 || d->tap_col_step != 0))
    return fail(VP3D_ERR_INVALID, "conv_gemm: int8 needs k_per_tap %% 128 == 0 and taps that step "
                "rows (tap_col_step 0)");
  if (d->out_u8 && (!f16 || d->out_u8_ld % 16 || d->out_u8_ld < d->n_pad ||
                    reinterpret_cast<uintptr_t>(d->out_u8) % 16))
    return fail(VP3D_ERR_INVALID, "conv_gemm: a u8 output needs fp16 or int8, a 16-byte aligned "
                "pointer and out_u8_ld >= n_pad, a multiple of 16");
  if ((i8 || d->out_u8) &&
      (!d->scale || !d->shift || !d->relu || d->out_f32 || d->res_col_begin || d->res_cols ||
       (d->res && d->res_planes > 1) || (i8 && d->res && !d->out) ||
       (i8 && !d->res && (d->out || !d->out_u8)) || (!i8 && (!d->out || d->res))))
    return fail(VP3D_ERR_UNSUPPORTED, "conv_gemm: int8 and u8 outputs exist for affine + ReLU "
                "[+ one-plane residual over every column] launches: int8 writes u8 alone or, with a "
                "residual, fp16 [+ u8]; fp16 without a residual writes fp16 + u8");
  if (pairs == 3 && a_planes != 2)
    return fail(VP3D_ERR_INVALID, "conv_gemm: bf16x3 needs hi/lo planes of A");
  const int w_planes = pairs == 3 ? 2 : 1;
  // 128-wide N tiles (a 128 x 128 tile per CTA: 64 x 128 wgmma per consumer warpgroup) while they
  // still fill half a wave of the SMs; small layers (few row tiles) fall back to 64-wide tiles so
  // that more SMs share the work.
  int& block_n = L->block_n;
  L->sms = num_sms();
  block_n = 64;
  {
    const long long m_tiles = d->per_sample_tiles
                                  ? (long long)d->samples * ((d->out_rows + kBlockM - 1) / kBlockM)
                                  : ((long long)d->out_rows + kBlockM - 1) / kBlockM;
    if (d->n_pad % 128 == 0 && m_tiles * (d->n_pad / 128) * 2 >= L->sms) block_n = 128;
  }

  CUtensorMap& ma = L->ma;
  CUtensorMap& mw = L->mw;
  const uint64_t a_rows = d->a_rows, a_ld = d->a_ld;
  // (an explicit plane stride when the A rows are a window into a larger buffer, e.g. a history ring)
  const uint64_t plane_stride = d->a_plane_stride > 0 ? (uint64_t)d->a_plane_stride
                                                      : (uint64_t)d->samples * a_rows * a_ld;
  VP3D_TRY(make_map_4d(&ma, d->a, a_ld, a_rows, a_ld, d->samples, a_rows * a_ld, a_planes,
                       plane_stride, kBlockM, i8 ? 1 : 2));
  ConvGemmArgs& g = L->g;
  memset(&g, 0, sizeof(g));
  g.dilated = d->per_sample_tiles ? 1 : 0;
  g.samples = d->samples;
  g.out_rows = d->out_rows;
  g.tiles_per_sample = (d->out_rows + kBlockM - 1) / kBlockM;
  g.taps = d->taps;
  g.kblocks_per_tap = d->k_per_tap / (i8 ? kBlockK8 : kBlockK);
  g.tap_row_step = d->tap_row_step;
  g.tap_col_step = d->tap_col_step;
  g.n_pad = d->n_pad;
  g.n_tiles = d->n_pad / block_n;
  g.pairs = pairs;
  g.f16 = f16;
  g.flags = 0;
  if (d->scale && d->shift) g.flags |= kEpiAffine;
  if (d->relu) g.flags |= kEpiRelu;
  if (d->res) g.flags |= kEpiResidual;
  if (d->stats) g.flags |= kEpiStats;
  if (d->out_f32) g.flags |= kEpiOutF32;
  g.scale = d->scale;
  g.shift = d->shift;
  g.res = static_cast<const __nv_bfloat16*>(d->res);
  g.res_plane_stride = d->res_plane_stride;
  g.res_planes = d->res ? (d->res_planes > 0 ? d->res_planes : 1) : 0;
  g.res_ld = d->res_ld;
  g.res_rows_per_sample = d->res_rows_per_sample;
  g.res_row_step = d->res_row_step;
  g.res_row_off = d->res_row_off;
  g.res_sample_div = d->res_sample_div;
  g.res_col_begin = d->res_col_begin;
  g.res_cols = d->res_cols > 0 ? d->res_cols : d->n_pad;
  g.res_check_rows = d->res_check_rows;
  g.out = static_cast<__nv_bfloat16*>(d->out);
  g.out_plane_stride = d->out_plane_stride;
  g.out_planes = d->out_planes > 0 ? d->out_planes : 1;
  g.out_ld = d->out_ld;
  g.out_f32 = d->out_f32;
  g.out_f32_ld = d->out_f32_ld;
  g.n_valid = d->n_valid > 0 ? d->n_valid : d->n_pad;
  g.stats = d->stats;
  g.lo_row_begin = d->lo_row_end > 0 ? d->lo_row_begin : 0;
  g.lo_row_end = d->lo_row_end > 0 ? d->lo_row_end : 0x7fffffff;
  g.i8 = i8;
  g.out_u8 = static_cast<uint8_t*>(d->out_u8);
  g.u8_inv_s = d->out_u8_inv_scale;
  if (!d->out && !d->out_f32 && !d->out_u8) return fail(VP3D_ERR_INVALID, "conv_gemm: no output");
  if (d->out && (d->out_ld % 8)) return fail(VP3D_ERR_INVALID, "conv_gemm: out_ld % 8 != 0");
  if (d->res && (d->res_ld % 8)) return fail(VP3D_ERR_INVALID, "conv_gemm: res_ld % 8 != 0");
  CUtensorMap& mo = L->mo;
  mo = ma;
  if (d->out) {
    const uint64_t o_rows = d->out_rows, o_ld = d->out_ld;
    const uint64_t o_samples = d->per_sample_tiles ? d->samples : 1;
    uint64_t o_plane = (uint64_t)d->out_plane_stride;
    if (g.out_planes == 1 || o_plane == 0) o_plane = o_samples * o_rows * o_ld;
    // (32-row boxes: every epilogue warp stores its own quarter of a tile)
    VP3D_TRY(make_map_4d(&mo, d->out, o_ld, o_rows, o_ld, o_samples, o_rows * o_ld, g.out_planes,
                         o_plane, 32));
  }
  // Residual through TMA (warp 3 prefetches each 128 x 64 residual tile into shared memory) whenever
  // the residual rows of a tile are one box of a strided row view:
  //   row(t) = sample*rows_per_sample + t*step + off  ==  view row (sample, t), column off*ld + c
  // with the view's rows `step*ld` elements long (strided layout: off < step), or rows shifted by
  // `off` (step == 1).  Other maps (flat tiles split over samples, bounds-checked rows) keep the
  // register path.
  CUtensorMap& mr = L->mr;
  mr = ma;
  g.res_tma = 0;
  // (per-sample maps zero-fill rows outside the sample, which is exactly what res_check_rows asks)
  if (d->res && (!d->res_check_rows || (d->per_sample_tiles && d->res_row_step == 1)) && d->out &&
      (d->per_sample_tiles || d->res_sample_div == 0) &&
      d->res_row_step >= 1 && (d->res_row_step == 1 || d->res_row_off < d->res_row_step)) {
    const uint64_t step = d->res_row_step, ld = d->res_ld;
    const uint64_t r_samples = d->per_sample_tiles ? d->samples : 1;
    uint64_t view_rows, col_off;
    long long row_off;
    if (step == 1) {
      view_rows = d->per_sample_tiles ? (uint64_t)d->res_rows_per_sample
                                      : (uint64_t)d->out_rows + d->res_row_off;
      col_off = 0;
      row_off = d->res_row_off;
    } else {
      view_rows = d->per_sample_tiles ? (uint64_t)d->res_rows_per_sample / step
                                      : (uint64_t)d->out_rows;
      col_off = (uint64_t)d->res_row_off * ld;
      row_off = 0;
    }
    const uint64_t inner = step * ld;
    const uint64_t sample_stride = d->per_sample_tiles ? (uint64_t)d->res_rows_per_sample * ld
                                                       : view_rows * inner;
    uint64_t r_plane = (uint64_t)d->res_plane_stride;
    if (g.res_planes == 1 || r_plane == 0) r_plane = r_samples * sample_stride;
    if (view_rows > 0 &&
        make_map_4d(&mr, d->res, inner, view_rows, inner, r_samples, sample_stride, g.res_planes,
                    r_plane, kBlockM) == VP3D_OK) {
      g.res_tma = 1;
      g.res_tma_col_off = (int)col_off;
      g.res_tma_row_off = (int)row_off;
    }
  }
  // fused BatchNorm-backward reductions: Z rides the auxiliary TMA path with the output's geometry
  CUtensorMap& mz = L->mz;
  mz = mo;
  g.bnb = 0;
  if (d->bnb_z) {
    if (!d->out || g.out_planes != 1 || (d->res && !g.res_tma) || d->bnb_c <= 0 || d->bnb_c % 64)
      return fail(VP3D_ERR_INVALID, "conv_gemm: fused BN-backward needs a single-plane bf16 output, "
                  "a TMA-loadable residual (if any) and bnb_c % 64 == 0");
    const uint64_t o_rows = d->out_rows, o_ld = d->out_ld;
    const uint64_t o_samples = d->per_sample_tiles ? d->samples : 1;
    VP3D_TRY(make_map_4d(&mz, d->bnb_z, o_ld, o_rows, o_ld, o_samples, o_rows * o_ld, 1,
                         o_samples * o_rows * o_ld, kBlockM));
    g.bnb = 1;
    g.bnb_c = d->bnb_c;
    g.bnb_scale = d->bnb_scale; g.bnb_shift = d->bnb_shift; g.bnb_mean = d->bnb_mean;
    g.bnb_invstd = d->bnb_invstd; g.bnb_sums = d->bnb_sums;
    g.bnb_p = d->bnb_p;
    g.bnb_seed_lo = (unsigned)(d->bnb_seed & 0xFFFFFFFFu);
    g.bnb_seed_hi = (unsigned)(d->bnb_seed >> 32);
    g.bnb_layer = (unsigned)d->bnb_layer;
  }
  if (d->out_u8) {
    // the u8 output rides the auxiliary map slot (u8 launches have no BatchNorm-backward Z):
    // 64 x 32 byte boxes, unswizzled like the kernel's u8 staging tiles
    const uint64_t rows = d->out_rows, ld = d->out_u8_ld;
    const uint64_t smp = d->per_sample_tiles ? d->samples : 1;
    VP3D_TRY(make_map_4d(&mz, d->out_u8, d->n_pad, rows, ld, smp, rows * ld, 1, smp * rows * ld, 32,
                         1, 64, CU_TENSOR_MAP_SWIZZLE_NONE));
  }
  if ((i8 || d->out_u8) && d->res && !g.res_tma)
    return fail(VP3D_ERR_UNSUPPORTED, "conv_gemm: int8 / u8-output launches need a residual that "
                "TMA can load (one box of a strided row view)");
  const uint64_t w_rows = (uint64_t)w_planes * d->taps * d->n_pad;
  VP3D_TRY(make_map_2d(&mw, d->w, d->k_per_tap, w_rows, block_n, i8 ? 1 : 2));
  L->mw64 = mw;
  if (block_n == 128) VP3D_TRY(make_map_2d(&L->mw64, d->w, d->k_per_tap, w_rows, 64, i8 ? 1 : 2));
  return VP3D_OK;
}

int run_conv(const vp3d_conv_desc* d, cudaStream_t stream) {
  ConvLaunch L;
  VP3D_TRY(prepare_conv(d, &L));
  if (L.empty) return VP3D_OK;
  CUDA_TRY(launch_conv_gemm(L.ma, L.mw, L.mw64, L.mo, L.mr, L.mz, L.g, L.block_n, L.sms, stream));
  return VP3D_OK;
}

static int conv_instance(const vp3d_conv_desc* d, int* key) {
  if (!key) return fail(VP3D_ERR_INVALID, "conv_gemm_instance: null key");
  ConvLaunch L;
  VP3D_TRY(prepare_conv(d, &L));
  if (L.empty) return fail(VP3D_ERR_INVALID, "conv_gemm_instance: no output rows, nothing is launched");
  if (!conv_gemm_instance(L.g, L.block_n, L.sms, key))
    return fail(VP3D_ERR_UNSUPPORTED, "conv_gemm_instance: the selected instance is not compiled");
  return VP3D_OK;
}

// ------------------------------------------------------------------ plan
int plan_alloc(vp3d_plan* p, void** out, size_t bytes) {
  void* q = nullptr;
  CUDA_TRY(cudaMalloc(&q, bytes));
  p->allocs.push_back(q);
  *out = q;
  return VP3D_OK;
}

// K per tap of layers_conv[l]'s forward pack: C, or in an int8 block C padded to the 128-element
// k-blocks of the u8 x s8 GEMM (zero weights)
static int conv_k_pad(const vp3d_plan* p, int l) {
  return block_is_int8(p, l / 2 + 1) ? round_up(p->C, kBlockK8) : p->C;
}

// Device bytes allocated for pack k: a block conv of an int8 plan holds either format, whichever
// vp3d_set_int8_blocks picks for its block; the 16-bit pack (K per tap C, 2 bytes) is the larger.
static size_t pack_capacity(const vp3d_plan* p, const PackedConv& k) {
  const size_t b = pack_bytes(p, k);
  if (!p->int8 || k.transposed || k.src < 0) return b;
  const size_t b16 = (size_t)k.stored_taps * k.n_pad * p->C * sizeof(__nv_bfloat16);
  return b > b16 ? b : b16;
}

// The pack table of a plan whose shape fields are set (internal.cuh, PackedConv).
static void plan_packs(vp3d_plan* p) {
  auto add = [p](int src, int c_out, int c_in, int taps, bool transposed, bool merged, int n_pad,
                 int k_pad) {
    PackedConv& k = p->packs[p->n_packs++];
    k.src = src; k.c_out = c_out; k.c_in = c_in; k.taps = taps;
    k.transposed = transposed; k.merged = merged;
    k.stored_taps = merged ? 1 : taps; k.n_pad = n_pad; k.k_pad = k_pad;
    return &k;
  };
  const int C = p->C, cr = p->c_real, w0 = p->cfg.filter_widths[0];
  auto layer_taps = [p](int l) { return l % 2 == 0 ? p->taps[l / 2 + 1] : 1; };
  p->expand_dil = add(kSrcExpand, cr, p->c_in_raw, w0, false, false, C, p->c_in_pad);
  p->expand_flat = add(kSrcExpand, cr, p->c_in_raw, w0, false, true, C, p->k0_pad);
  for (int l = 0; l < 2 * p->nb; ++l)
    p->conv[l] = add(l, cr, cr, layer_taps(l), false, false, C, conv_k_pad(p, l));
  p->shrink = add(kSrcShrink, p->c_out_raw, cr, 1, false, false, p->c_out_pad, C);
  for (int l = 0; l < 2 * p->nb; ++l) p->conv_t[l] = add(l, cr, cr, layer_taps(l), true, false, C, C);
  // K of the shrink data gradient (dY's columns) padded to 128: also the row pitch of the padded dY
  // in the training workspace
  p->shrink_t = add(kSrcShrink, p->c_out_raw, cr, 1, true, false, C, round_up(p->c_out_raw, 128));
  // the input gradient in the plan's own layout: tap-merged rows (tap*c_in + ci) for the strided model
  p->expand_t = p->cfg.variant == VP3D_VARIANT_STRIDED
                    ? add(kSrcExpand, cr, p->c_in_raw, w0, true, true, p->k0_pad, C)
                    : add(kSrcExpand, cr, p->c_in_raw, w0, true, false, p->c_in_pad, C);
}

// the fp32 weight pack k is made from, an error if w lacks it
static int pack_source(const PackedConv& k, const vp3d_weights* w, const float** src) {
  *src = conv_weight(w, k.src);
  if (!*src && k.src >= 0) return fail(VP3D_ERR_INVALID, "set_weights: missing layers_conv.%d", k.src);
  if (!*src)
    return fail(VP3D_ERR_INVALID, "set_weights: missing %s",
                k.src == kSrcExpand ? "expand_conv.weight" : "shrink.weight");
  return VP3D_OK;
}

int pack_weight(const vp3d_plan* p, const PackedConv& k, const vp3d_weights* w, cudaStream_t stream,
                const PackedConv* fwd) {
  const float* src = nullptr;
  VP3D_TRY(pack_source(k, w, &src));
  if (pack_is_s8(p, k))
    CUDA_TRY(launch_pack_conv_weight_s8(src, reinterpret_cast<int8_t*>(k.w), k.w_scale, k.c_out,
                                        k.c_in, k.taps, k.n_pad, k.k_pad, stream));
  else if (k.transposed)
    CUDA_TRY(launch_pack_conv_weight_t(src, k.w, p->planes, k.c_out, k.c_in, k.taps, k.n_pad, k.k_pad,
                                       stream, fwd ? fwd->w : nullptr, fwd ? fwd->n_pad : 0,
                                       fwd ? fwd->k_pad : 0, k.merged));
  else
    CUDA_TRY(launch_pack_conv_weight(src, k.w, p->planes, k.c_out, k.c_in, k.taps, k.n_pad, k.k_pad,
                                     k.merged, stream, p->f16));
  return VP3D_OK;
}

int pack_expand_forward(const vp3d_plan* p, const vp3d_weights* w, cudaStream_t stream) {
  VP3D_TRY(pack_weight(p, *p->expand_dil, w, stream));
  return pack_weight(p, *p->expand_flat, w, stream);
}

void use_pack(vp3d_conv_desc* d, const PackedConv& k) {
  d->w = k.w;
  d->taps = k.stored_taps;
  d->k_per_tap = k.k_pad;
  d->n_pad = k.n_pad;
}

}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) int vp3d_version(void) { return VP3D_VERSION; }
extern "C" __attribute__((visibility("default"))) int vp3d_set_pdl(int on) {
  vp3d::conv_gemm_set_pdl(on);
  return VP3D_OK;
}
extern "C" __attribute__((visibility("default"))) int vp3d_set_sm_limit(int n) {
  if (n != 0 && n < 2) return fail(VP3D_ERR_INVALID, "set_sm_limit: need 0 (no limit) or >= 2 SMs");
  vp3d::g_sm_limit = n;
  return VP3D_OK;
}
extern "C" __attribute__((visibility("default"))) const char* vp3d_last_error(void) { return g_err; }
#ifdef VP3D_TIMELINE
// debug build only (`make dbg`, tools/timeline.py): device buffer of [max_launches][2][32][2] u64
extern "C" __attribute__((visibility("default"))) int vp3d_debug_set_timeline(unsigned long long* buf,
                                                                                int max_launches) {
  vp3d::conv_gemm_debug_set_timeline(buf, max_launches);
  return VP3D_OK;
}
#endif

extern "C" __attribute__((visibility("default"))) int vp3d_plan_create(const vp3d_config* cfg, vp3d_plan** out_plan) {
  if (!cfg || !out_plan) return fail(VP3D_ERR_INVALID, "plan_create: null argument");
  if (cfg->num_widths < 1 || cfg->num_widths > VP3D_MAX_WIDTHS)
    return fail(VP3D_ERR_INVALID, "plan_create: len(filter_widths) must be in [1, %d]",
                VP3D_MAX_WIDTHS);
  for (int i = 0; i < cfg->num_widths; ++i)
    if (cfg->filter_widths[i] < 1 || cfg->filter_widths[i] % 2 == 0)
      return fail(VP3D_ERR_INVALID, "Only odd filter widths are supported");  // model.py:20-21
  if (cfg->num_joints_in < 1 || cfg->in_features < 1 || cfg->num_joints_out < 1)
    return fail(VP3D_ERR_INVALID, "plan_create: joint / feature counts must be positive");
  if (cfg->channels < 1)
    return fail(VP3D_ERR_INVALID, "channels must be positive (got %d)", cfg->channels);
  if (cfg->precision < VP3D_PRECISION_BF16 || cfg->precision > VP3D_PRECISION_INT8)
    return fail(VP3D_ERR_INVALID, "plan_create: unknown precision %d", cfg->precision);
  if (cfg->variant != VP3D_VARIANT_DILATED && cfg->variant != VP3D_VARIANT_STRIDED)
    return fail(VP3D_ERR_INVALID, "plan_create: unknown variant %d", cfg->variant);
  if (cfg->variant == VP3D_VARIANT_STRIDED && cfg->dense)
    return fail(VP3D_ERR_INVALID, "dense=True only exists for TemporalModel");
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaFree(0) != cudaSuccess)
    return fail(VP3D_ERR_CUDA, "no usable CUDA device: %s", cudaGetErrorString(cudaGetLastError()));

  vp3d_plan* p = new vp3d_plan();
  p->cfg = *cfg;
  p->nb = cfg->num_widths - 1;
  // any `channels` (the reference takes any -ch, arguments.py:47): activations and packed weights
  // are laid out with the channel count padded to 64; padding channels carry zero weights and a
  // zero affine, so they stay exactly zero through every layer
  p->c_real = cfg->channels;
  p->C = round_up(cfg->channels, 64);
  p->c_in_raw = cfg->num_joints_in * cfg->in_features;
  p->c_out_raw = cfg->num_joints_out * 3;
  p->c_in_pad = round_up(p->c_in_raw, 64);
  p->k0_pad = round_up(p->c_in_raw * cfg->filter_widths[0], 64);
  p->c_out_pad = round_up(p->c_out_raw, 64);
  p->int8 = cfg->precision == VP3D_PRECISION_INT8 ? 1 : 0;
  p->f16 = (cfg->precision == VP3D_PRECISION_FP16 || p->int8) ? 1 : 0;
  p->int8_mask = p->int8 ? (1u << p->nb) - 1u : 0u;
  p->planes = (cfg->precision == VP3D_PRECISION_BF16 || p->f16) ? 1 : 2;
  // model.py:31, 107-121 / :172-184
  p->pad[0] = cfg->filter_widths[0] / 2;
  p->shift_dil[0] = p->shift_str[0] = cfg->causal ? cfg->filter_widths[0] / 2 : 0;
  p->dilation[0] = 1;
  p->taps[0] = cfg->filter_widths[0];
  int next_dilation = cfg->filter_widths[0];
  for (int i = 1; i < cfg->num_widths; ++i) {
    const int w = cfg->filter_widths[i];
    p->pad[i] = (w - 1) * next_dilation / 2;
    p->shift_dil[i] = cfg->causal ? (w / 2) * next_dilation : 0;
    p->shift_str[i] = cfg->causal ? (w / 2) : 0;
    p->dilation[i] = cfg->dense ? 1 : next_dilation;
    p->taps[i] = cfg->dense ? 2 * p->pad[i] + 1 : w;
    next_dilation *= w;
  }

  // int8: every int32 sum is bounded by K * 255 * 127 (K = taps * channels); reject a plan where
  // that could overflow (only the dense ablation's widest blocks reach it)
  for (int i = 1; p->int8 && i <= p->nb; ++i) {
    if ((long long)p->taps[i] * p->c_real * 255 * 127 >= (1ll << 31)) {
      const int taps = p->taps[i];
      vp3d_plan_destroy(p);
      return fail(VP3D_ERR_UNSUPPORTED, "int8: block %d has K = %d x %d, whose int32 sums could "
                  "overflow (K * 255 * 127 >= 2^31)", i, taps, cfg->channels);
    }
  }

  plan_packs(p);

  int st = VP3D_OK;
  do {
    for (int i = 0; i < p->n_packs && !st; ++i)
      if (!p->packs[i].transposed)
        st = plan_alloc(p, reinterpret_cast<void**>(&p->packs[i].w), pack_capacity(p, p->packs[i]));
    if (st) break;
    // affine vectors: expand + 2*nb layers (C each) + shrink (c_out_pad)
    float* aff = nullptr;
    const size_t n_aff = (size_t)(2 * p->nb + 1) * 2 * p->C + 2 * p->c_out_pad;
    if ((st = plan_alloc(p, reinterpret_cast<void**>(&aff), n_aff * sizeof(float)))) break;
    p->expand_dil->scale = p->expand_flat->scale = aff;
    p->expand_dil->shift = p->expand_flat->shift = aff + p->C;
    for (int l = 0; l < 2 * p->nb; ++l) {
      p->conv[l]->scale = aff + (size_t)(l + 1) * 2 * p->C;
      p->conv[l]->shift = p->conv[l]->scale + p->C;
    }
    p->shrink->scale = aff + (size_t)(2 * p->nb + 1) * 2 * p->C;
    p->shrink->shift = p->shrink->scale + p->c_out_pad;
    if (p->int8 && p->nb > 0) {
      float* q = nullptr;
      if ((st = plan_alloc(p, reinterpret_cast<void**>(&q), (size_t)4 * p->nb * p->C * sizeof(float))))
        break;
      for (int l = 0; l < 2 * p->nb; ++l) {
        p->conv[l]->w_scale = q + (size_t)l * 2 * p->C;
        p->conv[l]->q_scale = p->conv[l]->w_scale + p->C;
      }
    }
  } while (0);
  if (st) {
    vp3d_plan_destroy(p);
    return st;
  }
  *out_plan = p;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) void vp3d_plan_destroy(vp3d_plan* p) {
  if (!p) return;
  for (void* q : p->allocs) cudaFree(q);
  for (cudaEvent_t e : p->prof_events) if (e) cudaEventDestroy(e);
  if (p->train) train_state_destroy(p->train);
  delete p;
}

extern "C" __attribute__((visibility("default"))) int vp3d_receptive_field(const vp3d_plan* p) {
  if (!p) return fail(VP3D_ERR_INVALID, "null plan");
  int frames = 0;
  for (int i = 0; i < p->cfg.num_widths; ++i) frames += p->pad[i];
  return 1 + 2 * frames;
}

extern "C" __attribute__((visibility("default"))) int vp3d_total_causal_shift(const vp3d_plan* p) {
  if (!p) return fail(VP3D_ERR_INVALID, "null plan");
  const int* cs = p->cfg.variant == VP3D_VARIANT_STRIDED ? p->shift_str : p->shift_dil;
  int frames = cs[0];
  int next_dilation = p->cfg.filter_widths[0];
  for (int i = 1; i < p->cfg.num_widths; ++i) {
    frames += cs[i] * next_dilation;
    next_dilation *= p->cfg.filter_widths[i];
  }
  return frames;
}

extern "C" __attribute__((visibility("default"))) int vp3d_set_weights(vp3d_plan* p, const vp3d_weights* w, int what, void* stream_) {
  if (!p || !w) return fail(VP3D_ERR_INVALID, "set_weights: null argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (what & VP3D_PACK_CONV) {
    const float* src = nullptr;
    for (int i = 0; i < p->n_packs; ++i) VP3D_TRY(pack_source(p->packs[i], w, &src));
    VP3D_TRY(pack_expand_forward(p, w, stream));
    // with VP3D_PACK_CONV_T the transposed-pack kernels below also write the other forward packs
    for (int i = 0; i < p->n_packs && !(what & VP3D_PACK_CONV_T); ++i)
      if (!p->packs[i].transposed && p->packs[i].src != kSrcExpand)
        VP3D_TRY(pack_weight(p, p->packs[i], w, stream));
    p->conv_packed = true;
  }
  if (what & VP3D_PACK_BN_EVAL) {
    const float eps = 1e-5f;  // nn.BatchNorm1d default, model.py:32
    for (int k = 0; k < 4; ++k)
      if (!w->expand_bn[k]) return fail(VP3D_ERR_INVALID, "set_weights: missing expand_bn");
    if (!w->shrink_bias) return fail(VP3D_ERR_INVALID, "set_weights: missing shrink.bias");
    CUDA_TRY(launch_bn_fold(w->expand_bn[0], w->expand_bn[1], w->expand_bn[2], w->expand_bn[3], eps,
                            p->expand_dil->scale, p->expand_dil->shift, p->c_real, p->C, stream));
    for (int l = 0; l < 2 * p->nb; ++l) {
      for (int k = 0; k < 4; ++k)
        if (!w->layers_bn[l][k]) return fail(VP3D_ERR_INVALID, "set_weights: missing layers_bn.%d", l);
      CUDA_TRY(launch_bn_fold(w->layers_bn[l][0], w->layers_bn[l][1], w->layers_bn[l][2],
                              w->layers_bn[l][3], eps, p->conv[l]->scale, p->conv[l]->shift,
                              p->c_real, p->C, stream));
    }
    CUDA_TRY(launch_bias_affine(w->shrink_bias, p->shrink->scale, p->shrink->shift, p->c_out_raw,
                                p->c_out_pad, stream));
    p->bn_packed = true;
  }
  if (p->int8 && (what & (VP3D_PACK_CONV | VP3D_PACK_BN_EVAL))) {
    // the int8 affine: the BatchNorm scale times both dequantisation factors
    p->int8_folded = false;
    if (p->int8_scales && p->conv_packed && p->bn_packed) {
      for (int l = 0; l < 2 * p->nb; ++l)
        if (block_is_int8(p, l / 2 + 1))
          CUDA_TRY(launch_int8_fold(p->conv[l]->scale, p->conv[l]->w_scale, p->act_scale[l],
                                    p->conv[l]->q_scale, p->C, stream));
      p->int8_folded = true;
    }
  }
  if ((what & VP3D_PACK_CONV_T) && p->f16)
    return fail(VP3D_ERR_UNSUPPORTED, "fp16 plans are inference-only (train with bf16 / bf16x3)");
  if (what & VP3D_PACK_CONV_T)
    VP3D_TRY(train_pack_transposed(p, w, stream, (what & VP3D_PACK_CONV) != 0));
  if ((what & VP3D_PACK_EXPAND_T) && p->f16)
    return fail(VP3D_ERR_UNSUPPORTED, "fp16 plans are inference-only (train with bf16 / bf16x3)");
  if (what & VP3D_PACK_EXPAND_T) VP3D_TRY(train_pack_expand_t(p, w, stream));
  return VP3D_OK;
}

// ------------------------------------------------------------------ eval schedules
// The strided ("flat") schedule is used for TemporalModelOptimized1f and for TemporalModel in eval
// mode when the input is exactly one receptive field long: with running statistics every output
// frame depends only on its own dependency cone, whose rows are exactly the stride-w rows
// Optimized1f computes (the reference states the weights are interchangeable, model.py:146-148).
namespace vp3d {
bool use_strided(const vp3d_plan* p, int T) {
  if (p->cfg.variant == VP3D_VARIANT_STRIDED) return true;
  return !p->cfg.dense && T == vp3d_receptive_field(p);
}

// rows per sample after each stage: L[0] = rows out of expand, L[i] = rows out of block i
int layer_rows(const vp3d_plan* p, int T, bool strided, int* L) {
  const int* fw = p->cfg.filter_widths;
  if (strided) {
    L[0] = T / fw[0];  // Conv1d(stride=w, kernel=w): floor((T - w)/w) + 1
    for (int i = 1; i <= p->nb; ++i) L[i] = L[i - 1] / fw[i];
    // (when T is not exactly one receptive field the floors drop trailing frames layer by layer;
    // strided_trim() below tells which rows the output actually depends on)
  } else {
    L[0] = T - (fw[0] - 1);
    for (int i = 1; i <= p->nb; ++i) L[i] = L[i - 1] - 2 * p->pad[i];
  }
  for (int i = 0; i <= p->nb; ++i)
    if (L[i] < 1) return 0;
  return L[p->nb];
}

}  // namespace vp3d

namespace vp3d {
// Strided model on an input whose length is not a multiple of the widths, as Conv1d(stride = w)
// handles it (model.py:167, 178, 191): every conv floors its output length, i.e. ignores trailing
// frames, and the residual slice x[:, :, shift + w//2 :: w] must come out with the conv's length
// (otherwise the reference's `res + x` raises a size mismatch -- reproduced here as an error).
// On success L[] is trimmed to the rows the output depends on: L[i-1] = w_i * L[i], so that the
// row-region (tap-major) schedule applies; in eval mode (running statistics) dropping the unused
// rows changes nothing.  Returns VP3D_OK / an error status with the reference's message.
int strided_trim(const vp3d_plan* p, int* L) {
  const int* fw = p->cfg.filter_widths;
  for (int i = 1; i <= p->nb; ++i) {
    const int first = p->shift_str[i] + fw[i] / 2;
    const int res_len = L[i - 1] > first ? (L[i - 1] - first + fw[i] - 1) / fw[i] : 0;
    if (res_len != L[i])
      return fail(VP3D_ERR_INVALID, "The size of tensor a (%d) must match the size of tensor b (%d) "
                  "at non-singleton dimension 2 (residual slice of block %d on %d frames, width %d)",
                  res_len, L[i], i, L[i - 1], fw[i]);
  }
  for (int i = p->nb; i >= 1; --i) L[i - 1] = fw[i] * L[i];
  return VP3D_OK;
}
}  // namespace vp3d

extern "C" __attribute__((visibility("default"))) int vp3d_output_frames(const vp3d_plan* p, int T) {
  if (!p) return fail(VP3D_ERR_INVALID, "null plan");
  int L[VP3D_MAX_WIDTHS];
  return layer_rows(p, T, p->cfg.variant == VP3D_VARIANT_STRIDED, L);
}

struct WsLayout {
  size_t a0 = 0, x0 = 0, x1 = 0, h = 0, q = 0, yf = 0, total = 0;
  size_t a0_plane = 0, x_plane = 0, h_plane = 0;  // elements per plane
};

// y_rows > 0 (vp3d_forward_clips only): an fp32 buffer of y_rows shrink rows at the end
static WsLayout ws_layout(const vp3d_plan* p, int N, int T, bool strided, const int* L,
                          size_t y_rows = 0) {
  WsLayout w;
  const size_t a0_rows = strided ? (size_t)N * L[0] : (size_t)N * T;
  const size_t a0_ld = strided ? p->k0_pad : p->c_in_pad;
  w.a0_plane = a0_rows * a0_ld;
  w.x_plane = (size_t)N * L[0] * p->C;
  w.h_plane = p->nb > 0 ? (size_t)N * L[1] * p->C : 0;
  Arena a{1024};
  w.a0 = a.take(w.a0_plane * p->planes * 2);
  w.x0 = a.take(w.x_plane * p->planes * 2);
  w.x1 = a.take(w.h_plane * p->planes * 2);  // block outputs are <= L[1] rows
  w.h = a.take(w.h_plane * p->planes * 2);
  // int8: H is stored as u8 only (in the fp16 H buffer), and one u8 buffer holds Q_i: block i + 1's
  // first conv reads it before its 1x1 conv writes Q_{i+1} (the next kernel of the stream)
  if (p->int8) w.q = a.take(w.x_plane);
  if (y_rows) w.yf = a.take(y_rows * p->c_out_raw * sizeof(float));
  w.total = a.total();
  return w;
}

extern "C" __attribute__((visibility("default"))) size_t vp3d_workspace_bytes(const vp3d_plan* p, int N, int T) {
  if (!p || N < 1) return 0;
  int L[VP3D_MAX_WIDTHS];
  const bool strided = use_strided(p, T);
  if (!layer_rows(p, T, strided, L)) return 0;
  if (strided && strided_trim(p, L) != VP3D_OK) return 0;
  return ws_layout(p, N, T, strided, L).total;
}

// ------------------------------------------------------------------ host-buffer staging
HostStaging::~HostStaging() {
  if (stream) cudaStreamDestroy(stream);
  if (copy_stream) cudaStreamDestroy(copy_stream);
  for (cudaEvent_t e : copy_events) if (e) cudaEventDestroy(e);
  for (Slot& s : slots) {
    if (s.copied) cudaEventDestroy(s.copied);
    if (s.done) cudaEventDestroy(s.done);
  }
}

// create *s (non-blocking) / *e on first use
static int lazy_stream(cudaStream_t* s) {
  if (!*s) CUDA_TRY(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
  return VP3D_OK;
}
static int lazy_event(cudaEvent_t* e, unsigned flags = cudaEventDisableTiming) {
  if (!*e) CUDA_TRY(cudaEventCreateWithFlags(e, flags));
  return VP3D_OK;
}

// measurement hook: record an event pair around launch number p->prof_launch
static int prof_event(vp3d_plan* p, int launch, bool begin, cudaStream_t stream) {
  if (p->prof_launch < 0 || launch != p->prof_launch) return VP3D_OK;
  const size_t idx = p->prof_used + (begin ? 0 : 1);
  if (p->prof_events.size() <= idx) p->prof_events.resize(idx + 1, nullptr);
  VP3D_TRY(lazy_event(&p->prof_events[idx], cudaEventDefault));
  CUDA_TRY(cudaEventRecord(p->prof_events[idx], stream));
  if (!begin) p->prof_used += 2;
  return VP3D_OK;
}

// expand (model.py:127 / :188), the residual blocks (:129-135 / :190-194), shrink (:137 / :196)
// writing (N, T_out, J_out, 3) directly (fuses :74-75)
int vp3d::run_infer_chain(vp3d_plan* p, const InferChain& c, cudaStream_t stream, int* launches) {
  const int C = p->C;
  // conv k + BN + ReLU of stage i in the chain's tiling
  auto conv = [&](int i, const PackedConv& k, const __nv_bfloat16* a, long long a_plane, int a_rows,
                  int a_ld) {
    vp3d_conv_desc d = conv_desc(p, c.precision[i]);
    d.a = a; d.a_plane_stride = a_plane; d.samples = c.samples; d.a_rows = a_rows; d.a_ld = a_ld;
    use_pack(&d, k);
    d.per_sample_tiles = c.per_sample_tiles; d.out_rows = c.st[i].out_rows;
    d.scale = k.scale; d.shift = k.shift; d.relu = 1;
    d.out_ld = C;
    return d;
  };
  auto launch = [&](const vp3d_conv_desc& d) -> int {
    if (c.profile) VP3D_TRY(prof_event(p, *launches, true, stream));
    VP3D_TRY(run_conv(&d, stream));
    if (c.profile) VP3D_TRY(prof_event(p, *launches, false, stream));
    ++*launches;
    return VP3D_OK;
  };
  // calibration: fold the maximum of a stored fp16 plane into amax[l], or add its real channels
  // to the histogram of layer l
  auto amax = [&](int l, const __nv_bfloat16* x, long long n) -> int {
    if (c.amax) CUDA_TRY(launch_amax_f16(x, n, c.amax + l, stream));
    if (c.hist)
      CUDA_TRY(launch_hist_f16(x, n / C, C, p->c_real, c.hist + (size_t)l * kHistBins,
                               c.hist + (size_t)2 * p->nb * kHistBins + l, num_sms(), stream));
    return VP3D_OK;
  };
  for (int i = 0; i < c.stages; ++i) {
    const ChainStage& s = c.st[i];
    // the planes of a stage's input lie where its producer wrote them, and must hold its rows
    const long long in_plane = i == 0 ? c.in_plane : c.st[i - 1].out_plane;
    const int in_ld = i == 0 ? c.expand->k_pad : C;
    if (in_plane < (long long)c.samples * s.in_rows * in_ld)
      return fail(VP3D_ERR_STATE, "internal: activation plane mismatch in block %d", i);
    if (i > 0 && c.precision[i] == VP3D_PRECISION_INT8) {
      // u8 x s8 block: Q_{i-1} -> H (u8 only) -> X_i (fp16, residual X_{i-1}) [+ Q_i]
      const PackedConv& k1 = *p->conv[2 * (i - 1)];
      const PackedConv& k2 = *p->conv[2 * (i - 1) + 1];
      if (!s.q_in || !c.hq) return fail(VP3D_ERR_STATE, "internal: int8 block %d has no u8 input", i);
      if (s.q_in_bytes < (long long)c.samples * s.in_rows * C)
        return fail(VP3D_ERR_STATE, "internal: u8 activation plane mismatch in block %d", i);
      vp3d_conv_desc d = conv(i, k1, nullptr, 0, s.in_rows, C);
      d.a = s.q_in;
      d.tap_row_step = s.tap_row_step;
      d.scale = k1.q_scale;
      d.out_u8 = c.hq; d.out_u8_ld = C; d.out_u8_inv_scale = p->act_inv[2 * (i - 1) + 1];
      VP3D_TRY(launch(d));
      d = conv(i, k2, nullptr, 0, s.out_rows, C);
      d.a = c.hq;
      d.scale = k2.q_scale;
      d.res = s.in; d.res_plane_stride = in_plane; d.res_ld = C; d.res_row_step = 1;
      d.res_row_off = s.res_row_off;
      d.res_rows_per_sample = c.per_sample_tiles ? s.in_rows : 0;
      d.out = s.out; d.out_plane_stride = s.out_plane;
      if (s.q_out) { d.out_u8 = s.q_out; d.out_u8_ld = C; d.out_u8_inv_scale = p->act_inv[2 * i]; }
      VP3D_TRY(launch(d));
      continue;
    }
    // the k-tap conv: the expand conv writes X_0, a block's first conv H
    vp3d_conv_desc d = conv(i, i == 0 ? *c.expand : *p->conv[2 * (i - 1)], s.in, in_plane,
                            s.in_rows, in_ld);
    d.tap_row_step = s.tap_row_step;
    if (i > 0) {
      // H only needs a lo plane when its consumer is split-bf16
      const int h_planes = c.precision[i] == VP3D_PRECISION_BF16X3 ? 2 : 1;
      d.out_planes = h_planes; d.out = c.h; d.out_plane_stride = s.h_plane;
      VP3D_TRY(launch(d));
      VP3D_TRY(amax(2 * (i - 1) + 1, c.h, (long long)c.samples * s.out_rows * C));
      // second conv: 1x1 + the block input's centre (causal: newest) tap as residual; with
      // per-sample tiles the residual rows of a tile are then one TMA box of the block input
      d = conv(i, *p->conv[2 * (i - 1) + 1], c.h, s.h_plane, s.out_rows, C);
      d.a_planes = h_planes;
      d.res = s.in; d.res_plane_stride = in_plane; d.res_ld = C; d.res_row_step = 1;
      d.res_row_off = s.res_row_off;
      d.res_rows_per_sample = c.per_sample_tiles ? s.in_rows : 0;
    }
    d.out = s.out; d.out_plane_stride = s.out_plane;
    d.lo_row_begin = s.lo_row_begin; d.lo_row_end = s.lo_row_end;
    // Q_i: the expand's epilogue writes Q_0 from its fp32 value; no GEMM writes fp16 + residual +
    // u8, so after an fp16 block a pass of its own quantises the stored fp16 X_i
    if (s.q_out && i == 0) {
      d.out_u8 = s.q_out; d.out_u8_ld = C; d.out_u8_inv_scale = p->act_inv[0];
    }
    VP3D_TRY(launch(d));
    if (s.q_out && i > 0) {
      if (c.profile) VP3D_TRY(prof_event(p, *launches, true, stream));
      CUDA_TRY(launch_quantize_u8(s.out, s.q_out, (long long)c.samples * s.out_rows, C, p->c_real,
                                  p->act_inv[2 * i], num_sms(), stream));
      if (c.profile) VP3D_TRY(prof_event(p, *launches, false, stream));
      ++*launches;
    }
    if (i < p->nb) VP3D_TRY(amax(2 * i, s.out, (long long)c.samples * s.out_rows * C));
  }
  if (!c.y) return VP3D_OK;
  // shrink: one flat GEMM over all rows of the last stage, the bias as its affine, fp32 out
  const ChainStage& s = c.st[c.stages - 1];
  vp3d_conv_desc d = conv_desc(p, c.precision[p->nb + 1]);
  d.a = s.out; d.a_plane_stride = s.out_plane; d.a_ld = C;
  d.a_rows = d.out_rows = (c.per_sample_tiles ? c.samples : 1) * s.out_rows;
  use_pack(&d, *p->shrink);
  d.scale = p->shrink->scale; d.shift = p->shrink->shift;
  d.out_f32 = c.y; d.out_f32_ld = p->c_out_raw; d.n_valid = p->c_out_raw;
  return launch(d);
}

// The two offline geometries, over the N * L[i] rows of stage i.
//
// Strided schedule: every activation is kept in tap-major row order (pack.cuh), so the w taps of
// block i are w contiguous row regions of R = N * L[i] rows: tap k of output row j is row k * R + j
// of the block input, and the residual of the block is its centre (or, causal, last) region.
static void strided_chain(const vp3d_plan* p, int N, const int* L, InferChain* c) {
  c->samples = 1;
  c->per_sample_tiles = 0;
  c->expand = p->expand_flat;
  for (int i = 0; i <= p->nb; ++i) {
    ChainStage& s = c->st[i];
    const int R = N * L[i];
    s.in_rows = i == 0 ? R : N * L[i - 1];
    s.out_rows = R;
    s.tap_row_step = i == 0 ? 0 : R;
    s.res_row_off = (p->cfg.filter_widths[i] / 2 + p->shift_str[i]) * R;
  }
}

// Dilated schedule: every GEMM but shrink tiles per sample, the 1x1 convs too; taps are rows
// `dilation` apart and the residual starts pad + shift rows into the sample.
static void dilated_chain(const vp3d_plan* p, int N, int T, const int* L, InferChain* c) {
  c->samples = N;
  c->per_sample_tiles = 1;
  c->expand = p->expand_dil;
  for (int i = 0; i <= p->nb; ++i) {
    ChainStage& s = c->st[i];
    s.in_rows = i == 0 ? T : L[i - 1];
    s.out_rows = L[i];
    s.tap_row_step = p->dilation[i];
    s.res_row_off = p->pad[i] + p->shift_dil[i];
  }
}

// What every offline chain needs of the plan: packed weights and, in int8, folded scales.
static int eval_ready(const vp3d_plan* p, const char* what) {
  if (!p->conv_packed || !p->bn_packed)
    return fail(VP3D_ERR_STATE, "%s: vp3d_set_weights has not been called", what);
  if (p->int8 && !p->int8_folded)
    return fail(VP3D_ERR_STATE, "%s: int8 plan without activation scales (call "
                "vp3d_set_int8_scales, then vp3d_set_weights)", what);
  return VP3D_OK;
}

// The offline chain in workspace layout wl over N samples with L[i] rows out of stage i: X_i
// alternates between the workspace's two X buffers, its planes and H's packed to the rows of stage
// i; and the per-layer operand precision.  The caller adds the geometry (strided_chain /
// dilated_chain), the shrink output and the measurement hooks.
static void eval_chain(const vp3d_plan* p, const WsLayout& wl, uint8_t* base, int N, const int* L,
                       InferChain* out) {
  const int* fw = p->cfg.filter_widths;
  const int C = p->C;
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(base + off); };
  InferChain& c = *out;
  memset(&c, 0, sizeof(c));
  c.stages = p->nb + 1;
  c.in_plane = (long long)wl.a0_plane;
  c.h = bf(wl.h);
  if (p->int8) c.hq = base + wl.h;
  for (int i = 0; i <= p->nb; ++i) {
    ChainStage& s = c.st[i];
    s.in = i == 0 ? bf(wl.a0) : c.st[i - 1].out;
    s.out = bf(i % 2 ? wl.x1 : wl.x0);
    s.out_plane = s.h_plane = (long long)N * L[i] * C;
    // Q_i exists where block i + 1 runs u8 x s8
    if (i < p->nb && block_is_int8(p, i + 1)) s.q_out = base + wl.q;
    if (i > 0) {
      s.q_in = c.st[i - 1].q_out;
      s.q_in_bytes = (long long)wl.x_plane;
    }
  }

  // Per-layer operand precision.  index 0 = expand, 1..nb = residual blocks, nb+1 = shrink.
  //   bf16   : every GEMM single-plane bf16.
  //   bf16x3 : every GEMM split-bf16 (3 MMAs per product).
  //   mixed  : the residual stream X keeps hi+lo planes (skip path exact); expand and shrink run
  //            split-bf16 (they carry most of the bf16 error, tools/precision_study.py),
  //            residual blocks run plain bf16 on the hi plane unless they hold < 0.5% of the
  //            forward FLOPs (negligible even at the narrow-tile rate of such layers).
  //   int8   : layer_precision: the residual blocks of int8_mask u8 x s8; expand, shrink and the
  //            other blocks fp16.
  {
    double fl[VP3D_MAX_WIDTHS + 1], total = 0.0;
    fl[0] = (double)N * L[0] * p->c_in_raw * fw[0] * C;
    for (int i = 1; i <= p->nb; ++i) fl[i] = (double)N * L[i] * (p->taps[i] + 1.0) * C * C;
    fl[p->nb + 1] = (double)N * L[p->nb] * C * p->c_out_raw;
    for (int i = 0; i <= p->nb + 1; ++i) total += fl[i];
    for (int i = 0; i <= p->nb + 1; ++i) {
      const bool x3 = i == 0 || i == p->nb + 1 || fl[i] < 0.005 * total;
      c.precision[i] = p->cfg.precision == VP3D_PRECISION_MIXED
                           ? (x3 ? VP3D_PRECISION_BF16X3 : VP3D_PRECISION_BF16)
                           : layer_precision(p, i);
    }
  }
}

// The offline eval forward (y != null) or, with `amax` or `hist`, the calibration pass of
// vp3d_calibrate_int8 / vp3d_calibrate_int8_hist (the chain without shrink, every quantised
// activation's maximum folded into amax or its values counted into hist).
static int eval_forward(vp3d_plan* p, const float* x, float* y, int N, int T, void* ws,
                        size_t ws_bytes, cudaStream_t stream, unsigned* amax,
                        unsigned long long* hist = nullptr) {
  if (N < 1) return fail(VP3D_ERR_INVALID, "forward_eval: batch must be >= 1");
  VP3D_TRY(eval_ready(p, "forward_eval"));
  const bool strided = use_strided(p, T);
  int L[VP3D_MAX_WIDTHS];
  if (!layer_rows(p, T, strided, L))
    return fail(VP3D_ERR_INVALID, "forward_eval: sequence of %d frames is shorter than the "
                "receptive field (%d)", T, vp3d_receptive_field(p));
  if (strided) VP3D_TRY(strided_trim(p, L));   // trailing frames the strided convs ignore
  const WsLayout wl = ws_layout(p, N, T, strided, L);
  if (!ws || ws_bytes < wl.total) return fail(VP3D_ERR_WORKSPACE, "workspace too small: %zu < %zu",
                                              ws_bytes, wl.total);
  uint8_t* base = ws_base(ws);
  const int* fw = p->cfg.filter_widths;
  auto bf = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(base + off); };
  InferChain c;
  eval_chain(p, wl, base, N, L, &c);
  c.y = y;
  c.profile = true;
  c.amax = amax;
  c.hist = hist;

  // ---- input packing (model.py:127 / :188), then the chain
  int launches = 0;
  if (strided && (long long)N * L[0] > 0x7fffffffll)
    return fail(VP3D_ERR_UNSUPPORTED, "forward_eval: too many rows (%lld)", (long long)N * L[0]);
  VP3D_TRY(prof_event(p, launches, true, stream));
  if (strided) {
    PackPerm perm;
    memset(&perm, 0, sizeof(perm));
    perm.levels = p->nb;
    perm.last_rows = L[p->nb];
    for (int i = 1; i <= p->nb; ++i) {
      perm.region[i - 1] = (unsigned)((long long)N * L[i]);
      perm.width[i - 1] = fw[i];
    }
    CUDA_TRY(launch_pack_input(x, bf(wl.a0), p->planes, N, T, p->c_in_raw, L[0], fw[0], fw[0], p->k0_pad,
                               (long long)wl.a0_plane, stream, &perm, p->f16));
    strided_chain(p, N, L, &c);
    // Only the residual region of X_i needs the lo plane when block i + 1 runs plain bf16 (`mixed`)
    for (int i = 0; i < p->nb; ++i) {
      if (p->planes != 2 || c.precision[i + 1] == VP3D_PRECISION_BF16X3) continue;
      const long long r = fw[i + 1] / 2 + p->shift_str[i + 1], R = (long long)N * L[i + 1];
      c.st[i].lo_row_begin = (int)(r * R);
      c.st[i].lo_row_end = (int)((r + 1) * R);
    }
  } else {
    CUDA_TRY(launch_pack_input(x, bf(wl.a0), p->planes, N, T, p->c_in_raw, T, 1, 1, p->c_in_pad,
                               (long long)wl.a0_plane, stream, nullptr, p->f16));
    dilated_chain(p, N, T, L, &c);
  }
  VP3D_TRY(prof_event(p, launches, false, stream));
  ++launches;
  VP3D_TRY(run_infer_chain(p, c, stream, &launches));
  p->last_launches = launches;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_forward_eval(vp3d_plan* p, const float* x, float* y, int N, int T, void* ws,
                                 size_t ws_bytes, void* stream_) {
  if (!p || !x || !y) return fail(VP3D_ERR_INVALID, "forward_eval: null argument");
  return eval_forward(p, x, y, N, T, ws, ws_bytes, static_cast<cudaStream_t>(stream_), nullptr);
}

// ------------------------------------------------------------------ clips (vp3d_forward_clips)
// The checks of a clip chain's flags and row count that need no plan.
static int clips_args(long long rows, int flags, const char* what) {
  if (flags & ~VP3D_CLIPS_AUGMENT)
    return fail(VP3D_ERR_INVALID, "%s: unknown flags 0x%x", what, (unsigned)flags);
  const int copies = flags & VP3D_CLIPS_AUGMENT ? 2 : 1;
  if (rows < 1 || rows % copies)
    return fail(VP3D_ERR_INVALID, "%s: rows (%lld) must be a positive multiple of %d", what, rows,
                copies);
  // the GEMMs index rows (and round them up to whole 128-row tiles) in int32
  if (rows > 0x7fffffffLL - kBlockM)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: %lld rows overflow the chain's int32 row indices", what,
                rows);
  return VP3D_OK;
}

// Geometry of a clip chain of `rows` packed rows: the offline dilated chain as one sample of `rows`
// frames.  Fails for plans and sizes the clip chain does not cover.
static int clips_geometry(const vp3d_plan* p, long long rows, int flags, const char* what, int* L) {
  VP3D_TRY(clips_args(rows, flags, what));
  if (p->cfg.variant != VP3D_VARIANT_DILATED)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: clip chains need the TemporalModel (dilated) variant; a "
                "TemporalModelOptimized1f state_dict loads into TemporalModel unchanged", what);
  if (p->cfg.precision == VP3D_PRECISION_MIXED)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: precision 'mixed' is not supported: its per-layer split "
                "depends on the geometry", what);
  const int rf = vp3d_receptive_field(p);
  if (rows < rf || !layer_rows(p, (int)rows, false, L))
    return fail(VP3D_ERR_INVALID, "%s: %lld rows are fewer than one clip takes (%d)", what, rows, rf);
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) size_t vp3d_clips_workspace_bytes(
    const vp3d_plan* p, int64_t rows, int flags) {
  int L[VP3D_MAX_WIDTHS];
  if (!p || clips_geometry(p, rows, flags, "clips_workspace_bytes", L) != VP3D_OK) return 0;
  return ws_layout(p, 1, (int)rows, false, L, (size_t)L[p->nb]).total;
}

extern "C" __attribute__((visibility("default"))) int vp3d_forward_clips(
    vp3d_plan* p, const float* x, const int64_t* clip_first, const int32_t* clip_len, int clips,
    int64_t rows, int flags, const int32_t* kps_src, const int32_t* joints_src, float* y,
    const int64_t* y_first, void* ws, size_t ws_bytes, void* stream_) {
  const char* what = "forward_clips";
  if (!x || !clip_first || !clip_len || !y || !y_first)
    return fail(VP3D_ERR_INVALID, "%s: null x, clip table or y", what);
  if (clips < 1) return fail(VP3D_ERR_INVALID, "%s: clips must be >= 1 (got %d)", what, clips);
  const bool aug = flags & VP3D_CLIPS_AUGMENT;
  if (!aug && (kps_src || joints_src))
    return fail(VP3D_ERR_INVALID, "%s: mirror maps given without VP3D_CLIPS_AUGMENT", what);
  if (aug && !kps_src) return fail(VP3D_ERR_INVALID, "%s: VP3D_CLIPS_AUGMENT needs kps_src", what);
  VP3D_TRY(clips_args(rows, flags, what));
  const int copies = aug ? 2 : 1;
  if (!p) return fail(VP3D_ERR_INVALID, "%s: null plan", what);
  int L[VP3D_MAX_WIDTHS];
  VP3D_TRY(clips_geometry(p, rows, flags, what, L));
  const int rf = vp3d_receptive_field(p);
  if (rows < (long long)copies * clips * rf)
    return fail(VP3D_ERR_INVALID, "%s: %lld rows cannot hold %d clips (each takes at least %d x "
                "%d rows)", what, (long long)rows, clips, copies, rf);
  const int j_in = p->cfg.num_joints_in, j_out = p->cfg.num_joints_out;
  if (aug) {
    if (j_in > kClipMaxJoints || j_out > kClipMaxJoints)
      return fail(VP3D_ERR_UNSUPPORTED, "%s: augment supports up to %d joints", what,
                  kClipMaxJoints);
    VP3D_TRY(check_mirror_map(kps_src, j_in, what, "kps_src"));
    if (joints_src) VP3D_TRY(check_mirror_map(joints_src, j_out, what, "joints_src"));
  }
  VP3D_TRY(eval_ready(p, what));
  const int T = (int)rows;
  const WsLayout wl = ws_layout(p, 1, T, false, L, (size_t)L[p->nb]);
  if (!ws || ws_bytes < wl.total)
    return fail(VP3D_ERR_WORKSPACE, "%s: workspace too small: %zu < %zu", what, ws_bytes, wl.total);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* base = ws_base(ws);
  InferChain c;
  eval_chain(p, wl, base, 1, L, &c);
  float* ybuf = reinterpret_cast<float*>(base + wl.yf);
  c.y = ybuf;
  dilated_chain(p, 1, T, L, &c);

  ClipChain t;
  t.first = reinterpret_cast<const long long*>(clip_first);
  t.len = clip_len;
  t.y_first = reinterpret_cast<const long long*>(y_first);
  t.clips = clips;
  t.copies = copies;
  t.rf = rf;
  t.front = (rf - 1) / 2 + (p->cfg.causal ? (rf - 1) / 2 : 0);   // run.py:186-193
  t.rows = rows;
  // ---- the clips' padded copies (generators.py:216-238), the chain, each clip's rows
  CUDA_TRY(launch_clip_pack(t, x, p->c_in_raw, p->cfg.in_features, aug ? kps_src : nullptr,
                            reinterpret_cast<__nv_bfloat16*>(base + wl.a0), p->c_in_pad, p->planes,
                            (long long)wl.a0_plane, p->f16, stream));
  int launches = 1;
  VP3D_TRY(run_infer_chain(p, c, stream, &launches));
  CUDA_TRY(launch_clip_output(t, ybuf, L[p->nb], p->c_out_raw, aug ? joints_src : nullptr, y,
                              stream));
  p->last_launches = launches + 1;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_calibrate_int8(
    vp3d_plan* p, const float* x, int N, int T, void* ws, size_t ws_bytes, float* amax,
    void* stream_) {
  if (!p || !x || !amax) return fail(VP3D_ERR_INVALID, "calibrate_int8: null argument");
  if (p->cfg.precision != VP3D_PRECISION_FP16)
    return fail(VP3D_ERR_INVALID, "calibrate_int8: needs an fp16 plan (the activations it measures "
                "are the fp16 forward's)");
  if (reinterpret_cast<uintptr_t>(amax) % 4)
    return fail(VP3D_ERR_INVALID, "calibrate_int8: amax not 4-byte aligned");
  // (fp32 values >= 0: their bit patterns order like the values)
  return eval_forward(p, x, nullptr, N, T, ws, ws_bytes, static_cast<cudaStream_t>(stream_),
                      reinterpret_cast<unsigned*>(amax));
}

extern "C" __attribute__((visibility("default"))) size_t vp3d_int8_hist_bytes(const vp3d_plan* p) {
  if (!p || p->nb < 1) return 0;
  return (size_t)2 * p->nb * (kHistBins + 1) * sizeof(uint64_t);
}

extern "C" __attribute__((visibility("default"))) int vp3d_calibrate_int8_hist(
    vp3d_plan* p, const float* x, int N, int T, void* ws, size_t ws_bytes, uint64_t* hist,
    void* stream_) {
  if (!p || !x || !hist) return fail(VP3D_ERR_INVALID, "calibrate_int8_hist: null argument");
  if (p->cfg.precision != VP3D_PRECISION_FP16)
    return fail(VP3D_ERR_INVALID, "calibrate_int8_hist: needs an fp16 plan (the activations it "
                "measures are the fp16 forward's)");
  if (p->nb < 1) return fail(VP3D_ERR_INVALID, "calibrate_int8_hist: the model has no residual block");
  if (reinterpret_cast<uintptr_t>(hist) % 8)
    return fail(VP3D_ERR_INVALID, "calibrate_int8_hist: hist not 8-byte aligned");
  if (N < 1) return fail(VP3D_ERR_INVALID, "calibrate_int8_hist: batch must be >= 1");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  unsigned long long* h = reinterpret_cast<unsigned long long*>(hist);
  VP3D_TRY(eval_forward(p, x, nullptr, N, T, ws, ws_bytes, stream, nullptr, h));
  // the input pack saturates inf and NaN to finite fp16, so no histogram would show them: they
  // count as invalid values of X_0
  CUDA_TRY(launch_count_nonfinite(x, (long long)N * T * p->c_in_raw, h + (size_t)2 * p->nb * kHistBins,
                                  num_sms(), stream));
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_int8_packs(
    const vp3d_plan* p, int layer, void* w_s8, float* w_scale, float* q_scale, void* stream_) {
  if (!p || !p->int8) return fail(VP3D_ERR_INVALID, "int8_packs: not an int8 plan");
  if (layer < 0 || layer >= 2 * p->nb) return fail(VP3D_ERR_INVALID, "int8_packs: no layer %d", layer);
  if (!block_is_int8(p, layer / 2 + 1))
    return fail(VP3D_ERR_INVALID, "int8_packs: layer %d is in block %d, which runs fp16 "
                "(vp3d_set_int8_blocks)", layer, layer / 2 + 1);
  if (!p->conv_packed) return fail(VP3D_ERR_STATE, "int8_packs: weights not packed yet");
  if (q_scale && !p->int8_folded) return fail(VP3D_ERR_STATE, "int8_packs: scales not folded yet");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const PackedConv& k = *p->conv[layer];
  if (w_s8) CUDA_TRY(cudaMemcpyAsync(w_s8, k.w, pack_bytes(p, k), cudaMemcpyDeviceToDevice, stream));
  if (w_scale)
    CUDA_TRY(cudaMemcpyAsync(w_scale, k.w_scale, k.n_pad * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  if (q_scale)
    CUDA_TRY(cudaMemcpyAsync(q_scale, k.q_scale, k.n_pad * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_set_int8_scales(vp3d_plan* p,
                                                                          const float* amax_host,
                                                                          int n) {
  if (!p || !amax_host) return fail(VP3D_ERR_INVALID, "set_int8_scales: null argument");
  if (!p->int8) return fail(VP3D_ERR_INVALID, "set_int8_scales: not an int8 plan");
  if (n != 2 * p->nb)
    return fail(VP3D_ERR_INVALID, "set_int8_scales: expected %d amax values, got %d", 2 * p->nb, n);
  for (int l = 0; l < n; ++l)
    if (!(amax_host[l] >= 0.0f) || !(amax_host[l] <= 3.0e38f))
      return fail(VP3D_ERR_INVALID, "set_int8_scales: amax[%d] = %g is not a finite value >= 0", l,
                  (double)amax_host[l]);
  for (int l = 0; l < n; ++l) {
    // s = amax / 255 and 1 / s, both in fp32 (round to nearest)
    const float s = amax_host[l] > 0.0f ? amax_host[l] / 255.0f : 1.0f;
    p->act_scale[l] = s;
    p->act_inv[l] = 1.0f / s;
  }
  p->int8_scales = true;
  p->int8_folded = false;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_set_int8_blocks(vp3d_plan* p,
                                                                          uint32_t mask) {
  if (!p) return fail(VP3D_ERR_INVALID, "set_int8_blocks: null plan");
  if (!p->int8) return fail(VP3D_ERR_INVALID, "set_int8_blocks: not an int8 plan");
  const uint32_t all = (1u << p->nb) - 1u;
  if (mask & ~all)
    return fail(VP3D_ERR_INVALID, "set_int8_blocks: mask 0x%x selects blocks beyond the plan's %d",
                (unsigned)mask, p->nb);
  if (mask == p->int8_mask) return VP3D_OK;
  p->int8_mask = mask;
  for (int l = 0; l < 2 * p->nb; ++l) p->conv[l]->k_pad = conv_k_pad(p, l);
  // the packs of the blocks that changed format are stale until the next vp3d_set_weights
  p->conv_packed = false;
  p->int8_folded = false;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_forward_eval_host(vp3d_plan* p, const float* x_host, float* y_host, int N,
                                      int T) {
  if (!p || !x_host || !y_host) return fail(VP3D_ERR_INVALID, "forward_eval_host: null argument");
  const int t_out = vp3d_output_frames(p, T);
  if (t_out < 1 || N < 1) return fail(VP3D_ERR_INVALID, "forward_eval_host: bad shape");
  HostStaging& h = p->host;
  VP3D_TRY(lazy_stream(&h.stream));
  const size_t xb = (size_t)N * T * p->c_in_raw * sizeof(float);
  const size_t yb = (size_t)N * t_out * p->c_out_raw * sizeof(float);
  VP3D_TRY(h.x.grow(xb));
  VP3D_TRY(h.y.grow(yb));
  VP3D_TRY(h.ws.grow(vp3d_workspace_bytes(p, N, T)));
  // Batch rows are independent in eval mode: split the batch into chunks so that the host->device
  // copy of chunk i+1 (copy stream) overlaps the kernels of chunk i (compute stream).  PCIe moves
  // 33.8 MB per 1024 x 243 batch, which is longer than the whole forward.
  int chunks = N >= 512 ? 2 : 1;
  if (const char* env = getenv("VP3D_HOST_CHUNKS")) {  // measurement knob
    const int c = atoi(env);
    if (c >= 1 && c <= kMaxHostChunks && c <= N) chunks = c;
  }
  if (chunks == 1) {
    CUDA_TRY(cudaMemcpyAsync(h.x.ptr, x_host, xb, cudaMemcpyHostToDevice, h.stream));
    VP3D_TRY(vp3d_forward_eval(p, h.x.ptr, h.y.ptr, N, T, h.ws.ptr, h.ws.bytes, h.stream));
  } else {
    VP3D_TRY(lazy_stream(&h.copy_stream));
    for (int c = 0; c < chunks; ++c) VP3D_TRY(lazy_event(&h.copy_events[c]));
    const size_t x_row = (size_t)T * p->c_in_raw, y_row = (size_t)t_out * p->c_out_raw;
    int launches = 0;
    // the previous call's kernels may still read h.x: order the copies behind them
    CUDA_TRY(cudaEventRecord(h.copy_events[0], h.stream));
    CUDA_TRY(cudaStreamWaitEvent(h.copy_stream, h.copy_events[0], 0));
    for (int c = 0; c < chunks; ++c) {
      const int n0 = (int)((long long)N * c / chunks), n1 = (int)((long long)N * (c + 1) / chunks);
      CUDA_TRY(cudaMemcpyAsync(h.x.ptr + n0 * x_row, x_host + n0 * x_row,
                               (size_t)(n1 - n0) * x_row * sizeof(float), cudaMemcpyHostToDevice,
                               h.copy_stream));
      CUDA_TRY(cudaEventRecord(h.copy_events[c], h.copy_stream));
    }
    for (int c = 0; c < chunks; ++c) {
      const int n0 = (int)((long long)N * c / chunks), n1 = (int)((long long)N * (c + 1) / chunks);
      CUDA_TRY(cudaStreamWaitEvent(h.stream, h.copy_events[c], 0));
      VP3D_TRY(vp3d_forward_eval(p, h.x.ptr + n0 * x_row, h.y.ptr + n0 * y_row, n1 - n0, T,
                                 h.ws.ptr, h.ws.bytes, h.stream));
      launches += p->last_launches;
    }
    p->last_launches = launches;
  }
  CUDA_TRY(cudaMemcpyAsync(y_host, h.y.ptr, yb, cudaMemcpyDeviceToHost, h.stream));
  CUDA_TRY(cudaStreamSynchronize(h.stream));
  return VP3D_OK;
}

// Pipelined host API: submit() enqueues H2D (copy stream) -> forward (compute stream) -> D2H for one
// batch and returns immediately; wait() blocks until that batch's output is in y_host.  With two
// slots the PCIe copy of batch i+1 overlaps the kernels of batch i, so the sustained rate is
// max(copy, compute) instead of their sum.
extern "C" __attribute__((visibility("default"))) int vp3d_forward_eval_host_submit(
    vp3d_plan* p, const float* x_host, float* y_host, int N, int T, int slot) {
  if (!p || !x_host || !y_host) return fail(VP3D_ERR_INVALID, "host_submit: null argument");
  if (slot < 0 || slot > 1) return fail(VP3D_ERR_INVALID, "host_submit: slot must be 0 or 1");
  const int t_out = vp3d_output_frames(p, T);
  if (t_out < 1 || N < 1) return fail(VP3D_ERR_INVALID, "host_submit: bad shape");
  HostStaging& h = p->host;
  HostStaging::Slot& s = h.slots[slot];
  if (s.busy) return fail(VP3D_ERR_STATE, "host_submit: slot %d still in flight (call wait first)", slot);
  VP3D_TRY(lazy_stream(&h.stream));
  VP3D_TRY(lazy_stream(&h.copy_stream));
  VP3D_TRY(lazy_event(&s.copied));
  VP3D_TRY(lazy_event(&s.done));
  const size_t xb = (size_t)N * T * p->c_in_raw * sizeof(float);
  const size_t yb = (size_t)N * t_out * p->c_out_raw * sizeof(float);
  const size_t wb = vp3d_workspace_bytes(p, N, T);
  VP3D_TRY(s.x.grow(xb));
  VP3D_TRY(s.y.grow(yb));
  if (wb > h.ws.bytes) {
    CUDA_TRY(cudaStreamSynchronize(h.stream));  // the other slot may be using the old workspace
    VP3D_TRY(h.ws.grow(wb));
  }
  CUDA_TRY(cudaMemcpyAsync(s.x.ptr, x_host, xb, cudaMemcpyHostToDevice, h.copy_stream));
  CUDA_TRY(cudaEventRecord(s.copied, h.copy_stream));
  CUDA_TRY(cudaStreamWaitEvent(h.stream, s.copied, 0));
  VP3D_TRY(vp3d_forward_eval(p, s.x.ptr, s.y.ptr, N, T, h.ws.ptr, h.ws.bytes, h.stream));
  CUDA_TRY(cudaMemcpyAsync(y_host, s.y.ptr, yb, cudaMemcpyDeviceToHost, h.stream));
  CUDA_TRY(cudaEventRecord(s.done, h.stream));
  s.busy = true;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_forward_eval_host_wait(vp3d_plan* p,
                                                                                 int slot) {
  if (!p || slot < 0 || slot > 1) return fail(VP3D_ERR_INVALID, "host_wait: bad argument");
  HostStaging::Slot& s = p->host.slots[slot];
  if (!s.busy) return fail(VP3D_ERR_STATE, "host_wait: slot %d has nothing in flight", slot);
  CUDA_TRY(cudaEventSynchronize(s.done));
  s.busy = false;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_last_launch_count(const vp3d_plan* p) { return p ? p->last_launches : 0; }

extern "C" __attribute__((visibility("default"))) int vp3d_profile_launch(vp3d_plan* p, int launch_index) {
  if (!p) return fail(VP3D_ERR_INVALID, "null plan");
  p->prof_launch = launch_index;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_profile_read(vp3d_plan* p, float* total_ms, int* count) {
  if (!p || !total_ms || !count) return fail(VP3D_ERR_INVALID, "profile_read: null argument");
  float sum = 0.0f;
  int n = 0;
  for (size_t i = 0; i + 1 < p->prof_used; i += 2) {
    CUDA_TRY(cudaEventSynchronize(p->prof_events[i + 1]));
    float ms = 0.0f;
    CUDA_TRY(cudaEventElapsedTime(&ms, p->prof_events[i], p->prof_events[i + 1]));
    sum += ms;
    ++n;
  }
  p->prof_used = 0;
  *total_ms = sum;
  *count = n;
  return VP3D_OK;
}

extern "C" __attribute__((visibility("default"))) int vp3d_conv_gemm(const vp3d_conv_desc* d, void* stream) {
  return run_conv(d, static_cast<cudaStream_t>(stream));
}
extern "C" __attribute__((visibility("default"))) int vp3d_conv_gemm_instance(const vp3d_conv_desc* d,
                                                                              int* key) {
  return conv_instance(d, key);
}
extern "C" __attribute__((visibility("default"))) int vp3d_conv_gemm_instances(int* keys, int max) {
  if (max > 0 && !keys) return fail(VP3D_ERR_INVALID, "conv_gemm_instances: null keys");
  return vp3d::conv_gemm_instances(keys, max);
}
