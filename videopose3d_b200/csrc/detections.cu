// Streaming sessions fed by a 2-D detector (vp3d_stream_pack_detections): the input rows of one
// push_detections call, built from the detector's pixel keypoints the way the reference's
// in-the-wild pipeline prepares them.
//
//   * data/prepare_data_2d_custom.py:39-49 (decode) fills the frames without a detection by
//     np.interp(indices, indices[mask], kp[mask, i, j]) per joint and coordinate, in float64, and
//     stores the result as float32: between detections ia < t < ib the value is
//     slope * (t - ia) + fp[ia] with slope = (fp[ib] - fp[ia]) / (ib - ia); before the first
//     detection np.interp's left value (the first detection), after the last its right value (the
//     last detection); a detected frame is its own value.
//   * run.py:93-97 / common/camera.py:14-18 then normalise: X / w * 2 - [1, h / w], where X / w and
//     * 2 are float32 operations (a float32 array and Python ints) and the subtraction is float64
//     (the list is a float64 array), rounded back to float32 when it is stored into the keypoints.
//
// Every operation below is an explicit round-to-nearest intrinsic, so nvcc cannot contract a
// multiply and an add into an FMA: numpy evaluates each of them on its own.
//
// The host (streaming.DetectionBook) decides which frames a call releases and from what; the table
// it builds has one record per output row, so the kernel only evaluates.  The last detection of
// every slot lives in a double-buffered device store: the kernel reads half `parity` (the
// detection a previous call left) and writes half 1 - parity, so no thread reads what another one
// writes in the same launch.
#include "internal.cuh"

namespace vp3d {

namespace {

constexpr int kDetThreads = 256;

struct DetRecord {
  int slot;    // the slot whose keypoints the row is made from
  int left;    // row of kps_px[slot] (< k) holding the left value, -1 = the last-detection store,
               // -2 = the row is no frame (zeros)
  int right;   // row of kps_px[slot] holding the right value of an interpolation, -1 = none (copy)
  int num;     // t - ia
  int den;     // ib - ia (> 0 with right >= 0)
};

__device__ __forceinline__ float interp(float l, float r, int num, int den) {
  const double dl = (double)l;
  const double slope = __ddiv_rn(__dsub_rn((double)r, dl), (double)den);
  return __double2float_rn(__dadd_rn(__dmul_rn(slope, (double)num), dl));
}

// X / w * 2 - off in the reference's precisions (off = 1 for x, h / w in float64 for y)
__device__ __forceinline__ float normalise(float v, int w, double off) {
  const float q = __fmul_rn(__fdiv_rn(v, (float)w), 2.0f);
  return __double2float_rn(__dsub_rn((double)q, off));
}

__global__ void __launch_bounds__(kDetThreads) stream_detections_kernel(
    const float2* __restrict__ kps, int S, int k, int J, const int* __restrict__ slot_tab,
    const DetRecord* __restrict__ rec, long long rows, const float2* last_in, float2* last_out,
    float2* __restrict__ out) {
  const long long n_rows = rows * J, n_all = n_rows + (long long)S * J;
  const long long nthr = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += nthr) {
    if (i >= n_rows) {
      // the last-detection store: the newest detection of this call, or the one kept from before
      const long long sj = i - n_rows;
      const int s = (int)(sj / J);
      const int keep = __ldg(slot_tab + 3 * s + 2);
      last_out[sj] = keep >= 0 && keep < k ? kps[((long long)s * k + keep) * J + (sj - (long long)s * J)]
                                           : last_in[sj];
      continue;
    }
    const long long r = i / J;
    const int j = (int)(i - r * J);
    const DetRecord d = rec[r];
    float2 v = make_float2(0.f, 0.f);
    if (d.slot >= 0 && d.slot < S && d.left >= -1 && d.left < k && d.right < k) {
      const long long base = (long long)d.slot * k;
      float2 p = d.left < 0 ? last_in[(long long)d.slot * J + j] : kps[(base + d.left) * J + j];
      if (d.right >= 0 && d.den > 0) {
        const float2 q = kps[(base + d.right) * J + j];
        p.x = interp(p.x, q.x, d.num, d.den);
        p.y = interp(p.y, q.y, d.num, d.den);
      }
      const int w = __ldg(slot_tab + 3 * d.slot), h = __ldg(slot_tab + 3 * d.slot + 1);
      if (w > 0 && h > 0) {
        v.x = normalise(p.x, w, 1.0);
        v.y = normalise(p.y, w, __ddiv_rn((double)h, (double)w));
      }
    }
    out[i] = v;
  }
}

}  // namespace

}  // namespace vp3d

#define VP3D_EXPORT extern "C" __attribute__((visibility("default")))

VP3D_EXPORT int vp3d_stream_pack_detections(const float* kps_px, int S, int k, int J,
                                            const int32_t* table, int64_t rows, float* last,
                                            int parity, float* out, void* stream) {
  using vp3d::fail;
  const char* what = "stream_pack_detections";
  if (S < 1 || k < 1 || J < 1)
    return fail(VP3D_ERR_INVALID, "%s: S (%d), k (%d) and J (%d) must be >= 1", what, S, k, J);
  if (rows < 0) return fail(VP3D_ERR_INVALID, "%s: rows must be >= 0 (got %lld)", what, (long long)rows);
  if (parity != 0 && parity != 1)
    return fail(VP3D_ERR_INVALID, "%s: parity must be 0 or 1 (got %d)", what, parity);
  if (!kps_px || !table || !last || (rows > 0 && !out))
    return fail(VP3D_ERR_INVALID, "%s: null kps_px, table, last or out", what);
  if ((reinterpret_cast<uintptr_t>(kps_px) | reinterpret_cast<uintptr_t>(table) |
       reinterpret_cast<uintptr_t>(last) | reinterpret_cast<uintptr_t>(out)) & 7)
    return fail(VP3D_ERR_INVALID, "%s: kps_px, table, last and out must be 8-byte aligned", what);
  const long long work = (rows + S) * (long long)J;
  long long blocks = (work + vp3d::kDetThreads - 1) / vp3d::kDetThreads;
  if (blocks > 132 * 8) blocks = 132 * 8;
  const float2* last2 = reinterpret_cast<const float2*>(last);
  const long long half = (long long)S * J;
  vp3d::stream_detections_kernel<<<(int)blocks, vp3d::kDetThreads, 0,
                                   static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float2*>(kps_px), S, k, J, table,
      reinterpret_cast<const vp3d::DetRecord*>(table + 3 * S), rows, last2 + parity * half,
      reinterpret_cast<float2*>(last) + (1 - parity) * half, reinterpret_cast<float2*>(out));
  CUDA_TRY(cudaGetLastError());
  return VP3D_OK;
}
