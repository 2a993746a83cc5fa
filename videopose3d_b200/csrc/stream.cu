// Streaming (frame-by-frame) inference of TemporalModel: common/model.py:63-77, 126-138 applied
// incrementally, with the edge padding of common/generators.py:216-238 done in place.
//
// A session holds S stream slots that advance in lockstep.  Every conv layer with history (the
// expand conv and the first conv of every residual block) keeps its INPUT in a time-major ring,
//   [plane][frame position][stream][ld]      (ld = padded channels of that input)
// so that tap j of the k*S new output rows is one contiguous block of k*S ring rows, a fixed
// dilation*S rows after tap j-1: exactly the flat geometry of conv_gemm_kernel (tap_row_step =
// dilation*S, M = k*S rows).  The residual of block i is a row offset into the same window.
//
// Ring maintenance (mirrored rings).  Ring l needs H_l = (taps-1)*dilation = 2*pad_l frames of
// history next to the k <= K new ones.  It has R_l = H_l + K + 1 frame positions, stored twice
// (positions [0, R) and [R, 2R) hold the same frames): frame t lives at t mod R and t mod R + R.
// The window of a push that starts at frame q is then always the contiguous span
// [w0, w0 + H + k) with w0 = (q - H) mod R, whatever q is.  New frames are written once by the
// GEMM epilogue (ring 0: by the input kernel, which writes both copies) and mirrored into the
// other half by the input kernel of the NEXT push, before any GEMM reads them.  Per push and ring
// this copies exactly the k*S new rows: O(k*S*C) per layer, no periodic compaction.
//
// Start of a sequence.  Every layer maps a constant input sequence to a constant sequence, so the
// history of a slot that starts with frame x0 (np.pad 'edge' of the generator) is one vector per
// ring, v_l(x0).  The v-pass computes it with the same GEMM kernel and every tap reading the same
// row (tap_row_step = 0), which is the very sum (pair -> tap -> k-block order, same operands) the
// offline forward evaluates on an edge-padded stretch; the broadcast kernel then writes it into
// the history positions of the starting slots only.
//
// Test-time flip augmentation (VP3D_STREAM_AUGMENT).  Slot s runs two physical rows: row s the
// plain copy, row S + s the mirrored one (common/generators.py:223-237), in every ring and buffer,
// so every layer is the same flat GEMM over P = 2S rows.  Only the frame bookkeeping and the
// output stay logical: the output kernel writes the flip average of rows s and S + s (run.py:
// 674-680).  The offline forward never mixes samples, so each physical row is the offline forward
// of its own padded sequence; the mirrored row's start history is v_l(mirror(x0)), the edge padding
// of the mirrored sequence.
//
// End of a sequence (vp3d_stream_push_ex's `end`).  A slot whose sequence ended is fed the
// generator's end padding, its last real frame repeated (common/generators.py:216-238), until frame
// length - 1 has come out lookahead frames later; then it is idle.  The per-slot bookkeeping (count,
// active, length) is double-buffered by push parity: the input kernel reads buffer `parity` and
// writes buffer `parity ^ 1`, so the pack, which depends on the bookkeeping of its slot, reads only
// values no block of the same launch writes, whatever order the blocks run in.
//
// Per-slot frame counts (vp3d_stream_push_counts's `count`).  Every push works from one invariant:
// at its start, positions [q - H_l, q) of ring l hold the slot's last H_l ring-l inputs.  A slot
// with n < k real frames still runs all k GEMM rows: rows f < n read only history and earlier real
// rows, so they are exact; rows f >= n are scratch.  The realign kernel then restores the invariant
// for the next push by moving the slot's last H_l positions forward by k - n in every ring: window
// positions [w0 + n, w0 + n + H) go to [w0 + k, w0 + k + H), so the newest real frame sits at the
// window end as after k real frames.  Source and destination overlap; the mirrored rings order the
// copy without scratch memory, because a window of H + k < R positions never holds a position
// together with its mirror (p +- R):
//   phase 1 reads the sources (window positions only) and writes them to the MIRROR copies of the
//     destination, none of which lies in the window: no block reads what another block writes.  It
//     also overwrites the mirror copies of history positions [w0 + k, w0 + H), which is safe because
//     phase 1 never reads a mirror position and phase 2 rewrites their window copies to match;
//   phase 2 (the next launch, after phase 1 has completed) copies those mirror copies back onto the
//     destination window positions, reading only mirror positions.  Both copies then agree, as the
//     next push's input kernel and its mirror pass expect.
// Both phases cover ring 0 and rings 1..nb, every plane and both physical rows of an AUGMENT slot.
//
// Provisional outputs (VP3D_STREAM_PROVISIONAL, vp3d_stream_push_provisional).  A push of k frames
// also returns what vp3d_stream_finish would return right after it, for the la = lookahead frames
// that are not final yet, without changing the session.  The chain of the push runs over k + T
// frame rows instead of k (T = la here): rows [k, k + T) (the tail) are fed the end padding, the
// slot's last real frame repeated, exactly as the rows f >= n of a counted or ending slot already
// are, so row n + j (n = slot_count) is the j-th row finish would compute, with the same operands in
// the same k-order.  The flag sizes every ring with R_l = H_l + K + tail + 1 positions (tail = la),
// so the window of such a push, [w0, w0 + H + k + T), still never holds a position together with its
// mirror.  The tail lands in positions [w0 + H + k, w0 + H + k + T) (ring 0: both copies); modulo R
// these are residues w0 + H + k + j, which lie outside the residues [w0, w0 + H + k) of this push's
// history and new rows because H + k + T < R.  So speculative writes never touch history, and never
// a row whose mirror copy is pending: the next push copies only rows [w0 + H, w0 + H + k) (prev_k =
// k), and its history [w0 + k, w0 + k + H) is H residues that again exclude the tail's (H + T < R).
// A later push reads a tail residue as history only after writing it as one of its new rows.  The
// realign of a counted push moves only window positions [w0, w0 + H + k) and writes their mirror
// copies, none of which lies in the tail's window copies.  The bookkeeping is double-buffered by
// parity as for every push, q / prev_q / prev_k / parity advance as for k frames, and the output
// kernel reads n from the two bookkeeping buffers (count after - count before), so nothing of the
// tail persists.
//
// Held frames (VP3D_STREAM_HELD, vp3d_stream_push_held).  A detector-fed slot may hold P pending
// frames after its last detection, which finish would first push as that detection repeated, then
// end-pad: to the network, la + P more copies of the slot's last real frame, the same end padding
// the tail packs.  So the provisional rows of such a slot are tail rows j < la + P.  Tail row j is
// frame c - la + j, whose input cone [c - la + j - pad - shift, c - la + j + pad - shift] lies in
// the constant end padding once j >= RF - 2 (= 2 pad - 1, causal or not); inside a constant cone
// every layer's rows have the same operands, hence the same bits (the v-pass argument above), so
// rows j >= RF - 2 are copies of row RF - 2 and a push computes T = min(la + max P, RF - 1) tail
// rows, whatever the gap.  The flag sizes the rings for tail = RF - 1 >= T: every argument of the
// previous paragraph holds with H + k + T <= H + K + tail < R.  T = 0 (a causal plan, nothing
// pending) computes no tail.
//
// int8 sessions (VP3D_STREAM_INT8).  Ring i >= 1 of a block in the plan's int8 mask also holds a u8
// plane Q_{i-1} with the positions of its 16-bit planes (frame t at t mod R and t mod R + R): block
// i's k-tap conv reads the window [w0, w0 + H + k) of it, while stage i - 1 writes the new rows at
// w0 + H into both planes (the expand's and an int8 block's epilogue; after an fp16 block a quantise
// pass over the stored 16-bit rows, as in the offline int8 chain).  The start pass makes the u8
// v_l(x0) the same way and the broadcast writes it next to the 16-bit one; the input kernel mirrors,
// and the realign kernel moves, the u8 rows with the 16-bit ones.  Every ordering argument above
// (mirror halves, tail residues, the two realign phases) is about positions, not planes, so it
// holds for each plane: the u8 plane is written and read at exactly the positions of the 16-bit
// planes, by the same kernels in the same order.  H is stored as u8 in `h`, as offline.
//
// Moving slots (vp3d_stream_export / vp3d_stream_import).  Everything a later push reads of logical
// slot s is, per physical row of it and ring l, the H_l history positions [q - H_l, q) of every
// plane (u8 planes too), plus its bookkeeping in buffer `parity`; h, xlast, ybuf and the v vectors
// are rebuilt by every push.  The blob stores them by their rank j = t - (q - H_l) in that window,
// not by ring position, so R, K, S and the tail sizing of the two sessions may differ.
//   Export reads the copy the last writer wrote.  After a push of prev_k frames from window start
//   prev_w0, positions [q - H, q) are the last H positions of that push's window: window index
//   prev_w0 + prev_k + j.  The newest prev_k of them exist in rings 1..nb only at that index (their
//   mirror copy is the next input kernel's job); the older ones were mirrored by the input kernel of
//   the last push, ring 0 and broadcast rows were written twice, and a realigned row had both
//   copies rewritten by its two phases.  So the window index holds frame t whatever wrote it.
//   Import writes both copies, w0' + j and its mirror (w0' = (q' - H) mod R'), of every history
//   position of the destination, and the bookkeeping into buffer parity'.  The destination's own
//   pending mirror copy (the rows [prev_w0' + H, + prev_k') of its last push, which overlap
//   [q' - H, q')) then copies imported values onto equal imported values, whichever half it reads.
//   Neither touches a tail residue or another slot's rows, and both are ordered with the pushes on
//   the caller's stream.
#include "internal.cuh"
#include "launch.cuh"

namespace vp3d {

int stream_lookahead(const vp3d_plan* p);

namespace {

constexpr int kMaxRings = VP3D_MAX_WIDTHS;   // ring 0 = network input, ring i = block i input
constexpr int kStreamFlags =
    VP3D_STREAM_AUGMENT | VP3D_STREAM_PROVISIONAL | VP3D_STREAM_INT8 | VP3D_STREAM_HELD;

struct StreamRing {
  __nv_bfloat16* base;   // plane 0, position 0
  long long plane;       // elements per plane (2R * P * ld, P physical rows per position)
  // VP3D_STREAM_INT8, ring i >= 1 of a block in the plan's int8_mask: the u8 plane Q_{i-1} block i
  // reads, 2R * P * ld bytes with the positions of the 16-bit planes; null otherwise
  uint8_t* q;
  int ld, H, R;
  int w0;                // first window position of the current push
  int prev_w0, prev_k;   // window start and new frames of the previous push (prev_k = 0: none)
};

struct StreamLayout {
  int rings = 0;
  int tail = 0;                 // the end-padding rows a push may append (stream_tail)
  int H[kMaxRings], R[kMaxRings], ld[kMaxRings];
  long long plane[kMaxRings];   // elements per ring plane
  size_t ring[kMaxRings];       // byte offsets
  size_t count = 0, active = 0, length = 0;   // per-slot bookkeeping, [2][S] (push parity)
  size_t h = 0, xlast = 0, ybuf = 0, total = 0;
  size_t v[kMaxRings];          // v_l(x0) of rings 1..nb: [plane][P][C]
  size_t kps = 0, jsrc = 0;     // AUGMENT: int32 mirror maps [J_in], [J_out]
  // INT8, rings 1..nb whatever the block mask (the size depends on plan, S, K and flags only): the
  // u8 plane [2R][P][C] and the u8 v_l(x0) [P][C]; H is stored as u8 in `h`.  After every other
  // buffer, so that a layout without the flag is the one it always was.
  size_t q[kMaxRings], vq[kMaxRings];
};

// rows every ring, activation and output buffer holds per frame position
inline int physical_rows(int S, int flags) { return flags & VP3D_STREAM_AUGMENT ? 2 * S : S; }

// end-padding rows a push may append to its k: PROVISIONAL the look-ahead, HELD the RF - 1 rows past
// which every tail row is a copy (header comment), else 0
inline int stream_tail(const vp3d_plan* p, int flags) {
  if (flags & VP3D_STREAM_HELD) return vp3d_receptive_field(p) - 1;
  return flags & VP3D_STREAM_PROVISIONAL ? stream_lookahead(p) : 0;
}

StreamLayout stream_layout(const vp3d_plan* p, int S, int K, int flags) {
  StreamLayout L;
  L.rings = p->nb + 1;
  L.tail = stream_tail(p, flags);
  const int planes = p->planes;
  const int P = physical_rows(S, flags);
  const int rows = K + L.tail;   // frame rows a push computes at most
  Arena a{1024};
  L.count = a.take((size_t)2 * S * 8);
  L.active = a.take((size_t)2 * S);
  L.length = a.take((size_t)2 * S * 8);
  for (int l = 0; l < L.rings; ++l) {
    L.H[l] = 2 * p->pad[l];
    L.R[l] = L.H[l] + rows + 1;
    L.ld[l] = l == 0 ? p->c_in_pad : p->C;
    L.plane[l] = 2LL * L.R[l] * P * L.ld[l];
    L.ring[l] = a.take((size_t)L.plane[l] * planes * 2);
  }
  const size_t act = (size_t)planes * rows * P * p->C * 2;
  L.h = a.take(act);
  L.xlast = a.take(act);
  L.v[0] = 0;
  for (int l = 1; l < L.rings; ++l) L.v[l] = a.take((size_t)planes * P * p->C * 2);
  L.ybuf = a.take((size_t)rows * P * p->c_out_raw * 4);
  if (flags & VP3D_STREAM_AUGMENT) {
    L.kps = a.take((size_t)p->cfg.num_joints_in * 4);
    L.jsrc = a.take((size_t)p->cfg.num_joints_out * 4);
  }
  L.q[0] = L.vq[0] = 0;
  for (int l = 1; l < L.rings; ++l) {
    L.q[l] = L.vq[l] = 0;
    if (!(flags & VP3D_STREAM_INT8)) continue;
    L.q[l] = a.take((size_t)L.plane[l]);
    L.vq[l] = a.take((size_t)P * p->C);
  }
  L.total = a.total();
  return L;
}

inline int pos_mod(long long a, int m) { return (int)(((a % m) + m) % m); }
__device__ __forceinline__ int pos_mod_dev(int a, int m) { return ((a % m) + m) % m; }
// the other copy of a ring position in [0, 2R)
__device__ __forceinline__ int mirror_pos(int a, int R) { return a < R ? a + R : a - R; }

struct StepArgs {
  StreamRing ring[kMaxRings];
  int rings, planes, f16, S, P, k, c_raw, feat;
  const float* x;          // (S, k, c_raw) fp32, or null: repeat each slot's newest frame (finish)
  const long long* x_rows; // (S,) or null: x is a flat (rows, c_raw) store, frame f of slot s at
                           // row x_rows[s] + f
  const int* kps;          // AUGMENT: [J_in] mirror source of every input joint; null: no rows >= S
  const uint8_t* start;    // (S,) or null
  const int* end;          // (S,) or null: the sequence ends after frame end[s] - 1 of this push
  const int* count;        // (S,) or null: real frames of an open sequence in this push (slot_count)
  // per slot, the buffer of this push's parity (read) and of the next one (written):
  const long long* count_in;    // frames of the current sequence pushed so far
  const uint8_t* active_in;     // 1 while the slot holds a sequence (also while it drains)
  const long long* length_in;   // length of the ended sequence, -1 while it is open
  long long* count_out;
  uint8_t* active_out;
  long long* length_out;
  long long* frame;        // (S, frame_ld) int64
  int frame_ld, frame_off, lookahead;
  int tail;                // provisional push: the T end-padding rows after the k (else 0)
  int prov_rows;           // rows of frame_prov per slot (0: no provisional request)
  long long* frame_prov;   // (S, prov_rows) int64, the frames of the provisional rows
  const int* held;         // (S,) or null: pending held frames of an open sequence (HELD push)
  int max_held;            // held values outside [0, max_held] read as 0
};

// Channel c of the mirrored input frame (generators.py:235-237) is source channel *src, negated when
// *neg: feature 0 negated, joint j read from kps[j].  Negation is exact, so the pack below rounds it
// as the offline pack rounds the generator's mirrored batch.
__device__ __forceinline__ void mirror_channel(int c, const StepArgs& a, int* src, bool* neg) {
  if (c >= a.c_raw) return;
  const int j = c / a.feat, e = c - j * a.feat;
  *src = __ldg(a.kps + j) * a.feat + e;
  *neg = e == 0;
}

// end[s] of this push, values outside [-1, k] read as -1 (a device array cannot be checked on the host)
__device__ __forceinline__ int slot_end(const StepArgs& a, int s) {
  if (!a.end) return -1;
  const int e = a.end[s];
  return e < -1 || e > a.k ? -1 : e;
}

// Frames slot s advances by in this push: count[s] for a slot that holds an open sequence (active,
// or starting in this push) that does not end in it, k for every other slot (an ending slot's real
// frames are its first end[s]; draining and idle slots advance as without counts).  Values outside
// [0, k], and 0 on a starting slot (a start needs its first frame), read as k.  The input kernel
// and the realign kernel both decide through this function, from pre-push values only.
__device__ __forceinline__ int slot_count(const StepArgs& a, int s) {
  if (!a.count) return a.k;
  const bool st = a.start && a.start[s];
  if (!st && (!a.active_in[s] || a.length_in[s] >= 0)) return a.k;
  if (slot_end(a, s) >= 0) return a.k;
  const int n = a.count[s];
  return n < (st ? 1 : 0) || n > a.k ? a.k : n;
}

// Frames of this push that row r packs from x: slot_count for an open sequence, end[s] for one that
// ends in this push, 0 once it has ended or in finish mode (the newest packed frame is repeated
// instead).  An idle slot packs its dense x as it always has; row-addressed x is not read for it.
// Only pre-push values are read: the bookkeeping loop of the same launch writes the other buffer.
__device__ __forceinline__ int packed_frames(const StepArgs& a, int s) {
  if (!a.x) return 0;
  const bool st = a.start && a.start[s];
  if (!st && !a.active_in[s]) return a.x_rows ? 0 : a.k;
  if (!st && a.length_in[s] >= 0) return 0;
  const int e = slot_end(a, s);
  return e >= 0 ? e : slot_count(a, s);
}

// One launch at the head of every push:
//   * frame bookkeeping: a starting slot resets its frame counter; an `end` fixes the sequence's
//     length; output row f of slot s is frame idx = count + f - lookahead of its sequence when
//     0 <= idx < length, else -1 (warm-up of the look-ahead, idle slot, frames past the end); a slot
//     whose frame length - 1 has come out becomes idle;
//   * the input pack: fp32 (S, k, J*F) -> 16-bit ring-0 rows (both copies), zero-padded channels,
//     rounded exactly as the offline input pack rounds (hi / lo split for bf16x3, saturating fp16);
//     with AUGMENT every frame is packed twice, plain into row s and mirrored into row S + s; in
//     finish mode, and for the frames of a slot after its sequence's end, each physical row's last
//     real frame is repeated instead (the generator's end padding, generators.py:216-238): packed
//     from x[s, end - 1] in the push that ends it, the newest ring-0 position after that;
//   * the mirror copy of the rows the previous push's GEMMs wrote into rings 1..nb;
//   * a provisional push: rows [k, k + tail) packed as the end padding of rows f >= n, and
//     frame_prov[s, j] = count after the push - lookahead + j for j < lookahead + held[s] (held
//     read for an open sequence only) under the rules of `frame`, with the bookkeeping after the
//     push: the frames vp3d_stream_finish would number right after it (after a detector-fed slot's
//     held frames).
__global__ void __launch_bounds__(256, 1) stream_input_kernel(const StepArgs a) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthr = (long long)gridDim.x * blockDim.x;
  for (long long s = tid; s < a.S; s += nthr) {
    long long c = a.count_in[s], len = a.length_in[s];
    uint8_t act = a.active_in[s];
    if (a.start && a.start[s]) { c = 0; act = 1; len = -1; }
    const int e = slot_end(a, (int)s);
    const int n = slot_count(a, (int)s);   // rows f >= n are no frame (a counted slot's scratch)
    if (act && len < 0 && e >= 0) len = c + e;
    for (int f = 0; f < a.k; ++f) {
      const long long idx = c + f - a.lookahead;
      a.frame[s * a.frame_ld + a.frame_off + f] =
          (act && f < n && idx >= 0 && (len < 0 || idx < len)) ? idx : -1;
    }
    c += n;
    // idle once frame length - 1 is out (at once for a sequence without frames: start with end 0)
    if (act && len >= 0 && (c - a.lookahead >= len || len == 0)) act = 0;
    a.count_out[s] = c;
    a.active_out[s] = act;
    a.length_out[s] = len;
    int held = act && len < 0 && a.held ? a.held[s] : 0;
    if (held < 0 || held > a.max_held) held = 0;
    for (int j = 0; j < a.prov_rows; ++j) {
      const long long idx = c - a.lookahead + j;
      a.frame_prov[s * a.prov_rows + j] =
          (act && j < a.lookahead + held && idx >= 0 && (len < 0 || idx < len)) ? idx : -1;
    }
  }

  const StreamRing& r0 = a.ring[0];
  const int pairs = r0.ld >> 1;
  // rows f >= k (the tail) take the f >= n branch below: x[s, n - 1], or the newest ring-0 position
  const long long n_pack = (long long)(a.k + a.tail) * a.P * pairs;
  const int src_pos = pos_mod_dev(r0.w0 + r0.H - 1, r0.R);
  for (long long i = tid; i < n_pack; i += nthr) {
    const int cp = (int)(i % pairs);
    const long long row = i / pairs;          // f * P + r
    const int r = (int)(row % a.P), f = (int)(row / a.P);
    const int pos = r0.w0 + r0.H + f;
    const long long d0 = ((long long)pos * a.P + r) * r0.ld + 2 * cp;
    const long long d1 = ((long long)mirror_pos(pos, r0.R) * a.P + r) * r0.ld + 2 * cp;
    const bool mirrored = r >= a.S;
    const int s = mirrored ? r - a.S : r;
    const int n = packed_frames(a, s);
    if (n > 0) {
      // frames past the end repeat x[s, n - 1], rounded as every pack is: the bits of a ring copy
      const long long xrow = (a.x_rows ? __ldg(a.x_rows + s) : (long long)s * a.k) + min(f, n - 1);
      const float* src = a.x + xrow * a.c_raw;
      const int c0 = 2 * cp;
      int i0 = c0, i1 = c0 + 1;   // source channels
      bool n0 = false, n1 = false;
      if (mirrored) {
        mirror_channel(c0, a, &i0, &n0);
        mirror_channel(c0 + 1, a, &i1, &n1);
      }
      float v0 = c0 < a.c_raw ? __ldg(src + i0) : 0.0f;
      float v1 = c0 + 1 < a.c_raw ? __ldg(src + i1) : 0.0f;
      if (n0) v0 = -v0;
      if (n1) v1 = -v1;
      const Bits16 b0 = to_bits16(v0, a.f16), b1 = to_bits16(v1, a.f16);
      const __nv_bfloat162 hi = __halves2bfloat162(b0.hi, b1.hi);
      const __nv_bfloat162 lo = __halves2bfloat162(b0.lo, b1.lo);
      *reinterpret_cast<__nv_bfloat162*>(r0.base + d0) = hi;
      *reinterpret_cast<__nv_bfloat162*>(r0.base + d1) = hi;
      if (a.planes == 2) {
        *reinterpret_cast<__nv_bfloat162*>(r0.base + r0.plane + d0) = lo;
        *reinterpret_cast<__nv_bfloat162*>(r0.base + r0.plane + d1) = lo;
      }
    } else {
      const long long sr = ((long long)src_pos * a.P + r) * r0.ld + 2 * cp;
      for (int pl = 0; pl < a.planes; ++pl) {
        const uint32_t v = *reinterpret_cast<const uint32_t*>(r0.base + pl * r0.plane + sr);
        *reinterpret_cast<uint32_t*>(r0.base + pl * r0.plane + d0) = v;
        *reinterpret_cast<uint32_t*>(r0.base + pl * r0.plane + d1) = v;
      }
    }
  }

#pragma unroll
  for (int l = 1; l < kMaxRings; ++l) {   // (unrolled: the ring table stays in parameter space)
    const StreamRing& r = a.ring[l];
    if (l >= a.rings || r.prev_k == 0) continue;
    const long long per_frame = (long long)a.P * r.ld / 8;   // 16-byte vectors
    const long long n = (long long)a.planes * r.prev_k * per_frame;
    for (long long i = tid; i < n; i += nthr) {
      const long long e = i % per_frame;
      const long long q = i / per_frame;
      const int f = (int)(q % r.prev_k), pl = (int)(q / r.prev_k);
      const int pos = r.prev_w0 + r.H + f;
      const uint4* src = reinterpret_cast<const uint4*>(r.base + pl * r.plane +
                                                        (long long)pos * a.P * r.ld) + e;
      uint4* dst = reinterpret_cast<uint4*>(r.base + pl * r.plane +
                                            (long long)mirror_pos(pos, r.R) * a.P * r.ld) + e;
      *dst = *src;
    }
    if (!r.q) continue;
    // the u8 plane of the same rows (INT8 sessions, rings of int8 blocks)
    const long long per_frame_q = (long long)a.P * r.ld / 16;
    const long long nq = r.prev_k * per_frame_q;
    for (long long i = tid; i < nq; i += nthr) {
      const long long e = i % per_frame_q;
      const int pos = r.prev_w0 + r.H + (int)(i / per_frame_q);
      const uint4* src = reinterpret_cast<const uint4*>(r.q + (long long)pos * a.P * r.ld) + e;
      uint4* dst = reinterpret_cast<uint4*>(r.q + (long long)mirror_pos(pos, r.R) * a.P * r.ld) + e;
      *dst = *src;
    }
  }
}

// One phase of the realign of a counted push (header comment): every physical row whose slot got
// n = slot_count < k real frames moves its last H positions of every ring forward by k - n.
// phase = 0 (the header comment's phase 1) copies window positions w0 + n + j to the mirror copies
// of w0 + k + j, phase = 1 (phase 2) those mirror copies back onto w0 + k + j (j < H).
// The rows are taken kRealignTile at a time: every block lists the tile's realigned rows in shared
// memory, in row order (a ballot prefix sum, so every block holds the same list: the grid splits
// one flat index over it), then the grid strides over their row_vecs 16-byte vectors each, so a
// few realigned rows still spread over every block and a push without any costs one scan of the
// counts.  Each thread loads four vectors before it stores any.  Launched with 256 threads.
constexpr int kRealignTile = 1024;

__global__ void __launch_bounds__(256) stream_realign_kernel(const StepArgs a, int phase,
                                                             int row_vecs) {
  pdl_entry();
  constexpr int kBatch = 4, kWarps = 8;
  __shared__ int rows[kRealignTile], frames[kRealignTile];
  __shared__ int warp_rows[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r0 = 0; r0 < a.P; r0 += kRealignTile) {
    int listed = 0;   // the same in every thread
    for (int c = 0; c < kRealignTile; c += kWarps * 32) {
      const int r = r0 + c + threadIdx.x;
      const int n = r < a.P ? slot_count(a, r < a.S ? r : r - a.S) : a.k;
      const unsigned take = __ballot_sync(0xffffffffu, n < a.k);
      if (lane == 0) warp_rows[warp] = __popc(take);
      __syncthreads();
      int at = listed;
      for (int w = 0; w < kWarps; ++w) {
        if (w < warp) at += warp_rows[w];
        listed += warp_rows[w];
      }
      if (n < a.k) {
        at += __popc(take & ((1u << lane) - 1));
        rows[at] = r;
        frames[at] = n;
      }
      __syncthreads();
    }
    const long long total = (long long)listed * row_vecs;
    for (long long i0 = (long long)blockIdx.x * blockDim.x * kBatch + threadIdx.x; i0 < total;
         i0 += (long long)gridDim.x * blockDim.x * kBatch) {
      uint4 v[kBatch];
      uint4* dst[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const long long i = i0 + u * blockDim.x;
        if (i >= total) break;
        const int at = (int)(i / row_vecs);
        int rem = (int)(i - (long long)at * row_vecs);
        const int r = rows[at], n = frames[at];
#pragma unroll
        for (int l = 0; l < kMaxRings; ++l) {   // (unrolled: the ring table stays in parameter space)
          if (l >= a.rings) break;
          const StreamRing& g = a.ring[l];
          // the ring's 16-bit planes (ld / 8 vectors per row), then its u8 plane (ld / 16)
          const int vec = g.ld / 8;
          const int m = a.planes * g.H * vec;
          const int m_all = m + (g.q ? g.H * (g.ld / 16) : 0);
          if (rem >= m_all) {
            rem -= m_all;
            continue;
          }
          const bool u8 = rem >= m;
          const int vr = u8 ? g.ld / 16 : vec;
          if (u8) rem -= m;
          const int e = rem % vr, q = rem / vr;
          const int j = q % g.H, pl = q / g.H;
          const int to = g.w0 + a.k + j;   // a window position, < 2R
          const int from = phase == 0 ? g.w0 + n + j : mirror_pos(to, g.R);
          const int row_bytes = u8 ? g.ld : 2 * g.ld;
          uint8_t* pb = u8 ? g.q : reinterpret_cast<uint8_t*>(g.base + pl * g.plane);
          v[u] = *(reinterpret_cast<const uint4*>(pb + ((long long)from * a.P + r) * row_bytes) + e);
          dst[u] = reinterpret_cast<uint4*>(
                       pb + ((long long)(phase == 0 ? mirror_pos(to, g.R) : to) * a.P + r) *
                                row_bytes) + e;
          break;
        }
      }
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        if (i0 + u * blockDim.x >= total) break;
        *dst[u] = v[u];
      }
    }
    __syncthreads();   // the lists of the next tile overwrite these
  }
}

struct BcastArgs {
  StreamRing ring[kMaxRings];
  const __nv_bfloat16* src[kMaxRings];   // [plane][S][ld] rows v_l(x0)
  const uint8_t* src_q[kMaxRings];       // rings with a u8 plane: [P][ld] u8 rows v_l(x0)
  long long src_plane[kMaxRings];
  int rings, planes, S, P;
  const uint8_t* start;
};

// Start of a sequence: history positions [w0, w0 + H) of every ring (both copies) of the starting
// slots' physical rows (row r belongs to slot r mod S) receive that row's v_l(x0).
__global__ void __launch_bounds__(256) stream_broadcast_kernel(const BcastArgs a) {
  pdl_entry();
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthr = (long long)gridDim.x * blockDim.x;
  for (int l = 0; l < a.rings; ++l) {
    const StreamRing& r = a.ring[l];
    const int vec = r.ld / 8;
    const long long n = (long long)a.planes * r.H * a.P * vec;
    for (long long i = tid; i < n; i += nthr) {
      const int e = (int)(i % vec);
      long long q = i / vec;
      const int row = (int)(q % a.P);
      q /= a.P;
      if (!a.start[row < a.S ? row : row - a.S]) continue;
      const int j = (int)(q % r.H), pl = (int)(q / r.H);
      const uint4 v = *(reinterpret_cast<const uint4*>(a.src[l] + pl * a.src_plane[l] +
                                                       (long long)row * r.ld) + e);
      const int pos = r.w0 + j;
      __nv_bfloat16* pbase = r.base + pl * r.plane;
      *(reinterpret_cast<uint4*>(pbase + ((long long)pos * a.P + row) * r.ld) + e) = v;
      *(reinterpret_cast<uint4*>(pbase + ((long long)mirror_pos(pos, r.R) * a.P + row) * r.ld) + e) = v;
    }
    if (!r.q) continue;
    const int vq = r.ld / 16;
    const long long nq = (long long)r.H * a.P * vq;
    for (long long i = tid; i < nq; i += nthr) {
      const int e = (int)(i % vq);
      const long long q = i / vq;
      const int row = (int)(q % a.P), j = (int)(q / a.P);
      if (!a.start[row < a.S ? row : row - a.S]) continue;
      const uint4 v = *(reinterpret_cast<const uint4*>(a.src_q[l] + (long long)row * r.ld) + e);
      const int pos = r.w0 + j;
      *(reinterpret_cast<uint4*>(r.q + ((long long)pos * a.P + row) * r.ld) + e) = v;
      *(reinterpret_cast<uint4*>(r.q + ((long long)mirror_pos(pos, r.R) * a.P + row) * r.ld) + e) = v;
    }
  }
}

// Shrink output rows are time-major; y is (S, y_frames, c_out) at frame offset f_off, or with
// y_rows a flat (rows, c_out) buffer that receives the returned frame t of slot s at row
// y_rows[s] + t (rows whose frame is -1 are not written).  Plain: rows f * S + s are copied.
// augment: rows f * 2S + s (plain) and f * 2S + S + s (mirrored) are flip-averaged (run.py:674-680),
// output joint j of the mirrored row read from joint_src[j] (null: no joint swap, the trajectory
// model).
// Provisional push (prov.tail > 0): prov.y (S, rows, c_out) receives row j of slot s from frame row
// n + min(j, tail - 1), n = the frames the slot advanced by (prov.count_out[s] minus
// prov.count_in[s], or minus 0 for a starting slot: the input kernel's bookkeeping of this push);
// tail rows past the last computed one are its copies (header comment, held frames).
struct ProvOut {
  float* y;
  const long long* count_in;
  const long long* count_out;
  const uint8_t* start;
  int tail, rows;
};

__global__ void __launch_bounds__(256) stream_output_kernel(const float* ybuf, float* y, int S, int k,
                                                            int c_out, int y_frames, int f_off,
                                                            int augment, const int* joint_src,
                                                            const long long* frame,
                                                            const long long* y_rows,
                                                            const ProvOut prov) {
  pdl_entry();
  const long long n = (long long)(k + (prov.tail ? prov.rows : 0)) * S * c_out;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c_out);
    const long long r = i / c_out;
    const int s = (int)(r % S);
    int f = (int)(r / S);   // the frame row of ybuf
    float* out;
    if (f < k) {
      out = y + ((long long)s * y_frames + f_off + f) * c_out + c;
      if (y_rows) {
        const long long t = frame[(long long)s * y_frames + f_off + f];
        if (t < 0) continue;
        out = y + (__ldg(y_rows + s) + t) * c_out + c;
      }
    } else {
      const int j = f - k;
      out = prov.y + ((long long)s * prov.rows + j) * c_out + c;
      f = (int)(prov.count_out[s] - (prov.start && prov.start[s] ? 0 : prov.count_in[s])) +
          min(j, prov.tail - 1);
    }
    float v;
    if (augment) {
      const int j = c / 3, e = c - 3 * j;
      const int js = joint_src ? __ldg(joint_src + j) : j;
      const float* row0 = ybuf + ((long long)f * 2 * S + s) * c_out;
      v = flip_average(row0[c], row0[(long long)S * c_out + js * 3 + e], e);
    } else {
      v = ybuf[((long long)f * S + s) * c_out + c];
    }
    *out = v;
  }
}

// Slot transfer (header comment, moving slots).  One blob record per listed slot: two bookkeeping
// vectors {count, length} {active, 0} (int64), then per physical row of the slot (row s, AUGMENT
// also S + s) its history, ring by ring: the 16-bit planes [plane][j < H][ld], then with INT8 the u8
// plane [j < H][ld] of rings 1..nb.  A launch takes at most kSlotChunk slots, listed in parameter
// space.
constexpr int kSlotChunk = 1024;
constexpr int kSlotBookVecs = 2;

struct SlotArgs {
  StreamRing ring[kMaxRings];   // q: the u8 plane of every ring >= 1 with INT8
  int rings, planes, S, phys;   // phys: physical rows per slot (2 with AUGMENT)
  int P, row_vecs;              // row_vecs: 16-byte vectors of one physical row's history
  long long slot_vecs;          // kSlotBookVecs + phys * row_vecs
  long long* count;             // bookkeeping buffer `parity` (S each)
  uint8_t* active;
  long long* length;
  uint4* blob;
  int n;
  int slot[kSlotChunk];
};

// Vector `rem` (< row_vecs) of physical row r's history: its address in the source window (export:
// the copy the last push wrote, window index prev_w0 + prev_k + j) or the two copies of the
// destination position (import: w0 + j and its mirror).
__device__ __forceinline__ void slot_hist_vec(const SlotArgs& a, int r, int rem, bool import,
                                              uint4** p0, uint4** p1) {
#pragma unroll
  for (int l = 0; l < kMaxRings; ++l) {   // (unrolled: the ring table stays in parameter space)
    if (l >= a.rings) break;
    const StreamRing& g = a.ring[l];
    const int vec = g.ld / 8;
    const int m = a.planes * g.H * vec;
    const int m_all = m + (g.q ? g.H * (g.ld / 16) : 0);
    if (rem >= m_all) {
      rem -= m_all;
      continue;
    }
    const bool u8 = rem >= m;
    const int vr = u8 ? g.ld / 16 : vec;
    if (u8) rem -= m;
    const int e = rem % vr, q = rem / vr;
    const int j = q % g.H, pl = q / g.H;
    const int row_bytes = u8 ? g.ld : 2 * g.ld;
    uint8_t* pb = u8 ? g.q : reinterpret_cast<uint8_t*>(g.base + pl * g.plane);
    const int pos = import ? g.w0 + j : g.prev_w0 + g.prev_k + j;   // < 2R
    *p0 = reinterpret_cast<uint4*>(pb + ((long long)pos * a.P + r) * row_bytes) + e;
    *p1 = reinterpret_cast<uint4*>(pb + ((long long)mirror_pos(pos, g.R) * a.P + r) * row_bytes) + e;
    return;
  }
}

__global__ void __launch_bounds__(256) stream_export_kernel(const SlotArgs a) {
  const long long total = (long long)a.n * a.slot_vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int at = (int)(i / a.slot_vecs);
    long long rem = i - (long long)at * a.slot_vecs;
    const int s = a.slot[at];
    uint4 v;
    if (rem < kSlotBookVecs) {
      const long long w0 = rem == 0 ? a.count[s] : (long long)a.active[s];
      const long long w1 = rem == 0 ? a.length[s] : 0;
      v = make_uint4((unsigned)w0, (unsigned)(w0 >> 32), (unsigned)w1, (unsigned)(w1 >> 32));
    } else {
      rem -= kSlotBookVecs;
      const int pr = (int)(rem / a.row_vecs);
      uint4 *src, *unused;
      slot_hist_vec(a, pr == 0 ? s : a.S + s, (int)(rem - (long long)pr * a.row_vecs), false, &src,
                    &unused);
      v = *src;
    }
    a.blob[i] = v;
  }
}

__global__ void __launch_bounds__(256) stream_import_kernel(const SlotArgs a) {
  const long long total = (long long)a.n * a.slot_vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int at = (int)(i / a.slot_vecs);
    long long rem = i - (long long)at * a.slot_vecs;
    const int s = a.slot[at];
    const uint4 v = a.blob[i];
    if (rem < kSlotBookVecs) {
      const long long w0 = (long long)(((unsigned long long)v.y << 32) | v.x);
      const long long w1 = (long long)(((unsigned long long)v.w << 32) | v.z);
      if (rem == 0) {
        a.count[s] = w0;
        a.length[s] = w1;
      } else {
        a.active[s] = (uint8_t)w0;
      }
    } else {
      rem -= kSlotBookVecs;
      const int pr = (int)(rem / a.row_vecs);
      uint4 *d0, *d1;
      slot_hist_vec(a, pr == 0 ? s : a.S + s, (int)(rem - (long long)pr * a.row_vecs), true, &d0,
                    &d1);
      *d0 = v;
      *d1 = v;
    }
  }
}

inline int grid_for(long long work) {
  long long b = (work + 255) / 256;
  if (b < 1) b = 1;
  if (b > 132 * 8) b = 132 * 8;
  return (int)b;
}

// rows of ring r from frame position pos on
inline __nv_bfloat16* ring_rows(const StreamRing& r, int pos, int P) {
  return r.base + (long long)pos * P * r.ld;
}
// the same rows of its u8 plane (null without one)
inline uint8_t* ring_rows_q(const StreamRing& r, int pos, int P) {
  return r.q ? r.q + (long long)pos * P * r.ld : nullptr;
}

// The push of k frames as a flat chain over ring windows.  The window of ring i is its frame
// positions [w0, w0 + H + k): tap j of the k * P new rows lies dilation * P rows after tap j - 1, the
// residual (the centre tap, causal: the newest; model.py:130-132) a row offset into the same window.
// Stage i writes the new rows of ring i + 1, the last stage the buffer shrink reads.  A provisional
// push appends its `tail` rows to the k: the same chain over k + tail frame rows.  An int8 block i
// reads the same window of ring i's u8 plane, which stage i - 1 fills at w0 + H as it writes the
// 16-bit rows (the expand's and int8 blocks' epilogues, or a quantise pass after an fp16 block).
void push_chain(const vp3d_plan* p, const StreamLayout& L, uint8_t* base, const StreamRing* ring,
                int P, int K, int k, int tail, float* y, InferChain* c) {
  memset(c, 0, sizeof(*c));
  c->stages = p->nb + 1;
  c->samples = 1;
  c->in_plane = ring[0].plane;
  c->expand = p->expand_dil;
  c->h = reinterpret_cast<__nv_bfloat16*>(base + L.h);
  if (p->int8) c->hq = base + L.h;
  c->y = y;
  for (int i = 0; i <= p->nb + 1; ++i) c->precision[i] = layer_precision(p, i);   // (never `mixed`)
  for (int i = 0; i <= p->nb; ++i) {
    ChainStage& s = c->st[i];
    s.in = ring_rows(ring[i], ring[i].w0, P);
    s.in_rows = (ring[i].H + k + tail) * P;
    if (i > 0) {
      s.q_in = ring_rows_q(ring[i], ring[i].w0, P);
      s.q_in_bytes = (long long)(2 * ring[i].R - ring[i].w0) * P * ring[i].ld;
    }
    const StreamRing* next = i < p->nb ? &ring[i + 1] : nullptr;
    s.q_out = next ? ring_rows_q(*next, next->w0 + next->H, P) : nullptr;
    s.out = next ? ring_rows(*next, next->w0 + next->H, P)
                 : reinterpret_cast<__nv_bfloat16*>(base + L.xlast);
    s.h_plane = (long long)(K + L.tail) * P * p->C;
    s.out_plane = next ? next->plane : s.h_plane;
    s.out_rows = (k + tail) * P;
    s.tap_row_step = p->dilation[i] * P;
    s.res_row_off = (p->pad[i] + p->shift_dil[i]) * P;
  }
}

// The start pass, from the push's chain: the same GEMMs on the P rows of the new frame with every
// tap (and the residual) on the same row, v_{i+1} the input of v_{i+2}; ring nb's vector is the last
// it needs, so block nb and shrink do not run.
void vpass_chain(const vp3d_plan* p, const StreamLayout& L, uint8_t* base, const StreamRing* ring,
                 int P, InferChain* c) {
  const long long v_plane = (long long)P * p->C;
  c->stages = p->nb;
  c->y = nullptr;
  for (int i = 0; i < p->nb; ++i) {
    ChainStage& s = c->st[i];
    s.in = i == 0 ? ring_rows(ring[0], ring[0].w0 + ring[0].H, P) : c->st[i - 1].out;
    s.in_rows = s.out_rows = P;
    s.out = reinterpret_cast<__nv_bfloat16*>(base + L.v[i + 1]);
    s.out_plane = v_plane;
    s.tap_row_step = s.res_row_off = 0;
    // the u8 v_l(x0) of the rings of int8 blocks, made and read as the push's u8 rows are
    s.q_in = i == 0 ? nullptr : c->st[i - 1].q_out;
    s.q_in_bytes = (long long)P * p->C;
    s.q_out = ring[i + 1].q ? base + L.vq[i + 1] : nullptr;
  }
}

// A push's provisional request (y null: none): y_prov (S, rows, c_out) / frame_prov (S, rows), the
// chain's tail rows (y_prov row j is tail row min(j, tail - 1)), and the pending held frames of
// every slot (null: none; values outside [0, max_held] read as 0).
struct ProvRequest {
  float* y = nullptr;
  long long* frame = nullptr;
  const int* held = nullptr;
  int max_held = 0, rows = 0, tail = 0;
};

}  // namespace

// run.py:186-193 pads pad + causal_shift frames in front and pad - causal_shift behind, with
// causal_shift = pad for a causal model (every block's shift, in frames, adds up to pad)
int stream_lookahead(const vp3d_plan* p) {
  return p->cfg.causal ? 0 : (vp3d_receptive_field(p) - 1) / 2;
}

// One push of k frames (x null: k copies of every slot's newest frame).  y receives rows
// [f_off, f_off + k) of a (S, y_frames, J_out, 3) tensor, or with y_rows the rows y_rows[s] + frame
// of a flat one; frame the matching (S, y_frames) entries.  The GEMMs run over P physical rows per
// frame (S, or 2S with AUGMENT).  A provisional request (pr.y non-null) also computes pr.tail
// end-padding rows and writes y_prov / frame_prov (ProvRequest).
static int stream_step(vp3d_plan* p, uint8_t* base, StreamHost& h, const float* x, int k,
                       const uint8_t* start, const int* end, const int* count,
                       const long long* x_rows,
                       const long long* y_rows, float* y, int y_frames, int f_off, long long* frame,
                       const ProvRequest& pr, cudaStream_t stream) {
  const int S = h.S, K = h.K, C = p->C, planes = p->planes;
  const bool aug = h.flags & VP3D_STREAM_AUGMENT;
  const int P = physical_rows(S, h.flags);
  const StreamLayout L = stream_layout(p, S, K, h.flags);
  const int tail = pr.y ? pr.tail : 0;
  int launches = 0;

  StepArgs a;
  memset(&a, 0, sizeof(a));
  StreamRing ring[kMaxRings];
  for (int l = 0; l < L.rings; ++l) {
    StreamRing& r = ring[l];
    r.base = reinterpret_cast<__nv_bfloat16*>(base + L.ring[l]);
    r.plane = L.plane[l];
    r.q = (h.flags & VP3D_STREAM_INT8) && l > 0 && block_is_int8(p, l) ? base + L.q[l] : nullptr;
    r.ld = L.ld[l];
    r.H = L.H[l];
    r.R = L.R[l];
    r.w0 = pos_mod(h.q - r.H, r.R);
    r.prev_w0 = pos_mod(h.prev_q - r.H, r.R);
    r.prev_k = h.prev_k;
    a.ring[l] = r;
  }
  a.rings = L.rings;
  a.planes = planes;
  a.f16 = p->f16;
  a.S = S;
  a.P = P;
  a.k = k;
  a.c_raw = p->c_in_raw;
  a.feat = p->cfg.in_features;
  a.x = x;
  a.x_rows = x_rows;
  a.kps = aug ? reinterpret_cast<const int*>(base + L.kps) : nullptr;
  a.start = start;
  a.end = end;
  a.count = count;
  {
    const int in = h.parity, out = h.parity ^ 1;
    long long* count = reinterpret_cast<long long*>(base + L.count);
    long long* length = reinterpret_cast<long long*>(base + L.length);
    a.count_in = count + (size_t)in * S;
    a.count_out = count + (size_t)out * S;
    a.active_in = base + L.active + (size_t)in * S;
    a.active_out = base + L.active + (size_t)out * S;
    a.length_in = length + (size_t)in * S;
    a.length_out = length + (size_t)out * S;
  }
  a.frame = frame;
  a.frame_ld = y_frames;
  a.frame_off = f_off;
  a.lookahead = stream_lookahead(p);
  a.tail = tail;
  a.prov_rows = pr.y ? pr.rows : 0;
  a.frame_prov = pr.frame;
  a.held = pr.held;
  a.max_held = pr.max_held;
  {
    long long work = (long long)(k + tail) * P * (p->c_in_pad / 2);
    for (int l = 1; l < L.rings; ++l)
      work += (long long)planes * h.prev_k * P * C / 8 + (ring[l].q ? (long long)h.prev_k * P * C / 16 : 0);
    if (work < S) work = S;
    // a plain launch: the first kernel of a push may follow a weight re-pack, which the GEMMs'
    // early weight loads must not overlap
    stream_input_kernel<<<grid_for(work), 256, 0, stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    ++launches;
  }

  const long long v_plane = (long long)P * C;
  auto vbuf = [&](int l) { return reinterpret_cast<__nv_bfloat16*>(base + L.v[l]); };
  // shrink straight into y when the time-major rows already are y's rows (k == 1 or S == 1, no
  // AUGMENT: the flip average always takes the output kernel, and so do row-addressed outputs and
  // provisional pushes)
  const bool direct = !aug && !y_rows && !pr.y && (y_frames == 1 || S == 1);
  float* ybuf = reinterpret_cast<float*>(base + L.ybuf);
  InferChain push;
  push_chain(p, L, base, ring, P, K, k, tail,
             direct ? y + (long long)f_off * p->c_out_raw : ybuf, &push);

  if (start && p->nb >= 1) {
    // ---- v-pass: v_1 = expand(x0), v_{i+1} = block_i(v_i)
    InferChain v = push;
    vpass_chain(p, L, base, ring, P, &v);
    VP3D_TRY(run_infer_chain(p, v, stream, &launches));
  }
  if (start) {
    BcastArgs b;
    memset(&b, 0, sizeof(b));
    long long work = 0;
    for (int l = 0; l < L.rings; ++l) {
      b.ring[l] = ring[l];
      if (l == 0) {
        // the starting slot's first frame, just packed
        b.src[0] = ring_rows(ring[0], ring[0].w0 + ring[0].H, P);
        b.src_plane[0] = ring[0].plane;
      } else {
        b.src[l] = vbuf(l);
        b.src_plane[l] = v_plane;
        b.src_q[l] = ring[l].q ? base + L.vq[l] : nullptr;
      }
      work += (long long)planes * ring[l].H * P * ring[l].ld / 8 +
              (ring[l].q ? (long long)ring[l].H * P * ring[l].ld / 16 : 0);
    }
    b.rings = L.rings;
    b.planes = planes;
    b.S = S;
    b.P = P;
    b.start = start;
    CUDA_TRY(launch_pdl(stream_broadcast_kernel, dim3(grid_for(work)), dim3(256), 0, stream, b));
    ++launches;
  }

  // ---- the push: expand (model.py:127), residual blocks (:129-135), shrink (:137)
  VP3D_TRY(run_infer_chain(p, push, stream, &launches));
  if (count) {
    // the slots with fewer real frames than k: both realign phases, after the last GEMM read the
    // rings (the host cannot see the counts, so they always run)
    int row_vecs = 0;   // 16-byte vectors a realigned row moves per phase
    for (int l = 0; l < L.rings; ++l)
      row_vecs += planes * ring[l].H * ring[l].ld / 8 + (ring[l].q ? ring[l].H * ring[l].ld / 16 : 0);
    // four vectors per thread over one full tile, at most four blocks per SM: enough loads in
    // flight for HBM bandwidth, and few blocks to scan the counts when no row realigns
    int grid = grid_for((long long)row_vecs * (P < kRealignTile ? P : kRealignTile) / 4);
    if (grid > 132 * 4) grid = 132 * 4;
    for (int phase = 0; phase < 2; ++phase) {
      CUDA_TRY(launch_pdl(stream_realign_kernel, dim3(grid), dim3(256), 0, stream, a, phase,
                          row_vecs));
      ++launches;
    }
  }
  if (!direct) {
    ProvOut prov;
    memset(&prov, 0, sizeof(prov));
    if (tail) {
      prov.y = pr.y;
      prov.count_in = a.count_in;
      prov.count_out = a.count_out;
      prov.start = start;
      prov.tail = tail;
      prov.rows = pr.rows;
    }
    CUDA_TRY(launch_pdl(stream_output_kernel,
                        dim3(grid_for((long long)(k + (tail ? pr.rows : 0)) * S * p->c_out_raw)),
                        dim3(256), 0,
                        stream, (const float*)ybuf, y, S, k, p->c_out_raw, y_frames, f_off, (int)aug,
                        h.joint_src ? (const int*)(base + L.jsrc) : (const int*)nullptr,
                        (const long long*)frame, y_rows, prov));
    ++launches;
  }
  h.parity ^= 1;
  h.prev_q = h.q;
  h.prev_k = k;
  h.q += k;
  p->last_launches = launches;
  return VP3D_OK;
}

static int stream_supported(const vp3d_plan* p, int flags, const char* what) {
  if (p->cfg.variant != VP3D_VARIANT_DILATED)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: streaming needs the TemporalModel (dilated) variant",
                what);
  if (p->cfg.precision == VP3D_PRECISION_MIXED)
    return fail(VP3D_ERR_UNSUPPORTED, "%s: precision 'mixed' is not supported for streaming", what);
  if (p->int8 && !(flags & VP3D_STREAM_INT8))
    return fail(VP3D_ERR_UNSUPPORTED, "%s: precision 'int8' streams only in a session initialised "
                "with VP3D_STREAM_INT8", what);
  if (!p->int8 && (flags & VP3D_STREAM_INT8))
    return fail(VP3D_ERR_INVALID, "%s: VP3D_STREAM_INT8 needs an int8 plan", what);
  return VP3D_OK;
}

// An INT8 session's history holds the quantisation of the plan's block mask and activation scales
// at its first push after init: later pushes need the same ones (and, as every int8 chain, folded
// scales).
static int stream_int8_ready(const vp3d_plan* p, StreamHost& h, const char* what) {
  if (!(h.flags & VP3D_STREAM_INT8)) return VP3D_OK;
  if (!p->int8_folded)
    return fail(VP3D_ERR_STATE, "%s: int8 plan without folded activation scales (call "
                "vp3d_set_int8_scales, then vp3d_set_weights)", what);
  const size_t scale_bytes = sizeof(float) * 2 * p->nb;
  if (!h.int8_snap) {
    h.int8_snap = true;
    h.int8_mask = p->int8_mask;
    memcpy(h.act_scale, p->act_scale, scale_bytes);
    return VP3D_OK;
  }
  if (h.int8_mask != p->int8_mask || memcmp(h.act_scale, p->act_scale, scale_bytes) != 0)
    return fail(VP3D_ERR_STATE, "%s: the plan's int8 blocks or activation scales changed since the "
                "session's first push; initialise the session again", what);
  return VP3D_OK;
}

// every row index of a session's rings and buffers fits an int
static bool stream_fits(const vp3d_plan* p, int S, int K, int flags) {
  const int tail = stream_tail(p, flags);
  return (long long)physical_rows(S, flags) * (K + tail + 2LL * vp3d_receptive_field(p)) <=
         0x7fffffffLL;
}

}  // namespace vp3d

using namespace vp3d;

#define VP3D_EXPORT extern "C" __attribute__((visibility("default")))

VP3D_EXPORT int vp3d_stream_lookahead(const vp3d_plan* p) {
  if (!p) return fail(VP3D_ERR_INVALID, "stream_lookahead: null plan");
  return stream_lookahead(p);
}

VP3D_EXPORT size_t vp3d_stream_state_bytes_ex(const vp3d_plan* p, int S, int K, int flags) {
  if (!p || S < 1 || K < 1 || (flags & ~kStreamFlags) || !stream_fits(p, S, K, flags))
    return 0;
  if ((flags & VP3D_STREAM_PROVISIONAL) && stream_lookahead(p) == 0) return 0;
  if ((flags & VP3D_STREAM_PROVISIONAL) && (flags & VP3D_STREAM_HELD)) return 0;
  if ((flags & VP3D_STREAM_INT8) && !p->int8) return 0;
  return stream_layout(p, S, K, flags).total;
}

VP3D_EXPORT size_t vp3d_stream_state_bytes(const vp3d_plan* p, int S, int K) {
  return vp3d_stream_state_bytes_ex(p, S, K, 0);
}

int vp3d::check_mirror_map(const int32_t* map, int n, const char* what, const char* name) {
  for (int j = 0; j < n; ++j)
    if (map[j] < 0 || map[j] >= n)
      return fail(VP3D_ERR_INVALID, "%s: %s[%d] = %d is not a joint index in [0, %d)", what, name, j,
                  map[j], n);
  return VP3D_OK;
}

static int stream_init(const char* what, vp3d_plan* p, void* state, size_t state_bytes, int S,
                       int K, int flags, const int32_t* kps_src, const int32_t* joints_src,
                       void* stream) {
  if (S < 1 || K < 1)
    return fail(VP3D_ERR_INVALID, "%s: streams (%d) and max_frames (%d) must be >= 1", what, S, K);
  if (flags & ~kStreamFlags)
    return fail(VP3D_ERR_INVALID, "%s: unknown flags 0x%x", what, (unsigned)flags);
  if ((flags & VP3D_STREAM_PROVISIONAL) && (flags & VP3D_STREAM_HELD))
    return fail(VP3D_ERR_INVALID, "%s: VP3D_STREAM_HELD and VP3D_STREAM_PROVISIONAL exclude each "
                "other (a HELD session's push_held with max_held = 0 is the provisional push)", what);
  const bool aug = flags & VP3D_STREAM_AUGMENT;
  if (!aug && (kps_src || joints_src))
    return fail(VP3D_ERR_INVALID, "%s: mirror maps given without VP3D_STREAM_AUGMENT", what);
  if (aug && !kps_src)
    return fail(VP3D_ERR_INVALID, "%s: VP3D_STREAM_AUGMENT needs kps_src", what);
  if (!p) return fail(VP3D_ERR_INVALID, "%s: null plan", what);
  if (!state) return fail(VP3D_ERR_INVALID, "%s: null state", what);
  VP3D_TRY(stream_supported(p, flags, what));
  if ((flags & VP3D_STREAM_PROVISIONAL) && stream_lookahead(p) == 0)
    return fail(VP3D_ERR_INVALID,
                "%s: VP3D_STREAM_PROVISIONAL on a causal model (lookahead 0: every output is final)",
                what);
  const int j_in = p->cfg.num_joints_in, j_out = p->cfg.num_joints_out;
  if (aug) {
    VP3D_TRY(check_mirror_map(kps_src, j_in, what, "kps_src"));
    if (joints_src) VP3D_TRY(check_mirror_map(joints_src, j_out, what, "joints_src"));
  }
  if (!stream_fits(p, S, K, flags))
    return fail(VP3D_ERR_UNSUPPORTED, "%s: %d streams x %d frames is too large", what, S, K);
  const StreamLayout L = stream_layout(p, S, K, flags);
  if (state_bytes < L.total)
    return fail(VP3D_ERR_WORKSPACE, "%s: state too small: %zu < %zu", what, state_bytes, L.total);
  StreamHost h;
  h.S = S;
  h.K = K;
  h.flags = flags;
  h.joint_src = aug && joints_src;
  p->streams[state] = h;
  uint8_t* base = ws_base(state);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(base, 0, L.total - 1024, s));
  // every sequence open (length -1) in both bookkeeping buffers
  CUDA_TRY(cudaMemsetAsync(base + L.length, 0xff, (size_t)2 * S * 8, s));
  if (aug) {
    // the maps live in the state from here on: pushes read them on the device
    CUDA_TRY(cudaMemcpyAsync(base + L.kps, kps_src, (size_t)j_in * 4, cudaMemcpyHostToDevice, s));
    if (joints_src)
      CUDA_TRY(cudaMemcpyAsync(base + L.jsrc, joints_src, (size_t)j_out * 4, cudaMemcpyHostToDevice, s));
  }
  return VP3D_OK;
}

VP3D_EXPORT int vp3d_stream_init_ex(vp3d_plan* p, void* state, size_t state_bytes, int S, int K,
                                    int flags, const int32_t* kps_src, const int32_t* joints_src,
                                    void* stream) {
  return stream_init("stream_init_ex", p, state, state_bytes, S, K, flags, kps_src, joints_src,
                     stream);
}

VP3D_EXPORT int vp3d_stream_init(vp3d_plan* p, void* state, size_t state_bytes, int S, int K,
                                 void* stream) {
  return stream_init("stream_init", p, state, state_bytes, S, K, 0, nullptr, nullptr, stream);
}

VP3D_EXPORT int vp3d_stream_release(vp3d_plan* p, void* state) {
  if (!p || !state) return fail(VP3D_ERR_INVALID, "stream_release: null argument");
  p->streams.erase(state);
  return VP3D_OK;
}

static int stream_lookup(vp3d_plan* p, void* state, const char* what, StreamHost** out) {
  auto it = p->streams.find(state);
  if (it == p->streams.end())
    return fail(VP3D_ERR_STATE, "%s: state was not initialised with vp3d_stream_init", what);
  *out = &it->second;
  return VP3D_OK;
}

// 16-byte vectors of one physical row's history in a slot blob (SlotArgs)
static int slot_row_vecs(const vp3d_plan* p, int flags) {
  int v = 0;
  for (int l = 0; l <= p->nb; ++l) {
    const int H = 2 * p->pad[l], ld = l == 0 ? p->c_in_pad : p->C;
    v += p->planes * H * ld / 8 + ((flags & VP3D_STREAM_INT8) && l > 0 ? H * ld / 16 : 0);
  }
  return v;
}

static long long slot_vecs(const vp3d_plan* p, int flags) {
  return kSlotBookVecs + (long long)(flags & VP3D_STREAM_AUGMENT ? 2 : 1) * slot_row_vecs(p, flags);
}

// The checks both transfer entries make before any device work (argument errors under `what`, then
// the session's slots), and the kernel arguments of the session's current position.
static int slot_transfer_args(const char* what, vp3d_plan* p, void* state, const int32_t* slots,
                              int n, const void* blob, size_t blob_bytes, const void* header,
                              bool import, StreamHost** hp, SlotArgs* a) {
  if (!state) return fail(VP3D_ERR_INVALID, "%s: null state", what);
  if (!p) return fail(VP3D_ERR_INVALID, "%s: null plan", what);
  if (n < 1) return fail(VP3D_ERR_INVALID, "%s: n must be >= 1 (got %d)", what, n);
  if (!slots || !blob || !header) return fail(VP3D_ERR_INVALID, "%s: null slots, blob or header", what);
  if (reinterpret_cast<uintptr_t>(blob) % 16)
    return fail(VP3D_ERR_INVALID, "%s: blob is not 16-byte aligned", what);
  VP3D_TRY(stream_lookup(p, state, what, hp));
  const StreamHost& h = **hp;
  for (int i = 0; i < n; ++i) {
    if (slots[i] < 0 || slots[i] >= h.S)
      return fail(VP3D_ERR_INVALID, "%s: slots[%d] = %d is not a slot in [0, %d)", what, i, slots[i],
                  h.S);
    if (import)
      for (int j = 0; j < i; ++j)
        if (slots[j] == slots[i])
          return fail(VP3D_ERR_INVALID, "%s: slot %d is listed twice (slots[%d], slots[%d])", what,
                      slots[i], j, i);
  }
  const long long need = (long long)n * slot_vecs(p, h.flags) * 16;
  if ((long long)blob_bytes < need)
    return fail(VP3D_ERR_WORKSPACE, "%s: blob too small: %zu < %lld bytes for %d slots", what,
                blob_bytes, need, n);
  const StreamLayout L = stream_layout(p, h.S, h.K, h.flags);
  uint8_t* base = ws_base(state);
  memset(a, 0, sizeof(*a));
  a->rings = L.rings;
  a->planes = p->planes;
  a->S = h.S;
  a->phys = h.flags & VP3D_STREAM_AUGMENT ? 2 : 1;
  a->P = physical_rows(h.S, h.flags);
  a->row_vecs = slot_row_vecs(p, h.flags);
  a->slot_vecs = slot_vecs(p, h.flags);
  for (int l = 0; l < L.rings; ++l) {
    StreamRing& r = a->ring[l];
    r.base = reinterpret_cast<__nv_bfloat16*>(base + L.ring[l]);
    r.plane = L.plane[l];
    r.q = (h.flags & VP3D_STREAM_INT8) && l > 0 ? base + L.q[l] : nullptr;
    r.ld = L.ld[l];
    r.H = L.H[l];
    r.R = L.R[l];
    r.w0 = pos_mod(h.q - r.H, r.R);
    r.prev_w0 = pos_mod(h.prev_q - r.H, r.R);
    r.prev_k = h.prev_k;
  }
  a->count = reinterpret_cast<long long*>(base + L.count) + (size_t)h.parity * h.S;
  a->active = base + L.active + (size_t)h.parity * h.S;
  a->length = reinterpret_cast<long long*>(base + L.length) + (size_t)h.parity * h.S;
  return VP3D_OK;
}

// One launch per kSlotChunk listed slots; the blob record of slots[i] starts at vector
// i * slot_vecs.
template <typename Kernel>
static int slot_transfer_launch(Kernel kernel, vp3d_plan* p, SlotArgs& a, const int32_t* slots,
                                int n, void* blob, cudaStream_t stream) {
  int launches = 0;
  for (int i0 = 0; i0 < n; i0 += kSlotChunk) {
    a.n = n - i0 < kSlotChunk ? n - i0 : kSlotChunk;
    memcpy(a.slot, slots + i0, sizeof(int) * a.n);
    a.blob = reinterpret_cast<uint4*>(blob) + (long long)i0 * a.slot_vecs;
    kernel<<<grid_for((long long)a.n * a.slot_vecs), 256, 0, stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    ++launches;
  }
  p->last_launches = launches;
  return VP3D_OK;
}

static int stream_push(const char* what, vp3d_plan* p, void* state, const float* x, int k,
                       const uint8_t* start_mask, const int32_t* end, const int32_t* count,
                       const int64_t* x_rows, const int64_t* y_rows, float* y, int64_t* frame,
                       int prov_flag, ProvRequest pr, void* stream) {
  if (!state) return fail(VP3D_ERR_INVALID, "%s: null state", what);
  if (k < 1) return fail(VP3D_ERR_INVALID, "%s: k must be >= 1 (got %d)", what, k);
  if (!p) return fail(VP3D_ERR_INVALID, "%s: null plan", what);
  if (y_rows && !frame)
    return fail(VP3D_ERR_INVALID, "%s: y_rows needs frame (the row of every output is its frame)",
                what);
  if (!x || !y || !frame) return fail(VP3D_ERR_INVALID, "%s: null x, y or frame", what);
  StreamHost* h = nullptr;
  VP3D_TRY(stream_lookup(p, state, what, &h));
  if (prov_flag && !(h->flags & prov_flag))
    return fail(VP3D_ERR_STATE, "%s: the session was not initialised with %s", what,
                prov_flag == VP3D_STREAM_HELD ? "VP3D_STREAM_HELD" : "VP3D_STREAM_PROVISIONAL");
  if (k > h->K)
    return fail(VP3D_ERR_INVALID, "%s: k = %d frames exceeds max_frames = %d", what, k, h->K);
  const int la = stream_lookahead(p);
  if (prov_flag == VP3D_STREAM_PROVISIONAL) pr.rows = pr.tail = la;
  if (prov_flag == VP3D_STREAM_HELD) {
    if ((long long)pr.rows < (long long)la + pr.max_held)
      return fail(VP3D_ERR_INVALID, "%s: rows = %d < lookahead %d + max_held %d", what, pr.rows, la,
                  pr.max_held);
    const long long t = (long long)la + pr.max_held;
    pr.tail = (int)(t < vp3d_receptive_field(p) - 1 ? t : vp3d_receptive_field(p) - 1);
  }
  if (!p->conv_packed || !p->bn_packed)
    return fail(VP3D_ERR_STATE, "%s: vp3d_set_weights has not been called", what);
  VP3D_TRY(stream_int8_ready(p, *h, what));
  return stream_step(p, ws_base(state), *h, x, k, start_mask, end, count,
                     reinterpret_cast<const long long*>(x_rows),
                     reinterpret_cast<const long long*>(y_rows), y, k, 0,
                     reinterpret_cast<long long*>(frame), pr, static_cast<cudaStream_t>(stream));
}

VP3D_EXPORT int vp3d_stream_push_counts(vp3d_plan* p, void* state, const float* x, int k,
                                        const uint8_t* start_mask, const int32_t* end,
                                        const int64_t* x_rows, const int64_t* y_rows, float* y,
                                        int64_t* frame, const int32_t* count, void* stream) {
  return stream_push("stream_push_counts", p, state, x, k, start_mask, end, count, x_rows, y_rows,
                     y, frame, 0, ProvRequest(), stream);
}

VP3D_EXPORT int vp3d_stream_push_provisional(vp3d_plan* p, void* state, const float* x, int k,
                                             const uint8_t* start_mask, const int32_t* end,
                                             const int32_t* count, float* y, int64_t* frame,
                                             float* y_prov, int64_t* frame_prov, void* stream) {
  if (!y_prov || !frame_prov)
    return fail(VP3D_ERR_INVALID, "stream_push_provisional: null y_prov or frame_prov");
  ProvRequest pr;
  pr.y = y_prov;
  pr.frame = reinterpret_cast<long long*>(frame_prov);
  return stream_push("stream_push_provisional", p, state, x, k, start_mask, end, count, nullptr,
                     nullptr, y, frame, VP3D_STREAM_PROVISIONAL, pr, stream);
}

VP3D_EXPORT int vp3d_stream_push_held(vp3d_plan* p, void* state, const float* x, int k,
                                      const uint8_t* start_mask, const int32_t* end,
                                      const int32_t* count, const int32_t* held, int max_held,
                                      int rows, float* y, int64_t* frame, float* y_prov,
                                      int64_t* frame_prov, void* stream) {
  if (!y_prov || !frame_prov || !held)
    return fail(VP3D_ERR_INVALID, "stream_push_held: null y_prov, frame_prov or held");
  if (max_held < 0)
    return fail(VP3D_ERR_INVALID, "stream_push_held: max_held must be >= 0 (got %d)", max_held);
  ProvRequest pr;
  pr.y = y_prov;
  pr.frame = reinterpret_cast<long long*>(frame_prov);
  pr.held = held;
  pr.max_held = max_held;
  pr.rows = rows;
  return stream_push("stream_push_held", p, state, x, k, start_mask, end, count, nullptr, nullptr,
                     y, frame, VP3D_STREAM_HELD, pr, stream);
}

VP3D_EXPORT int vp3d_stream_push_ex(vp3d_plan* p, void* state, const float* x, int k,
                                    const uint8_t* start_mask, const int32_t* end,
                                    const int64_t* x_rows, const int64_t* y_rows, float* y,
                                    int64_t* frame, void* stream) {
  return stream_push("stream_push_ex", p, state, x, k, start_mask, end, nullptr, x_rows, y_rows, y,
                     frame, 0, ProvRequest(), stream);
}

VP3D_EXPORT int vp3d_stream_push(vp3d_plan* p, void* state, const float* x, int k,
                                 const uint8_t* start_mask, float* y, int64_t* frame,
                                 void* stream) {
  return stream_push("stream_push", p, state, x, k, start_mask, nullptr, nullptr, nullptr, nullptr,
                     y, frame, 0, ProvRequest(), stream);
}

VP3D_EXPORT int vp3d_stream_finish(vp3d_plan* p, void* state, float* y, int64_t* frame,
                                   void* stream) {
  if (!state) return fail(VP3D_ERR_INVALID, "stream_finish: null state");
  if (!p) return fail(VP3D_ERR_INVALID, "stream_finish: null plan");
  StreamHost* h = nullptr;
  VP3D_TRY(stream_lookup(p, state, "stream_finish", &h));
  if (!p->conv_packed || !p->bn_packed)
    return fail(VP3D_ERR_STATE, "stream_finish: vp3d_set_weights has not been called");
  const int la = stream_lookahead(p);
  if (la > 0 && (!y || !frame)) return fail(VP3D_ERR_INVALID, "stream_finish: null y or frame");
  VP3D_TRY(stream_int8_ready(p, *h, "stream_finish"));
  uint8_t* base = ws_base(state);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int launches = 0;
  for (int off = 0; off < la; off += h->K) {
    const int k = la - off < h->K ? la - off : h->K;
    VP3D_TRY(stream_step(p, base, *h, nullptr, k, nullptr, nullptr, nullptr, nullptr, nullptr, y,
                         la, off, reinterpret_cast<long long*>(frame), ProvRequest(), s));
    launches += p->last_launches;
  }
  // every slot idle in the buffer the next push reads
  CUDA_TRY(cudaMemsetAsync(base + stream_layout(p, h->S, h->K, h->flags).active +
                               (size_t)h->parity * h->S, 0, h->S, s));
  p->last_launches = launches;
  return VP3D_OK;
}

// Bytes of one slot's record in a slot blob (the `flags` of its session; AUGMENT and INT8 shape it).
VP3D_EXPORT size_t vp3d_stream_slot_bytes(const vp3d_plan* p, int flags) {
  if (!p || (flags & ~kStreamFlags) || ((flags & VP3D_STREAM_INT8) && !p->int8)) return 0;
  return (size_t)slot_vecs(p, flags) * 16;
}

VP3D_EXPORT int vp3d_stream_export(vp3d_plan* p, void* state, const int32_t* slots, int n,
                                   void* blob, size_t blob_bytes,
                                   vp3d_stream_slots_header* header, void* stream) {
  const char* what = "stream_export";
  StreamHost* h = nullptr;
  SlotArgs a;
  VP3D_TRY(slot_transfer_args(what, p, state, slots, n, blob, blob_bytes, header, false, &h, &a));
  memset(header, 0, sizeof(*header));
  header->version = VP3D_STREAM_SLOTS_VERSION;
  header->n = n;
  header->cfg = p->cfg;
  header->flags = h->flags & (VP3D_STREAM_AUGMENT | VP3D_STREAM_INT8);
  header->rings = a.rings;
  header->planes = p->planes;
  header->f16 = p->f16;
  header->lookahead = stream_lookahead(p);
  for (int l = 0; l < a.rings; ++l) {
    header->H[l] = a.ring[l].H;
    header->ld[l] = a.ring[l].ld;
  }
  header->int8_snap = h->int8_snap;
  header->int8_mask = h->int8_mask;
  memcpy(header->act_scale, h->act_scale, sizeof(header->act_scale));
  header->slot_bytes = a.slot_vecs * 16;
  return slot_transfer_launch(stream_export_kernel, p, a, slots, n, blob,
                              static_cast<cudaStream_t>(stream));
}

VP3D_EXPORT int vp3d_stream_import(vp3d_plan* p, void* state, const int32_t* slots, int n,
                                   const void* blob, size_t blob_bytes,
                                   const vp3d_stream_slots_header* header, void* stream) {
  const char* what = "stream_import";
  StreamHost* h = nullptr;
  SlotArgs a;
  VP3D_TRY(slot_transfer_args(what, p, state, slots, n, blob, blob_bytes, header, true, &h, &a));
  if (header->version != VP3D_STREAM_SLOTS_VERSION)
    return fail(VP3D_ERR_STATE, "%s: header version %d, expected %d", what, header->version,
                VP3D_STREAM_SLOTS_VERSION);
  if (header->n != n)
    return fail(VP3D_ERR_STATE, "%s: the blob holds %d slots, %d listed", what, header->n, n);
  const vp3d_config &c0 = header->cfg, &c1 = p->cfg;
  bool same = c0.num_joints_in == c1.num_joints_in && c0.in_features == c1.in_features &&
              c0.num_joints_out == c1.num_joints_out && c0.num_widths == c1.num_widths &&
              c0.causal == c1.causal && c0.channels == c1.channels && c0.dense == c1.dense &&
              c0.variant == c1.variant && c0.precision == c1.precision;
  for (int i = 0; same && i < c1.num_widths && i < VP3D_MAX_WIDTHS; ++i)
    same = c0.filter_widths[i] == c1.filter_widths[i];
  if (!same)
    return fail(VP3D_ERR_STATE, "%s: the blob comes from another model configuration or precision",
                what);
  const int shape = VP3D_STREAM_AUGMENT | VP3D_STREAM_INT8;
  if (header->flags != (h->flags & shape))
    return fail(VP3D_ERR_STATE, "%s: the blob has flags 0x%x (AUGMENT | INT8), the session 0x%x", what,
                (unsigned)header->flags, (unsigned)(h->flags & shape));
  bool geometry = header->rings == a.rings && header->planes == p->planes &&
                  header->f16 == p->f16 && header->lookahead == stream_lookahead(p) &&
                  header->slot_bytes == a.slot_vecs * 16;
  for (int l = 0; geometry && l < a.rings; ++l)
    geometry = header->H[l] == a.ring[l].H && header->ld[l] == a.ring[l].ld;
  if (!geometry)
    return fail(VP3D_ERR_STATE, "%s: the blob's ring geometry differs from the session's", what);
  if (header->int8_snap) {
    // the imported history holds this quantisation: the plan's and the session's must be it
    const size_t scale_bytes = sizeof(float) * 2 * p->nb;
    if (header->int8_mask != p->int8_mask || memcmp(header->act_scale, p->act_scale, scale_bytes))
      return fail(VP3D_ERR_STATE, "%s: the blob's int8 blocks or activation scales differ from the "
                  "plan's", what);
    if (h->int8_snap &&
        (h->int8_mask != header->int8_mask || memcmp(h->act_scale, header->act_scale, scale_bytes)))
      return fail(VP3D_ERR_STATE, "%s: the blob's int8 blocks or activation scales differ from the "
                  "session's", what);
  }
  VP3D_TRY(slot_transfer_launch(stream_import_kernel, p, a, slots, n, const_cast<void*>(blob),
                                static_cast<cudaStream_t>(stream)));
  if (header->int8_snap && !h->int8_snap) {
    h->int8_snap = true;
    h->int8_mask = header->int8_mask;
    memcpy(h->act_scale, header->act_scale, sizeof(h->act_scale));
  }
  return VP3D_OK;
}
