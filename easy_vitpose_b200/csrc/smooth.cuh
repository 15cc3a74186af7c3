// Keypoint smoothing on the device (vpb_smoother_update): the reference's OneEuroFilter
// (easy_ViTPose/vit_utils/post_processing/one_euro_filter.py) kept per track id, for S streams in two launches, equal to the
// reference class composed per id as float64 values.  oracle/one_euro_oracle.py states the composition; in short, per
// stream and update u (the stream's count of accepted updates) with clock c:
//
//   1. forget every id absent from more than max_gap updates in a row (u - u_last - 1 > max_gap);
//   2. a known id outputs f(x, t_e): fps mode t_e = c - c_last (c defaults to u), realtime mode t_e = (c - c_last) * d_cutoff;
//   3. a new id takes a free slot and outputs x unchanged (the constructor filters nothing);
//   4. every id of the update gets c_last = c, u_last = u.
//
// The filter follows numpy's promotion: on the first call after construction x_prev is still float32, so x - x_prev is a
// float32 subtraction; afterwards it is float64.  Every float64 add, multiply and divide is a __d*_rn intrinsic, which nvcc
// never contracts into an FMA, in the reference's evaluation order ((2 pi) cutoff) t_e, r / (r + 1), a x + (1 - a) x_prev.
// A coordinate with x <= 0 outputs -10 and stores it as x_prev; NaN is not masked.
//
// smooth_assign: one CTA per stream, one thread per slot and per row.  The stream's row offset (a prefix of the counts
//   before it), the limits, the forget step, the id match against the 128-slot table, duplicates, the free slots handed to
//   new ids in row order (ballot prefix on both sides), each row's (slot, t_e, mode), the slot table and the update count.
// smooth_apply: one thread per (row, keypoint) of each stream.  Runs the filter on both coordinates, writes the float64
//   result when asked and the float32 (y, x) of the caller's [n, K, 3] keypoints in place, and stores the slot state.
// A stream whose count is negative or above SMOOTH_MAX, whose rows would run past the caller's n, that names an id twice,
// or that would hold more than SMOOTH_MAX ids is left as it was (no rows written, update count kept) and sets a status bit.
// Both launches read everything from device memory, so they can be captured in a CUDA graph.
#pragma once
#include <cstdint>

constexpr int SMOOTH_MAX = 128;                  // VPB_SMOOTH_MAX: rows and live ids per stream; one thread each
constexpr int SMOOTH_THREADS = 128;
constexpr int SMOOTH_APPLY_THREADS = 256;
constexpr int SMOOTH_MAX_K = 144;
constexpr int SMOOTH_DUPLICATE_ID = 1;           // VPB_SMOOTH_DUPLICATE_ID
constexpr int SMOOTH_OVER_CAPACITY = 2;          // VPB_SMOOTH_OVER_CAPACITY
constexpr int SMOOTH_NEW = 0, SMOOTH_FIRST = 1, SMOOTH_KNOWN = 2;   // row modes: new id, first filter call, later call
static_assert(SMOOTH_THREADS == SMOOTH_MAX, "one thread per slot and per row");

struct SmoothParams {
  float* kpts;                 // [n, K, 3] (y, x, score) in/out, rows concatenated stream by stream
  const int32_t* counts;       // [S]
  const int32_t* ids;          // [n]
  const double* clock;         // [S] or null (the update count)
  double* out;                 // [n, K, 2] or null
  double* x_prev;              // [S, SMOOTH_MAX, K, 2]
  double* dx_prev;             // [S, SMOOTH_MAX, K, 2]
  double* c_last;              // [S, SMOOTH_MAX]
  int32_t* slot_id;            // [S, SMOOTH_MAX]
  int32_t* slot_u;             // [S, SMOOTH_MAX] u_last, -1 = free
  int32_t* slot_first;         // [S, SMOOTH_MAX] the first filter call is pending
  int32_t* updates;            // [S] accepted updates
  int32_t* row_slot;           // [S, SMOOTH_MAX] scratch: each row's slot
  int32_t* row_mode;           // [S, SMOOTH_MAX] scratch: SMOOTH_NEW / FIRST / KNOWN
  double* row_te;              // [S, SMOOTH_MAX] scratch: each row's t_e
  int32_t* rows;               // [S] rows to filter, -1 = stream skipped
  int32_t* row0;               // [S] the stream's first row
  int32_t* status;
  int num_streams, k, n, max_gap, realtime;
  double min_cutoff, beta, d_cutoff, deriv_cutoff, dx0;   // deriv_cutoff: fps in fps mode, d_cutoff in realtime mode
};

__device__ __forceinline__ double s_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double s_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double s_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double s_div(double a, double b) { return __ddiv_rn(a, b); }

// smoothing_factor: r = 2 * np.pi * cutoff * t_e (left to right), r / (r + 1)
__device__ __forceinline__ double smooth_factor(double te, double cutoff) {
  const double r = s_mul(s_mul(2.0 * 3.141592653589793, cutoff), te);
  return s_div(r, s_add(r, 1.0));
}

// exclusive prefix count of `flag` over the block's threads in thread order; *total gets the block's count
__device__ __forceinline__ int smooth_scan(bool flag, int* warp_cnt, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_cnt[warp] = __popc(m);
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < SMOOTH_THREADS / 32; ++w) {
    before += w < warp ? warp_cnt[w] : 0;
    all += warp_cnt[w];
  }
  __syncthreads();
  *total = all;
  return before + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(SMOOTH_THREADS) smooth_assign(SmoothParams q) {
  __shared__ long long red[SMOOTH_THREADS / 32];
  __shared__ int warp_cnt[SMOOTH_THREADS / 32];
  __shared__ int tab_id[SMOOTH_MAX], tab_u[SMOOTH_MAX], row_id[SMOOTH_MAX], free_slot[SMOOTH_MAX];
  __shared__ int new_first[SMOOTH_MAX];
  __shared__ double new_c[SMOOTH_MAX];
  const int st = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long M = SMOOTH_MAX;

  // the stream's first row: the rows of the streams before it (a negative count holds none)
  long long before = 0;
  for (int j = tid; j < st; j += SMOOTH_THREADS) before += q.counts[j] > 0 ? q.counts[j] : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) before += __shfl_down_sync(0xffffffffu, before, o);
  if (lane == 0) red[warp] = before;
  __syncthreads();
  before = 0;
#pragma unroll
  for (int w = 0; w < SMOOTH_THREADS / 32; ++w) before += red[w];
  const int n = q.counts[st];
  if (n < 0 || n > SMOOTH_MAX || before + n > q.n) {     // uniform over the block
    if (tid == 0) { atomicOr(q.status, SMOOTH_OVER_CAPACITY); q.rows[st] = -1; }
    return;
  }

  // forget (step 1), then match the rows' ids against the live slots
  const int u = q.updates[st];
  const int su = q.slot_u[st * M + tid];
  const bool live = su >= 0 && static_cast<long long>(u) - su - 1 <= q.max_gap;
  tab_id[tid] = q.slot_id[st * M + tid];
  tab_u[tid] = live ? su : -1;
  const int id = tid < n ? q.ids[before + tid] : 0;
  row_id[tid] = id;
  __syncthreads();
  int slot = -1;
  bool dup = false;
  if (tid < n) {
    for (int j = 0; j < SMOOTH_MAX; ++j)
      if (tab_u[j] >= 0 && tab_id[j] == id) slot = j;
    for (int j = 0; j < n; ++j) dup |= j != tid && row_id[j] == id;
  }
  if (__syncthreads_or(dup)) {
    if (tid == 0) { atomicOr(q.status, SMOOTH_DUPLICATE_ID); q.rows[st] = -1; }
    return;
  }
  const bool is_new = tid < n && slot < 0;
  int num_new, num_free;
  const int rank_new = smooth_scan(is_new, warp_cnt, &num_new);
  const int rank_free = smooth_scan(!live, warp_cnt, &num_free);
  if (num_new > num_free) {                      // live ids + new ids > SMOOTH_MAX
    if (tid == 0) { atomicOr(q.status, SMOOTH_OVER_CAPACITY); q.rows[st] = -1; }
    return;
  }
  if (!live) free_slot[rank_free] = tid;
  new_first[tid] = 0;
  __syncthreads();
  if (is_new) slot = free_slot[rank_new];

  // each row's slot, mode and t_e; the slots of this update take id, u_last = u, c_last = c
  const double c = q.clock ? q.clock[st] : static_cast<double>(u);
  if (tid < n) {
    int mode = SMOOTH_NEW;
    double te = 0.0;
    if (!is_new) {
      mode = q.slot_first[st * M + slot] ? SMOOTH_FIRST : SMOOTH_KNOWN;
      te = s_sub(c, q.c_last[st * M + slot]);
      if (q.realtime) te = s_mul(te, q.d_cutoff);
    }
    q.row_slot[st * M + tid] = slot;
    q.row_mode[st * M + tid] = mode;
    q.row_te[st * M + tid] = te;
    tab_id[slot] = id;
    tab_u[slot] = u;
    new_first[slot] = is_new ? 1 : 0;
    new_c[slot] = c;
  }
  __syncthreads();
  const bool used = tab_u[tid] == u;             // in this update
  q.slot_id[st * M + tid] = tab_id[tid];
  q.slot_u[st * M + tid] = tab_u[tid];
  if (used) {
    q.slot_first[st * M + tid] = new_first[tid];
    q.c_last[st * M + tid] = new_c[tid];
  }
  if (tid == 0) {
    q.rows[st] = n;
    q.row0[st] = static_cast<int>(before);
    q.updates[st] = u + 1;
  }
}

// grid (ceil(SMOOTH_MAX * K / SMOOTH_APPLY_THREADS), S)
__global__ void __launch_bounds__(SMOOTH_APPLY_THREADS) smooth_apply(SmoothParams q) {
  const int st = blockIdx.y, K = q.k;
  const int n = q.rows[st];
  const int e = blockIdx.x * SMOOTH_APPLY_THREADS + threadIdx.x;
  if (e >= n * K) return;                        // also n = -1: the stream was skipped
  const int j = e / K, kp = e - j * K;
  const long long M = SMOOTH_MAX;
  const int slot = q.row_slot[st * M + j], mode = q.row_mode[st * M + j];
  const double te = q.row_te[st * M + j];
  const long long r = q.row0[st] + j;
  float* x_io = q.kpts + (r * K + kp) * 3;
  double* xp = q.x_prev + ((st * M + slot) * K + kp) * 2;
  double* dxp = q.dx_prev + ((st * M + slot) * K + kp) * 2;
  double res[2];
  if (mode == SMOOTH_NEW) {                      // OneEuroFilter(x0, dx0, ...): x_prev = x0, dx_prev = dx0, output x0
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      res[c] = static_cast<double>(x_io[c]);
      xp[c] = res[c];
      dxp[c] = q.dx0;
    }
  } else {
    const double a_d = smooth_factor(te, q.deriv_cutoff);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float xf = x_io[c];
      const double x = static_cast<double>(xf), x_prev = xp[c];
      // first call: float32 x - float32 x_prev, then the float64 division
      const double diff = mode == SMOOTH_FIRST ? static_cast<double>(__fsub_rn(xf, static_cast<float>(x_prev))) : s_sub(x, x_prev);
      const double dx = s_div(diff, te);
      const double dx_hat = s_add(s_mul(a_d, dx), s_mul(s_sub(1.0, a_d), dxp[c]));
      const double cutoff = s_add(q.min_cutoff, s_mul(q.beta, fabs(dx_hat)));
      const double a = smooth_factor(te, cutoff);
      double x_hat = s_add(s_mul(a, x), s_mul(s_sub(1.0, a), x_prev));
      if (xf <= 0.0f) x_hat = -10.0;             // missing keypoint (NaN is not masked)
      xp[c] = x_hat;
      dxp[c] = dx_hat;
      res[c] = x_hat;
      x_io[c] = __double2float_rn(x_hat);
    }
  }
  if (q.out) {
    double* o = q.out + (r * K + kp) * 2;
    o[0] = res[0];
    o[1] = res[1];
  }
}
