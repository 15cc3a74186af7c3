// SORT on the device (vpb_tracker_update): easy_ViTPose/sort.py's Sort.update for S streams in two launches, equal to the
// reference as float64 values.  oracle/sort_oracle.py states the contract and the reasons; in short:
//
//   - P keeps an exact block structure ((x, vx), (y, vy), (s, vs) 2 x 2 blocks and the scalar r; everything else stays +-0), S
//     is diagonal, and every sum filterpy forms has at most two nonzero terms.  So the per-element formulas below give the
//     values the dense np.dot / np.linalg.inv filter gives, provided each operation rounds once: every add, multiply, divide
//     and square root here is a __d*_rn intrinsic, which nvcc never contracts into an FMA.  A track carries 13 P doubles.
//   - Association is scipy's linear_sum_assignment (Crouse's shortest augmenting path) with its tie rule, because zero IoU is
//     everywhere and the tie decides which detections become new tracks, and so their ids.
//
// track_associate: one CTA per stream, one thread per track or detection.  Predict, stable compaction of NaN tracks, the IoU
//   matrix in shared memory (fp64, at most 128 x 128), the one-to-one shortcut, else the LSAP (column scan as a block
//   reduction, augmentation serial), the unmatched detections in reference order, and the Kalman update of the matched
//   tracks.  Records how many tracks each stream creates and which detections they come from.
// track_emit: one CTA per stream.  Exclusive scan of the new-track counts over the streams (ids in stream order, then
//   creation order), the new tracks' states, the output rows in reversed list order, the death rule, the id counter.
// A stream with a negative count, more than TRACK_MAX detections, a non-finite row or x2 <= x1 or y2 <= y1, or that would
// hold more than TRACK_MAX tracks is left as it was, emits no rows and sets a status bit.  Both launches read everything
// from device memory, so they can be captured in a CUDA graph.
#pragma once
#include <cstdint>

constexpr int TRACK_MAX = 128;                   // VPB_TRACK_MAX: detections and live tracks per stream; one thread each
constexpr int TRACK_THREADS = 128;
constexpr int TRACK_FIELDS = 21;                 // x[7], P[13] (3 blocks of (pp, pv, vp, vv), then P33), score
constexpr int TRACK_BAD_ROW = 1;                 // VPB_TRACK_BAD_ROW
constexpr int TRACK_OVER_CAPACITY = 2;           // VPB_TRACK_OVER_CAPACITY
static_assert(TRACK_THREADS == TRACK_MAX, "one thread per track slot");

struct TrackParams {
  const double* dets;          // [S, TRACK_MAX, 5] (x1, y1, x2, y2, score)
  const int32_t* counts;       // [S]
  double* rows;                // [S, TRACK_MAX, 6] out (x1, y1, x2, y2, score, id + 1)
  int32_t* boxes;              // [S, TRACK_MAX, 4] out, rows rounded half to even
  int32_t* out_counts;         // [S] out
  double* state;               // [S, TRACK_FIELDS, TRACK_MAX]
  long long* ids;              // [S, TRACK_MAX]
  int32_t* tsu;                // [S, TRACK_MAX] time_since_update
  int32_t* hits;               // [S, TRACK_MAX] hit_streak
  int32_t* num_tracks;         // [S]
  int32_t* frame_count;        // [S]
  int32_t* num_new;            // [S] tracks created by the last update, -1 = stream skipped
  int32_t* new_det;            // [S, TRACK_MAX] the detections they come from, in creation order
  long long* next_id;          // KalmanBoxTracker.count
  long long* id_base;          // next_id as the update found it
  int32_t* status;
  int num_streams, max_age, min_hits;
  double iou_threshold;
};

struct TrackSmem {
  double iou[TRACK_MAX * TRACK_MAX];             // [det][track]
  double det[TRACK_MAX][5];
  double tbox[TRACK_MAX][4];                     // predicted boxes of the kept tracks
  double u[TRACK_MAX], v[TRACK_MAX], spc[TRACK_MAX];
  double red_val[TRACK_THREADS / 32];
  int red_it[TRACK_THREADS / 32], red_free[TRACK_THREADS / 32];
  int path[TRACK_MAX], col4row[TRACK_MAX], row4col[TRACK_MAX], remaining[TRACK_MAX];
  int det_match[TRACK_MAX], trk_det[TRACK_MAX], new_det[TRACK_MAX];
  int warp_cnt[TRACK_THREADS / 32];
  int num_new;
  unsigned char sr[TRACK_MAX], sc[TRACK_MAX];
};

// ------------------------------------------------------------------------------------------------ IEEE helpers (no FMA)
__device__ __forceinline__ double t_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double t_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double t_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double t_div(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double t_max(double a, double b) { return a > b ? a : b; }
__device__ __forceinline__ double t_min(double a, double b) { return a < b ? a : b; }

// convert_x_to_bbox (sort.py:81-91)
__device__ __forceinline__ void x_to_bbox(const double* x, double* b) {
  const double w = __dsqrt_rn(t_mul(x[2], x[3]));
  const double h = t_div(x[2], w);
  b[0] = t_sub(x[0], t_div(w, 2.0));
  b[1] = t_sub(x[1], t_div(h, 2.0));
  b[2] = t_add(x[0], t_div(w, 2.0));
  b[3] = t_add(x[1], t_div(h, 2.0));
}
// convert_bbox_to_z (sort.py:66-78)
__device__ __forceinline__ void bbox_to_z(const double* d, double* z) {
  const double w = t_sub(d[2], d[0]), h = t_sub(d[3], d[1]);
  z[0] = t_add(d[0], t_div(w, 2.0));
  z[1] = t_add(d[1], t_div(h, 2.0));
  z[2] = t_mul(w, h);
  z[3] = t_div(w, h);
}
// iou_batch (sort.py:47-63), one element
__device__ __forceinline__ double iou_one(const double* d, const double* t) {
  const double w = t_max(0.0, t_sub(t_min(d[2], t[2]), t_max(d[0], t[0])));
  const double h = t_max(0.0, t_sub(t_min(d[3], t[3]), t_max(d[1], t[1])));
  const double wh = t_mul(w, h);
  return t_div(wh, t_sub(t_add(t_mul(t_sub(d[2], d[0]), t_sub(d[3], d[1])), t_mul(t_sub(t[2], t[0]), t_sub(t[3], t[1]))), wh));
}

// KalmanBoxTracker.predict's filter part: the x[6] + x[2] <= 0 guard, x = Fx, P = 1.0 (F P F^T) + Q
__device__ __forceinline__ void kf_predict(double* x, double* P) {
  const double q_vel[3] = {1.0 * 0.01, 1.0 * 0.01, (1.0 * 0.01) * 0.01};
  if (t_add(x[6], x[2]) <= 0.0) x[6] = t_mul(x[6], 0.0);
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    x[b] = t_add(x[b], x[b + 4]);
    const double a = P[4 * b], u = P[4 * b + 1], c = P[4 * b + 2], d = P[4 * b + 3];
    P[4 * b] = t_add(t_add(t_add(a, c), t_add(u, d)), 1.0);
    P[4 * b + 1] = t_add(u, d);
    P[4 * b + 2] = t_add(c, d);
    P[4 * b + 3] = t_add(d, q_vel[b]);
  }
  P[12] = t_add(P[12], 1.0);
}

// filterpy 1.4.5 KalmanFilter.update with H = [I4 0], R = diag(1, 1, 10, 10), the Joseph form
__device__ __forceinline__ void kf_update(double* x, double* P, const double* z) {
  const double r[4] = {1.0, 1.0, 10.0, 10.0};
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    const double a = P[4 * b], u = P[4 * b + 1], c = P[4 * b + 2], d = P[4 * b + 3];
    const double y = t_sub(z[b], x[b]);
    const double si = t_div(1.0, t_add(a, r[b]));
    const double kp = t_mul(a, si), kv = t_mul(c, si), nkv = -kv;
    x[b] = t_add(x[b], t_mul(kp, y));
    x[b + 4] = t_add(x[b + 4], t_mul(kv, y));
    const double ik = t_sub(1.0, kp);
    const double a00 = t_mul(ik, a), a01 = t_mul(ik, u);                          // (I - KH) P
    const double a10 = t_add(t_mul(nkv, a), c), a11 = t_add(t_mul(nkv, u), d);
    const double krp = t_mul(kp, r[b]), krv = t_mul(kv, r[b]);                    // K R
    P[4 * b] = t_add(t_mul(a00, ik), t_mul(krp, kp));
    P[4 * b + 1] = t_add(t_add(t_mul(a00, nkv), a01), t_mul(krp, kv));
    P[4 * b + 2] = t_add(t_mul(a10, ik), t_mul(krv, kp));
    P[4 * b + 3] = t_add(t_add(t_mul(a10, nkv), a11), t_mul(krv, kv));
  }
  const double p = P[12];
  const double k = t_mul(p, t_div(1.0, t_add(p, r[3])));
  x[3] = t_add(x[3], t_mul(k, t_sub(z[3], x[3])));
  const double ik = t_sub(1.0, k);
  P[12] = t_add(t_mul(t_mul(ik, p), ik), t_mul(t_mul(k, r[3]), k));
}

// exclusive prefix count of `flag` over the block's threads in thread order; *total gets the block's count
__device__ __forceinline__ int track_scan(bool flag, int* warp_cnt, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_cnt[warp] = __popc(m);
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < TRACK_THREADS / 32; ++w) {
    before += w < warp ? warp_cnt[w] : 0;
    all += warp_cnt[w];
  }
  __syncthreads();
  *total = all;
  return before + __popc(m & ((1u << lane) - 1u));
}

// The LSAP column pick: the minimum of the shortest-path costs; among equal minima the LAST position of an unassigned
// column, else the FIRST position.  `a` better than `b`?
__device__ __forceinline__ bool lsap_better(double av, int ai, int af, double bv, int bi, int bf) {
  if (ai < 0) return false;
  if (bi < 0) return true;
  if (av != bv) return av < bv;
  if (af != bf) return af > bf;
  return af ? ai > bi : ai < bi;
}

// scipy's rectangular_lsap on cost = -iou (rows = dets unless that is the taller side), leaving s.det_match[d] = track or -1
__device__ void track_lsap(TrackSmem& s, int n, int nt) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool tr = nt < n;                        // tall matrix: solve the transpose
  const int nr = tr ? nt : n, nc = tr ? n : nt;
  s.u[tid] = 0.0; s.v[tid] = 0.0;
  s.path[tid] = -1; s.col4row[tid] = -1; s.row4col[tid] = -1;
  for (int cur = 0; cur < nr; ++cur) {
    s.remaining[tid] = nc - 1 - tid;
    s.spc[tid] = __longlong_as_double(0x7ff0000000000000LL);
    s.sr[tid] = 0; s.sc[tid] = 0;
    __syncthreads();
    int i = cur, num = nc, sink = -1;
    double min_val = 0.0;
    while (sink < 0) {
      if (tid == 0) s.sr[i] = 1;
      double val = 0.0;
      int it = -1, fr = 0;
      if (tid < num) {
        const int j = s.remaining[tid];
        const double c = -(tr ? s.iou[j * TRACK_MAX + i] : s.iou[i * TRACK_MAX + j]);
        const double r = t_sub(t_sub(t_add(min_val, c), s.u[i]), s.v[j]);
        if (r < s.spc[j]) { s.path[j] = i; s.spc[j] = r; }
        val = s.spc[j]; it = tid; fr = s.row4col[j] == -1;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_down_sync(0xffffffffu, val, o);
        const int oi = __shfl_down_sync(0xffffffffu, it, o), of = __shfl_down_sync(0xffffffffu, fr, o);
        if (lsap_better(ov, oi, of, val, it, fr)) { val = ov; it = oi; fr = of; }
      }
      if (lane == 0) { s.red_val[warp] = val; s.red_it[warp] = it; s.red_free[warp] = fr; }
      __syncthreads();
      double bv = s.red_val[0];
      int bi = s.red_it[0], bf = s.red_free[0];
#pragma unroll
      for (int w = 1; w < TRACK_THREADS / 32; ++w)
        if (lsap_better(s.red_val[w], s.red_it[w], s.red_free[w], bv, bi, bf)) { bv = s.red_val[w]; bi = s.red_it[w]; bf = s.red_free[w]; }
      min_val = bv;
      const int j = s.remaining[bi];
      if (s.row4col[j] == -1) sink = j; else i = s.row4col[j];
      --num;
      __syncthreads();                           // everyone has read remaining[] and row4col[]
      if (tid == 0) { s.sc[j] = 1; s.remaining[bi] = s.remaining[num]; }
      __syncthreads();
    }
    if (tid < nr && s.sr[tid] && tid != cur) s.u[tid] = t_add(s.u[tid], t_sub(min_val, s.spc[s.col4row[tid]]));
    if (tid == cur) s.u[tid] = t_add(s.u[tid], min_val);
    if (tid < nc && s.sc[tid]) s.v[tid] = t_sub(s.v[tid], t_sub(min_val, s.spc[tid]));
    __syncthreads();
    if (tid == 0) {
      int j = sink;
      while (true) {
        const int r = s.path[j];
        s.row4col[j] = r;
        const int prev = s.col4row[r];
        s.col4row[r] = j;
        j = prev;
        if (r == cur) break;
      }
    }
    __syncthreads();
  }
  s.det_match[tid] = -1;
  __syncthreads();
  if (tid < nr) {
    if (tr) s.det_match[s.col4row[tid]] = tid;
    else s.det_match[tid] = s.col4row[tid];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(TRACK_THREADS, 1) track_associate(TrackParams q) {
  extern __shared__ __align__(16) unsigned char track_smem_raw[];
  TrackSmem& s = *reinterpret_cast<TrackSmem*>(track_smem_raw);
  const int st = blockIdx.x, tid = threadIdx.x;
  if (st == 0 && tid == 0) *q.id_base = *q.next_id;
  const int n = q.counts[st];
  if (n < 0 || n > TRACK_MAX) {                  // uniform over the block
    if (tid == 0) { atomicOr(q.status, TRACK_OVER_CAPACITY); q.num_new[st] = -1; }
    return;
  }
  bool bad = false;
  if (tid < n) {
    const double* d = q.dets + ((long long)st * TRACK_MAX + tid) * 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) { s.det[tid][k] = d[k]; bad |= !isfinite(d[k]); }
    bad |= !(d[2] > d[0]) || !(d[3] > d[1]);
  }
  if (__syncthreads_or(bad)) {
    if (tid == 0) { atomicOr(q.status, TRACK_BAD_ROW); q.num_new[st] = -1; }
    return;
  }

  // predict every track (list order = thread order), then drop the NaN ones keeping the order of the rest
  const int T = q.num_tracks[st];
  double* sb = q.state + (long long)st * TRACK_FIELDS * TRACK_MAX;
  double x[7], P[13], score = 0.0;
  long long id = 0;
  int tsu = 0, hs = 0;
  bool keep = false;
  double b[4];
  if (tid < T) {
#pragma unroll
    for (int k = 0; k < 7; ++k) x[k] = sb[k * TRACK_MAX + tid];
#pragma unroll
    for (int k = 0; k < 13; ++k) P[k] = sb[(7 + k) * TRACK_MAX + tid];
    score = sb[20 * TRACK_MAX + tid];
    id = q.ids[st * TRACK_MAX + tid];
    tsu = q.tsu[st * TRACK_MAX + tid];
    hs = q.hits[st * TRACK_MAX + tid];
    kf_predict(x, P);
    if (tsu > 0) hs = 0;
    ++tsu;
    x_to_bbox(x, b);
    keep = !(isnan(b[0]) || isnan(b[1]) || isnan(b[2]) || isnan(b[3]));
  }
  int nt;
  const int pos = track_scan(keep, s.warp_cnt, &nt);   // the track's place in the compacted list
  if (keep) {
#pragma unroll
    for (int k = 0; k < 4; ++k) s.tbox[pos][k] = b[k];
  }
  s.trk_det[tid] = -1;
  s.det_match[tid] = -1;
  __syncthreads();

  // association (sort.py:158-200)
  const double thr = q.iou_threshold;
  if (n > 0 && nt > 0) {
    for (int e = tid; e < n * nt; e += TRACK_THREADS) {
      const int i = e / nt, j = e - i * nt;
      s.iou[i * TRACK_MAX + j] = iou_one(s.det[i], s.tbox[j]);
    }
    __syncthreads();
    int row_cnt = 0, row_j = -1, col_cnt = 0;
    if (tid < n)
      for (int j = 0; j < nt; ++j)
        if (s.iou[tid * TRACK_MAX + j] > thr) { ++row_cnt; row_j = j; }
    if (tid < nt)
      for (int i = 0; i < n; ++i) col_cnt += s.iou[i * TRACK_MAX + tid] > thr;
    const bool row_many = __syncthreads_or(row_cnt > 1), row_one = __syncthreads_or(row_cnt == 1);
    const bool col_many = __syncthreads_or(col_cnt > 1);
    if (!row_many && row_one && !col_many) {     // a.sum(1).max() == 1 and a.sum(0).max() == 1: np.where(a)
      s.det_match[tid] = tid < n && row_cnt == 1 ? row_j : -1;
      __syncthreads();
    } else {
      track_lsap(s, n, nt);
    }
  }

  // unmatched detections: never assigned (ascending), then the low-IoU pairs in matched (= detection) order
  if (tid == 0) {
    int k = 0;
    for (int d = 0; d < n; ++d)
      if (s.det_match[d] < 0) s.new_det[k++] = d;
    for (int d = 0; d < n; ++d) {
      const int t = s.det_match[d];
      if (t < 0) continue;
      if (s.iou[d * TRACK_MAX + t] < thr) s.new_det[k++] = d;
      else s.trk_det[t] = d;
    }
    s.num_new = k;
  }
  __syncthreads();
  const int k_new = s.num_new;
  if (nt + k_new > TRACK_MAX) {
    if (tid == 0) { atomicOr(q.status, TRACK_OVER_CAPACITY); q.num_new[st] = -1; }
    return;
  }

  // update the matched tracks, write the kept ones back in order
  if (keep) {
    const int d = s.trk_det[pos];
    if (d >= 0) {
      double z[4];
      bbox_to_z(s.det[d], z);
      kf_update(x, P, z);
      tsu = 0;
      ++hs;
      score = s.det[d][4];
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) sb[k * TRACK_MAX + pos] = x[k];
#pragma unroll
    for (int k = 0; k < 13; ++k) sb[(7 + k) * TRACK_MAX + pos] = P[k];
    sb[20 * TRACK_MAX + pos] = score;
    q.ids[st * TRACK_MAX + pos] = id;
    q.tsu[st * TRACK_MAX + pos] = tsu;
    q.hits[st * TRACK_MAX + pos] = hs;
  }
  if (tid < k_new) q.new_det[st * TRACK_MAX + tid] = s.new_det[tid];
  if (tid == 0) {
    q.num_tracks[st] = nt;
    q.num_new[st] = k_new;
    q.frame_count[st] += 1;
  }
}

__global__ void __launch_bounds__(TRACK_THREADS, 1) track_emit(TrackParams q) {
  __shared__ int warp_cnt[TRACK_THREADS / 32];
  __shared__ long long red[TRACK_THREADS / 32][2];
  const int st = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // ids: exclusive scan of the created tracks over the streams
  long long before = 0, all = 0;
  for (int j = tid; j < q.num_streams; j += TRACK_THREADS) {
    const long long c = q.num_new[j] > 0 ? q.num_new[j] : 0;
    all += c;
    before += j < st ? c : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    before += __shfl_down_sync(0xffffffffu, before, o);
    all += __shfl_down_sync(0xffffffffu, all, o);
  }
  if (lane == 0) { red[warp][0] = before; red[warp][1] = all; }
  __syncthreads();
  before = 0; all = 0;
#pragma unroll
  for (int w = 0; w < TRACK_THREADS / 32; ++w) { before += red[w][0]; all += red[w][1]; }
  const long long base = *q.id_base;
  if (st == 0 && tid == 0) *q.next_id = base + all;
  const int k_new = q.num_new[st];
  if (k_new < 0) {
    if (tid == 0) q.out_counts[st] = 0;
    return;
  }
  double* sb = q.state + (long long)st * TRACK_FIELDS * TRACK_MAX;
  const int T = q.num_tracks[st], L = T + k_new;
  // new tracks (KalmanBoxTracker.__init__): x = [z, 0, 0, 0], P0 = diag(10, 10, 10, 10, 1e4, 1e4, 1e4)
  if (tid < k_new) {
    const int t = T + tid;
    const double* d = q.dets + ((long long)st * TRACK_MAX + q.new_det[st * TRACK_MAX + tid]) * 5;
    double z[4];
    bbox_to_z(d, z);
    const double p0 = 1.0 * 10.0, p0v = (1.0 * 1000.0) * 10.0;
    const double P[13] = {p0, 0.0, 0.0, p0v, p0, 0.0, 0.0, p0v, p0, 0.0, 0.0, p0v, p0};
#pragma unroll
    for (int k = 0; k < 4; ++k) sb[k * TRACK_MAX + t] = z[k];
#pragma unroll
    for (int k = 4; k < 7; ++k) sb[k * TRACK_MAX + t] = 0.0;
#pragma unroll
    for (int k = 0; k < 13; ++k) sb[(7 + k) * TRACK_MAX + t] = P[k];
    sb[20 * TRACK_MAX + t] = d[4];
    q.ids[st * TRACK_MAX + t] = base + before + tid;
    q.tsu[st * TRACK_MAX + t] = 0;
    q.hits[st * TRACK_MAX + t] = 0;
  }
  __syncthreads();

  // rows from the reversed list (sort.py:249-266): thread r takes list entry L - 1 - r
  const int fc = q.frame_count[st];
  const int t = L - 1 - tid;
  bool emit = false;
  double row[6];
  if (tid < L) {
    double x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = sb[k * TRACK_MAX + t];
    x_to_bbox(x, row);
    row[4] = sb[20 * TRACK_MAX + t];
    row[5] = static_cast<double>(q.ids[st * TRACK_MAX + t] + 1);
    emit = q.tsu[st * TRACK_MAX + t] < 1 && (q.hits[st * TRACK_MAX + t] >= q.min_hits || fc <= q.min_hits);
  }
  const bool any = __syncthreads_or(emit);
  if (!any && q.counts[st] == 0) emit = tid < L;    // the empty-detections branch: every track, the dying ones included
  int m;
  const int p = track_scan(emit, warp_cnt, &m);
  if (emit) {
    double* o = q.rows + ((long long)st * TRACK_MAX + p) * 6;
    int32_t* ob = q.boxes + ((long long)st * TRACK_MAX + p) * 4;
#pragma unroll
    for (int k = 0; k < 6; ++k) o[k] = row[k];
#pragma unroll
    for (int k = 0; k < 4; ++k) ob[k] = __double2int_rn(row[k]);
  }
  if (tid == 0) q.out_counts[st] = m;

  // remove dead tracklets (time_since_update > max_age), keeping the order of the rest
  const bool alive = tid < L && q.tsu[st * TRACK_MAX + tid] <= q.max_age;
  double f[TRACK_FIELDS];
  long long id = 0;
  int tsu = 0, hs = 0;
  if (alive) {
#pragma unroll
    for (int k = 0; k < TRACK_FIELDS; ++k) f[k] = sb[k * TRACK_MAX + tid];
    id = q.ids[st * TRACK_MAX + tid];
    tsu = q.tsu[st * TRACK_MAX + tid];
    hs = q.hits[st * TRACK_MAX + tid];
  }
  int live;
  const int to = track_scan(alive, warp_cnt, &live);   // its barriers also order the reads above before the writes below
  if (alive && to != tid) {
#pragma unroll
    for (int k = 0; k < TRACK_FIELDS; ++k) sb[k * TRACK_MAX + to] = f[k];
    q.ids[st * TRACK_MAX + to] = id;
    q.tsu[st * TRACK_MAX + to] = tsu;
    q.hits[st * TRACK_MAX + to] = hs;
  }
  if (tid == 0) q.num_tracks[st] = live;
}
