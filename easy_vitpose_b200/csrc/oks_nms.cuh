// OKS NMS on the device (vpb_oks_nms, vpb_oks_iou): the reference's oks_iou, oks_nms and soft_oks_nms
// (easy_ViTPose/vit_utils/post_processing/nms.py:51-207) for F frames in one launch, one CTA per frame.
// oracle/oks_nms_oracle.py restates the arithmetic in numpy; in short, per frame of n people with keypoints [K, 3] float32,
// area and score float64:
//
//   order   the reference's scores.argsort()[::-1] evaluated with a stable argsort: descending, NaN above +inf, and among
//           equal scores the later position first.  soft_oks_nms re-sorts the remaining order every round, so its ties are
//           broken by position in that order, which is why the order array is kept rather than re-derived from indices.
//   OKS     dx, dy float32; dx*dx + dy*dy float32 (no FMA); / vars[k] / ((a_g + a_d) / 2 + 2^-52) / 2 in float64, left to
//           right; exp; numpy's pairwise sum over the candidate's visible keypoints (the `list(vg > t) and list(vd > t)` of
//           oks_iou keeps the candidate's mask alone); / count; rounded to float32.  No visible keypoint gives 0.
//   hard    keep the head of the order, drop every remaining person whose OKS against it is not <= thr (float32 compare,
//           so a NaN OKS drops), repeat until the order is empty.
//   soft    keep the head, rescale the rest by exp(-(o*o) / thr) in float32 times the float64 score, re-sort, repeat until
//           the order is empty or max_dets people are kept.
//   rescore (optional, before the sort) HRNet's evaluation rescoring: mean of the keypoint scores above rescore_vis_thr
//           (float32 sum in keypoint order, float32 divide, 0 when none) times the box score rounded to float32.
//
// Everything before exp is a __f*_rn / __d*_rn intrinsic, which nvcc never contracts into an FMA.  CUDA's exp / expf are not
// numpy's, so an OKS may differ from the reference's by one float32 ulp; kept lists are identical except where such an ulp
// decides (oracle.flag_ambiguous).
// A frame whose count is negative, above NMS_MAX_PEOPLE, or whose rows run past the caller's n_rows keeps nothing and sets a
// status bit; the other frames are unaffected.  Every launch reads its sizes from device memory (no host synchronisation),
// so the calls can be captured in a CUDA graph.
#pragma once
#include <cstdint>

#include "pairwise.cuh"

constexpr int NMS_MAX_PEOPLE = 256;              // VPB_NMS_MAX_PEOPLE: one thread per person
constexpr int NMS_MAX_K = 144;                   // VPB_NMS_MAX_K
constexpr int NMS_MAX_DETS = 256;                // VPB_NMS_MAX_DETS
constexpr int NMS_THREADS = NMS_MAX_PEOPLE;
constexpr int NMS_TOO_MANY_PEOPLE = 1;           // VPB_NMS_TOO_MANY_PEOPLE
constexpr int NMS_BAD_ROWS = 2;                  // VPB_NMS_BAD_ROWS
static_assert(NMS_MAX_K < 256, "visible keypoint lists are uint8");

struct OksNmsParams {
  const float* kpts;           // [n_rows, K, 3]
  const int32_t* counts;       // [F]
  const double* areas;         // [n_rows]
  const double* scores;        // [n_rows] (box scores when rescoring)
  int32_t* keep;               // [n_rows] frame-local kept indices, then -1 over the rest of the frame's rows
  int32_t* keep_counts;        // [F]
  double* scores_out;          // [n_rows] the score each row entered the sort with, or null
  float* oks;                  // vpb_oks_iou: [n_rows, NMS_MAX_PEOPLE]
  int32_t* status;
  double vars[NMS_MAX_K];      // (2 sigma)^2
  int n_rows, k, num_frames, soft, max_dets, use_vis, rescore;
  float thr, vis_thr, rescore_vis_thr;
};

// numpy's descending order (reversed ascending, NaN last): does a come before b, and are they equal?
__device__ __forceinline__ bool nms_above(double a, double b) { return a > b || (isnan(a) && !isnan(b)); }
__device__ __forceinline__ bool nms_same(double a, double b) { return a == b || (isnan(a) && isnan(b)); }

// exclusive prefix count of `flag` over the block's threads; *total gets the block's count
__device__ __forceinline__ int nms_scan(bool flag, int* warp_cnt, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_cnt[warp] = __popc(m);
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < NMS_THREADS / 32; ++w) {
    before += w < warp ? warp_cnt[w] : 0;
    all += warp_cnt[w];
  }
  __syncthreads();
  *total = all;
  return before + __popc(m & ((1u << lane) - 1u));
}

struct NmsFrame {
  int row0, n;
  bool ok;
};

// The frame's first row (the rows of the frames before it; a negative count holds none) and its limits; uniform over the
// block.  A frame over a limit sets its status bit, keeps nothing and writes -1 over whatever of its rows lie in the buffer.
// Every CTA sums the counts before it, so the grid reads O(F^2) counts in all: sized for the tens to a few thousand frames
// of a video step or an evaluation batch (64 frames: 2 K reads), where a separate prefix launch would cost more than it saves.
__device__ __forceinline__ NmsFrame nms_frame(const OksNmsParams& q, long long* red) {
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long before = 0;
  for (int j = tid; j < f; j += NMS_THREADS) before += q.counts[j] > 0 ? q.counts[j] : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) before += __shfl_down_sync(0xffffffffu, before, o);
  if (lane == 0) red[warp] = before;
  __syncthreads();
  before = 0;
#pragma unroll
  for (int w = 0; w < NMS_THREADS / 32; ++w) before += red[w];
  const int n = q.counts[f];
  NmsFrame fr{static_cast<int>(before < q.n_rows ? before : q.n_rows), n, true};
  if (n < 0 || before + n > q.n_rows || n > NMS_MAX_PEOPLE) {
    fr.ok = false;
    if (tid == 0) {
      atomicOr(q.status, n > NMS_MAX_PEOPLE && before + n <= q.n_rows ? NMS_TOO_MANY_PEOPLE : NMS_BAD_ROWS);
      if (q.keep_counts) q.keep_counts[f] = 0;
    }
    if (q.keep && n > 0)
      for (long long r = before + tid; r < before + n && r < q.n_rows; r += NMS_THREADS) q.keep[r] = -1;
  }
  return fr;
}

// Each person's visible keypoints (the candidate mask of oks_iou), in keypoint order: vis[t][0..cnt[t])
__device__ __forceinline__ void nms_visible(const OksNmsParams& q, const float* kp, int t, int n, uint8_t (*vis)[NMS_MAX_K], int* cnt) {
  if (t >= n) return;
  int c = 0;
  for (int k = 0; k < q.k; ++k) {
    if (q.use_vis && !(kp[k * 3 + 2] > q.vis_thr)) continue;
    vis[t][c++] = static_cast<uint8_t>(k);
  }
  cnt[t] = c;
}

// exp(-e) of keypoint k of the pair: ((dx*dx + dy*dy) / vars[k] / den) / 2
__device__ __forceinline__ double oks_term(const OksNmsParams& q, const float* g, const float* d, int k, double den) {
  const float dx = __fsub_rn(d[k * 3], g[k * 3]), dy = __fsub_rn(d[k * 3 + 1], g[k * 3 + 1]);
  const float s = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
  const double e = __dmul_rn(__ddiv_rn(__ddiv_rn(static_cast<double>(s), q.vars[k]), den), 0.5);
  return exp(-e);
}

// oks_iou(g, d): g the kept person, d the candidate, v / m the candidate's visible keypoints (m <= NMS_MAX_K < 256: at most
// one pairwise split)
__device__ __forceinline__ float oks_pair(const OksNmsParams& q, const float* g, const float* d, double a_g, double a_d, const uint8_t* v, int m) {
  if (m == 0) return 0.0f;
  const double den = __dadd_rn(__dmul_rn(__dadd_rn(a_g, a_d), 0.5), 2.220446049250313e-16);
  const double sum = pairwise_sum<1>([&](int i) { return oks_term(q, g, d, v[i], den); }, 0, m);
  return __double2float_rn(__ddiv_rn(sum, static_cast<double>(m)));
}

// rank of `key` at position t among positions [lo, hi) of `keys` in the stable descending order
__device__ __forceinline__ int nms_rank(const double* keys, int lo, int hi, int t, double key) {
  int r = 0;
  for (int u = lo; u < hi; ++u) {
    const double b = keys[u];
    r += nms_above(b, key) || (nms_same(b, key) && u > t);
  }
  return r;
}

struct NmsShared {
  uint8_t vis[NMS_MAX_PEOPLE][NMS_MAX_K];
  int vis_cnt[NMS_MAX_PEOPLE];
  double key[2][NMS_MAX_PEOPLE];                 // scores by position in the order (two buffers)
  int ord[2][NMS_MAX_PEOPLE];                    // frame-local person by position in the order
  double fresh[NMS_MAX_PEOPLE];                  // soft: the rescaled scores before the re-sort
  long long red[NMS_THREADS / 32];
  int warp_cnt[NMS_THREADS / 32];
};

__global__ void __launch_bounds__(NMS_THREADS) oks_nms_kernel(OksNmsParams q) {
  __shared__ NmsShared sm;
  const int tid = threadIdx.x, K = q.k;
  const NmsFrame fr = nms_frame(q, sm.red);
  if (!fr.ok) return;
  const int n = fr.n;
  const long long row0 = fr.row0;
  const float* kp = q.kpts + (row0 + tid) * K * 3;

  // the score each person enters the sort with
  double s = 0.0;
  if (tid < n) {
    s = q.scores[row0 + tid];
    if (q.rescore) {
      float sum = 0.0f;
      int c = 0;
      for (int k = 0; k < K; ++k) {
        const float ts = kp[k * 3 + 2];
        if (ts > q.rescore_vis_thr) { sum = __fadd_rn(sum, ts); ++c; }
      }
      const float mean = c ? __fdiv_rn(sum, static_cast<float>(c)) : 0.0f;
      s = static_cast<double>(__fmul_rn(mean, __double2float_rn(s)));
    }
    if (q.scores_out) q.scores_out[row0 + tid] = s;
    sm.key[1][tid] = s;
  }
  nms_visible(q, kp, tid, n, sm.vis, sm.vis_cnt);
  __syncthreads();
  if (tid < n) {
    const int r = nms_rank(sm.key[1], 0, n, tid, s);
    sm.ord[0][r] = tid;
    sm.key[0][r] = s;
  }
  __syncthreads();

  int rem = n, kept = 0, b = 0;
  const int limit = q.soft ? q.max_dets : NMS_MAX_PEOPLE;
  while (rem > 0 && kept < limit) {              // uniform over the block
    const int head = sm.ord[b][0];
    const float* g = q.kpts + (row0 + head) * K * 3;
    const double a_g = q.areas[row0 + head];
    const bool mine = tid >= 1 && tid < rem;
    float o = 0.0f;
    int j = 0;
    if (mine) {
      j = sm.ord[b][tid];
      o = oks_pair(q, g, q.kpts + (row0 + j) * K * 3, a_g, q.areas[row0 + j], sm.vis[j], sm.vis_cnt[j]);
    }
    if (tid == 0) q.keep[row0 + kept] = head;
    ++kept;
    if (!q.soft) {
      const bool stay = mine && o <= q.thr;
      int total;
      const int p = nms_scan(stay, sm.warp_cnt, &total);
      if (stay) sm.ord[b ^ 1][p] = j;
      rem = total;
    } else {
      double ns = 0.0;
      if (mine) {
        ns = __dmul_rn(sm.key[b][tid], static_cast<double>(expf(__fdiv_rn(-__fmul_rn(o, o), q.thr))));
        sm.fresh[tid] = ns;
      }
      __syncthreads();
      if (mine) {
        const int r = nms_rank(sm.fresh, 1, rem, tid, ns);
        sm.ord[b ^ 1][r] = j;
        sm.key[b ^ 1][r] = ns;
      }
      rem -= 1;
    }
    b ^= 1;
    __syncthreads();
  }
  for (int r = kept + tid; r < n; r += NMS_THREADS) q.keep[row0 + r] = -1;
  if (tid == 0) q.keep_counts[blockIdx.x] = kept;
}

// vpb_oks_iou: oks[row0 + i][j] = oks_iou(person i, person j) of each frame, j < n (the rest of the row is left alone)
__global__ void __launch_bounds__(NMS_THREADS) oks_iou_kernel(OksNmsParams q) {
  __shared__ NmsShared sm;
  const int tid = threadIdx.x, K = q.k;
  const NmsFrame fr = nms_frame(q, sm.red);
  if (!fr.ok) return;
  const int n = fr.n;
  const long long row0 = fr.row0;
  nms_visible(q, q.kpts + (row0 + tid) * K * 3, tid, n, sm.vis, sm.vis_cnt);
  __syncthreads();
  if (tid >= n) return;
  const float* d = q.kpts + (row0 + tid) * K * 3;
  const double a_d = q.areas[row0 + tid];
  for (int i = 0; i < n; ++i)
    q.oks[(row0 + i) * NMS_MAX_PEOPLE + tid] = oks_pair(q, q.kpts + (row0 + i) * K * 3, d, q.areas[row0 + i], a_d, sm.vis[tid], sm.vis_cnt[tid]);
}
