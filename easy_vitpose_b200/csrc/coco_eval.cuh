// COCO keypoint evaluation on the device (vpb_coco_eval): pycocotools' COCOeval(iouType='keypoints') evaluate, accumulate and
// summarize for category 1 over I images in one enqueue.  oracle/coco_oks_eval.py restates the algorithm in numpy and
// oracle/coco_eval_oracle.py adds the arrays compared here.  Parameters are Params.setKpParams's: maxDets 20, the ten OKS
// thresholds .5:.05:.95, the 101 recall thresholds 0:.01:1, the area ranges all / medium / large.
//
//   coco_frames_kernel   one CTA: each detection frame's first row (the rows of the frames before it, as vpb_oks_nms lays
//                        them out) and its checks.
//   coco_image_kernel    one CTA per image.  Gathers the image's detection rows (frames in call order, each frame's rows or
//                        its keep list in order), orders them by argsort(-score, kind='mergesort') (descending, stable, NaN
//                        last), keeps the first 20, computes loadRes's area from the keypoint extent and computeOks in float64
//                        against the image's ground truths, then for each area range sets _ignore, orders the ground truths
//                        stably by it and runs evaluateImg's greedy matching at each threshold.  Writes the image's ordered
//                        scores into slots [i*20, i*20+20) (padding after them), a matched and an ignored bit per (area,
//                        threshold) per detection, and the non-ignored ground-truth count per area.
//   coco_merge_kernel    ceil(log2 I) passes of a stable merge (merge path by binary search, the left run winning ties)
//                        turn the image-ordered runs into accumulate's argsort(-scores, kind='mergesort') over all images.
//   coco_accumulate_kernel one CTA per (area, threshold): inclusive scans of tp and fp, rc = tp / npig and
//                        pr = tp / (fp + tp + 2^-52), the backward running max of pr, searchsorted(rc, recThrs, 'left') and
//                        recall = rc[-1] (0 with no detection; -1 everywhere when npig = 0).
//   coco_summarize_kernel the ten numbers of summarize(): np.mean over the entries > -1, in numpy's pairwise order.
//
// Exactness: everything before exp is a __d*_rn intrinsic (no FMA contraction) and everything after it is integer counting,
// IEEE division, comparison and numpy's sum order, so the device equals the numpy statement bit for bit except where CUDA's
// exp moves an OKS by an ulp across a threshold or across another OKS it is compared with (oracle flag_ambiguous).
// Limits: COCO_MAX_GTS ground truths and COCO_MAX_ROWS detection rows (before the truncation to 20) per image, K <= COCO_MAX_K.
// An image over a limit, a frame with a negative count, rows past the buffer, a keep entry outside its frame, a frame of no
// image or a ground-truth offset table out of order sets a status bit, and the ten stats are then NaN.  Every launch reads its
// sizes from device memory: no host synchronisation, no allocation, so the call can be captured in a CUDA graph.
#pragma once
#include <cstdint>

#include "pairwise.cuh"

constexpr int COCO_MAX_GTS = 256;                // VPB_COCO_MAX_GTS: ground truths per image
constexpr int COCO_MAX_ROWS = 1024;              // VPB_COCO_MAX_ROWS: detection rows per image before the truncation
constexpr int COCO_MAX_K = 144;                  // VPB_COCO_MAX_K
constexpr int COCO_MAX_DETS = 20;                // maxDets
constexpr int COCO_T = 10, COCO_R = 101, COCO_A = 3;
constexpr int COCO_TOO_MANY_GTS = 1;             // VPB_COCO_TOO_MANY_GTS
constexpr int COCO_TOO_MANY_ROWS = 2;            // VPB_COCO_TOO_MANY_ROWS
constexpr int COCO_BAD_INPUT = 4;                // VPB_COCO_BAD_INPUT
constexpr int COCO_THREADS = 256;                // coco_image_kernel and coco_merge_kernel
constexpr int COCO_ACC_THREADS = 1024;
constexpr int COCO_SUMMARY_TERMS = COCO_T * COCO_R;
static_assert(COCO_MAX_GTS <= 256, "ground-truth orders are uint8");
static_assert(COCO_MAX_K < 256, "visible keypoint lists are uint8");
static_assert(COCO_A * COCO_T <= 32, "one matched and one ignored bit per (area, threshold) in a 64-bit word");

// np.linspace(.5, 0.95, 10): arange * ((0.95 - .5) / 9) + .5, the last entry set to 0.95
__constant__ double kCocoIouThrs[COCO_T] = {0x1.0000000000000p-1, 0x1.199999999999ap-1, 0x1.3333333333333p-1, 0x1.4cccccccccccdp-1,
                                            0x1.6666666666666p-1, 0x1.8000000000000p-1, 0x1.999999999999ap-1, 0x1.b333333333333p-1,
                                            0x1.cccccccccccccp-1, 0x1.e666666666666p-1};
// np.linspace(.0, 1.00, 101): r * 0.01, the last entry set to 1.0
__device__ __forceinline__ double coco_rec_thr(int r) { return r == COCO_R - 1 ? 1.0 : __dmul_rn(static_cast<double>(r), 0.01); }
// areaRng: all [0, 1e10], medium [32^2, 96^2], large [96^2, 1e10]; outside means area < lo or area > hi
__device__ __forceinline__ bool coco_out_of_range(double area, int a) {
  const double lo = a == 2 ? 9216.0 : (a == 1 ? 1024.0 : 0.0), hi = a == 1 ? 9216.0 : 1e10;
  return area < lo || area > hi;
}

struct CocoEvalParams {
  // ground truths, CSR by image: image i holds rows [gt_offsets[i], gt_offsets[i + 1])
  const int32_t* gt_offsets;     // [num_images + 1]
  const double* gt_kpts;         // [num_gts, k, 3] x, y, v
  const double* gt_area;         // [num_gts]
  const double* gt_bbox;         // [num_gts, 4] x, y, w, h
  const int32_t* gt_iscrowd;     // [num_gts]
  const int32_t* gt_num_kpts;    // [num_gts]
  // detections: frame f holds the next counts[f] rows and belongs to image frame_image[f]
  const double* dt_kpts;         // [n_rows, k, 2] x, y
  const double* dt_scores;       // [n_rows]
  const int32_t* counts;         // [num_frames]
  const int32_t* frame_image;    // [num_frames]
  const int32_t* keep;           // [n_rows] frame-local rows in order (vpb_oks_nms's d_keep), or null: every row
  const int32_t* keep_counts;    // [num_frames]
  // workspace
  int32_t* frame_row0;           // [num_frames] first row, -1 for a frame that failed its checks
  double* key[2];                // [num_images * 20] scores by slot, merge ping-pong
  int32_t* slot[2];              // [num_images * 20] slot of each sorted position, -1 for padding
  unsigned long long* bits;      // [num_images * 20] bit a*10+t: matched; bit 32+a*10+t: dtIgnore
  int32_t* num_dets;             // [num_images]
  int32_t* npig;                 // [3, num_images]
  double* summary;               // [10, COCO_SUMMARY_TERMS] the entries > -1 of each mean
  // outputs
  double* stats;                 // [10]
  double* precision;             // [3, 10, 101]
  double* recall;                // [3, 10]
  int32_t* status;
  double vars[COCO_MAX_K];       // (2 sigma)^2
  int k, num_images, num_gts, num_frames, n_rows;
};

// ------------------------------------------------------------------------------------------------------------ frame table
__global__ void __launch_bounds__(1024) coco_frames_kernel(CocoEvalParams q) {
  __shared__ long long warp_sum[32];
  __shared__ long long carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  int bad = 0;
  for (int base = 0; base < q.num_frames; base += 1024) {
    const int f = base + tid;
    const int n = f < q.num_frames ? q.counts[f] : 0;
    long long x = n > 0 ? n : 0, incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    long long before = carry;
    for (int w = 0; w < warp; ++w) before += warp_sum[w];
    before += incl - x;
    if (f < q.num_frames) {
      const int img = q.frame_image[f];
      const int kc = q.keep ? q.keep_counts[f] : n;
      const bool ok = n >= 0 && before + n <= q.n_rows && img >= 0 && img < q.num_images && kc >= 0 && kc <= n;
      q.frame_row0[f] = ok ? static_cast<int32_t>(before) : -1;
      bad |= !ok;
    }
    __syncthreads();
    if (tid == 1023) carry = before + x;
    __syncthreads();
  }
  if (__syncthreads_or(bad) && tid == 0) atomicOr(q.status, COCO_BAD_INPUT);
}

// ------------------------------------------------------------------------------------------------------------ per image
struct CocoImageShared {
  double oks[COCO_MAX_DETS][COCO_MAX_GTS];       // [sorted detection][ground truth in input order]
  double score[COCO_MAX_ROWS];
  int32_t row[COCO_MAX_ROWS];
  uint8_t vis[COCO_MAX_GTS][COCO_MAX_K];         // each ground truth's keypoints with v > 0, in order
  int16_t vis_cnt[COCO_MAX_GTS];
  uint8_t order[COCO_A][COCO_MAX_GTS];           // ground truths stably ordered by _ignore, per area range
  uint8_t ignore[COCO_A][COCO_MAX_GTS];          // _ignore by input order
  unsigned int gt_matched[COCO_A * COCO_T][COCO_MAX_GTS / 32];
  unsigned long long det_bits[COCO_MAX_DETS];
  double det_area[COCO_MAX_DETS];
  int top[COCO_MAX_DETS];                        // gathered index of each sorted detection
  int frames[COCO_THREADS];
  int warp_cnt[COCO_THREADS / 32];
  int npig[COCO_A];
  int n_rows, n_frames, flag;
};

// argsort(-score, kind='mergesort'): does a come before b (descending, NaN last)?
__device__ __forceinline__ bool coco_before(double a, double b) { return a > b || (!isnan(a) && isnan(b)); }
__device__ __forceinline__ bool coco_same(double a, double b) { return a == b || (isnan(a) && isnan(b)); }

// np.max((0, v)) of computeOks's bbox branch: NaN propagates
__device__ __forceinline__ double coco_pos(double v) { return isnan(v) ? v : (v > 0.0 ? v : 0.0); }

// np.min / np.max of a coordinate over the keypoints (NaN propagates)
__device__ __forceinline__ void coco_extent(const double* kp, int k, int c, double* lo, double* hi) {
  double a = kp[c], b = kp[c];
  for (int j = 1; j < k; ++j) {
    const double v = kp[j * 2 + c];
    if (isnan(a)) break;
    if (isnan(v)) { a = b = v; break; }
    a = v < a ? v : a;
    b = v > b ? v : b;
  }
  *lo = a;
  *hi = b;
}

// computeOks for one (detection, ground truth): e = (dx^2 + dy^2) / vars / (area + 2^-52) / 2, exp(-e), numpy's sum over the
// ground truth's visible keypoints (every keypoint, with the bbox-distance dx, dy, when none is visible), / their count
__device__ __forceinline__ double coco_oks(const CocoEvalParams& q, const double* d, const double* g, const double* bb, double area,
                                           const uint8_t* vis, int m) {
  const double den = __dadd_rn(area, 2.220446049250313e-16);
  if (m > 0) {
    const double sum = pairwise_sum<1>([&](int i) {
      const int k = vis[i];
      const double dx = __dsub_rn(d[k * 2], g[k * 3]), dy = __dsub_rn(d[k * 2 + 1], g[k * 3 + 1]);
      const double e = __ddiv_rn(__ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), q.vars[k]), den), 2.0);
      return exp(-e);
    }, 0, m);
    return __ddiv_rn(sum, static_cast<double>(m));
  }
  const double x0 = __dsub_rn(bb[0], bb[2]), x1 = __dadd_rn(bb[0], __dmul_rn(bb[2], 2.0));
  const double y0 = __dsub_rn(bb[1], bb[3]), y1 = __dadd_rn(bb[1], __dmul_rn(bb[3], 2.0));
  const double sum = pairwise_sum<1>([&](int k) {
    const double xd = d[k * 2], yd = d[k * 2 + 1];
    const double dx = __dadd_rn(coco_pos(__dsub_rn(x0, xd)), coco_pos(__dsub_rn(xd, x1)));
    const double dy = __dadd_rn(coco_pos(__dsub_rn(y0, yd)), coco_pos(__dsub_rn(yd, y1)));
    const double e = __ddiv_rn(__ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), q.vars[k]), den), 2.0);
    return exp(-e);
  }, 0, q.k);
  return __ddiv_rn(sum, static_cast<double>(q.k));
}

__global__ void __launch_bounds__(COCO_THREADS, 2) coco_image_kernel(CocoEvalParams q) {
  extern __shared__ __align__(16) unsigned char coco_smem[];
  CocoImageShared& sm = *reinterpret_cast<CocoImageShared*>(coco_smem);
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, K = q.k;
  const long long slot0 = static_cast<long long>(img) * COCO_MAX_DETS;
  if (tid == 0) { sm.n_rows = 0; sm.flag = 0; }
  if (tid < COCO_A) sm.npig[tid] = 0;
  if (tid < COCO_MAX_DETS) sm.det_bits[tid] = 0ull;

  // the image's ground truths
  const int g0 = q.gt_offsets[img], g1 = q.gt_offsets[img + 1];
  const bool gts_ok = g0 >= 0 && g0 <= g1 && g1 <= q.num_gts;
  const int G = gts_ok ? g1 - g0 : 0;
  if (tid == 0 && !gts_ok) sm.flag = COCO_BAD_INPUT;
  if (tid == 0 && G > COCO_MAX_GTS) sm.flag = COCO_TOO_MANY_GTS;

  // the image's detection rows: its frames in call order, each frame's rows (or keep list) in order
  __syncthreads();
  for (int base = 0; base < q.num_frames; base += COCO_THREADS) {
    const int f = base + tid;
    const bool mine = f < q.num_frames && q.frame_image[f] == img && q.frame_row0[f] >= 0;
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) sm.warp_cnt[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < COCO_THREADS / 32; ++w) {
      before += w < warp ? sm.warp_cnt[w] : 0;
      total += sm.warp_cnt[w];
    }
    if (mine) sm.frames[before + __popc(m & ((1u << lane) - 1u))] = f;
    __syncthreads();
    for (int j = 0; j < total; ++j) {
      const int fj = sm.frames[j], r0 = q.frame_row0[fj], n = q.counts[fj];
      const int c = q.keep ? q.keep_counts[fj] : n;
      const int have = sm.n_rows;
      for (int u = tid; u < c && have + u < COCO_MAX_ROWS; u += COCO_THREADS) {
        int local = u;
        if (q.keep) {
          local = q.keep[r0 + u];
          if (local < 0 || local >= n) { atomicOr(&sm.flag, COCO_BAD_INPUT); local = 0; }
        }
        sm.row[have + u] = r0 + local;
      }
      __syncthreads();
      if (tid == 0) {
        if (have + c > COCO_MAX_ROWS) atomicOr(&sm.flag, COCO_TOO_MANY_ROWS);
        sm.n_rows = min(have + c, COCO_MAX_ROWS);
      }
      __syncthreads();
    }
  }
  __syncthreads();
  const int flag = sm.flag;
  if (flag) {                                    // the stats will be NaN; leave this image empty
    if (tid == 0) atomicOr(q.status, flag);
    if (tid < COCO_MAX_DETS) {
      q.key[0][slot0 + tid] = 0.0;
      q.slot[0][slot0 + tid] = -1;
      q.bits[slot0 + tid] = 0ull;
    }
    if (tid == 0) q.num_dets[img] = 0;
    if (tid < COCO_A) q.npig[tid * q.num_images + img] = 0;
    return;
  }
  const int n = sm.n_rows;
  for (int u = tid; u < n; u += COCO_THREADS) sm.score[u] = q.dt_scores[sm.row[u]];
  __syncthreads();
  // the first 20 of argsort(-score, kind='mergesort')
  for (int u = tid; u < n; u += COCO_THREADS) {
    const double s = sm.score[u];
    int r = 0;
    for (int v = 0; v < n && r < COCO_MAX_DETS; ++v) {
      const double b = sm.score[v];
      r += coco_before(b, s) || (coco_same(b, s) && v < u);
    }
    if (r < COCO_MAX_DETS) sm.top[r] = u;
  }
  const int D = n < COCO_MAX_DETS ? n : COCO_MAX_DETS;
  // ground truths: visible keypoints and _ignore per area range
  for (int g = tid; g < G; g += COCO_THREADS) {
    const double* gk = q.gt_kpts + static_cast<long long>(g0 + g) * K * 3;
    int c = 0;
    for (int k = 0; k < K; ++k)
      if (gk[k * 3 + 2] > 0.0) sm.vis[g][c++] = static_cast<uint8_t>(k);
    sm.vis_cnt[g] = static_cast<int16_t>(c);
    const bool ign = q.gt_iscrowd[g0 + g] != 0 || q.gt_num_kpts[g0 + g] == 0;
    const double area = q.gt_area[g0 + g];
#pragma unroll
    for (int a = 0; a < COCO_A; ++a) sm.ignore[a][g] = ign || coco_out_of_range(area, a);
  }
  __syncthreads();
  // loadRes's area of the kept detections: (max x - min x) * (max y - min y)
  if (tid < D) {
    const double* dk = q.dt_kpts + static_cast<long long>(sm.row[sm.top[tid]]) * K * 2;
    double x0, x1, y0, y1;
    coco_extent(dk, K, 0, &x0, &x1);
    coco_extent(dk, K, 1, &y0, &y1);
    sm.det_area[tid] = __dmul_rn(__dsub_rn(x1, x0), __dsub_rn(y1, y0));
  }
  if (tid < COCO_A) {                            // np.argsort(_ignore, kind='mergesort'), and the non-ignored count
    int p = 0;
    for (int g = 0; g < G; ++g)
      if (!sm.ignore[tid][g]) sm.order[tid][p++] = static_cast<uint8_t>(g);
    sm.npig[tid] = p;
    for (int g = 0; g < G; ++g)
      if (sm.ignore[tid][g]) sm.order[tid][p++] = static_cast<uint8_t>(g);
  }
  for (int u = tid; u < COCO_A * COCO_T * (COCO_MAX_GTS / 32); u += COCO_THREADS) (&sm.gt_matched[0][0])[u] = 0u;
  for (int p = tid; p < D * G; p += COCO_THREADS) {
    const int d = p / G, g = p % G;
    sm.oks[d][g] = coco_oks(q, q.dt_kpts + static_cast<long long>(sm.row[sm.top[d]]) * K * 2, q.gt_kpts + static_cast<long long>(g0 + g) * K * 3,
                            q.gt_bbox + static_cast<long long>(g0 + g) * 4, q.gt_area[g0 + g], sm.vis[g], sm.vis_cnt[g]);
  }
  __syncthreads();
  // evaluateImg's greedy matching, one thread per (area range, threshold)
  if (tid < COCO_A * COCO_T) {
    const int a = tid / COCO_T, t = tid % COCO_T;
    unsigned int* matched = sm.gt_matched[tid];
    const double thr = kCocoIouThrs[t] < 1.0 - 1e-10 ? kCocoIouThrs[t] : 1.0 - 1e-10;
    for (int d = 0; d < D; ++d) {
      double iou = thr;
      int m = -1;
      for (int j = 0; j < G; ++j) {
        const int g = sm.order[a][j];
        if (((matched[g >> 5] >> (g & 31)) & 1u) && !q.gt_iscrowd[g0 + g]) continue;
        if (m > -1 && !sm.ignore[a][m] && sm.ignore[a][g]) break;
        const double o = sm.oks[d][g];
        if (o < iou) continue;
        iou = o;
        m = g;
      }
      bool ign;
      if (m >= 0) {
        matched[m >> 5] |= 1u << (m & 31);
        ign = sm.ignore[a][m];
        atomicOr(&sm.det_bits[d], 1ull << tid);
      } else {
        ign = coco_out_of_range(sm.det_area[d], a);
      }
      if (ign) atomicOr(&sm.det_bits[d], 1ull << (32 + tid));
    }
  }
  __syncthreads();
  if (tid < COCO_MAX_DETS) {
    const bool real = tid < D;
    q.key[0][slot0 + tid] = real ? sm.score[sm.top[tid]] : 0.0;
    q.slot[0][slot0 + tid] = real ? static_cast<int32_t>(slot0 + tid) : -1;
    q.bits[slot0 + tid] = real ? sm.det_bits[tid] : 0ull;
  }
  if (tid == 0) q.num_dets[img] = D;
  if (tid < COCO_A) q.npig[tid * q.num_images + img] = sm.npig[tid];
}

// ------------------------------------------------------------------------------------------------------------ merge
// strict order of (key, slot) entries: real scores descending with NaN last, padding (slot -1) after every real entry
__device__ __forceinline__ bool coco_entry_before(double ka, int sa, double kb, int sb) {
  if (sa < 0) return false;
  if (sb < 0) return true;
  return coco_before(ka, kb);
}

// one pass: runs of `width` entries become runs of 2 * width; in a pair of runs the left run wins ties (stable)
__global__ void __launch_bounds__(COCO_THREADS) coco_merge_kernel(CocoEvalParams q, int src, long long width) {
  const long long N = static_cast<long long>(q.num_images) * COCO_MAX_DETS;
  const long long x = static_cast<long long>(blockIdx.x) * COCO_THREADS + threadIdx.x;
  if (x >= N) return;
  const double* key = q.key[src];
  const int32_t* slot = q.slot[src];
  const long long s = x - x % (2 * width), mid = min(s + width, N), end = min(s + 2 * width, N);
  const double k = key[x];
  const int sl = slot[x];
  long long pos;
  if (x < mid) {                                 // count the right run's entries strictly before this one
    long long lo = mid, hi = end;
    while (lo < hi) {
      const long long c = (lo + hi) >> 1;
      if (coco_entry_before(key[c], slot[c], k, sl)) lo = c + 1; else hi = c;
    }
    pos = (x - s) + (lo - mid);
  } else {                                       // count the left run's entries not after this one
    long long lo = s, hi = mid;
    while (lo < hi) {
      const long long c = (lo + hi) >> 1;
      if (!coco_entry_before(k, sl, key[c], slot[c])) lo = c + 1; else hi = c;
    }
    pos = (x - mid) + (lo - s);
  }
  q.key[src ^ 1][s + pos] = k;
  q.slot[src ^ 1][s + pos] = sl;
}

// ------------------------------------------------------------------------------------------------------------ accumulate
// block-wide exclusive scan of a 64-bit value (1024 threads); *total gets the sum
__device__ __forceinline__ long long coco_block_scan(long long v, long long* warp_sum, long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  long long before = 0, all = 0;
  for (int w = 0; w < COCO_ACC_THREADS / 32; ++w) {
    before += w < warp ? warp_sum[w] : 0;
    all += warp_sum[w];
  }
  __syncthreads();
  *total = all;
  return before + incl - v;
}

__global__ void __launch_bounds__(COCO_ACC_THREADS) coco_accumulate_kernel(CocoEvalParams q, int src) {
  __shared__ long long warp_sum[COCO_ACC_THREADS / 32];
  __shared__ double chunk_max[COCO_ACC_THREADS];
  __shared__ double prec[COCO_R];
  __shared__ int need[COCO_R];                   // the tp count where rc first reaches recThrs[r]
  const int a = blockIdx.x / COCO_T, t = blockIdx.x % COCO_T, bit = a * COCO_T + t, tid = threadIdx.x;
  const int32_t* slot = q.slot[src];
  long long nd_part = 0, npig_part = 0;
  for (int i = tid; i < q.num_images; i += COCO_ACC_THREADS) {
    nd_part += q.num_dets[i];
    npig_part += q.npig[a * q.num_images + i];
  }
  long long nd, npig;
  coco_block_scan(nd_part, warp_sum, &nd);
  coco_block_scan(npig_part, warp_sum, &npig);
  double* P = q.precision + (a * COCO_T + t) * COCO_R;
  if (npig == 0) {
    if (tid < COCO_R) P[tid] = -1.0;
    if (tid == 0) q.recall[a * COCO_T + t] = -1.0;
    return;
  }
  const double np_d = static_cast<double>(npig);
  if (tid < COCO_R) {
    const double thr = coco_rec_thr(tid);
    long long lo = 0, hi = npig;                 // smallest v with v / npig >= thr (npig / npig = 1 >= every threshold)
    while (lo < hi) {
      const long long c = (lo + hi) >> 1;
      if (__ddiv_rn(static_cast<double>(c), np_d) >= thr) hi = c; else lo = c + 1;
    }
    need[tid] = static_cast<int>(lo);
    prec[tid] = 0.0;
  }
  // each thread takes a contiguous chunk of the sorted detections
  const long long per = (nd + COCO_ACC_THREADS - 1) / COCO_ACC_THREADS;
  const long long i0 = min(nd, tid * per), i1 = min(nd, i0 + per);
  long long tp_c = 0, fp_c = 0;
  for (long long i = i0; i < i1; ++i) {
    const unsigned long long b = q.bits[slot[i]];
    const bool m = (b >> bit) & 1ull, ig = (b >> (32 + bit)) & 1ull;
    tp_c += m && !ig;
    fp_c += !m && !ig;
  }
  long long tp_all, fp_all;
  const long long tp0 = coco_block_scan(tp_c, warp_sum, &tp_all);
  const long long fp0 = coco_block_scan(fp_c, warp_sum, &fp_all);
  // pr of each entry, the chunk's maximum, then the running maximum from the end
  double mx = -1.0;
  {
    long long tp = tp0, fp = fp0;
    for (long long i = i0; i < i1; ++i) {
      const unsigned long long b = q.bits[slot[i]];
      const bool m = (b >> bit) & 1ull, ig = (b >> (32 + bit)) & 1ull;
      tp += m && !ig;
      fp += !m && !ig;
      const double td = static_cast<double>(tp);
      const double pr = __ddiv_rn(td, __dadd_rn(__dadd_rn(static_cast<double>(fp), td), 2.220446049250313e-16));
      mx = pr > mx ? pr : mx;
    }
  }
  chunk_max[tid] = mx;
  __syncthreads();
  double after = -1.0;                           // max of pr over the later chunks
  for (int u = tid + 1; u < COCO_ACC_THREADS; ++u) after = chunk_max[u] > after ? chunk_max[u] : after;
  {
    long long tp = tp0 + tp_c, fp = fp0 + fp_c;  // inclusive counts at i1 - 1, walked back
    double run = after;
    for (long long i = i1 - 1; i >= i0; --i) {
      const double td = static_cast<double>(tp);
      const double pr = __ddiv_rn(td, __dadd_rn(__dadd_rn(static_cast<double>(fp), td), 2.220446049250313e-16));
      run = pr > run ? pr : run;
      const unsigned long long b = q.bits[slot[i]];
      const bool m = (b >> bit) & 1ull, ig = (b >> (32 + bit)) & 1ull;
      const bool is_tp = m && !ig;
      // searchsorted(rc, thr, 'left') = the first i with tp[i] >= need: the need-th true positive, or 0 when need is 0
      if (is_tp || i == 0)
        for (int r = 0; r < COCO_R; ++r)
          if ((is_tp && need[r] == tp) || (i == 0 && need[r] == 0)) prec[r] = run;
      tp -= is_tp;
      fp -= !m && !ig;
    }
  }
  __syncthreads();
  if (tid < COCO_R) P[tid] = prec[tid];
  if (tid == 0) q.recall[a * COCO_T + t] = nd ? __ddiv_rn(static_cast<double>(tp_all), np_d) : 0.0;
}

// ------------------------------------------------------------------------------------------------------------ summarize
// thread s computes stat s: AP, AP50, AP75, AP_medium, AP_large, AR, AR50, AR75, AR_medium, AR_large
__global__ void __launch_bounds__(32) coco_summarize_kernel(CocoEvalParams q) {
  const int s = threadIdx.x;
  if (s >= 10) return;
  const bool ap = s < 5;
  const int which = s % 5;                       // 0 all thresholds, 1 t = .5, 2 t = .75, 3 medium, 4 large
  const int a = which == 3 ? 1 : (which == 4 ? 2 : 0);
  const int t0 = which == 1 ? 0 : (which == 2 ? 5 : 0), nt = (which == 1 || which == 2) ? 1 : COCO_T;
  const int per_t = ap ? COCO_R : 1;
  const double* src = ap ? q.precision + (a * COCO_T + t0) * COCO_R : q.recall + a * COCO_T + t0;
  double* kept = q.summary + s * COCO_SUMMARY_TERMS;
  int m = 0;
  for (int u = 0; u < nt * per_t; ++u)
    if (src[u] > -1.0) kept[m++] = src[u];
  double v = -1.0;
  if (m > 0) v = __ddiv_rn(pairwise_sum<4>([&](int i) { return kept[i]; }, 0, m), static_cast<double>(m));
  q.stats[s] = *q.status ? __longlong_as_double(0x7ff8000000000000ll) : v;
}
