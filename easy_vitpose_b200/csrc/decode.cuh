// Heatmap decode: [N,K,64,48] f32 -> keypoints [N,K,3] (y, x, score) + flat argmax [N,K] i32.
// HBM-bound (12 288 B read per map, 16 B written); one warp per map, 128-bit coalesced loads.
//
// Restates the branch VitInference takes (unbiased=True, use_udp=True, GaussianHeatmap):
//   _get_max_preds            vit_utils/top_down_eval.py:82-114   first-index argmax, (-1,-1) if max <= 0
//   post_dark_udp(kernel=11)  vit_utils/top_down_eval.py:354-415  cv2.GaussianBlur 11x11 -> clip -> log ->
//                                                                 7-point Taylor step with a float64 2x2 inverse
//   transform_preds(use_udp)  vit_utils/post_processing/post_transforms.py:183-192
//   VitInference.postprocess  easy_ViTPose/inference.py:187-205   centre = org // 2, output order (y, x, score)
//   VitInference.inference    easy_ViTPose/inference.py:270       optional integer (y, x) offset back to the frame
// The blur is only evaluated at the (at most) 7 stencil points the Taylor step reads, with cv2's exact
// float32 accumulation order (row pass: sequential fmaf left to right; column pass: centre tap then
// fmaf of symmetric pairs), so blurred values are bit-identical to cv2 4.13 (oracle/make_golden.py).
#pragma once
#include "ptx.cuh"

namespace vpb {

constexpr int HM_H = 64, HM_W = 48, HM_PIX = HM_H * HM_W;

// float32(cv2.getGaussianKernel(11, 0)) taps 0..5 (symmetric), sigma = 0.3*((11-1)*0.5-1)+0.8 = 2.0
__device__ __constant__ float c_gauss11[6] = {0x1.20c256p-7f, 0x1.bcb86ap-6f, 0x1.0ab50ap-4f,
                                              0x1.f2464cp-4f, 0x1.6a7e1ep-3f, 0x1.9ac20ap-3f};

// Modulation kernels other than 11 (keypoints_from_heatmaps' `kernel` argument, top_down_eval.py:499; 17 for sigma = 3): taps by
// distance from the centre, filled on the host (engine.cu: gauss_taps) the way cv2.getGaussianKernel(k, 0) returns them (the
// formula from 11 taps on, fixed tables below).
constexpr int MAX_RADIUS = 17;                              // kernel sizes up to 35
struct GaussTaps {
  int radius = 5;
  float t[MAX_RADIUS + 1] = {};                             // t[d] = tap at distance d from the centre
};

__device__ __forceinline__ int reflect101(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}
// Row pass of cv2's separable float32 filter at one output sample; at(j) = the input sample at offset j - R, t[d] = the tap at
// distance d.  7 taps and more accumulate left to right (acc = 0; acc = fmaf(k[j], x[j], acc)); 3 and 5 taps take cv2's
// small-kernel row filter, which starts with the inner pair: acc = (x[-1] + x[+1]) * k1; acc = fmaf(k0, x[0], acc);
// acc = fmaf(k2, x[-2] + x[+2], acc)  (oracle/vitpose_oracle.py: row_pass, pinned on cv2 bit for bit).
template <typename F>
__device__ __forceinline__ float blur_row(const float* t, int R, F&& at) {
  if (R == 1 || R == 2) {
    float acc = __fmul_rn(__fadd_rn(at(R - 1), at(R + 1)), t[1]);
    acc = __fmaf_rn(t[0], at(R), acc);
    if (R == 2) acc = __fmaf_rn(t[2], __fadd_rn(at(0), at(4)), acc);
    return acc;
  }
  float acc = 0.0f;
  for (int j = 0; j <= 2 * R; ++j) acc = __fmaf_rn(t[j < R ? R - j : j - R], at(j), acc);
  return acc;
}
// `_gaussian_blur` (top_down_eval.py:443-455) blurs the map inside a zero border of width R; cv2's column filter is vectorised
// over x in steps of 8 and the columns of the (48 + 2R)-wide image past the last full step run through its scalar loop, whose
// products are not fused.  First visible column handled that way (HM_W if none: only 5 and 7 taps reach visible columns).
__host__ __device__ __forceinline__ int zero_padded_tail_start(int R) {
  if (R < 2) return 48;
  const int s = 8 * ((48 + 2 * R) / 8) - R;
  return s < 48 ? s : 48;
}
__device__ __forceinline__ bool arg_better(float v, int i, float bv, int bi) {
  // np.argmax order: NaN beats everything, first index wins among equals
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return i < bi;
}

struct DecodeParams {
  const float* heatmaps;   // [N,K,64,48]
  const int* org_wh;       // [N,2] crop (width, height)
  float* kpts;             // [N,K,3]
  int* idx;                // [N,K] (may be nullptr)
  const int* offs_yx;      // [N,2] integer (y, x) added to the keypoints: crop -> frame coordinates (inference.py:270); may be nullptr
  int n, k;
  int wrap_batch;          // sentinel quirk: 0 = previous map wraps inside the crop, 1 = inside the whole call
  // maps / keypoint rows between consecutive crops in heatmaps, kpts and idx (0 = k): a multi-head call decodes each
  // segment's K_head maps out of crops laid out K_max apart.  With wrap_batch = 1 the "previous map" is taken over the
  // compact n * k maps of the call (one reference call on the segment's own [n, K_head] array), read at its strided slot.
  int kstride = 0;
  // general transform_preds (post_transforms.py:150-194) for callers other than VitInference.postprocess: per crop
  // (centre_x, centre_y, scale_x, scale_y) either as float32 (numpy keeps the whole expression in float32) or as float64
  // (int64 / float64 arrays promote it to float64); both null = the VitInference form above (scale = org, centre = org // 2)
  const float* cs32 = nullptr;
  const double* cs64 = nullptr;
  GaussTaps taps;          // read by the GENERIC instantiation only (kernel != 11)
};

// coords (heatmap pixels) -> image pixels: x * (scale / (W-1 or W)) + centre - scale * 0.5, evaluated left to right with one
// rounding per operation in the type numpy would use (no FMA contraction)
__device__ __forceinline__ void transform_cs(float xr, float yr, int n_i, const float* cs32, const double* cs64, bool use_udp,
                                             float& X, float& Y) {
  if (cs32 != nullptr) {
    const float cx = cs32[4 * n_i], cy = cs32[4 * n_i + 1], sx = cs32[4 * n_i + 2], sy = cs32[4 * n_i + 3];
    const float kx = __fdiv_rn(sx, use_udp ? HM_W - 1.0f : static_cast<float>(HM_W));
    const float ky = __fdiv_rn(sy, use_udp ? HM_H - 1.0f : static_cast<float>(HM_H));
    X = __fsub_rn(__fadd_rn(__fmul_rn(xr, kx), cx), __fmul_rn(sx, 0.5f));
    Y = __fsub_rn(__fadd_rn(__fmul_rn(yr, ky), cy), __fmul_rn(sy, 0.5f));
  } else {
    const double cx = cs64[4 * n_i], cy = cs64[4 * n_i + 1], sx = cs64[4 * n_i + 2], sy = cs64[4 * n_i + 3];
    const double kx = __ddiv_rn(sx, use_udp ? HM_W - 1.0 : static_cast<double>(HM_W));
    const double ky = __ddiv_rn(sy, use_udp ? HM_H - 1.0 : static_cast<double>(HM_H));
    X = static_cast<float>(__dsub_rn(__dadd_rn(__dmul_rn(static_cast<double>(xr), kx), cx), __dmul_rn(sx, 0.5)));
    Y = static_cast<float>(__dsub_rn(__dadd_rn(__dmul_rn(static_cast<double>(yr), ky), cy), __dmul_rn(sy, 0.5)));
  }
}

// warps (= maps) per CTA: 4 gives 272 CTAs for 64 x 17 maps, i.e. about two per SM with 8 warps of 16-byte loads in flight;
// wider CTAs would leave SMs idle at this size
// GENERIC = false: the 11x11 kernel every reference config uses, taps and trip counts compiled in (the engine's hot path);
// GENERIC = true: radius and taps from p.taps.
constexpr int DECODE_WARPS = 4;
template <bool GENERIC>
__global__ void __launch_bounds__(DECODE_WARPS * 32) decode_heatmaps(const DecodeParams p) {
  __shared__ float s_rowpass[DECODE_WARPS][7][GENERIC ? 2 * MAX_RADIUS + 1 : 11];
  const int R = GENERIC ? p.taps.radius : 5, KS = 2 * R + 1;
  auto tap = [&](int d) { return GENERIC ? p.taps.t[d] : c_gauss11[5 - d]; };
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g0 = blockIdx.x * DECODE_WARPS + wib;           // map index n*K + k
  const int total = p.n * p.k;
  pdl_launch_dependents();
  pdl_wait();
  if (g0 >= total) return;
  const int g = p.kstride ? (g0 / p.k) * p.kstride + g0 % p.k : g0;   // the map's slot in heatmaps / kpts / idx
  const float* hm = p.heatmaps + static_cast<size_t>(g) * HM_PIX;

  // ---- first-index argmax over 3072 values.  The scan is branch-free so that the loads can run ahead of it (ptxas keeps a
  // rolling window of seven 16-byte loads per lane in flight): the first version's early-return comparison compiled to
  // divergent branches between the loads, which left ONE load in flight per lane.  A lane sees its elements in increasing index order, so "first index wins"
  // is "replace only when strictly better"; a NaN replaces a number and is never replaced (np.argmax: the first NaN).
  float bv;
  int bi;
  {
    const float4* h4 = reinterpret_cast<const float4*>(hm);
    constexpr int NL = HM_PIX / 128;                         // 24 float4 per lane
    float4 v[NL];
#pragma unroll
    for (int j = 0; j < NL; ++j) v[j] = __ldg(h4 + j * 32 + lane);
    bv = v[0].x; bi = lane * 4;
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int base = (j * 32 + lane) * 4;
      const float vv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool take = (vv[e] > bv) | ((vv[e] != vv[e]) & (bv == bv));   // bitwise: no short-circuit branches
        bv = take ? vv[e] : bv;
        bi = take ? base + e : bi;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (arg_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  const float mx = bv;
  const int amax = bi;
  const bool positive = mx > 0.0f;

  // ---- stencil points (map, x, y), order: c, x+1, y+1, x+1y+1, x-1, y-1, x-1y-1
  int x = -1, y = -1;
  const float* pmap[7];
  int ptx[7], pty[7];
  if (positive) {
    x = amax % HM_W;
    y = amax / HM_W;
    const int xm = max(x - 1, 0), xp = min(x + 1, HM_W - 1), ym = max(y - 1, 0), yp = min(y + 1, HM_H - 1);
    const int xs[7] = {x, xp, x, xp, xm, x, xm};
    const int ys[7] = {y, y, yp, yp, y, ym, ym};
#pragma unroll
    for (int i = 0; i < 7; ++i) { pmap[i] = hm; ptx[i] = xs[i]; pty[i] = ys[i]; }
  } else {
    // (-1,-1): four reads land on this map's top-left pad corner (= l(0,0)); the three "minus" reads
    // underflow into the previous map's padded slab: l_prev(W-1,H-1) twice and l_prev(0,H-1).
    const int n_i = g0 / p.k, k_i = g0 % p.k, ks = p.kstride ? p.kstride : p.k;
    const int pc = (g0 + total - 1) % total;                // wrap_batch: the previous compact map of the whole call
    const int prev = p.wrap_batch ? (pc / p.k) * ks + pc % p.k : n_i * ks + (k_i + p.k - 1) % p.k;
    const float* hp = p.heatmaps + static_cast<size_t>(prev) * HM_PIX;
#pragma unroll
    for (int i = 0; i < 4; ++i) { pmap[i] = hm; ptx[i] = 0; pty[i] = 0; }
    pmap[4] = hp; ptx[4] = HM_W - 1; pty[4] = HM_H - 1;     // ix1_   (index - 1)
    pmap[5] = hp; ptx[5] = 0;        pty[5] = HM_H - 1;     // iy1_   (index - W - 2)
    pmap[6] = hp; ptx[6] = HM_W - 1; pty[6] = HM_H - 1;     // ix1_y1_(index - W - 3)
  }

  // ---- row pass of the separable blur: 7 points x 11 rows, one (point,row) per lane per round
  for (int tsk = lane; tsk < 7 * KS; tsk += 32) {
    const int pt = tsk / KS, r = tsk % KS;
    const float* m = pmap[0];
    int cx = ptx[0], cy = pty[0];
#pragma unroll
    for (int i = 1; i < 7; ++i)
      if (pt == i) { m = pmap[i]; cx = ptx[i]; cy = pty[i]; }
    const float* rowp = m + reflect101(cy - R + r, HM_H) * HM_W;
    float acc = 0.0f;
    if constexpr (GENERIC) {
      acc = blur_row(p.taps.t, R, [&](int j) { return __ldg(rowp + reflect101(cx - R + j, HM_W)); });
    } else {
#pragma unroll
      for (int j = 0; j < KS; ++j) acc = __fmaf_rn(tap(j < R ? R - j : j - R), __ldg(rowp + reflect101(cx - R + j, HM_W)), acc);
    }
    s_rowpass[wib][pt][r] = acc;
  }
  __syncwarp();
  // ---- column pass + clip + log on lanes 0..6
  float l = 0.0f;
  if (lane < 7) {
    const float* rp = s_rowpass[wib][lane];
    float acc = __fmul_rn(tap(0), rp[R]);
#pragma unroll
    for (int d = 1; d <= R; ++d) acc = __fmaf_rn(tap(d), __fadd_rn(rp[R + d], rp[R - d]), acc);
    l = logf(acc != acc ? acc : fminf(fmaxf(acc, 1e-3f), 50.0f));   // np.clip keeps NaN (fminf / fmaxf alone would not)
  }
  const float i_ = __shfl_sync(0xffffffffu, l, 0), ix1 = __shfl_sync(0xffffffffu, l, 1);
  const float iy1 = __shfl_sync(0xffffffffu, l, 2), ix1y1 = __shfl_sync(0xffffffffu, l, 3);
  const float ix1_ = __shfl_sync(0xffffffffu, l, 4), iy1_ = __shfl_sync(0xffffffffu, l, 5);
  const float ix1_y1_ = __shfl_sync(0xffffffffu, l, 6);

  if (lane == 0) {
    const float dx = __fmul_rn(0.5f, __fsub_rn(ix1, ix1_));
    const float dy = __fmul_rn(0.5f, __fsub_rn(iy1, iy1_));
    const float two_i = __fmul_rn(2.0f, i_);
    const float dxx = __fadd_rn(__fsub_rn(ix1, two_i), ix1_);
    const float dyy = __fadd_rn(__fsub_rn(iy1, two_i), iy1_);
    float t = __fsub_rn(ix1y1, ix1);
    t = __fsub_rn(t, iy1);
    t = __fadd_rn(t, i_);
    t = __fadd_rn(t, i_);
    t = __fsub_rn(t, ix1_);
    t = __fsub_rn(t, iy1_);
    t = __fadd_rn(t, ix1_y1_);
    const float dxy = __fmul_rn(0.5f, t);
    // float64 2x2 inverse of H + eps*I (top_down_eval.py:413), then coords -= H^-1 g (:414)
    const double eps = 1.1920928955078125e-07;
    const double a = static_cast<double>(dxx) + eps, b = static_cast<double>(dxy), d = static_cast<double>(dyy) + eps;
    const double det = a * d - b * b;
    const double offx = (d * static_cast<double>(dx) - b * static_cast<double>(dy)) / det;
    const double offy = (a * static_cast<double>(dy) - b * static_cast<double>(dx)) / det;
    const float xr = static_cast<float>(static_cast<double>(x) - offx);
    const float yr = static_cast<float>(static_cast<double>(y) - offy);
    const int n_i = g0 / p.k;
    float X, Y;
    if (p.cs32 != nullptr || p.cs64 != nullptr) {
      transform_cs(xr, yr, n_i, p.cs32, p.cs64, true, X, Y);
    } else {
      const int ow = p.org_wh[2 * n_i], oh = p.org_wh[2 * n_i + 1];
      X = static_cast<float>(static_cast<double>(xr) * (ow / (HM_W - 1.0)) + static_cast<double>(ow / 2) - ow * 0.5);
      Y = static_cast<float>(static_cast<double>(yr) * (oh / (HM_H - 1.0)) + static_cast<double>(oh / 2) - oh * 0.5);
    }
    float* o = p.kpts + static_cast<size_t>(g) * 3;
    float Yf = Y, Xf = X;
    if (p.offs_yx != nullptr) {
      // numpy adds the int64 offsets in float64 and casts back: one rounding of an exact sum, which is what a float32
      // add of an exactly representable integer does.  Zero offsets are skipped so that -0.0 survives.
      const int oy = p.offs_yx[2 * n_i], ox = p.offs_yx[2 * n_i + 1];
      if (oy != 0) Yf = __fadd_rn(Y, static_cast<float>(oy));
      if (ox != 0) Xf = __fadd_rn(X, static_cast<float>(ox));
    }
    o[0] = Yf; o[1] = Xf; o[2] = mx;
    if (p.idx != nullptr) p.idx[g] = amax;
  }
}

// ------------------------------------------------------------------------------------------------
// The decode modes VitInference never selects (SURVEY.md section 8 row f4), for mmpose-style callers of
// keypoints_from_heatmaps (vit_utils/top_down_eval.py:493-641):
//   mode 0  post_process=None       argmax only                                           :598
//   mode 1  'default'               +-0.25 px towards the higher neighbour                  :617-631
//   mode 2  'unbiased'              zero-padded Gaussian modulation + log + _taylor          :600-607, :315-350, :416-456
//   mode 3  'megvii'                modulation first, argmax of the modulated map, +-0.25 + 0.5, score / 255 + 0.5   :573-574,:629-639
//   mode 5  use_udp + 'CombinedTarget'  (:580-593) maps come in triples (response, offset x, offset y): the response map is
//           blurred with a (2*kernel+1)^2 Gaussian and arg-maxed, the two offset maps with kernel^2; the offsets at the arg-max,
//           times valid_radius_factor * H, are added to the integer location; transform_preds in its UDP form.
// One CTA per map (the modulation needs every pixel and the global maximum of the blurred map); the map lives in shared memory.
// Modes 2/3 blur with a zero border (what `_gaussian_blur`'s padding amounts to), mode 5 with cv2's default BORDER_REFLECT_101;
// same accumulation order as above.
enum : int { DECODE_NONE = 0, DECODE_DEFAULT = 1, DECODE_UNBIASED = 2, DECODE_MEGVII = 3, DECODE_DARK_UDP = 4, DECODE_COMBINED = 5 };

struct DecodeModesParams {
  const float* heatmaps;   // [N,K,64,48]; mode 5: [N,3K,64,48]
  const float* cs32;       // [N,4] (centre_x, centre_y, scale_x, scale_y) float32, or
  const double* cs64;      // the same as float64 (exactly one of the two is non-null)
  float* kpts;             // [N,K,3] (y, x, score)
  int* idx;                // [N,K] flat argmax of the map the coordinates were read from (may be nullptr)
  int n, k, mode;
  GaussTaps taps;          // `kernel`
  GaussTaps taps_wide;     // 2 * kernel + 1 (mode 5: the response map)
  float valid_radius;      // mode 5: float32(valid_radius_factor * H)
};

// np.argmax / np.amax over the 3072 values in shared memory; result broadcast to every thread
__device__ __forceinline__ void block_argmax(const float* s_map, float* s_rv, int* s_ri, float& bv, int& bi) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  bv = -INFINITY; bi = 0x7fffffff;
  for (int i = tid; i < HM_PIX; i += 256)
    if (arg_better(s_map[i], i, bv, bi)) { bv = s_map[i]; bi = i; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (arg_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  __syncthreads();                                         // previous users of s_rv / s_ri are done
  if (lane == 0) { s_rv[w] = bv; s_ri[w] = bi; }
  __syncthreads();
  bv = s_rv[0]; bi = s_ri[0];
#pragma unroll
  for (int j = 1; j < 8; ++j)
    if (arg_better(s_rv[j], s_ri[j], bv, bi)) { bv = s_rv[j]; bi = s_ri[j]; }
}

// cv2.GaussianBlur(map, (k, k), 0) (BORDER_REFLECT_101) at one point, by one warp; the value is returned on every lane
__device__ __forceinline__ float blur_point_reflect(const float* m, int cx, int cy, const GaussTaps& tp, float* s_rows) {
  const int lane = threadIdx.x & 31, R = tp.radius;
  for (int r = lane; r <= 2 * R; r += 32) {
    const float* rowp = m + reflect101(cy - R + r, HM_H) * HM_W;
    s_rows[r] = blur_row(tp.t, R, [&](int j) { return __ldg(rowp + reflect101(cx - R + j, HM_W)); });
  }
  __syncwarp();
  float acc = __fmul_rn(tp.t[0], s_rows[R]);
  for (int d = 1; d <= R; ++d) acc = __fmaf_rn(tp.t[d], __fadd_rn(s_rows[R + d], s_rows[R - d]), acc);
  return acc;
}

// mode 5, one CTA per keypoint: g = n * K + k, maps 3g (response), 3g + 1 (offset x), 3g + 2 (offset y)
__device__ __forceinline__ void decode_combined(const DecodeModesParams& p, float* s_a, float* s_b, float* s_rv, int* s_ri) {
  __shared__ float s_rows[2][2 * MAX_RADIUS + 1];
  __shared__ float s_off[2];
  const int g = blockIdx.x, tid = threadIdx.x;
  {
    const float4* h4 = reinterpret_cast<const float4*>(p.heatmaps + static_cast<size_t>(3 * g) * HM_PIX);
    for (int i = tid; i < HM_PIX / 4; i += 256) reinterpret_cast<float4*>(s_a)[i] = __ldg(h4 + i);
  }
  __syncthreads();
  const int R = p.taps_wide.radius;
  for (int i = tid; i < HM_PIX; i += 256) {
    const int y = i / HM_W, x = i % HM_W;
    s_b[i] = blur_row(p.taps_wide.t, R, [&](int j) { return s_a[y * HM_W + reflect101(x - R + j, HM_W)]; });
  }
  __syncthreads();
  for (int i = tid; i < HM_PIX; i += 256) {
    const int y = i / HM_W, x = i % HM_W;
    float acc = __fmul_rn(p.taps_wide.t[0], s_b[i]);
    for (int d = 1; d <= R; ++d)
      acc = __fmaf_rn(p.taps_wide.t[d], __fadd_rn(s_b[reflect101(y + d, HM_H) * HM_W + x], s_b[reflect101(y - d, HM_H) * HM_W + x]), acc);
    s_a[i] = acc;
  }
  __syncthreads();
  float mx; int amax;
  block_argmax(s_a, s_rv, s_ri, mx, amax);
  // offsets are read at flat index x + y*W + W*H*g of the [N*K, H*W] offset planes (:588-591); with the (-1,-1) sentinel that
  // index is one row and one pixel before this keypoint's plane: pixel (W-1, H-2) of the previous keypoint's plane, and for
  // g = 0 numpy's negative index wraps to the last plane of the call
  int src = g, ox = amax % HM_W, oy = amax / HM_W;
  float cx = static_cast<float>(ox), cy = static_cast<float>(oy);
  if (!(mx > 0.0f)) {
    cx = cy = -1.0f;
    src = (g + p.n * p.k - 1) % (p.n * p.k); ox = HM_W - 1; oy = HM_H - 2;
  }
  const int w = tid >> 5;
  if (w < 2) {
    const float v = blur_point_reflect(p.heatmaps + static_cast<size_t>(3 * src + 1 + w) * HM_PIX, ox, oy, p.taps, s_rows[w]);
    if ((tid & 31) == 0) s_off[w] = __fmul_rn(v, p.valid_radius);
  }
  __syncthreads();
  if (tid != 0) return;
  float X, Y;
  transform_cs(__fadd_rn(cx, s_off[0]), __fadd_rn(cy, s_off[1]), g / p.k, p.cs32, p.cs64, true, X, Y);
  float* o = p.kpts + static_cast<size_t>(g) * 3;
  o[0] = Y; o[1] = X; o[2] = mx;
  if (p.idx != nullptr) p.idx[g] = amax;
}

__global__ void __launch_bounds__(256) decode_modes(const DecodeModesParams p) {
  __shared__ float s_a[HM_PIX];
  __shared__ float s_b[HM_PIX];
  __shared__ float s_rv[8];
  __shared__ int s_ri[8];
  const int g = blockIdx.x, tid = threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  if (p.mode == DECODE_COMBINED) { decode_combined(p, s_a, s_b, s_rv, s_ri); return; }
  {
    const float4* h4 = reinterpret_cast<const float4*>(p.heatmaps + static_cast<size_t>(g) * HM_PIX);
    for (int i = tid; i < HM_PIX / 4; i += 256) reinterpret_cast<float4*>(s_a)[i] = __ldg(h4 + i);
  }
  __syncthreads();
  float mx; int amax;
  block_argmax(s_a, s_rv, s_ri, mx, amax);                  // raw map: np.argmax, np.amax (= np.max: NaN wins both)
  if (p.mode == DECODE_UNBIASED || p.mode == DECODE_MEGVII) {
    // _gaussian_blur (:416-456): zero-padded kernel x kernel blur, then *= origin_max / max(blurred)
    const int R = p.taps.radius;
    for (int i = tid; i < HM_PIX; i += 256) {
      const int y = i / HM_W, x = i % HM_W;
      s_b[i] = blur_row(p.taps.t, R, [&](int j) {
        const int xx = x - R + j;
        return (xx >= 0 && xx < HM_W) ? s_a[y * HM_W + xx] : 0.0f;
      });
    }
    __syncthreads();
    for (int i = tid; i < HM_PIX; i += 256) {
      const int y = i / HM_W, x = i % HM_W;
      float acc = __fmul_rn(p.taps.t[0], s_b[i]);
      const bool unfused = x >= zero_padded_tail_start(R);      // cv2's scalar tail (5 and 7 taps: the last visible columns)
      for (int d = 1; d <= R; ++d) {
        const float lo = y - d >= 0 ? s_b[(y - d) * HM_W + x] : 0.0f, hi = y + d < HM_H ? s_b[(y + d) * HM_W + x] : 0.0f;
        acc = unfused ? __fadd_rn(acc, __fmul_rn(p.taps.t[d], __fadd_rn(hi, lo))) : __fmaf_rn(p.taps.t[d], __fadd_rn(hi, lo), acc);
      }
      s_a[i] = acc;                                          // the raw map is no longer needed
    }
    __syncthreads();
    float bmax; int bidx;
    block_argmax(s_a, s_rv, s_ri, bmax, bidx);
    const float ratio = __fdiv_rn(mx, bmax);
    for (int i = tid; i < HM_PIX; i += 256) {
      float v = __fmul_rn(s_a[i], ratio);
      if (p.mode == DECODE_UNBIASED) v = logf(v != v ? v : fmaxf(v, 1e-10f));      // np.log(np.maximum(., 1e-10)), NaN propagates
      s_a[i] = v;
    }
    __syncthreads();
    if (p.mode == DECODE_MEGVII) block_argmax(s_a, s_rv, s_ri, mx, amax);          // megvii reads everything from the modulated map
  }
  if (tid != 0) return;
  float cx = -1.0f, cy = -1.0f;
  if (mx > 0.0f) { cx = static_cast<float>(amax % HM_W); cy = static_cast<float>(amax / HM_W); }
  const int px = static_cast<int>(cx), py = static_cast<int>(cy);
  auto at = [&](int yy, int xx) { return s_a[yy * HM_W + xx]; };
  if (p.mode == DECODE_DEFAULT || p.mode == DECODE_MEGVII) {
    if (1 < px && px < HM_W - 1 && 1 < py && py < HM_H - 1) {
      const float dx = __fsub_rn(at(py, px + 1), at(py, px - 1)), dy = __fsub_rn(at(py + 1, px), at(py - 1, px));
      const float sx = dx != dx ? dx : (dx > 0.f ? 1.f : (dx < 0.f ? -1.f : 0.f));      // np.sign (NaN stays NaN)
      const float sy = dy != dy ? dy : (dy > 0.f ? 1.f : (dy < 0.f ? -1.f : 0.f));
      cx = __fadd_rn(cx, __fmul_rn(sx, 0.25f)); cy = __fadd_rn(cy, __fmul_rn(sy, 0.25f));
      if (p.mode == DECODE_MEGVII) { cx = __fadd_rn(cx, 0.5f); cy = __fadd_rn(cy, 0.5f); }
    }
  } else if (p.mode == DECODE_UNBIASED) {
    if (1 < px && px < HM_W - 2 && 1 < py && py < HM_H - 2) {                           // _taylor (:315-350), float32 derivatives
      const float c2 = __fmul_rn(2.0f, at(py, px));
      const float dx = __fmul_rn(0.5f, __fsub_rn(at(py, px + 1), at(py, px - 1)));
      const float dy = __fmul_rn(0.5f, __fsub_rn(at(py + 1, px), at(py - 1, px)));
      const float dxx = __fmul_rn(0.25f, __fadd_rn(__fsub_rn(at(py, px + 2), c2), at(py, px - 2)));
      const float dyy = __fmul_rn(0.25f, __fadd_rn(__fsub_rn(at(py + 2, px), c2), at(py - 2, px)));
      const float dxy = __fmul_rn(0.25f, __fadd_rn(__fsub_rn(__fsub_rn(at(py + 1, px + 1), at(py - 1, px + 1)), at(py + 1, px - 1)),
                                                   at(py - 1, px - 1)));
      if (__fsub_rn(__fmul_rn(dxx, dyy), __fmul_rn(dxy, dxy)) != 0.0f) {
        // the reference inverts the float32 2x2 with LAPACK; closed form in float64 here (tolerance stated in the tests)
        const double a = dxx, b = dxy, d = dyy, det = a * d - b * b;
        cx = static_cast<float>(static_cast<double>(cx) - (d * dx - b * dy) / det);
        cy = static_cast<float>(static_cast<double>(cy) - (a * dy - b * dx) / det);
      }
    }
  }
  float X, Y;
  transform_cs(cx, cy, g / p.k, p.cs32, p.cs64, false, X, Y);
  float score = mx;
  if (p.mode == DECODE_MEGVII) score = __fadd_rn(__fdiv_rn(mx, 255.0f), 0.5f);
  float* o = p.kpts + static_cast<size_t>(g) * 3;
  o[0] = Y; o[1] = X; o[2] = score;
  if (p.idx != nullptr) p.idx[g] = amax;
}

}  // namespace vpb
