// Crop pre-processing (SURVEY.md section 8 row f1): frame uint8 RGB [H,W,3] + int boxes [n,4]  ->  normalised crops
// f32 [n,3,256,192], canvas sizes [n,2] (w,h) and frame offsets [n,2] (y,x), one launch for all people of a frame.
// HBM/L2-bound: 589 824 B written per crop; the gather side re-reads frame pixels that stay in L2.
//
// Restates, per box, what VitInference.inference does on the CPU:
//   easy_ViTPose/inference.py:259-261   box +-10 px, clipped to the frame
//   easy_ViTPose/inference.py:264-265   crop, then pad_image(crop, 3/4): zero-pad to a 3:4 canvas (vit_utils/inference.py:41-70);
//                                       the canvas is never materialised here, out-of-crop taps read 0
//   easy_ViTPose/inference.py:314-318   pre_img: cv2.resize(.., (192,256), INTER_LINEAR) on uint8, /255, (x-MEAN)/STD in
//                                       float64, HWC -> CHW, astype(float32)
//   easy_ViTPose/inference.py:270       offset (y0 - top_pad, x0 - left_pad) that maps crop keypoints back to the frame
// cv2's uint8 bilinear resize is fixed-point; the arithmetic below is its exact integer pipeline (oracle/preproc_oracle.py
// documents and pins it): int16 coefficients rint(frac * 2048), horizontal sums in int32, vertical
// (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.  The horizontal pass clamps (index, fraction) at the
// borders, the vertical pass clamps only the row indices.  Normalisation is a 3x256 table computed in float64, so the
// crops are bit-identical to the reference's.
#pragma once
#include <cuda_bf16.h>

#include <cstdint>

#include "ptx.cuh"

namespace vpb {

constexpr int PP_W = 192, PP_H = 256, PP_ROWS = 16;     // one CTA: 192 columns x 16 output rows of one crop

struct PreprocParams {
  const uint8_t* frame;       // [fh, fw, 3] RGB, row pitch `pitch` bytes
  long long pitch;
  int fh, fw;
  const int* bboxes;          // [n,4] (x0, y0, x1, y1), already rounded to int (inference.py:253)
  int n, pad;
  float* crops;               // [n,3,256,192]
  int* org_wh;                // [n,2] canvas (w, h)
  int* offs_yx;               // [n,2] (y0 - top_pad, x0 - left_pad)
  int* status;                // bit 0 set if any box is empty after clipping (may be nullptr)
};

struct PpAxis { int i0, i1, a0, a1; };

// cv2: scale = 1 / (dst / src) in double
__device__ __forceinline__ double pp_scale(int dn, int sn) {
  return __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(dn), static_cast<double>(sn)));
}
// destination index d -> the two source indices and int16 weights over a source of `sn` samples
__device__ __forceinline__ PpAxis pp_axis(int d, double scale, int sn, bool clamp_fraction) {
  const float f = static_cast<float>(__dadd_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), -0.5));
  int s = __float2int_rd(f);
  float fr = __fsub_rn(f, static_cast<float>(s));
  if (clamp_fraction) {
    if (s < 0) { s = 0; fr = 0.f; }
    if (s >= sn - 1) { s = sn - 1; fr = 0.f; }
  }
  PpAxis a;
  a.a1 = __float2int_rn(__fmul_rn(fr, 2048.f));
  a.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fr), 2048.f));
  a.i0 = min(max(s, 0), sn - 1);
  a.i1 = min(max(s + 1, 0), sn - 1);
  return a;
}

__global__ void __launch_bounds__(PP_W) crop_resize_normalise(const PreprocParams p) {
  __shared__ float s_lut[3][256];
  __shared__ PpAxis s_ay[PP_ROWS];
  const int crop = blockIdx.x, dx = threadIdx.x, dy0 = blockIdx.y * PP_ROWS;
  for (int i = dx; i < 768; i += PP_W) {                   // inference.py:32-33 MEAN / STD, float64 as in pre_img
    const int c = i >> 8, v = i & 255;
    const double mean = c == 0 ? 0.485 : (c == 1 ? 0.456 : 0.406), stdv = c == 0 ? 0.229 : (c == 1 ? 0.224 : 0.225);
    s_lut[c][v] = static_cast<float>(__ddiv_rn(__dsub_rn(__ddiv_rn(static_cast<double>(v), 255.0), mean), stdv));
  }
  const int* bb = p.bboxes + 4 * crop;
  const int x0 = min(max(bb[0] - p.pad, 0), p.fw), x1 = min(max(bb[2] + p.pad, 0), p.fw);
  const int y0 = min(max(bb[1] - p.pad, 0), p.fh), y1 = min(max(bb[3] + p.pad, 0), p.fh);
  const int w = x1 - x0, h = y1 - y0;
  __syncthreads();
  float* out = p.crops + static_cast<size_t>(crop) * 3 * PP_H * PP_W;
  if (w <= 0 || h <= 0) {                                   // the reference raises here; flag it, emit a black crop
    if (dx == 0 && blockIdx.y == 0) {
      if (p.status) atomicOr(p.status, 1);
      p.org_wh[2 * crop] = 0; p.org_wh[2 * crop + 1] = 0;
      p.offs_yx[2 * crop] = y0; p.offs_yx[2 * crop + 1] = x0;
    }
    for (int r = 0; r < PP_ROWS; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) out[(c * PP_H + dy0 + r) * PP_W + dx] = s_lut[c][0];
    return;
  }
  // pad_image: w / h < 3 / 4  <=>  4w < 3h;  int(0.75 * h) = 3h / 4,  int(w / 0.75) = 4w / 3
  int cw = w, ch = h, left = 0, top = 0;
  if (4 * w < 3 * h) { cw = (3 * h) / 4; left = (cw - w) / 2; }
  else { ch = (4 * w) / 3; top = (ch - h) / 2; }
  if (dx == 0 && blockIdx.y == 0) {
    p.org_wh[2 * crop] = cw; p.org_wh[2 * crop + 1] = ch;
    p.offs_yx[2 * crop] = y0 - top; p.offs_yx[2 * crop + 1] = x0 - left;
  }
  if (dx < PP_ROWS) s_ay[dx] = pp_axis(dy0 + dx, pp_scale(PP_H, ch), ch, false);   // the row weights are shared by the CTA
  const PpAxis ax = pp_axis(dx, pp_scale(PP_W, cw), cw, true);
  __syncthreads();
  const int cx0 = ax.i0 - left, cx1 = ax.i1 - left;          // canvas column -> crop column
  const bool vx0 = cx0 >= 0 && cx0 < w, vx1 = cx1 >= 0 && cx1 < w;
  const uint8_t* col0 = p.frame + static_cast<size_t>(vx0 ? x0 + cx0 : 0) * 3;   // only dereferenced when valid
  const uint8_t* col1 = p.frame + static_cast<size_t>(vx1 ? x0 + cx1 : 0) * 3;
#pragma unroll 4
  for (int r = 0; r < PP_ROWS; ++r) {
    const int dy = dy0 + r;
    const PpAxis ay = s_ay[r];
    const int cy0 = ay.i0 - top, cy1 = ay.i1 - top;
    const bool vy0 = cy0 >= 0 && cy0 < h, vy1 = cy1 >= 0 && cy1 < h;
    const size_t r0 = static_cast<size_t>(vy0 ? y0 + cy0 : 0) * p.pitch, r1 = static_cast<size_t>(vy1 ? y0 + cy1 : 0) * p.pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int p00 = (vy0 && vx0) ? col0[r0 + c] : 0, p01 = (vy0 && vx1) ? col1[r0 + c] : 0;
      const int p10 = (vy1 && vx0) ? col0[r1 + c] : 0, p11 = (vy1 && vx1) ? col1[r1 + c] : 0;
      const int s0 = p00 * ax.a0 + p01 * ax.a1, s1 = p10 * ax.a0 + p11 * ax.a1;
      int v = (((ay.a0 * (s0 >> 4)) >> 16) + ((ay.a1 * (s1 >> 4)) >> 16) + 2) >> 2;
      v = min(max(v, 0), 255);
      out[(c * PP_H + dy) * PP_W + dx] = s_lut[c][v];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The same pre-processing fused with the patch-embedding im2col (pointwise.cuh: patch_im2col): frame + boxes -> bf16 patch
// rows [n*192, 768] directly, so the f32 crops (589 824 B each) are never written or re-read.  Values are bf16(table[v]),
// i.e. exactly what patch_im2col produces from crop_resize_normalise's output.  One CTA = one crop x one patch row (16 image
// rows incl. the conv's 2-pixel zero border): the 16 x 192 x 3 pixels are gathered with lanes along the image row into a
// shared bf16 tile, which is then written out as 16-byte chunks of the im2col rows.
// Like patch_im2col, the launch also seeds the fp32 token stream with pos_embed + conv bias (vit.py:382).
// Flip test: a grid of (2 pp.n, 16) CTAs; crop c >= pp.n is the mirror image of crop c - pp.n (box c - pp.n, pixel dx stored at
// tile column 2 + (191 - dx)), i.e. the patch rows of flip(crop, dims=[3]).  Mirrored CTAs leave org_wh / offs_yx / status alone.
// Frames: the boxes may come from up to FP_MAX_FRAMES frames (vpb_infer_frames).  Frame j owns boxes first_box[j] ..
// first_box[j+1]-1 (first_box strictly increasing, frames[0].first_box = 0); a single-frame call is a one-entry table.  The
// table travels in the kernel's parameter block (64 x 32 B of the 4 KB): nothing to allocate or copy per call, and no shared
// device buffer that two calls in flight could race on.  The entry is picked by a run-time index; __grid_constant__ guarantees
// that this reads the parameter block in place, where a plain by-value parameter would allow the compiler to copy it to
// local memory (ptxas reports no stack frame for the kernel either way with CUDA 12.9).
// YUV frames (vpb_infer_frames_yuv, vpb_infer_frames_nv12): the kernels are templated on the table entry; a YuvEntry tap
// reads its Y byte and the (U, V) pair of its chroma block and converts them to RGB (yuv_rgb) before the unchanged resize /
// warp arithmetic, so the result is that of cv2.cvtColor(COLOR_YUV2RGB_<layout>) (or the full-range conversion) followed
// by the RGB path.  Taps outside the crop or frame still read RGB 0.
// Rotated frames (vpb_frame.rotation): an entry's fh / fw, pitches and planes describe the STORED frame, and `rot` (0..3 =
// 0, 90, 180, 270 degrees counter-clockwise) turns it into the VIEW the boxes and matrices are given in, the frame that
// cv2.rotate(stored, ROTATE_90_COUNTERCLOCKWISE | ROTATE_180 | ROTATE_90_CLOCKWISE) would produce.  Clipping, padding and
// bounds tests use the view's size (view_hw); each tap maps its view pixel to the stored pixel (stored_px) only to address
// it, so a rotated call reads exactly the bytes an upright call on the rotated copy reads.
constexpr int FP_MAX_FRAMES = 64;
struct FrameEntry {
  static constexpr bool kYuv = false;
  const uint8_t* data;          // [fh, fw, 3] RGB, row pitch `pitch` bytes
  long long pitch;
  int fh, fw;
  int first_box;
  int rot;                      // 0..3: the view is the stored frame turned by 90 rot degrees counter-clockwise
};
static_assert(sizeof(FrameEntry) == 32, "frame table entry layout");
// Every 8-bit layout is described by pointers and steps, with no per-layout branch in the kernels:
//   luma of pixel (x, row)    y[row * y_pitch + x * y_step]
//   chroma of pixel (x, row)  u[(row >> c_vshift) * c_pitch + (x >> 1) * c_step], and v at the same offset from its pointer
// The host fills them per layout (engine.cu: yuv_entry):
//   NV12  Y plane, 1 | uv, uv + 1 | 2 | 1        I420  Y plane, 1 | U plane, V plane | 1 | 1
//   NV21  Y plane, 1 | vu + 1, vu | 2 | 1        YV12  the same (V is stored first)
//   YUYV  base, 2 | base + 1, base + 3 | 4 | 0   UYVY  base + 1, 2 | base, base + 2 | 4 | 0
constexpr int YUV_BT601 = 0, YUV_BT709 = 1;
constexpr int YUV_LIMITED = 0, YUV_FULL = 1;
struct YuvEntry {
  static constexpr bool kYuv = true;
  const uint8_t* y;
  const uint8_t* u;
  const uint8_t* v;
  long long y_pitch, c_pitch;   // row pitches in bytes; U and V share one
  int fh, fw;                   // fw even; fh even for 4:2:0
  int first_box;
  uint8_t y_step, c_step, c_vshift;
  uint8_t conv : 2;             // matrix | range << 1 (YUV_BT601 | YUV_BT709, YUV_LIMITED | YUV_FULL), the same for every entry of a call
  uint8_t rot : 2;              // as FrameEntry::rot
};
static_assert(sizeof(YuvEntry) == 56, "YUV frame table entry layout");

// (view height, view width) of an entry: the stored size, swapped for 90 and 270 degrees
template <class Entry>
__device__ __forceinline__ int2 view_hw(const Entry& f) { return f.rot & 1 ? make_int2(f.fw, f.fh) : make_int2(f.fh, f.fw); }
// view pixel (x, y) -> the stored pixel (sx, sy) it shows, for a view pixel inside the view; np.rot90(stored, rot)[y, x]:
//   rot 0: (x, y)   1: (fw-1-y, x)   2: (fw-1-x, fh-1-y)   3: (y, fh-1-x)
// i.e. an axis swap for 90 / 270 and a reflection of stored x (90, 180) and of stored y (180, 270).
template <class Entry>
__device__ __forceinline__ int2 stored_px(const Entry& f, int x, int y) {
  const int rot = f.rot, a = rot & 1 ? y : x, b = rot & 1 ? x : y;
  return make_int2(rot == 1 || rot == 2 ? f.fw - 1 - a : a, rot & 2 ? f.fh - 1 - b : b);
}
// byte offset of view pixel (x, y) in an RGB entry
__device__ __forceinline__ size_t rgb_offset(const FrameEntry& f, int x, int y) {
  const int2 s = stored_px(f, x, y);
  return static_cast<size_t>(s.y) * f.pitch + s.x * 3;
}

// Both conversions as one fixed-point form: out = clamp((max(Y - y0, 0) * cy + half + c_v (V - 128) + c_u (U - 128)) >> shift).
//   limited range: cv2's COLOR_YUV2RGB_NV12 (SHIFT 20, y0 = 16): oracle/nv12_oracle.py pins the formula.  The BT.709 set is
//                  round(2^20 x (1.164, 1.793, -0.533, -0.213, 2.112)), the 3-decimal form cv2 uses for BT.601.
//   full range:    cv2's COLOR_YCrCb2RGB (SHIFT 14): Y + ((c (C - 128) + 2^13) >> 14), written with y0 = 0 and cy = 2^14, since
//                  (Y 2^14 + s) >> 14 = Y + (s >> 14) exactly.  BT.709 is round(2^14 x (1.575, -0.468, -0.187, 1.856)).
struct YuvCoef { int y0, cy, half, shift, cvr, cvg, cug, cub; };
__device__ __forceinline__ YuvCoef yuv_coef(int conv) {
  switch (conv) {
    case YUV_BT709: return {16, 1220542, 1 << 19, 20, 1880097, -558891, -223347, 2214593};
    case YUV_BT601 | YUV_FULL << 1: return {0, 1 << 14, 1 << 13, 14, 22987, -11698, -5636, 29049};
    case YUV_BT709 | YUV_FULL << 1: return {0, 1 << 14, 1 << 13, 14, 25805, -7668, -3064, 30409};
    default: return {16, 1220542, 1 << 19, 20, 1673527, -852492, -409993, 2116026};
  }
}
// view pixel (vx, vy) of a YUV frame -> RGB: the stored pixel's Y and its stored chroma block; every intermediate fits in
// int32 (|sum| < 2^30)
__device__ __forceinline__ void yuv_rgb(const YuvEntry& f, const YuvCoef& k, int vx, int vy, int rgb[3]) {
  const int2 s = stored_px(f, vx, vy);
  const int x = s.x, y = s.y;
  const int Y = f.y[static_cast<size_t>(y) * f.y_pitch + x * f.y_step];
  const size_t c = static_cast<size_t>(y >> f.c_vshift) * f.c_pitch + (x >> 1) * f.c_step;
  const int u = f.u[c] - 128, v = f.v[c] - 128;
  const int yy = max(Y - k.y0, 0) * k.cy + k.half;
  rgb[0] = min(max((yy + k.cvr * v) >> k.shift, 0), 255);
  rgb[1] = min(max((yy + k.cvg * v + k.cug * u) >> k.shift, 0), 255);
  rgb[2] = min(max((yy + k.cub * u) >> k.shift, 0), 255);
}

template <class Entry>
struct FramePatchParamsT {
  PreprocParams pp;             // frame / pitch / fh / fw / crops unused (the table holds the frames); pp.n = number of boxes
  __nv_bfloat16* rows;          // [n*192, 768]
  const float4* pos_bias;       // [192*D/4]
  float4* stream;               // [n*192*D/4]
  int D;
  int num_frames;               // 1..FP_MAX_FRAMES
  Entry frames[FP_MAX_FRAMES];
};
using FramePatchParams = FramePatchParamsT<FrameEntry>;
static_assert(sizeof(FramePatchParamsT<FrameEntry>) <= 4096 && sizeof(FramePatchParamsT<YuvEntry>) <= 4096,
              "the frame table travels in the 4 KB parameter block");

template <class Entry>
__global__ void __launch_bounds__(384) frame_to_patch_rows(const __grid_constant__ FramePatchParamsT<Entry> q) {
  constexpr int FP_PITCH = 208;                               // 2 + 192 + 14 bf16 per tile row: 16-byte aligned rows
  __shared__ uint16_t s_lut[3][256];
  __shared__ PpAxis s_ay[16];
  __shared__ PpAxis s_ax[PP_W];
  __shared__ __align__(16) uint16_t s_tile[3 * 16 * FP_PITCH];
  const PreprocParams& p = q.pp;
  const int crop = blockIdx.x, py = blockIdx.y, tid = threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();                                               // the previous step may still be reading patch rows / the stream
  {
    const int per_crop4 = 192 * q.D / 4, per_cta4 = per_crop4 / 16;      // this CTA seeds 1/16 of its crop's tokens
    const float4* src = q.pos_bias + py * per_cta4;
    float4* dst = q.stream + static_cast<size_t>(crop) * per_crop4 + py * per_cta4;
    for (int j = tid; j < per_cta4; j += 384) dst[j] = __ldg(src + j);
  }
  for (int i = tid; i < 768; i += 384) {
    const int c = i >> 8, v = i & 255;
    const double mean = c == 0 ? 0.485 : (c == 1 ? 0.456 : 0.406), stdv = c == 0 ? 0.229 : (c == 1 ? 0.224 : 0.225);
    const float f = static_cast<float>(__ddiv_rn(__dsub_rn(__ddiv_rn(static_cast<double>(v), 255.0), mean), stdv));
    s_lut[c][v] = __bfloat16_as_ushort(__float2bfloat16_rn(f));
  }
  const bool mirror = crop >= p.n;
  const int box = mirror ? crop - p.n : crop;
  int lo = 0, hi = q.num_frames;                              // the last frame whose first_box <= box
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (q.frames[mid].first_box <= box) lo = mid; else hi = mid;
  }
  const Entry& fr = q.frames[lo];
  const int2 vhw = view_hw(fr);                               // boxes are clipped to the view
  const int fh = vhw.x, fw = vhw.y;
  const int* bb = p.bboxes + 4 * box;
  const int x0 = min(max(bb[0] - p.pad, 0), fw), x1 = min(max(bb[2] + p.pad, 0), fw);
  const int y0 = min(max(bb[1] - p.pad, 0), fh), y1 = min(max(bb[3] + p.pad, 0), fh);
  int w = x1 - x0, h = y1 - y0;
  const bool empty = w <= 0 || h <= 0;
  if (empty) { w = 0; h = 0; }
  int cw = max(w, 1), ch = max(h, 1), left = 0, top = 0;    // an empty box reads nothing: a black crop, as in crop_resize_normalise
  if (!empty) {
    if (4 * w < 3 * h) { cw = (3 * h) / 4; left = (cw - w) / 2; }
    else { ch = (4 * w) / 3; top = (ch - h) / 2; }
  }
  if (tid == 0 && py == 0 && !mirror) {
    if (empty && p.status) atomicOr(p.status, 1);
    p.org_wh[2 * crop] = empty ? 0 : cw; p.org_wh[2 * crop + 1] = empty ? 0 : ch;
    p.offs_yx[2 * crop] = y0 - top; p.offs_yx[2 * crop + 1] = x0 - left;
  }
  if (tid < PP_W) s_ax[tid] = pp_axis(tid, pp_scale(PP_W, cw), cw, true);
  else if (tid < PP_W + 16) {
    const int dy = 16 * py - 2 + (tid - PP_W);
    if (dy >= 0) s_ay[tid - PP_W] = pp_axis(dy, pp_scale(PP_H, ch), ch, false);
  }
  __syncthreads();
  // Phase 1: one (row, column) pixel per thread-iteration with consecutive lanes on consecutive output columns, so that a
  // warp's byte gathers fall into neighbouring sectors; bf16 values go to a shared tile laid out [channel][ky][2 + dx]
  // (column 0,1 and 194..207 = the conv's zero padding / alignment).
  for (int i = tid; i < 3 * 16 * 8; i += 384) {              // zero the padding columns once: 16 bf16 per (c, ky) row
    const int row = i >> 3, e = i & 7;
    s_tile[row * FP_PITCH + (e < 2 ? e : 192 + e)] = 0;
  }
  for (int i = tid; i < 16 * PP_W; i += 384) {
    const int ky = i / PP_W, dx = i % PP_W;
    const int dy = 16 * py - 2 + ky;
    uint16_t v3[3] = {0, 0, 0};
    if (dy >= 0) {
      const PpAxis ay = s_ay[ky];
      const PpAxis ax = s_ax[dx];
      const int cy0 = ay.i0 - top, cy1 = ay.i1 - top, cx0 = ax.i0 - left, cx1 = ax.i1 - left;
      const bool vy0 = cy0 >= 0 && cy0 < h, vy1 = cy1 >= 0 && cy1 < h, vx0 = cx0 >= 0 && cx0 < w, vx1 = cx1 >= 0 && cx1 < w;
      if constexpr (Entry::kYuv) {
        const YuvCoef k = yuv_coef(fr.conv);
        int t00[3] = {0, 0, 0}, t01[3] = {0, 0, 0}, t10[3] = {0, 0, 0}, t11[3] = {0, 0, 0};   // out-of-crop taps: RGB 0
        if (vy0 && vx0) yuv_rgb(fr, k, x0 + cx0, y0 + cy0, t00);
        if (vy0 && vx1) yuv_rgb(fr, k, x0 + cx1, y0 + cy0, t01);
        if (vy1 && vx0) yuv_rgb(fr, k, x0 + cx0, y0 + cy1, t10);
        if (vy1 && vx1) yuv_rgb(fr, k, x0 + cx1, y0 + cy1, t11);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int s0 = t00[c] * ax.a0 + t01[c] * ax.a1, s1 = t10[c] * ax.a0 + t11[c] * ax.a1;
          int v = (((ay.a0 * (s0 >> 4)) >> 16) + ((ay.a1 * (s1 >> 4)) >> 16) + 2) >> 2;
          v3[c] = s_lut[c][min(max(v, 0), 255)];
        }
      } else {
        const int X0 = vx0 ? x0 + cx0 : 0, X1 = vx1 ? x0 + cx1 : 0;           // view pixels, only dereferenced when valid
        const int Y0 = vy0 ? y0 + cy0 : 0, Y1 = vy1 ? y0 + cy1 : 0;
        const uint8_t *t00 = fr.data + rgb_offset(fr, X0, Y0), *t01 = fr.data + rgb_offset(fr, X1, Y0);
        const uint8_t *t10 = fr.data + rgb_offset(fr, X0, Y1), *t11 = fr.data + rgb_offset(fr, X1, Y1);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int p00 = (vy0 && vx0) ? t00[c] : 0, p01 = (vy0 && vx1) ? t01[c] : 0;
          const int p10 = (vy1 && vx0) ? t10[c] : 0, p11 = (vy1 && vx1) ? t11[c] : 0;
          const int s0 = p00 * ax.a0 + p01 * ax.a1, s1 = p10 * ax.a0 + p11 * ax.a1;
          int v = (((ay.a0 * (s0 >> 4)) >> 16) + ((ay.a1 * (s1 >> 4)) >> 16) + 2) >> 2;
          v3[c] = s_lut[c][min(max(v, 0), 255)];
        }
      }
    }
    const int tx = 2 + (mirror ? PP_W - 1 - dx : dx);
#pragma unroll
    for (int c = 0; c < 3; ++c) s_tile[(c * 16 + ky) * FP_PITCH + tx] = v3[c];
  }
  __syncthreads();
  // Phase 2: the im2col rows of this patch row, 16 bytes (8 kx) per store: element (px, c, ky, kx) = tile[c][ky][16 px + kx]
  for (int i = tid; i < 12 * 3 * 16 * 2; i += 384) {
    const int hf = i & 1, ky = (i >> 1) & 15, c = (i >> 5) % 3, px = i / 96;
    const uint4 v = *reinterpret_cast<const uint4*>(&s_tile[(c * 16 + ky) * FP_PITCH + 16 * px + 8 * hf]);
    *reinterpret_cast<uint4*>(q.rows + ((static_cast<size_t>(crop) * 16 + py) * 12 + px) * 768 + c * 256 + ky * 16 + 8 * hf) = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Affine top-down crops (the mmpose / HRNet data path of the reference's datasets/COCO.py:288-302): per box a 2x3 matrix
// M (what the caller hands to cv2.warpAffine), cv2.warpAffine(frame, M, (192, 256), INTER_LINEAR, constant 0 border), then
// torchvision ToTensor + Normalize in float32.  cv2's uint8 path is fixed-point and restated exactly (oracle/affine_oracle.py
// pins it against cv2 4.13):
//   the inverse of M in double (D = M0 M4 - M1 M3, 1/D or 0 for a singular M), then with AB_BITS = 10, INTER_BITS = 5
//   adelta[x] = cvRound(M0' x 1024), X0(y) = cvRound((M1' y + M2') 1024) + 16, X = (X0 + adelta) >> 5 (same for Y):
//   integer tap X >> 5 (int16-saturated), fraction X & 31; int16 weights (32 - f | f)_y (32 - f | f)_x 32, which sum to 32768
//   exactly; pixel (sum w p + 2^14) >> 15 with taps outside the frame reading 0.
// The double arithmetic is spelled with __dmul_rn / __dadd_rn so that nothing contracts into an FMA (cv2 rounds each step).
struct AffineInv { double m[6]; };     // the inverted matrix (M0', M1', M2', M3', M4', M5')
__device__ __forceinline__ AffineInv affine_invert(const double* M) {
  const double m0 = M[0], m1 = M[1], m2 = M[2], m3 = M[3], m4 = M[4], m5 = M[5];
  double d = __dsub_rn(__dmul_rn(m0, m4), __dmul_rn(m1, m3));
  d = d != 0.0 ? __ddiv_rn(1.0, d) : 0.0;
  AffineInv r;
  r.m[0] = __dmul_rn(m4, d);
  r.m[1] = __dmul_rn(m1, -d);
  r.m[3] = __dmul_rn(m3, -d);
  r.m[4] = __dmul_rn(m0, d);
  r.m[2] = __dsub_rn(__dmul_rn(-r.m[0], m2), __dmul_rn(r.m[1], m5));
  r.m[5] = __dsub_rn(__dmul_rn(-r.m[3], m2), __dmul_rn(r.m[4], m5));
  return r;
}
// adelta / bdelta of output column x
__device__ __forceinline__ int2 affine_col(const AffineInv& a, int x) {
  return make_int2(__double2int_rn(__dmul_rn(__dmul_rn(a.m[0], static_cast<double>(x)), 1024.0)),
                   __double2int_rn(__dmul_rn(__dmul_rn(a.m[3], static_cast<double>(x)), 1024.0)));
}
// X0 / Y0 of output row y (the +16 = round_delta of INTER_BITS)
__device__ __forceinline__ int2 affine_row(const AffineInv& a, int y) {
  const double yd = static_cast<double>(y);
  return make_int2(__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[1], yd), a.m[2]), 1024.0)) + 16,
                   __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[4], yd), a.m[5]), 1024.0)) + 16);
}
// one output pixel from its fixed-point source coordinates (view pixels): the three warped bytes
__device__ __forceinline__ void affine_pixel(const FrameEntry& f, int X, int Y, int v[3]) {
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767), fx = X & 31, fy = Y & 31;
  const int2 vhw = view_hw(f);
  const int fh = vhw.x, fw = vhw.y;
  const bool vx0 = sx >= 0 && sx < fw, vx1 = sx + 1 >= 0 && sx + 1 < fw, vy0 = sy >= 0 && sy < fh, vy1 = sy + 1 >= 0 && sy + 1 < fh;
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
  const int X0 = vx0 ? sx : 0, X1 = vx1 ? sx + 1 : 0, Y0 = vy0 ? sy : 0, Y1 = vy1 ? sy + 1 : 0;   // only dereferenced when valid
  const uint8_t *t00 = f.data + rgb_offset(f, X0, Y0), *t01 = f.data + rgb_offset(f, X1, Y0);
  const uint8_t *t10 = f.data + rgb_offset(f, X0, Y1), *t11 = f.data + rgb_offset(f, X1, Y1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int p00 = (vy0 && vx0) ? t00[c] : 0, p01 = (vy0 && vx1) ? t01[c] : 0;
    const int p10 = (vy1 && vx0) ? t10[c] : 0, p11 = (vy1 && vx1) ? t11[c] : 0;
    v[c] = (p00 * w00 + p01 * w01 + p10 * w10 + p11 * w11 + (1 << 14)) >> 15;
  }
}
// the same from a YUV frame: each tap converted to RGB first, the constant border is RGB 0
__device__ __forceinline__ void affine_pixel_yuv(const YuvEntry& f, const YuvCoef& k, int X, int Y, int v[3]) {
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767), fx = X & 31, fy = Y & 31;
  const int2 vhw = view_hw(f);
  const int fh = vhw.x, fw = vhw.y;
  const bool vx0 = sx >= 0 && sx < fw, vx1 = sx + 1 >= 0 && sx + 1 < fw, vy0 = sy >= 0 && sy < fh, vy1 = sy + 1 >= 0 && sy + 1 < fh;
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
  int t00[3] = {0, 0, 0}, t01[3] = {0, 0, 0}, t10[3] = {0, 0, 0}, t11[3] = {0, 0, 0};
  if (vy0 && vx0) yuv_rgb(f, k, sx, sy, t00);
  if (vy0 && vx1) yuv_rgb(f, k, sx + 1, sy, t01);
  if (vy1 && vx0) yuv_rgb(f, k, sx, sy + 1, t10);
  if (vy1 && vx1) yuv_rgb(f, k, sx + 1, sy + 1, t11);
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = (t00[c] * w00 + t01[c] * w01 + t10[c] * w10 + t11[c] * w11 + (1 << 14)) >> 15;
}
// torchvision ToTensor + Normalize (COCO.py:120-123): float32 throughout, IEEE division
__device__ __forceinline__ float affine_norm(int c, int v) {
  const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f), stdv = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
  return __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v), 255.f), mean), stdv);
}

// Launch parameters of both affine kernels.  The frame table is frame_to_patch_rows' (same binary search on first_box).
template <class Entry>
struct AffineParamsT {
  const double* mats;           // [n,6] f64: the matrix given to cv2.warpAffine (image -> crop)
  const float* cs;              // [n,4] (cx, cy, sx, sy) of the decode, checked for sx, sy > 0 (may be nullptr)
  int n;
  int* status;                  // bit 1 set if a matrix entry is not finite or a scale <= 0 (may be nullptr)
  float* crops;                 // crop_warp_normalise: [n,3,256,192]
  __nv_bfloat16* rows;          // frame_to_patch_rows_affine: [n*192, 768] (or [2n*192, 768] with the mirrors)
  const float4* pos_bias;
  float4* stream;
  int D;
  int num_frames;
  Entry frames[FP_MAX_FRAMES];
};
using AffineParams = AffineParamsT<FrameEntry>;
static_assert(sizeof(AffineParamsT<FrameEntry>) <= 4096 && sizeof(AffineParamsT<YuvEntry>) <= 4096,
              "the frame table travels in the 4 KB parameter block");
template <class Entry>
__device__ __forceinline__ const Entry& affine_frame(const AffineParamsT<Entry>& q, int box) {
  int lo = 0, hi = q.num_frames;                              // the last frame whose first_box <= box
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (q.frames[mid].first_box <= box) lo = mid; else hi = mid;
  }
  return q.frames[lo];
}
// the device forms cannot return an error for a bad matrix without a sync: flag it (the arithmetic stays in bounds)
template <class Entry>
__device__ __forceinline__ void affine_check(const AffineParamsT<Entry>& q, int box) {
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) ok = ok && isfinite(q.mats[6 * box + i]);
  if (q.cs) ok = ok && q.cs[4 * box + 2] > 0.f && q.cs[4 * box + 3] > 0.f;
  if (!ok && q.status) atomicOr(q.status, 2);
}

// f32 crops [n,3,256,192]: one CTA = one crop x 16 output rows, one thread per column
__global__ void __launch_bounds__(PP_W) crop_warp_normalise(const __grid_constant__ AffineParams q) {
  __shared__ int2 s_row[PP_ROWS];
  const int crop = blockIdx.x, dx = threadIdx.x, dy0 = blockIdx.y * PP_ROWS;
  const FrameEntry& fr = affine_frame(q, crop);
  const AffineInv a = affine_invert(q.mats + 6 * crop);
  if (dx < PP_ROWS) s_row[dx] = affine_row(a, dy0 + dx);
  if (dx == 0 && blockIdx.y == 0) affine_check(q, crop);
  const int2 col = affine_col(a, dx);
  __syncthreads();
  float* out = q.crops + static_cast<size_t>(crop) * 3 * PP_H * PP_W;
  for (int r = 0; r < PP_ROWS; ++r) {
    int v[3];
    affine_pixel(fr, (s_row[r].x + col.x) >> 5, (s_row[r].y + col.y) >> 5, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[(c * PP_H + dy0 + r) * PP_W + dx] = affine_norm(c, v[c]);
  }
}

// The same warp fused with the patch-embedding im2col: frame_to_patch_rows with a matrix per box instead of an int box.
// Same grid ((n or 2n) x 16 CTAs, crop c >= n the mirror image of crop c - n), bf16 tile, im2col store and pos_embed + bias
// seeding; each CTA inverts its matrix once and keeps adelta / bdelta of the 192 columns and X0 / Y0 of its 16 rows in shared
// memory.  Rows 16 py - 2 < 0 are the conv's zero padding and are never warped.
template <class Entry>
__global__ void __launch_bounds__(384) frame_to_patch_rows_affine(const __grid_constant__ AffineParamsT<Entry> q) {
  constexpr int FP_PITCH = 208;                               // as frame_to_patch_rows
  __shared__ uint16_t s_lut[3][256];
  __shared__ int2 s_row[16];
  __shared__ int2 s_col[PP_W];
  __shared__ __align__(16) uint16_t s_tile[3 * 16 * FP_PITCH];
  const int crop = blockIdx.x, py = blockIdx.y, tid = threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();                                               // the previous step may still be reading patch rows / the stream
  {
    const int per_crop4 = 192 * q.D / 4, per_cta4 = per_crop4 / 16;
    const float4* src = q.pos_bias + py * per_cta4;
    float4* dst = q.stream + static_cast<size_t>(crop) * per_crop4 + py * per_cta4;
    for (int j = tid; j < per_cta4; j += 384) dst[j] = __ldg(src + j);
  }
  for (int i = tid; i < 768; i += 384) s_lut[i >> 8][i & 255] = __bfloat16_as_ushort(__float2bfloat16_rn(affine_norm(i >> 8, i & 255)));
  const bool mirror = crop >= q.n;
  const int box = mirror ? crop - q.n : crop;
  const Entry& fr = affine_frame(q, box);
  if (tid < PP_W + 16) {
    const AffineInv a = affine_invert(q.mats + 6 * box);
    if (tid < PP_W) s_col[tid] = affine_col(a, tid);
    else {
      const int dy = 16 * py - 2 + (tid - PP_W);
      if (dy >= 0) s_row[tid - PP_W] = affine_row(a, dy);
    }
  }
  if (tid == 0 && py == 0 && !mirror) affine_check(q, box);
  for (int i = tid; i < 3 * 16 * 8; i += 384) {              // zero the padding columns once
    const int row = i >> 3, e = i & 7;
    s_tile[row * FP_PITCH + (e < 2 ? e : 192 + e)] = 0;
  }
  __syncthreads();
  for (int i = tid; i < 16 * PP_W; i += 384) {
    const int ky = i / PP_W, dx = i % PP_W;
    const int dy = 16 * py - 2 + ky;
    uint16_t v3[3] = {0, 0, 0};
    if (dy >= 0) {
      int v[3];
      const int2 r = s_row[ky], c = s_col[dx];
      if constexpr (Entry::kYuv) affine_pixel_yuv(fr, yuv_coef(fr.conv), (r.x + c.x) >> 5, (r.y + c.y) >> 5, v);
      else affine_pixel(fr, (r.x + c.x) >> 5, (r.y + c.y) >> 5, v);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) v3[ch] = s_lut[ch][v[ch]];
    }
    const int tx = 2 + (mirror ? PP_W - 1 - dx : dx);
#pragma unroll
    for (int c = 0; c < 3; ++c) s_tile[(c * 16 + ky) * FP_PITCH + tx] = v3[c];
  }
  __syncthreads();
  for (int i = tid; i < 12 * 3 * 16 * 2; i += 384) {
    const int hf = i & 1, ky = (i >> 1) & 15, c = (i >> 5) % 3, px = i / 96;
    const uint4 v = *reinterpret_cast<const uint4*>(&s_tile[(c * 16 + ky) * FP_PITCH + 16 * px + 8 * hf]);
    *reinterpret_cast<uint4*>(q.rows + ((static_cast<size_t>(crop) * 16 + py) * 12 + px) * 768 + c * 256 + ky * 16 + 8 * hf) = v;
  }
}

}  // namespace vpb
