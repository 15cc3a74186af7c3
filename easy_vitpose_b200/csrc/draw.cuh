// Pose overlay (vpb_draw_poses): the pose layer of VitInference.draw() (easy_ViTPose/inference.py:283-312,
// vit_utils/visualization.py:360-481) for the people of many frames in two launches, bit-exact with cv2 4.13.
//
// Per person, in the reference's painter's order: every limb (a, b) of the skeleton whose two scores are > threshold as
// cv2.line(img, (int(x_a), int(y_a)), (int(x_b), int(y_b)), limb_colour[idx % L], 2), then every keypoint i with score >
// threshold as cv2.circle(img, (int(x), int(y)), radius, point_colour[i % P], -1).  oracle/draw_oracle.py restates both
// primitives as pixel coverage and is pinned against live cv2; the arithmetic here is that restatement:
//   circle   Circle(fill=1): the midpoint loop's spans, tabulated per radius (draw_half_widths);
//   line     clipLine of the integer end points against Rect(-2, -2, w + 4, h + 4) (nothing when it misses), then
//            ThickLine in 16.16 fixed point: dp = cvRound((dy, dx) * 65536 / |p1 - p0|) in double without contraction, the
//            quad p0 +- dp, p1 -+ dp through FillConvexPoly(shift 16) -- four Line2 edges (clipLine on the image scaled by
//            2^16, a fixed-point DDA and its end pixel) and scanlines stepped by each edge's int64 dx -- and a radius-1
//            filled circle at both ends.
//
// draw_setup: one thread per candidate primitive (person p, slot s < E: limb s, s >= E: keypoint s - E) writes a DrawRec
// (everything the coverage test needs, in closed form) and an inclusive pixel box, empty for a primitive that is not drawn.
// draw_raster: one 32 x 8 pixel tile per block over every frame of the call.  The block gathers the records of its frame
// whose boxes overlap the tile, newest first, and each pixel takes the colour of the LAST primitive covering it in
// painter's order -- which is what painting in order leaves there, as nothing blends.  Every covered pixel is written once
// and by one thread, uncovered pixels are not touched, and there are no atomics: the result does not depend on scheduling.
#pragma once
#include <cstdint>

constexpr int DRAW_MAX_LIMBS = 128;
constexpr int DRAW_MAX_COLORS = 64;
constexpr int DRAW_MAX_FRAMES = 64;
constexpr int DRAW_MAX_RADIUS = 1023;
constexpr int DRAW_TILE_W = 32, DRAW_TILE_H = 8;             // 256 threads, one pixel each
constexpr int DRAW_SETUP_THREADS = 128;

struct DrawFrame {
  uint8_t* data;                // [h, w, 3], row pitch `pitch` bytes
  long long pitch;
  int h, w;
  int first_person, num_people; // rows of kpts
  int radius;                   // keypoint circle radius of this frame
  int first_tile;               // tiles of the frames before this one
};
static_assert(sizeof(DrawFrame) == 40, "draw frame table entry layout");

struct DrawParams {
  DrawFrame frames[DRAW_MAX_FRAMES];
  uint16_t limbs[DRAW_MAX_LIMBS][2];
  uint8_t point_rgb[DRAW_MAX_COLORS][3];                      // already in the frames' channel order
  uint8_t limb_rgb[DRAW_MAX_COLORS][3];
  const float* kpts;            // [n, k, 3] (y, x, score)
  const int32_t* person_index;  // [n] or nullptr (position within the frame)
  struct DrawRec* recs;         // [n * (E + k)]
  int4* boxes;                  // [n * (E + k)] inclusive (x0, y0, x1, y1); x0 > x1 = not drawn
  int n, k, num_limbs, num_point_colors, num_limb_colors, num_frames, total_tiles;
  float threshold;
};
static_assert(sizeof(DrawParams) <= 4096, "the draw tables travel in the 4 KB parameter block");

struct DrawSeg {                // rows y0 <= y < y1 of one side of the quad: edge at x + (y - y0) * dx (16.16)
  long long x, dx;
  int y0, y1, side, pad;
};
struct DrawEdge {               // Line2 after clipping: pixel t in [0, count] is (a0 + t, (b0 + t * step) >> 16) for an x-major
  long long b0, step;           // edge, ((b0 + t * step) >> 16, a0 + t) otherwise, plus the end pixel; count < 0: nothing
  int a0, count, end_x, end_y, x_major, pad;
};
struct DrawRec {
  uint8_t rgb[4];               // colour in the frame's channel order
  int kind;                     // 1 limb, 2 keypoint
  int cx0, cy0, cx1, cy1;       // limb: centres of the end circles (radius 1); keypoint: centre (cx0, cy0), radius cx1
  int nseg;
  DrawSeg seg[4];
  DrawEdge edge[4];
};

__device__ __forceinline__ int draw_frame_of(const DrawParams& q, int person) {
  int lo = 0, hi = q.num_frames - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (q.frames[mid].first_person <= person) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// int(v) of the reference (truncation toward zero); false for a coordinate cv2 cannot take (non-finite, outside int32)
__device__ __forceinline__ bool draw_coord(float v, int* out) {
  if (!(v >= -2147483648.0f && v < 2147483648.0f)) return false;
  *out = __float2int_rz(v);
  return true;
}

// drawing.cpp clipLine on a w x h image (int64 end points, double intercepts truncated as (int64) casts)
__device__ bool draw_clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
  if (w <= 0 || h <= 0) return false;
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(a - y1), __ll2double_rn(x2 - x1)), __ll2double_rn(y2 - y1)));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(a - y2), __ll2double_rn(x2 - x1)), __ll2double_rn(y2 - y1)));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(a - x1), __ll2double_rn(y2 - y1)), __ll2double_rn(x2 - x1)));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += __double2ll_rz(__ddiv_rn(__dmul_rn(__ll2double_rn(a - x2), __ll2double_rn(y2 - y1)), __ll2double_rn(x2 - x1)));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// Union of pixel rectangles, kept in int (clamped to [-1, 2^31 - 2]; the frame clip follows)
struct DrawBox {
  int x0 = 0x7fffffff, y0 = 0x7fffffff, x1 = -0x7fffffff, y1 = -0x7fffffff;
  static __device__ __forceinline__ int clamp(long long v) { return (int)max(-1LL, min(v, 0x7ffffffeLL)); }
  __device__ void add(long long xa, long long ya, long long xb, long long yb) {
    x0 = min(x0, clamp(min(xa, xb))); y0 = min(y0, clamp(min(ya, yb)));
    x1 = max(x1, clamp(max(xa, xb))); y1 = max(y1, clamp(max(ya, yb)));
  }
};

// Line2's DDA of the 16.16 segment p1 -> p2 on an h x w image
__device__ void draw_line2(int h, int w, long long x1, long long y1, long long x2, long long y2, DrawEdge& e, DrawBox& box) {
  e.count = -1;
  if (!draw_clip_line((long long)w << 16, (long long)h << 16, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long step;
  e.x_major = ax > ay;
  if (e.x_major) {
    if (dx < 0) { dy = -dy; long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    step = (dy * 65536) / (ax | 1);
    e.count = (int)((x2 - x1) >> 16);
  } else {
    if (dy < 0) { dx = -dx; long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    step = (dx * 65536) / (ay | 1);
    e.count = (int)((y2 - y1) >> 16);
  }
  e.end_x = (int)((x2 + 32768) >> 16);
  e.end_y = (int)((y2 + 32768) >> 16);
  x1 += 32768;
  y1 += 32768;
  e.step = step;
  e.a0 = (int)((e.x_major ? x1 : y1) >> 16);
  e.b0 = e.x_major ? y1 : x1;
  const long long m0 = e.b0 >> 16, m1 = (e.b0 + e.count * step) >> 16;
  if (e.x_major) box.add(e.a0, m0, e.a0 + e.count, m1); else box.add(m0, e.a0, m1, e.a0 + e.count);
  box.add(e.end_x, e.end_y, e.end_x, e.end_y);
}

// FillConvexPoly(shift 16, LINE_8)'s scanline walk over the quad v, as at most 4 edge segments
__device__ void draw_fill(int h, int w, const long long (&v)[4][2], DrawRec& r, DrawBox& box) {
  constexpr long long delta = 32768;
  r.nseg = 0;
  int imin = 0;
  long long xmn = v[0][0], xmx = v[0][0], ymx = v[0][1];
  for (int i = 1; i < 4; ++i) {
    if (v[i][1] < v[imin][1]) imin = i;
    xmn = min(xmn, v[i][0]); xmx = max(xmx, v[i][0]); ymx = max(ymx, v[i][1]);
  }
  xmn = (xmn + delta) >> 16; xmx = (xmx + delta) >> 16; ymx = (ymx + delta) >> 16;
  const long long ymn = (v[imin][1] + delta) >> 16;
  if (xmx < 0 || ymx < 0 || xmn >= w || ymn >= h) return;
  ymx = min(ymx, (long long)h - 1);
  int edges = 4;
  int idx[2] = {imin, imin}, open[2] = {-1, -1};
  const int di[2] = {1, 3};
  long long ye[2] = {ymn, ymn};
  long long y = ymn;
  for (;;) {
    for (int i = 0; i < 2; ++i) {
      if (y < ye[i]) continue;
      int idx0 = idx[i], id = (idx0 + di[i]) & 3;
      while (edges-- > 0) {
        const long long ty = (v[id][1] + delta) >> 16;
        if (ty > y) {
          if (open[i] >= 0) r.seg[open[i]].y1 = (int)y;
          DrawSeg& s = r.seg[r.nseg];
          s.side = i;
          s.y0 = (int)y;
          s.x = v[idx0][0];
          s.dx = ((v[id][0] - v[idx0][0]) * 2 + (ty - y)) / (2 * (ty - y));
          open[i] = r.nseg++;
          ye[i] = ty;
          idx[i] = id;
          break;
        }
        idx0 = id;
        id = (id + di[i]) & 3;
      }
    }
    if (edges < 0) break;
    y = min(min(ye[0], ye[1]), ymx + 1);
    if (y > ymx) break;
  }
  for (int i = 0; i < 2; ++i)
    if (open[i] >= 0) r.seg[open[i]].y1 = (int)y;
  for (int s = 0; s < r.nseg; ++s) {        // the spans lie between the edges' extremes over the rows inside the frame
    const DrawSeg& g = r.seg[s];
    const long long ra = max((long long)g.y0, 0LL), rb = min((long long)g.y1, (long long)h) - 1;
    if (ra > rb) continue;
    const long long xa = (g.x + (ra - g.y0) * g.dx + delta) >> 16, xb = (g.x + (rb - g.y0) * g.dx + delta) >> 16;
    box.add(xa, ra, xb, rb);
  }
}

__global__ void __launch_bounds__(DRAW_SETUP_THREADS) draw_setup(const __grid_constant__ DrawParams q) {
  const int per = q.num_limbs + q.k;
  const long long g = (long long)blockIdx.x * DRAW_SETUP_THREADS + threadIdx.x;
  if (g >= (long long)q.n * per) return;
  const int p = (int)(g / per), s = (int)(g % per);
  const DrawFrame& F = q.frames[draw_frame_of(q, p)];
  const int idx = q.person_index ? q.person_index[p] : p - F.first_person;
  const float* kp = q.kpts + (long long)p * q.k * 3;
  DrawRec& r = q.recs[g];
  int4 out = make_int4(0, 0, -1, -1);
  DrawBox box;
  if (s < q.num_limbs) {
    const int a = q.limbs[s][0], b = q.limbs[s][1];
    int xa, ya, xb, yb;
    if (kp[a * 3 + 2] > q.threshold && kp[b * 3 + 2] > q.threshold && draw_coord(kp[a * 3 + 1], &xa) && draw_coord(kp[a * 3], &ya) &&
        draw_coord(kp[b * 3 + 1], &xb) && draw_coord(kp[b * 3], &yb)) {
      long long x0 = (long long)xa + 2, y0 = (long long)ya + 2, x1 = (long long)xb + 2, y1 = (long long)yb + 2;
      if (draw_clip_line((long long)F.w + 4, (long long)F.h + 4, x0, y0, x1, y1)) {   // cv2.line's clip to the grown image
        x0 -= 2; y0 -= 2; x1 -= 2; y1 -= 2;
        const int c = ((idx % q.num_limb_colors) + q.num_limb_colors) % q.num_limb_colors;
        r.rgb[0] = q.limb_rgb[c][0]; r.rgb[1] = q.limb_rgb[c][1]; r.rgb[2] = q.limb_rgb[c][2]; r.rgb[3] = 0;
        r.kind = 1;
        r.cx0 = (int)x0; r.cy0 = (int)y0; r.cx1 = (int)x1; r.cy1 = (int)y1;
        box.add(x0 - 1, y0 - 1, x0 + 1, y0 + 1);
        box.add(x1 - 1, y1 - 1, x1 + 1, y1 + 1);
        r.nseg = 0;
        for (int e = 0; e < 4; ++e) r.edge[e].count = -1;
        const long long P0x = x0 << 16, P0y = y0 << 16, P1x = x1 << 16, P1y = y1 << 16;
        const double dx = __dmul_rn(__ll2double_rn(P0x - P1x), 1.0 / 65536), dy = __dmul_rn(__ll2double_rn(P1y - P0y), 1.0 / 65536);
        double rr = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        if (fabs(rr) > 2.220446049250313e-16) {
          rr = __ddiv_rn(65536.0, __dsqrt_rn(rr));
          const long long dpx = __double2int_rn(__dmul_rn(dy, rr)), dpy = __double2int_rn(__dmul_rn(dx, rr));
          const long long v[4][2] = {{P0x + dpx, P0y + dpy}, {P0x - dpx, P0y - dpy}, {P1x - dpx, P1y - dpy}, {P1x + dpx, P1y + dpy}};
          for (int e = 0; e < 4; ++e) {
            const int pe = (e + 3) & 3;
            draw_line2(F.h, F.w, v[pe][0], v[pe][1], v[e][0], v[e][1], r.edge[e], box);
          }
          draw_fill(F.h, F.w, v, r, box);
        }
      }
    }
  } else {
    const int i = s - q.num_limbs;
    int x, y;
    if (kp[i * 3 + 2] > q.threshold && draw_coord(kp[i * 3 + 1], &x) && draw_coord(kp[i * 3], &y)) {
      const int c = i % q.num_point_colors;
      r.rgb[0] = q.point_rgb[c][0]; r.rgb[1] = q.point_rgb[c][1]; r.rgb[2] = q.point_rgb[c][2]; r.rgb[3] = 0;
      r.kind = 2;
      r.cx0 = x; r.cy0 = y; r.cx1 = F.radius;
      box.add((long long)x - F.radius, (long long)y - F.radius, (long long)x + F.radius, (long long)y + F.radius);
    }
  }
  if (box.x0 <= box.x1) {
    out.x = max(box.x0, 0); out.y = max(box.y0, 0);
    out.z = min(box.x1, F.w - 1); out.w = min(box.y1, F.h - 1);
    if (out.x > out.z || out.y > out.w) out = make_int4(0, 0, -1, -1);
  }
  q.boxes[g] = out;
}

// hw[o] = half width of a filled circle's span on rows centre +- o (Circle()'s midpoint loop)
__device__ void draw_half_widths(int radius, int* hw) {
  for (int o = 0; o <= radius; ++o) hw[o] = -1;
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  while (dx >= dy) {
    hw[dy] = max(hw[dy], dx);
    hw[dx] = max(hw[dx], dy);
    dy++;
    err += plus;
    plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask;
    dx += mask;
    minus -= mask & 2;
  }
}

__device__ __forceinline__ bool draw_covers(const DrawRec& r, int x, int y, const int* hw) {
  if (r.kind == 2) {
    const int o = abs(y - r.cy0);
    return o <= r.cx1 && abs(x - r.cx0) <= hw[o];
  }
  if (abs(x - r.cx0) + abs(y - r.cy0) <= 1 || abs(x - r.cx1) + abs(y - r.cy1) <= 1) return true;
  long long xa = 0, xb = 0;
  int found = 0;
  for (int s = 0; s < r.nseg; ++s) {
    const DrawSeg& g = r.seg[s];
    if (y >= g.y0 && y < g.y1) {
      const long long xr = g.x + (long long)(y - g.y0) * g.dx;
      if (g.side) xb = xr; else xa = xr;
      found |= 1 << g.side;
    }
  }
  if (found == 3) {
    const long long lo = min(xa, xb), hi = max(xa, xb);
    if (x >= ((lo + 32768) >> 16) && x <= ((hi + 32768) >> 16)) return true;
  }
  for (int e = 0; e < 4; ++e) {
    const DrawEdge& d = r.edge[e];
    if (d.count < 0) continue;
    if (x == d.end_x && y == d.end_y) return true;
    const long long t = (long long)(d.x_major ? x : y) - d.a0;
    if (t >= 0 && t <= d.count && ((d.b0 + t * d.step) >> 16) == (d.x_major ? y : x)) return true;
  }
  return false;
}

__global__ void __launch_bounds__(DRAW_TILE_W * DRAW_TILE_H) draw_raster(const __grid_constant__ DrawParams q) {
  __shared__ int s_hw[DRAW_MAX_RADIUS + 1];
  __shared__ int s_list[DRAW_TILE_W * DRAW_TILE_H];
  __shared__ int s_warp[DRAW_TILE_W * DRAW_TILE_H / 32];
  int f = 0;
  {
    int lo = 0, hi = q.num_frames - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (q.frames[mid].first_tile <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    f = lo;
  }
  const DrawFrame& F = q.frames[f];
  const int tiles_x = (F.w + DRAW_TILE_W - 1) / DRAW_TILE_W;
  const int tile = (int)blockIdx.x - F.first_tile;
  const int tx0 = (tile % tiles_x) * DRAW_TILE_W, ty0 = (tile / tiles_x) * DRAW_TILE_H;
  const int tx1 = min(tx0 + DRAW_TILE_W, F.w) - 1, ty1 = min(ty0 + DRAW_TILE_H, F.h) - 1;
  const int x = tx0 + (threadIdx.x % DRAW_TILE_W), y = ty0 + (threadIdx.x / DRAW_TILE_W);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) draw_half_widths(F.radius, s_hw);
  bool done = x > tx1 || y > ty1;
  const int per = q.num_limbs + q.k;
  const int lo = F.first_person * per, hi = (F.first_person + F.num_people) * per;
  for (int end = hi; end > lo; end -= DRAW_TILE_W * DRAW_TILE_H) {
    if (!__syncthreads_or(!done)) break;                     // also orders the reuse of s_list / s_warp (and s_hw's fill)
    const int ri = end - 1 - (int)threadIdx.x;
    bool hit = false;
    if (ri >= lo) {
      const int4 b = q.boxes[ri];
      hit = b.x <= tx1 && b.z >= tx0 && b.y <= ty1 && b.w >= ty0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int off = 0, total = 0;
#pragma unroll
    for (int w = 0; w < DRAW_TILE_W * DRAW_TILE_H / 32; ++w) {
      off += w < warp ? s_warp[w] : 0;
      total += s_warp[w];
    }
    if (hit) s_list[off + __popc(m & ((1u << lane) - 1))] = ri;   // newest record first
    __syncthreads();
    if (done) continue;
    for (int i = 0; i < total; ++i) {
      const DrawRec& r = q.recs[s_list[i]];
      if (draw_covers(r, x, y, s_hw)) {
        uint8_t* px = F.data + (long long)y * F.pitch + 3LL * x;
        px[0] = r.rgb[0]; px[1] = r.rgb[1]; px[2] = r.rgb[2];
        done = true;
        break;
      }
    }
  }
}
