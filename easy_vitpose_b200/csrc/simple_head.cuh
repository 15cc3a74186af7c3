// The ViTPose simple decoder on sm_90a: relu -> 4x bilinear upsample (align_corners=False) -> 3x3 conv (padding 1), one kernel.
//
// Conv and upsample are both linear, so the conv's nine taps can be applied at the backbone's 16 x 12 token resolution:
//     out[k, y, x] = bias[k] + sum_{t = (dy, dx)} sum_{(i, j)} Ry[y + dy, i] Rx[x + dx, j] Y_t[(i, j), k],   Y_t = relu(xn) W_t^T
// with W_t[k, c] = weight[k, c, dy + 1, dx + 1] and Ry / Rx the bilinear row / column weights (zero outside the 64 x 48 map: the
// conv pads the UPSAMPLED map).  One CTA = one (crop, group of up to 16 keypoints):
//   warpgroups 0-2   rows 0-63 / 64-127 / 128-191 of the crop's 192 tokens: relu on their rows of each smem stage, then wgmma
//                    m64nNTk16 against the group's packed taps (N = 9 * keypoints of the group, rounded up to a wgmma width)
//   warp 12          TMA producer: xn k-blocks (192 x 64, 128B-swizzled) and W k-blocks (NT x 64) into a ring
// After the K loop the group's Y tile [192, NT] goes to shared memory (over the drained ring) and the same 384 threads apply the
// separable stencil: thread (keypoint, column x) sums the three column taps into H[dy][i] for all 16 token rows (48 registers), then
// walks the 64 output rows with the three row taps from registers, writing straight to the NCHW heatmap rows.
// Packed weights: rows n = g * 144 + t * Kg + k (Kg = keypoints of group g: 16, or K % 16 for the last group), bf16 [*, D].
#pragma once
#include <cuda.h>

#include "ptx.cuh"
#include "wgmma.cuh"

namespace vpb {

constexpr int SH_GROUP = 16;                 // keypoints per group: 9 taps x 16 = 144 = one wgmma N
constexpr int SH_NFULL = 9 * SH_GROUP;
constexpr int SH_BK = 64;
constexpr int SH_STAGES = 4;
constexpr int SH_THREADS = 3 * 128 + 32;
constexpr int SH_A_BYTES = 192 * SH_BK * 2;
constexpr int SH_STAGE_BYTES = SH_A_BYTES + SH_NFULL * SH_BK * 2;
constexpr int SH_PITCH = SH_NFULL + 1;       // odd fp32 pitch of the Y tile: rows read by one warp fall in distinct banks
constexpr int SH_SMEM = SH_STAGES * SH_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(192 * SH_PITCH * 4 <= SH_STAGES * SH_STAGE_BYTES, "the Y tile reuses the ring");

struct SimpleHeadParams {
  const float* bias;   // [K]
  float* out;          // heatmaps: crop b, keypoint k at out + (b * ch_stride + k) * 3072
  int D, K, c0;        // c0 = first crop of the segment in the xn workspace
  int ch_stride;
};

// The smallest wgmma width this kernel is built for that holds `rows` tap rows
__host__ __device__ constexpr int sh_width(int rows) { return rows <= 32 ? 32 : rows <= 64 ? 64 : rows <= 96 ? 96 : rows <= 128 ? 128 : 144; }

// Bilinear source rows of output row (or column) Y of a 4x upsample, align_corners=False: weights (3/8, 5/8), (1/8, 7/8),
// (7/8, 1/8), (5/8, 3/8) for Y % 4 = 0..3, source indices clamped to [0, n - 1].
__host__ __device__ __forceinline__ void sh_taps(int Y, int n, int& i0, int& i1, float& w0, float& w1) {
  const int q = Y >> 2, s = Y & 3;
  i0 = s < 2 ? (q > 0 ? q - 1 : 0) : q;
  i1 = s < 2 ? q : (q + 1 < n ? q + 1 : n - 1);
  w0 = s == 0 ? 0.375f : s == 1 ? 0.125f : s == 2 ? 0.875f : 0.625f;
  w1 = 1.0f - w0;
}

template <int NT>
__device__ __forceinline__ void simple_head_group(const CUtensorMap* ta, const CUtensorMap* tw, const SimpleHeadParams& p, int b, int g,
                                                  int kg, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = p.D / SH_BK;
  if (warp == 12) {                                               // producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* s = ring + stage * SH_STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], SH_A_BYTES + NT * SH_BK * 2);
        tma_load_2d(s, ta, &full_bar[stage], kb * SH_BK, (p.c0 + b) * 192);
        tma_load_2d(s + SH_A_BYTES, tw, &full_bar[stage], kb * SH_BK, g * SH_NFULL);
        if (++stage == SH_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  float acc[NT / 2];
  {
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      uint8_t* sa = ring + stage * SH_STAGE_BYTES + wg * 64 * 128;
      // relu on this warpgroup's 64 rows of the stage (8 KB); xn itself stays as the backbone left it.  NaN stays NaN.
      uint4* v = reinterpret_cast<uint4*>(sa);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint4 w = v[tid + 128 * i];
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&w);
        const __nv_bfloat162 z = __float2bfloat162_rn(0.f);
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __hmax2_nan(h[e], z);
        v[tid + 128 * i] = w;
      }
      fence_proxy_async_smem();                                   // generic writes -> the async proxy wgmma reads through
      named_bar_sync(1 + wg, 128);
      const uint64_t ad = wgmma_desc<128>(smem_u32(sa));
      const uint64_t bd = wgmma_desc<128>(smem_u32(ring + stage * SH_STAGE_BYTES + SH_A_BYTES));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < SH_BK / 16; ++k) wgmma_ss<NT>(acc, ad + 2 * k, bd + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == SH_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }
  named_bar_sync(4, 384);                                         // every warpgroup's MMAs have read the ring
  float* ys = reinterpret_cast<float*>(ring);
  {  // thread (warp w of the warpgroup, lane l): rows 16 w + l / 4 (+ 8), columns 8 j + 2 (l % 4) + {0, 1}
    const int r = 64 * wg + 16 * (tid >> 5) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      ys[r * SH_PITCH + 8 * j + cq] = acc[4 * j];
      ys[r * SH_PITCH + 8 * j + cq + 1] = acc[4 * j + 1];
      ys[(r + 8) * SH_PITCH + 8 * j + cq] = acc[4 * j + 2];
      ys[(r + 8) * SH_PITCH + 8 * j + cq + 1] = acc[4 * j + 3];
    }
  }
  named_bar_sync(4, 384);
  for (int item = threadIdx.x; item < kg * 48; item += 384) {
    const int k = item / 48, x = item - 48 * k;
    // column taps of output column x: source columns and weights for dx = -1, 0, 1 (none outside the 48 columns: conv padding)
    int j0[3], j1[3];
    float u0[3], u1[3];
    bool ok[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int X = x + d - 1;
      ok[d] = X >= 0 && X < 48;
      sh_taps(ok[d] ? X : 0, 12, j0[d], j1[d], u0[d], u1[d]);
    }
    float H[3][16];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float h = 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d)
          if (ok[d]) {
            const int col = (3 * dy + d) * kg + k;
            h += u0[d] * ys[(12 * i + j0[d]) * SH_PITCH + col];
            h += u1[d] * ys[(12 * i + j1[d]) * SH_PITCH + col];
          }
        H[dy][i] = h;
      }
    const int kk = g * SH_GROUP + k;
    const float bk = __ldg(p.bias + kk);
    float* o = p.out + (static_cast<size_t>(b) * p.ch_stride + kk) * 3072 + x;
#pragma unroll
    for (int y = 0; y < 64; ++y) {
      float v = bk;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const int Y = y + dy - 1;
        if (Y < 0 || Y >= 64) continue;
        int i0, i1;
        float w0, w1;
        sh_taps(Y, 16, i0, i1, w0, w1);
        v += w0 * H[dy][i0];
        v += w1 * H[dy][i1];
      }
      o[48 * y] = v;
    }
  }
}

// grid (crops, groups); the last group runs at width NT_REM when K % 16 != 0
template <int NT_REM>
__global__ void __launch_bounds__(SH_THREADS, 1)
    simple_head_kernel(const __grid_constant__ CUtensorMap ta, const __grid_constant__ CUtensorMap tw_full,
                       const __grid_constant__ CUtensorMap tw_rem, const SimpleHeadParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + SH_STAGES * SH_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + SH_STAGES;
  const int b = blockIdx.x, g = blockIdx.y;
  const int kg = min(SH_GROUP, p.K - g * SH_GROUP);
  if (threadIdx.x == 0) {
    for (int s = 0; s < SH_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 12); }
    fence_mbar_init();
    tma_prefetch_desc(&ta);
    tma_prefetch_desc(kg == SH_GROUP ? &tw_full : &tw_rem);
  }
  __syncthreads();
  pdl_wait();
  if (kg == SH_GROUP) simple_head_group<SH_NFULL>(&ta, &tw_full, p, b, g, kg, ring, full_bar, empty_bar);
  else simple_head_group<NT_REM>(&ta, &tw_rem, p, b, g, kg, ring, full_bar, empty_bar);
  pdl_launch_dependents();
}

// fp32 final_layer.weight [K, D, 3, 3] -> bf16 tap rows [ceil(K / 16) * 144, D] (layout above; rows past a group's 9 * Kg are zero)
__global__ void pack_simple_head(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int K, int D) {
  const long long tot = static_cast<long long>((K + SH_GROUP - 1) / SH_GROUP) * SH_NFULL * D;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < tot; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(i / D), c = static_cast<int>(i - static_cast<long long>(n) * D);
    const int g = n / SH_NFULL, r = n - g * SH_NFULL;
    const int kg = min(SH_GROUP, K - g * SH_GROUP);
    float v = 0.f;
    if (r < 9 * kg) {
      const int t = r / kg, k = g * SH_GROUP + r - t * kg;
      v = w[(static_cast<long long>(k) * D + c) * 9 + t];
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace vpb
