// Grouped expert GEMM for sm_90a: the dataset-expert columns of ViTPose+'s fc2 for a batch whose crops use different experts.
//
// ViTPose+ splits each block's fc2 output [D] into shared columns [0, D-P) and expert columns [D-P, D); crop c's expert columns
// come from expert e(c).  A call's crops form segments, runs of consecutive crops with one expert (rows row_begin .. row_end-1
// of the token matrix).  This kernel computes, for every segment s at once,
//     x[r, D-P + n] += A[r, :] * W[w_row0 + e_s * P + n, :]^T + bias[w_row0 + e_s * P + n]      r in segment s, n < P
// with W the stacked [shared; expert 0; expert 1; ...] fc2 weight.  Structure and ring as gemm_bf16_wgmma (gemm.cuh): warp 8
// loads A and W tiles by TMA, two consumer warpgroups run wgmma into fp32 registers.  The segment table travels in the
// __grid_constant__ parameter block (the frame-table pattern of preprocess.cuh); a CTA finds its tile's segment by a binary
// search on first_tile.  Segments start at row 192 c, not 128-aligned, so a tile may read rows of the next segment or past M
// (TMA zero-fills those) and columns of the next expert: the epilogue stores only its own segment's rows and columns n < P, as
// a direct load + add + store (a TMA store cannot mask rows).  Each element still receives one fp32 add of (acc + bias), acc
// accumulated in k order: the same two roundings as the single-expert fc2 launch, so the results are bit-identical to it.
#pragma once
#include "gemm.cuh"

namespace vpb {

// 128: a flip-test call of VPB_MAX_SEGMENTS segments runs its crops, then their mirror images, as twice that many (2 KB of the
// 4 KB parameter block)
constexpr int EXPERT_MAX_SEGMENTS = 128;

struct ExpertSegment {
  int row_begin, row_end;   // token rows of the segment (192 per crop)
  int expert;               // 0 .. H-1
  int first_tile;           // first tile index of the segment (prefix sum of the segments' tile counts)
};

struct ExpertParams {
  int K;                    // reduction (4D); K % 64 == 0
  int P;                    // expert width = output columns per segment; P % 32 == 0
  int col0;                 // first output column of the experts in x (D - P)
  int ldx;                  // row pitch of x (D)
  int w_row0;               // first expert row of the stacked W / bias (D - P)
  int n_tiles;              // column tiles per 128-row block: ceil(P / BN)
  int num_tiles;            // tiles of all segments
  int num_segs;             // 1 .. EXPERT_MAX_SEGMENTS
  int stages;               // debug: use at most this many ring stages (0 = all), as GemmParams::stages_limit
  const float* bias;        // stacked fc2 bias [D - P + H * P]
  float* x;                 // fp32 residual stream [M, ldx]
  ExpertSegment seg[EXPERT_MAX_SEGMENTS];
};

// the segment that owns `tile`: the last one whose first_tile <= tile
__device__ __forceinline__ const ExpertSegment& expert_segment(const ExpertParams& p, int tile) {
  int lo = 0, hi = p.num_segs;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (p.seg[mid].first_tile <= tile) lo = mid; else hi = mid;
  }
  return p.seg[lo];
}

// x[r, col0 + n] += acc + bias[n] for rows r_begin <= r < r_end and columns n < P; accumulator layout as epilogue_f32_rmw
template <int BN>
__device__ __forceinline__ void epilogue_expert(const float (&acc)[BN / 2], int n0, int row0, int r_begin, int r_end, const ExpertParams& p,
                                                const float* __restrict__ bias, int tid) {
  const int lane = tid & 31, wq = tid >> 5;
  const int r_lo = row0 + 16 * wq + (lane >> 2);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + cq;                  // even; P % 32 == 0, so n < P implies n + 1 < P
    if (n >= p.P) continue;
    const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_lo + 8 * h;
      if (r >= r_begin && r < r_end) {
        float2* px = reinterpret_cast<float2*>(p.x + static_cast<size_t>(r) * p.ldx + p.col0 + n);
        const float2 xv = __ldcg(px);
        __stcg(px, make_float2(xv.x + (acc[4 * j + 2 * h] + b2.x), xv.y + (acc[4 * j + 2 * h + 1] + b2.y)));
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_expert_segments(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ ExpertParams p) {
  using Cfg = TileCfg<BN, false>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int num_kb = p.K / GEMM_BK;
  const int num_stages = (p.stages > 0 && p.stages < Cfg::STAGES) ? p.stages : Cfg::STAGES;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                                       // the previous kernel's outputs (A = the fc1 activations, x) are complete

  if (warp >= GEMM_CONSUMER_WARPS) {
    setmaxnreg_dec<40>();
    if (warp != GEMM_CONSUMER_WARPS) return;
    RingPos rp;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const ExpertSegment& sg = expert_segment(p, tile);
      const int t = tile - sg.first_tile;
      const int m0 = sg.row_begin + (t / p.n_tiles) * GEMM_BM;         // rows past M are zero-filled by TMA
      const int wrow = p.w_row0 + sg.expert * p.P + (t % p.n_tiles) * BN;
      for (int kb = 0; kb < num_kb; ++kb) {
        ring_wait_slot(empty_bar, rp);
        uint8_t* sa = ring + rp.stage * Cfg::STAGE_BYTES;
        if (elect_one()) {
          mbar_expect_tx(&full_bar[rp.stage], Cfg::STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, &full_bar[rp.stage], kb * GEMM_BK, m0);
          tma_load_2d(sa + Cfg::A_BYTES, &tmap_w, &full_bar[rp.stage], kb * GEMM_BK, wrow);
        }
        __syncwarp();
        rp.next(num_stages);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int tid = threadIdx.x & 127;
    RingPos rp;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const ExpertSegment& sg = expert_segment(p, tile);
      const int t = tile - sg.first_tile;
      const int m0 = sg.row_begin + (t / p.n_tiles) * GEMM_BM;
      const int n0 = (t % p.n_tiles) * BN;
      tile_mainloop<BN>(acc, ring, Cfg::STAGE_BYTES, full_bar, empty_bar, num_kb, num_stages, rp, wg, lane, nullptr);
      epilogue_expert<BN>(acc, n0, m0 + 64 * wg, sg.row_begin, sg.row_end, p, p.bias + p.w_row0 + sg.expert * p.P, tid);
    }
  }
}

}  // namespace vpb
