// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = A[M,K] * W[N,K]^T  (+ fused epilogue)
//
//   warpgroups 0, 1    consumers: rows 0..63 / 64..127 of the 128 x BN tile, wgmma m64nBNk16 with fp32 accumulators in
//                      registers, then the epilogue straight from those registers: bias / GELU / ReLU -> swizzled smem
//                      staging -> TMA store (bf16) or TMA reduce-add (fp32 residual, the add happens in L2)
//   warp 8             TMA producer: A / W tiles -> 128B-swizzled smem ring, mbarrier full / empty
//
// Both operands are K-major (nn.Linear keeps W as [N,K]), so no transposes anywhere.  Tiles are handed out statically
// (tile = blockIdx.x + i * gridDim.x, n fastest: the CTAs running together cover a few A row-blocks x all W column-blocks,
// which keeps the big streaming operand A hot in L2).  The producer runs ahead of the consumers by the ring depth, across
// tile boundaries, so the next tile's operands arrive while the consumers run the epilogue of the current one.
// The accumulation order of an output element is the k order, whatever the tile width: every BN gives the same bits.
#pragma once
#include <cuda.h>

#include "ptx.cuh"
#include "wgmma.cuh"

namespace vpb {

enum Epilogue : int {
  EPI_BF16 = 0,         // out bf16 [M,ldc]   = acc + bias                              (qkv)            TMA store
  EPI_BF16_GELU = 1,    // out bf16 [M,ldc]   = gelu_erf(acc + bias)                    (fc1)            TMA store
  EPI_BF16_RELU_UP = 2, // implicit-GEMM deconv: A = shifted NHWC boxes (4-D TMA), all 4 sub-pixel phases in one launch,
                        // out bf16 NHWC (b,2y+py,2x+px) = relu(acc + bias)                                direct
  EPI_F32_NCHW = 4,     // out f32 [b,n,pix]  = acc + bias for n < n_valid              (1x1 conv)       direct
  EPI_F32_ADD = 5,      // out f32 [M,ldc]   += acc + bias                 (patch embed, proj, fc2)      TMA reduce-add
  EPI_BF16_GELU_ERF = 6,// like EPI_BF16_GELU with erf evaluated by Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7) instead of the fitted
                        // tanh form: the A/B switch for the GELU approximation (engine option "gelu_erf")
};

struct GemmParams {
  int M, N, K;            // problem (rows of A, rows of W, reduction); K % 64 == 0
  const float* bias;      // [N] (padded to the N tile) or nullptr
  void* out;              // direct epilogues only
  int ldc;                // row pitch of out in elements (direct row-major epilogues)
  int n_valid;            // EPI_F32_NCHW: number of real output channels
  int pix;                // EPI_F32_NCHW: pixels per image (rows per batch item)
  int ch_stride;          // EPI_F32_NCHW: channels between consecutive images of out (0 = n_valid; a multi-head call: K_max)
  int up_h, up_w;         // EPI_BF16_RELU_UP: input grid (H, W)
  int up_tr, up_tw;       // EPI_BF16_RELU_UP: an M tile is a up_tr x up_tw patch of positions (96 = 8x12 or 128 = 16x8)
  int up_c;               // EPI_BF16_RELU_UP: input channels (K = 4 taps * up_c)
  // Fused LayerNorm tail (EPI_F32_ADD, ln_out != nullptr): the CTA that completes the LAST column tile of a
  // 128-row block of the fp32 stream (atomic counter per block) normalises those rows out of L2 and writes the bf16 rows
  // the next GEMM consumes -- no separate LayerNorm launch, no second trip of x through HBM.
  const float* ln_gamma;  // [N]
  const float* ln_beta;   // [N]
  __nv_bfloat16* ln_out;  // [M, N] or nullptr
  int* ln_counters;       // [ceil(M/128)] zero before the first launch; the last arriver resets its entry
  float ln_eps;
  int rmw;                // EPI_F32_ADD: 1 = load + add + store in the generic proxy (needs out = the fp32 stream), 0 = TMA reduce-add
  int stages_limit;       // debug: use at most this many ring stages (0 = all)
  int dbg_flags;          // debug (results become wrong!): 1 = every CTA loads the SAME A rows, 2 = the same W rows
                          //        (probes whether L2 reads or SM-side delivery bound the loop); 4 = m-fastest tile order
  long long* dbg;         // debug: per-CTA cycle counters [8] (nullptr = off): 0 consumer (thread 0) total, 1 its wait for
                          //        operands, 3 producer total, 4 producer wait for free ring slots, 7 CTA lifetime
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_CONSUMER_WARPS = 8;     // two warpgroups of 64 rows
constexpr int GEMM_STAGE_TILE = 8192;      // one staging buffer: 64 rows x 128 B (two per consumer warpgroup)
constexpr int GEMM_BAR_EPI = 1;            // named barrier of the 256 consumer threads (2, 3: the warpgroups' staging barriers)

__host__ __device__ constexpr bool epi_uses_tma(int epi) { return epi == EPI_BF16 || epi == EPI_BF16_GELU || epi == EPI_F32_ADD || epi == EPI_BF16_GELU_ERF; }

// Ring and staging layout of a 128 x BN tile, shared by the standalone GEMM and the chained launches (chain.cuh).
template <int BN, bool STAGED>
struct TileCfg {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGING = STAGED ? 4 * GEMM_STAGE_TILE : 0;
  static constexpr int STAGES_RAW = (227 * 1024 - 2048 - STAGING) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(B_BYTES % 1024 == 0, "W tiles must keep 1024-byte alignment of the ring");
  static_assert(BN % 16 == 0 && BN >= 16 && BN <= 256, "wgmma N");
  static_assert(!STAGED || BN % 64 == 0, "TMA epilogues stage 64 bf16 / 32 f32 columns at a time");
  static_assert(STAGES >= 3, "ring too shallow");
};
template <int BN, int EPI>
using GemmCfg = TileCfg<BN, epi_uses_tma(EPI)>;

__device__ __forceinline__ float gelu_erf_as(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752440f)); }
#ifdef VPB_GELU_ERF
__device__ __forceinline__ float gelu_fast(float x) { return gelu_erf_as(x); }
#else
__device__ __forceinline__ float gelu_fast(float x) { return gelu_tanh_fit(x); }
#endif

// ---------------------------------------------------------------- ring: producer and consumer sides
// The ring position (stage, phase) runs on across tiles; both sides walk the same sequence of k-blocks.
struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next(int stages) { if (++stage == stages) { stage = 0; phase ^= 1; } }
};

// Producer side: wait until the consumers have released the slot at `rp` (a fresh barrier passes on parity 1).  Whole warp.
__device__ __forceinline__ void ring_wait_slot(uint64_t* empty_bar, const RingPos& rp) { mbar_wait(&empty_bar[rp.stage], rp.phase ^ 1); }

// Consumer warpgroup `wg`: acc = A[64 wg .. 64 wg + 63, :] * W[0 .. BN-1, :]^T over num_kb k-blocks of the ring.  Every
// consumer warp releases a slot once the MMAs that read it have retired (empty barriers count GEMM_CONSUMER_WARPS arrivals).
template <int BN>
__device__ __forceinline__ void tile_mainloop(float (&acc)[BN / 2], uint8_t* ring, int stage_bytes, uint64_t* full_bar, uint64_t* empty_bar,
                                              int num_kb, int stages, RingPos& rp, int wg, int lane, long long* t_wait) {
  constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    const long long w0 = t_wait ? clock64() : 0;
    mbar_wait(&full_bar[rp.stage], rp.phase);
    if (t_wait) *t_wait += clock64() - w0;
    const uint32_t sa = smem_u32(ring + rp.stage * stage_bytes) + wg * 64 * 128;
    const uint32_t sb = smem_u32(ring + rp.stage * stage_bytes + A_BYTES);
    const uint64_t ad = wgmma_desc<128>(sa), bd = wgmma_desc<128>(sb);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, ad + 2 * k, bd + 2 * k, (kb | k) != 0);   // +32 B per K = 16 step
    wgmma_commit();
    wgmma_wait<1>();                                  // k-block kb-1 has retired: its slot may be refilled
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = rp.stage;
    rp.next(stages);
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

// ---------------------------------------------------------------- epilogues from the accumulator registers
// Thread (warp w of the warpgroup, lane l) holds rows 16 w + l / 4 and + 8 of the warpgroup's 64, columns 8 j + 2 (l % 4) + {0, 1}.
template <int EPI>
__device__ __forceinline__ float epi_act(float v) {
  if constexpr (EPI == EPI_BF16_GELU) return gelu_fast(v);
  else if constexpr (EPI == EPI_BF16_GELU_ERF) return gelu_erf_as(v);
  else if constexpr (EPI == EPI_BF16_RELU_UP) return relu_keep_nan(v);
  else return v;
}

// TMA epilogues: 64 bf16 / 32 f32 columns (one 128-byte staging row) per round, two staging buffers per warpgroup in turn.
// `stiles` = this warpgroup's two buffers; `tid` = thread index inside the warpgroup (thread 0 issues and owns the bulk groups).
// `first` = the buffer of round 0: with an odd number of rounds per tile (BN = 192, bf16) the caller alternates it from tile to
// tile, so that round 0 never reuses the buffer of the previous tile's last round, whose store may still be reading it.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tma(const float (&acc)[BN / 2], int n0, int row0, int N, const float* __restrict__ bias, uint8_t* stiles,
                                             int wg, int tid, const CUtensorMap* tmap_out, int first = 0) {
  constexpr int COLS = (EPI == EPI_F32_ADD) ? 32 : 64;
  constexpr int JPC = COLS / 8;                       // accumulator column groups per round
  const int lane = tid & 31, wq = tid >> 5;
  const int r_lo = 16 * wq + (lane >> 2);             // staging rows r_lo and r_lo + 8 (same swizzle phase: (r + 8) % 8 = r % 8)
  const int sw = r_lo & 7;
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int c = 0; c < BN / COLS; ++c) {
    uint8_t* st = stiles + ((c ^ first) & 1) * GEMM_STAGE_TILE;
    const uint32_t sa = smem_u32(st);                 // st.shared with 32-bit addresses: generic 64-bit ones made ptxas spill BN = 256
    if (tid == 0) tma_store_wait_read<1>();           // the store that used this buffer two rounds ago has read it
    named_bar_sync(GEMM_BAR_EPI + 1 + wg, 128);
#pragma unroll
    for (int jl = 0; jl < JPC; ++jl) {
      const int j = c * JPC + jl;
      const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n0 + 8 * j + cq));
      const float v0 = epi_act<EPI>(acc[4 * j] + b2.x), v1 = epi_act<EPI>(acc[4 * j + 1] + b2.y);
      const float v2 = epi_act<EPI>(acc[4 * j + 2] + b2.x), v3 = epi_act<EPI>(acc[4 * j + 3] + b2.y);
      if constexpr (EPI == EPI_F32_ADD) {
        const int off = (((2 * jl + ((lane & 3) >> 1)) ^ sw) << 4) + (lane & 1) * 8;
        sts_f32x2(sa + r_lo * 128 + off, v0, v1);
        sts_f32x2(sa + (r_lo + 8) * 128 + off, v2, v3);
      } else {
        const int off = ((jl ^ sw) << 4) + (lane & 3) * 4;
        sts_u32(sa + r_lo * 128 + off, pack_bf16(v0, v1));
        sts_u32(sa + (r_lo + 8) * 128 + off, pack_bf16(v2, v3));
      }
    }
    fence_proxy_async_smem();                         // staging writes -> visible to the TMA engine
    named_bar_sync(GEMM_BAR_EPI + 1 + wg, 128);
    const int n = n0 + c * COLS;
    if (tid == 0 && n < N) {
      if constexpr (EPI == EPI_F32_ADD) tma_reduce_add_2d(tmap_out, st, n, row0);
      else tma_store_2d(tmap_out, st, n, row0);       // rows past M are clipped by the tensor map
    }
    if (tid == 0) tma_store_commit();
  }
}

// fp32 residual epilogue as LOAD + ADD + STORE (option "resid_rmw"): every element of the stream has exactly ONE writer per
// launch (no split-K), so that writer can do the add itself: fl(x + fl(acc + bias)), the very two roundings of the reduce-add
// form, hence bit-identical to it.
template <int BN>
__device__ __forceinline__ void epilogue_f32_rmw(const float (&acc)[BN / 2], int n0, int row0, int M, const float* __restrict__ bias,
                                                 float* __restrict__ x, int ldx, int tid) {
  const int lane = tid & 31, wq = tid >> 5;
  const int r_lo = row0 + 16 * wq + (lane >> 2);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + cq;
    if (n >= ldx) continue;
    const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_lo + 8 * h;
      if (r < M) {
        float2* px = reinterpret_cast<float2*>(x + static_cast<size_t>(r) * ldx + n);
        const float2 xv = __ldcg(px);
        __stcg(px, make_float2(xv.x + (acc[4 * j + 2 * h] + b2.x), xv.y + (acc[4 * j + 2 * h + 1] + b2.y)));
      }
    }
  }
}

// One warp normalises one row of the fp32 stream (D = 128*V columns) straight out of L2 (ld.global.cg: the row was just
// written by other SMs' TMA reduce-adds / stores) -> bf16.  nn.LayerNorm(eps), biased variance (backbone/vit.py:190,198,304).
template <int V>
__device__ __forceinline__ void ln_row_l2(const float* __restrict__ xrow, const float* __restrict__ gamma, const float* __restrict__ beta,
                                          __nv_bfloat16* __restrict__ yrow, float eps, int lane) {
  constexpr int D = 128 * V;
  float4 v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = __ldcg(reinterpret_cast<const float4*>(xrow) + i * 32 + lane);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / D;                           // divided, as layernorm_f32_to_bf16 (bit-identical to it)
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
    q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * (1.0f / D) + eps);
  uint2* yr = reinterpret_cast<uint2*>(yrow);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i * 32 + lane);
    const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + i * 32 + lane);
    uint2 o;
    o.x = pack_bf16(v[i].x * rstd * g.x + b.x, v[i].y * rstd * g.y + b.y);
    o.y = pack_bf16(v[i].z * rstd * g.z + b.z, v[i].w * rstd * g.w + b.w);
    yr[i * 32 + lane] = o;
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                const __grid_constant__ CUtensorMap tmap_out, const GemmParams p) {
  using Cfg = GemmCfg<BN, EPI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;
  uint8_t* staging = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  volatile int* ln_flag = reinterpret_cast<volatile int*>(empty_bar + Cfg::STAGES);   // "this CTA finishes the row block" broadcast

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);     // warp-uniform for the compiler (see elect_one in ptx.cuh)
  const int lane = threadIdx.x & 31;
  constexpr bool kDeconv = (EPI == EPI_BF16_RELU_UP);
  // deconv: an M tile is a up_tr x up_tw patch (96 or 128 positions) of one crop, p.M counts positions; the 4 phases play the n-blocks
  const int up_pos = kDeconv ? p.up_tr * p.up_tw : GEMM_BM;
  const int num_m = kDeconv ? p.M / up_pos : (p.M + GEMM_BM - 1) / GEMM_BM;
  const int num_n = kDeconv ? 4 : (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = p.K / GEMM_BK;
  const int num_stages = (p.stages_limit > 0 && p.stages_limit < Cfg::STAGES) ? p.stages_limit : Cfg::STAGES;
  auto tile_mn = [&](int tile, int& mt, int& nb) {
    if (p.dbg_flags & 4) { mt = tile % num_m; nb = tile / num_m; }
    else { mt = tile / num_n; nb = tile % num_n; }
  };

  const long long t_cta0 = (p.dbg && threadIdx.x == 0) ? clock64() : 0;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    if constexpr (epi_uses_tma(EPI)) tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);                     // the producer's expect_tx arrival
      mbar_init(&empty_bar[s], GEMM_CONSUMER_WARPS);  // every consumer warp releases the slot
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();                          // the next kernel may start its prologue as SMs free up
  pdl_wait();                                       // previous kernel's outputs (our A operand / residual) are complete

  // Register split: the producer warpgroup (warps 8..11; only warp 8 issues) needs few registers, the consumers' accumulators
  // (BN / 2 per thread) and epilogue need many.  384 threads start at 168 each; 128 x 40 + 256 x 232 = 64512 <= 65536.
  if (warp >= GEMM_CONSUMER_WARPS) {
    setmaxnreg_dec<40>();
    if (warp != GEMM_CONSUMER_WARPS) return;        // warps 9..11 only take part in the warpgroup-wide dec
    // ------------------------------------------------------------ TMA producer: the whole warp runs the (uniform) loop, one
    // elected lane issues
    RingPos rp;
    long long t_wait = 0;
    const long long t_begin = p.dbg ? clock64() : 0;
    const int tiles_x = kDeconv ? p.up_w / p.up_tw : 1;
    const int tiles_per_img = kDeconv ? (p.up_h / p.up_tr) * tiles_x : 1;
    const int kb_per_tap = kDeconv ? p.up_c / GEMM_BK : 1;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mt, nb;
      tile_mn(tile, mt, nb);
      const int m0 = (p.dbg_flags & 1) ? 0 : mt * GEMM_BM;   // may lie past M: TMA zero-fills
      const int n0 = (p.dbg_flags & 2) ? 0 : nb * BN;
      for (int kb = 0; kb < num_kb; ++kb) {
        const long long w0 = p.dbg ? clock64() : 0;
        ring_wait_slot(empty_bar, rp);
        if (p.dbg) t_wait += clock64() - w0;
        uint8_t* sa = ring + rp.stage * Cfg::STAGE_BYTES;
        if (elect_one()) {
          if constexpr (kDeconv) {
            // A tile = a up_tr x up_tw patch of the input map shifted by the tap's (dy, dx); the 4-D box is zero filled
            // outside the map (= the transposed conv's border).  With 96-position tiles rows 96..127 of the smem tile are
            // never written: they only feed accumulator rows nobody stores.
            const int tap = kb / kb_per_tap, c0 = (kb % kb_per_tap) * GEMM_BK;
            const int py = nb >> 1, px = nb & 1, iy = tap >> 1, ix = tap & 1;
            const int dy = py ? (iy ? 0 : 1) : (iy ? -1 : 0);
            const int dx = px ? (ix ? 0 : 1) : (ix ? -1 : 0);
            mbar_expect_tx(&full_bar[rp.stage], up_pos * 128 + Cfg::B_BYTES);
            const int ti = mt % tiles_per_img;
            tma_load_4d(sa, &tmap_a, &full_bar[rp.stage], c0, (ti % tiles_x) * p.up_tw + dx, (ti / tiles_x) * p.up_tr + dy, mt / tiles_per_img);
          } else {
            mbar_expect_tx(&full_bar[rp.stage], Cfg::STAGE_BYTES);
            tma_load_2d(sa, &tmap_a, &full_bar[rp.stage], kb * GEMM_BK, m0);
          }
          tma_load_2d(sa + Cfg::A_BYTES, &tmap_w, &full_bar[rp.stage], kb * GEMM_BK, n0);
        }
        __syncwarp();
        rp.next(num_stages);
      }
    }
    if (p.dbg && lane == 0) { p.dbg[blockIdx.x * 8 + 3] = clock64() - t_begin; p.dbg[blockIdx.x * 8 + 4] = t_wait; }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------------------------------------ consumers: MMA + epilogue, warpgroup wg owns rows 64 wg ..
    const int wg = warp >> 2;
    const int tid = threadIdx.x & 127;
    const int wq = warp & 3;
    uint8_t* stiles = staging + wg * 2 * GEMM_STAGE_TILE;
    RingPos rp;
    int sfirst = 0;                                   // staging buffer of the next tile's first epilogue round
    long long t_full = 0;
    const long long t_begin = p.dbg ? clock64() : 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mt, nb;
      tile_mn(tile, mt, nb);
      const int m0 = mt * GEMM_BM;
      const int n0 = kDeconv ? 0 : nb * BN;
      tile_mainloop<BN>(acc, ring, Cfg::STAGE_BYTES, full_bar, empty_bar, num_kb, num_stages, rp, wg, lane,
                        (p.dbg && threadIdx.x == 0) ? &t_full : nullptr);
      const int row0 = m0 + 64 * wg;                  // first row of this warpgroup

      if constexpr (epi_uses_tma(EPI)) {
        if (EPI == EPI_F32_ADD && p.rmw) epilogue_f32_rmw<BN>(acc, n0, row0, p.M, p.bias, reinterpret_cast<float*>(p.out), p.ldc, tid);
        else {
          epilogue_tma<BN, EPI>(acc, n0, row0, p.N, p.bias, stiles, wg, tid, &tmap_out, sfirst);
          sfirst ^= (BN / (EPI == EPI_F32_ADD ? 32 : 64)) & 1;
        }
      } else {
        // ---- direct epilogues (scattered / transposed outputs)
        const int cq = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 64 * wg + 16 * wq + (lane >> 2) + 8 * h;     // row inside the tile
          if constexpr (EPI == EPI_BF16_RELU_UP) {
            if (r >= up_pos || mt >= num_m) continue;
            const int tiles_x = p.up_w / p.up_tw;
            const int tiles_per_img = (p.up_h / p.up_tr) * tiles_x;
            const int b = mt / tiles_per_img, ti = mt % tiles_per_img;
            const int y = (ti / tiles_x) * p.up_tr + r / p.up_tw, x = (ti % tiles_x) * p.up_tw + r % p.up_tw;
            const size_t out_row = (static_cast<size_t>(b) * (2 * p.up_h) + (2 * y + (nb >> 1))) * (2 * p.up_w) + (2 * x + (nb & 1));
            uint32_t* o = reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + out_row * p.ldc);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int n = 8 * j + cq;
              if (n >= p.N) continue;
              const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias + n));
              o[n >> 1] = pack_bf16(relu_keep_nan(acc[4 * j + 2 * h] + b2.x), relu_keep_nan(acc[4 * j + 2 * h + 1] + b2.y));
            }
          } else {  // EPI_F32_NCHW
            const int row = m0 + r;
            if (row >= p.M) continue;
            const int b = row / p.pix, pix = row % p.pix;
            float* o = reinterpret_cast<float*>(p.out) + (static_cast<size_t>(b) * (p.ch_stride ? p.ch_stride : p.n_valid)) * p.pix + pix;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int n = n0 + 8 * j + cq;
              float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              if (p.bias != nullptr) { v0 += p.bias[n]; v1 += p.bias[n + 1]; }
              if (n < p.n_valid) o[static_cast<size_t>(n) * p.pix] = v0;
              if (n + 1 < p.n_valid) o[static_cast<size_t>(n + 1) * p.pix] = v1;
            }
          }
        }
      }

      if constexpr (EPI == EPI_F32_ADD) {
        if (p.ln_out != nullptr && mt < num_m) {
          // ---- fused LayerNorm tail
          if (tid == 0) tma_store_wait_all<0>();            // this warpgroup's reduce-adds have been performed in L2
          named_bar_sync(GEMM_BAR_EPI, 256);                // both consumer warpgroups are done with the tile
          if (threadIdx.x == 0) {
            __threadfence();
            const int old = atomicAdd(p.ln_counters + mt, 1);
            const int last = (old == num_n - 1);
            if (last) p.ln_counters[mt] = 0;                // every column tile has arrived: reset for the next launch
            *ln_flag = last;
          }
          named_bar_sync(GEMM_BAR_EPI, 256);
          if (*ln_flag) {
            __threadfence();                                // acquire side of the counter hand-off
            const int r_end = min(GEMM_BM, p.M - m0);
            const float* xb = reinterpret_cast<const float*>(p.out) + static_cast<size_t>(m0) * p.N;
            __nv_bfloat16* yb = p.ln_out + static_cast<size_t>(m0) * p.N;
            for (int r = warp; r < r_end; r += GEMM_CONSUMER_WARPS) {
              const float* xr = xb + static_cast<size_t>(r) * p.N;
              __nv_bfloat16* yr = yb + static_cast<size_t>(r) * p.N;
              switch (p.N) {
                case 384: ln_row_l2<3>(xr, p.ln_gamma, p.ln_beta, yr, p.ln_eps, lane); break;
                case 768: ln_row_l2<6>(xr, p.ln_gamma, p.ln_beta, yr, p.ln_eps, lane); break;
                case 1024: ln_row_l2<8>(xr, p.ln_gamma, p.ln_beta, yr, p.ln_eps, lane); break;
                default: ln_row_l2<10>(xr, p.ln_gamma, p.ln_beta, yr, p.ln_eps, lane); break;   // 1280
              }
            }
          }
          named_bar_sync(GEMM_BAR_EPI, 256);                // ln_flag is rewritten at the next tile
        }
      }
    }
    if constexpr (epi_uses_tma(EPI)) {
      if (tid == 0) tma_store_wait_all<0>();        // staging must stay alive until the TMA engine is done with it
    }
    if (p.dbg && threadIdx.x == 0) { p.dbg[blockIdx.x * 8 + 0] = clock64() - t_begin; p.dbg[blockIdx.x * 8 + 1] = t_full; }
  }
  if (p.dbg && threadIdx.x == 0) p.dbg[blockIdx.x * 8 + 7] = clock64() - t_cta0;
}

}  // namespace vpb
