// One persistent launch for a CHAIN of dependent GEMMs of a transformer block, with the LayerNorms between them:
//
//     [proj (+= x)] -> LN -> [fc1 + GELU] -> [fc2 (+= x)] -> LN -> [qkv of the next block]        (backbone/vit.py:202-205,164-180)
//
// Run as 4 GEMM launches + 2 LayerNorm launches, every launch pays a head (barrier init, first TMA round trip) and a tail (last
// tile's epilogue, idle SMs in the last wave) that programmatic dependent launch cannot hide (a CTA near the 227 KB shared
// memory limit leaves no room for the next grid), and every LayerNorm is a separate pass of the fp32 stream through all SMs
// with nothing else running.  Here the tiles of all phases form ONE list, handed out statically (tile g -> CTA g mod grid,
// phase-major, n fastest), and what used to be a kernel boundary is a counter:
//
//   * every 128-row block `mt` of an activation has a counter that the producing consumer warpgroups bump once their TMA
//     stores / reduce-adds of a tile have COMPLETED (cp.async.bulk.wait_group 0, cross-proxy fence, release);
//   * the TMA-producer warp of a consuming tile spins (acquire) on the counter of its A rows before its first load;
//   * LayerNorm runs on four dedicated warps of every CTA, concurrently with that CTA's tensor-core tiles: 16-row jobs handed
//     out statically (job j -> CTA j mod grid), each waiting for its row block's residual adds to complete; they read the fp32
//     stream out of L2 (ld.global.cg) and write the bf16 operand rows; the gpu-scope part of a job -- polling the residual
//     counter, the acquire, the cross-proxy fence and the release that bumps the "normalised rows ready" counter -- runs on a
//     control warp (ln_ctl, default) so that the LayerNorm warps only load, normalise and store.
//
// Dependencies only point to tiles that come earlier in the list (and LN jobs only to tiles), all CTAs are resident (one per
// SM, grid <= #SMs), every role walks its own list in order (see "Tile list" in the kernel for the order): the smallest
// unfinished tile can always run, so the waits cannot deadlock; a counter that never arrives traps (VPB_HANG_TRAP_SPINS)
// instead of hanging the GPU.
// The arithmetic of every phase is that of gemm.cuh's kernels and of layernorm_f32_to_bf16, in the same order: results are
// bit-identical to the unchained path (tests/test_gpu_engine.py::test_chain_is_bit_identical).
//
//   warps 0..7   consumers: two warpgroups, wgmma into registers, then the TMA epilogue of gemm.cuh
//   warp  8      TMA producer (+ dependency waits)
//   warp  9      LayerNorm control (ln_ctl): polls the residual counters / publishes the jobs for warps 10..13
//   warps 10..13 LayerNorm jobs
#pragma once
#include "gemm.cuh"

namespace vpb {

constexpr int CHAIN_MAX_PHASES = 4;
constexpr int CHAIN_MAX_LN = 2;
constexpr int CHAIN_THREADS = 448;       // 8 consumer warps, producer, LayerNorm control, 4 LayerNorm warps
constexpr int CHAIN_LN_WARPS = 4;
constexpr int CHAIN_LN_JOB_ROWS = 16;      // default rows per LayerNorm job (ChainParams::ln_job_rows: 8 or 16): 4 per warp

struct ChainPhase {
  int N, K;                 // W is [N,K]; N % BN == 0, K % 64 == 0
  int epi;                  // EPI_BF16 | EPI_BF16_GELU | EPI_BF16_GELU_ERF | EPI_F32_ADD
  const float* bias;        // [N]
  const int* a_ready;       // per 128-row block: A rows are complete once a_ready[mt] >= target (nullptr: produced by an earlier launch)
  int a_target;             // > 0: that many arrivals (GEMM-produced A: one per column tile of the producing phase);
                            // 0: LayerNorm-produced A: one arrival per 16-row job of the block
  int* out_done;            // per 128-row block, += 1 per tile once the CTA's stores of it have completed (nullptr: nobody waits)
};
struct ChainLn {
  const int* src_done;      // out_done of the residual phase that completes the fp32 rows
  int src_target;           // column tiles of that phase
  const float* gamma;       // [D]
  const float* beta;        // [D]
  int* ready;               // per 128-row block, += 1 per finished job
};
struct ChainParams {
  int M;                    // rows (tokens) of every phase
  int D;                    // LayerNorm width = row pitch of x / xn
  int num_phases, num_ln;
  const float* x;           // fp32 stream [M, D]
  __nv_bfloat16* xn;        // LayerNorm output [M, D]
  float eps;
  int wave_lag[2];          // tile order: lag (in 128-row blocks) of the second phase behind the first inside wavefronts {0,1} and {2,3}
  int ln_job_rows;          // rows per LayerNorm job: 16 (two 2-row iterations per warp) or 8 (one)
  int ln_ctl;               // 1 = the counter polls / publishes of the LayerNorm jobs run on a control warp (warp 9), 0 = on warp 10
  int rmw;                  // fp32 residual phases: 1 = load + add + store in the generic proxy (gemm.cuh: epilogue_f32_rmw), 0 = TMA reduce-add
  int dbg_nowait;           // measurement only (results may be wrong): publish tiles without waiting for their stores to complete
  long long* dbg;           // measurement: per CTA [CHAIN_MAX_PHASES][12] cycle counters or nullptr (8..10: LayerNorm stage s under
                            //   phase 2s, warp 10: wait for the residual rows, busy, jobs):
                            //   1 consumer wait for operands, 3 producer dependency wait, 4 producer wait for ring slots, 5 epilogue
                            //   (thread 0), 7 tiles, 11 dependency wait of the CTA's first tile of the phase
  ChainPhase ph[CHAIN_MAX_PHASES];
  ChainLn ln[CHAIN_MAX_LN];
};
struct alignas(64) ChainMaps {
  CUtensorMap a[CHAIN_MAX_PHASES], w[CHAIN_MAX_PHASES], out[CHAIN_MAX_PHASES];
};

template <int BN>
using ChainCfg = TileCfg<BN, true>;

// ---------------------------------------------------------------- counters in global memory
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// generic proxy <-> async proxy (TMA) ordering for global memory
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ int ld_relaxed_gpu(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Whole warp spins (one coalesced load per probe) until *p >= target.  The probes are RELAXED loads and one acquire fence
// follows the successful one: an acquire load at gpu scope is compiled to LDG + CCTL.IVALL, i.e. every probe of every waiting
// warp would invalidate the SM's L1 under the consumer warps' bias loads.
__device__ __forceinline__ void wait_counter(const int* p, int target) {
  uint32_t spins = 0;
  while (ld_relaxed_gpu(p) < target) {
    __nanosleep(64);
    if (++spins > (VPB_HANG_TRAP_SPINS >> 3)) __trap();
  }
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
}
__host__ __device__ __forceinline__ int chain_ln_jobs_in_block(int M, int mt, int job_rows) {
  const int rows = M - mt * GEMM_BM < GEMM_BM ? M - mt * GEMM_BM : GEMM_BM;
  return (rows + job_rows - 1) / job_rows;
}

// ---------------------------------------------------------------- LayerNorm rows (same arithmetic, same order as
// layernorm_f32_to_bf16 in pointwise.cuh: fp32 mean, centred biased variance, rsqrtf; backbone/vit.py:190,198,304)
template <int V>
struct LnRow {
  float4 v[V];
  float rstd;
  __device__ __forceinline__ void load(const float* __restrict__ xrow, int lane) {
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = __ldcg(reinterpret_cast<const float4*>(xrow) + i * 32 + lane);    // L2: written by other SMs
  }
  // centres v in place and leaves 1/sqrt(var + eps) in rstd
  __device__ __forceinline__ void stats(float eps) {
    constexpr int D = 128 * V;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / D;                         // divided, as layernorm_f32_to_bf16 (bit-identical to it)
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    rstd = rsqrtf(q * (1.0f / D) + eps);
  }
  __device__ __forceinline__ uint2 out(int i, const float4& g, const float4& b) const {
    uint2 o;
    o.x = pack_bf16(v[i].x * rstd * g.x + b.x, v[i].y * rstd * g.y + b.y);
    o.y = pack_bf16(v[i].z * rstd * g.z + b.z, v[i].w * rstd * g.w + b.w);
    return o;
  }
};
// rows [r0, r1) of one warp's share of a job; two rows in flight while they fit in registers (D <= 768), else one.
// gamma / beta are fetched once per 128-column slice and shared by the rows in flight.
template <int V>
__device__ __forceinline__ void chain_ln_rows(const ChainParams& p, const ChainLn& ln, int r0, int r1, int lane) {
  constexpr int D = 128 * V;
  constexpr int R = V <= 6 ? 2 : 1;
  for (int r = r0; r < r1; r += R) {
    LnRow<V> row[R];
    const bool two = R == 2 && r + 1 < r1;
    row[0].load(p.x + static_cast<size_t>(r) * D, lane);
    if constexpr (R == 2) { if (two) row[1].load(p.x + static_cast<size_t>(r + 1) * D, lane); }
    // gamma / beta are requested together with the rows (one exposed memory latency per job instead of two: the SM's L1 is
    // invalidated by every acquire fence of the CTA, so these are L2 round trips more often than not)
    float4 g[V], b[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
      g[i] = __ldg(reinterpret_cast<const float4*>(ln.gamma) + i * 32 + lane);
      b[i] = __ldg(reinterpret_cast<const float4*>(ln.beta) + i * 32 + lane);
    }
    row[0].stats(p.eps);
    if constexpr (R == 2) { if (two) row[1].stats(p.eps); }
    uint2* y0 = reinterpret_cast<uint2*>(p.xn + static_cast<size_t>(r) * D);
    uint2* y1 = reinterpret_cast<uint2*>(p.xn + static_cast<size_t>(r + 1) * D);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      y0[i * 32 + lane] = row[0].out(i, g[i], b[i]);
      if constexpr (R == 2) { if (two) y1[i * 32 + lane] = row[1].out(i, g[i], b[i]); }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(CHAIN_THREADS, 1)
gemm_chain_wgmma(const __grid_constant__ ChainMaps maps, const __grid_constant__ ChainParams p) {
  using Cfg = ChainCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;
  uint8_t* staging = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  uint64_t* ln_done = empty_bar + Cfg::STAGES;      // [2] LayerNorm warps -> control warp: the job's rows are written

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int num_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  // Tile list.  Default (lag >= #row blocks): PHASE-MAJOR, inside a phase tile = mt * num_n + nb (n fastest).  The general form pairs
  // the phases into two wavefronts, {0, 1} then {2, 3}: slot s holds the tiles of the first phase for row block s and those of the
  // second phase for row block s - lag, so that a CTA alternates between a reduce-add phase (proj, fc2) and its consumer.
  // Dependencies only point backwards for any lag (tests/test_chain_order.py); kept as an experiment (engine.cu: VPB_CHAIN_LAG0/1).
  int n_of[CHAIN_MAX_PHASES];
#pragma unroll
  for (int i = 0; i < CHAIN_MAX_PHASES; ++i) n_of[i] = i < p.num_phases ? p.ph[i].N / BN : 0;
  const int lag0 = p.wave_lag[0] < num_m ? p.wave_lag[0] : num_m, lag1 = p.wave_lag[1] < num_m ? p.wave_lag[1] : num_m;
  const int wave0_tiles = num_m * (n_of[0] + n_of[1]);
  const int total_tiles = wave0_tiles + num_m * (n_of[2] + n_of[3]);
  auto locate = [&](int g, int& ph, int& mt, int& nb) {
    const bool w1 = g >= wave0_tiles;
    const int gg = w1 ? g - wave0_tiles : g;
    const int na = w1 ? n_of[2] : n_of[0], nbb = w1 ? n_of[3] : n_of[1];
    const int lag = nbb == 0 ? num_m : (w1 ? lag1 : lag0);
    const int pa = w1 ? 2 : 0;
    const int head = na * lag;                               // slots [0, lag): first phase only
    const int mid = (num_m - lag) * (na + nbb);              // slots [lag, num_m): both
    if (gg < head) { ph = pa; mt = gg / na; nb = gg % na; }
    else if (gg < head + mid) {
      const int q = gg - head, s = lag + q / (na + nbb), r = q % (na + nbb);
      if (r < na) { ph = pa; mt = s; nb = r; }
      else { ph = pa + 1; mt = s - lag; nb = r - na; }
    } else {
      const int q = gg - head - mid;                         // slots [num_m, num_m + lag): second phase only
      ph = pa + 1; mt = num_m - lag + q / nbb; nb = q % nbb;
    }
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.num_phases; ++i) {
      tma_prefetch_desc(&maps.a[i]);
      tma_prefetch_desc(&maps.w[i]);
      tma_prefetch_desc(&maps.out[i]);
    }
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_CONSUMER_WARPS);
    }
    for (int s = 0; s < 2; ++s) mbar_init(&ln_done[s], CHAIN_LN_WARPS);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                                       // the previous kernel's outputs (first phase's A operand, x) are complete

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer (+ the waits that replace kernel boundaries)
    RingPos rp;
    int prev_ph = -1;
    for (int g = blockIdx.x; g < total_tiles; g += gridDim.x) {
      int ph, mt, nb;
      locate(g, ph, mt, nb);
      const ChainPhase& P = p.ph[ph];
      const int m0 = mt * GEMM_BM, n0 = nb * BN;
      const bool first_of_phase = ph != prev_ph;
      prev_ph = ph;
      const int num_kb = P.K / GEMM_BK;
      long long c0 = p.dbg ? clock64() : 0, w_dep = 0, w_ring = 0;
      if (P.a_ready != nullptr) {
        wait_counter(P.a_ready + mt, P.a_target > 0 ? P.a_target : chain_ln_jobs_in_block(p.M, mt, p.ln_job_rows));
        fence_proxy_async_all();                    // the rows were written through the generic / async proxy of other SMs
      }
      if (p.dbg) w_dep = clock64() - c0;
      for (int kb = 0; kb < num_kb; ++kb) {
        if (p.dbg) c0 = clock64();
        ring_wait_slot(empty_bar, rp);
        if (p.dbg) w_ring += clock64() - c0;
        uint8_t* sa = ring + rp.stage * Cfg::STAGE_BYTES;
        if (elect_one()) {
          mbar_expect_tx(&full_bar[rp.stage], Cfg::STAGE_BYTES);
          tma_load_2d(sa, &maps.a[ph], &full_bar[rp.stage], kb * GEMM_BK, m0);
          tma_load_2d(sa + Cfg::A_BYTES, &maps.w[ph], &full_bar[rp.stage], kb * GEMM_BK, n0);
        }
        __syncwarp();
        rp.next(Cfg::STAGES);
      }
      if (p.dbg && lane == 0) {
        long long* d = p.dbg + (blockIdx.x * CHAIN_MAX_PHASES + ph) * 12;
        d[3] += w_dep;
        if (first_of_phase) d[11] += w_dep;
        d[4] += w_ring;
      }
    }
  } else if (warp < GEMM_CONSUMER_WARPS) {
    // ------------------------------------------------------------ consumers: MMA + epilogue
    const int wg = warp >> 2;
    const int tid = threadIdx.x & 127;
    uint8_t* stiles = staging + wg * 2 * GEMM_STAGE_TILE;
    RingPos rp;
    float acc[BN / 2];
    for (int g = blockIdx.x; g < total_tiles; g += gridDim.x) {
      int ph, mt, nb;
      locate(g, ph, mt, nb);
      const ChainPhase& P = p.ph[ph];
      const int n0 = nb * BN, row0 = mt * GEMM_BM + 64 * wg;
      long long w_full = 0;
      tile_mainloop<BN>(acc, ring, Cfg::STAGE_BYTES, full_bar, empty_bar, P.K / GEMM_BK, Cfg::STAGES, rp, wg, lane,
                        (p.dbg && threadIdx.x == 0) ? &w_full : nullptr);
      const long long e0 = p.dbg ? clock64() : 0;
      if (P.epi == EPI_F32_ADD && p.rmw) epilogue_f32_rmw<BN>(acc, n0, row0, p.M, P.bias, const_cast<float*>(p.x), p.D, tid);
      else if (P.epi == EPI_F32_ADD) epilogue_tma<BN, EPI_F32_ADD>(acc, n0, row0, P.N, P.bias, stiles, wg, tid, &maps.out[ph]);
      else if (P.epi == EPI_BF16_GELU) epilogue_tma<BN, EPI_BF16_GELU>(acc, n0, row0, P.N, P.bias, stiles, wg, tid, &maps.out[ph]);
      else if (P.epi == EPI_BF16_GELU_ERF) epilogue_tma<BN, EPI_BF16_GELU_ERF>(acc, n0, row0, P.N, P.bias, stiles, wg, tid, &maps.out[ph]);
      else epilogue_tma<BN, EPI_BF16>(acc, n0, row0, P.N, P.bias, stiles, wg, tid, &maps.out[ph]);
      if (P.out_done != nullptr) {
        // publish the tile ONCE per CTA: each warpgroup's issuing thread waits until its stores / reduce-adds have been
        // PERFORMED (not just read out of smem) and fences them across the proxies (the load + add + store form's plain stores
        // are ordered by the release below); the two warpgroups meet on a named barrier; one thread does the gpu-scope release
        if (tid == 0) {
          if (!p.dbg_nowait) tma_store_wait_all<0>();
          fence_proxy_async_all();
        }
        named_bar_sync(GEMM_BAR_EPI, 256);
        if (threadIdx.x == 0) red_release_gpu_add(P.out_done + mt, 1);
      }
      if (p.dbg && threadIdx.x == 0) {
        long long* d = p.dbg + (blockIdx.x * CHAIN_MAX_PHASES + ph) * 12;
        d[1] += w_full; d[5] += clock64() - e0; d[7] += 1;
      }
    }
    if (tid == 0) tma_store_wait_all<0>();
  } else if (warp == 9 && p.ln_ctl != 0) {
    // ------------------------------------------------------------ LayerNorm control warp
    // The gpu-scope fences around a job -- the acquire after the poll of the residual phase's counter, fence.proxy.async +
    // red.release to publish the normalised rows -- are latency the LayerNorm warps would otherwise sit in, and the LayerNorm
    // stages are what the consumer phases wait for.  This warp takes both over: it walks the CTA's job list (job j -> CTA j mod grid, stage-major), polls
    // job i + 1 while the LayerNorm warps work on job i and publishes job i when they have arrived on ln_done.  Two slots each
    // way (slot = job sequence number & 1; "ready": named barriers 4 / 5, "done": mbarriers); "ready" for job i + 2 is only
    // signalled after "done" of job i was seen, so neither barrier can run a phase ahead.  Neither probe blocks: the first job of stage 1 waits for fc2 tiles that may
    // themselves wait for this CTA's last job of stage 0, which must be publishable in the meantime.
    const int jobs = (p.M + p.ln_job_rows - 1) / p.ln_job_rows;
    const int first = static_cast<int>(blockIdx.x), step = static_cast<int>(gridDim.x);
    const int end_s = first < jobs ? p.num_ln : 0;
    int a_s = 0, a_job = first, a_seq = 0;            // poll cursor
    int b_s = 0, b_job = first, b_seq = 0;            // publish cursor
    uint32_t idle = 0;
    while (b_s < end_s) {
      bool progressed = false;
      // neither probe blocks: a job that is done is published even while the next one's source rows are still outstanding
      if (a_s < end_s && a_seq <= b_seq + 1) {
        const ChainLn& L = p.ln[a_s];
        if (__shfl_sync(0xffffffffu, ld_relaxed_gpu(L.src_done + (a_job * p.ln_job_rows) / GEMM_BM), 0) >= L.src_target) {
          asm volatile("fence.acq_rel.gpu;" ::: "memory");
          __syncwarp();
          // "ready" is a NAMED barrier (ids 4 / 5 by slot, 4 LayerNorm warps + this one): the LayerNorm warps sleep in
          // bar.sync without taking issue slots (polling an mbarrier with try_wait would add four spinning warps per SM
          // that share schedulers with the consumer warps).
          if (a_seq & 1) asm volatile("bar.arrive 5, 160;" ::: "memory");
          else asm volatile("bar.arrive 4, 160;" ::: "memory");
          ++a_seq;
          a_job += step;
          if (a_job >= jobs) { ++a_s; a_job = first; }
          progressed = true;
        }
      }
      if (b_seq < a_seq && __shfl_sync(0xffffffffu, mbar_test_wait(&ln_done[b_seq & 1], (b_seq >> 1) & 1) ? 1 : 0, 0)) {
        if (lane == 0) {
          fence_proxy_async_all();                    // consumed by TMA loads (async proxy) of other SMs
          red_release_gpu_add(p.ln[b_s].ready + (b_job * p.ln_job_rows) / GEMM_BM, 1);
        }
        __syncwarp();
        ++b_seq;
        b_job += step;
        if (b_job >= jobs) { ++b_s; b_job = first; }
        progressed = true;
      }
      if (progressed) idle = 0;
      else {
        __nanosleep(96);                              // this warp shares a scheduler with two epilogue warps
        if (++idle > (VPB_HANG_TRAP_SPINS >> 3)) __trap();
      }
    }
  } else if (warp >= 10) {
    // ------------------------------------------------------------ LayerNorm jobs
    const int lw = warp - 10;
    const int jobs = (p.M + p.ln_job_rows - 1) / p.ln_job_rows;
    const int ROWS_PER_WARP = p.ln_job_rows / CHAIN_LN_WARPS;
    const bool ctl = p.ln_ctl != 0;                  // polls / publishes on the control warp (warp 9)
    uint32_t seq = 0;                                 // job sequence number of this CTA over both stages (mbarrier slot / parity)
    for (int s = 0; s < p.num_ln; ++s) {
      const ChainLn& L = p.ln[s];
      for (int job = blockIdx.x; job < jobs; job += gridDim.x, ++seq) {
        const int mt = (job * p.ln_job_rows) / GEMM_BM;
        const long long l0 = p.dbg ? clock64() : 0;
        if (ctl) {
          // the control warp has acquired the rows at gpu scope and arrived on the slot's named barrier
          if (seq & 1) asm volatile("bar.sync 5, 160;" ::: "memory");
          else asm volatile("bar.sync 4, 160;" ::: "memory");
        } else {
          // one warp polls the counter, the other three sleep on a named barrier (bar.sync carries the acquired state over)
          if (lw == 0) wait_counter(L.src_done + mt, L.src_target);
          asm volatile("bar.sync 4, 128;" ::: "memory");
        }
        const long long l1 = p.dbg ? clock64() : 0;
        const int r0 = job * p.ln_job_rows + lw * ROWS_PER_WARP;
        const int r1 = min(r0 + ROWS_PER_WARP, p.M);
        switch (p.D) {
          case 384: chain_ln_rows<3>(p, L, r0, r1, lane); break;
          case 768: chain_ln_rows<6>(p, L, r0, r1, lane); break;
          case 1024: chain_ln_rows<8>(p, L, r0, r1, lane); break;
          default: chain_ln_rows<10>(p, L, r0, r1, lane); break;     // 1280
        }
        // one gpu-scope release per job and CTA (a gpu-scope fence on an SM with TMA traffic in flight is expensive):
        // the four warps meet on a named barrier (orders their row stores before the releasing thread), warp 10 publishes
        const long long l2 = p.dbg ? clock64() : 0;
        if (ctl) {
          __syncwarp();                                                // every lane's row stores precede the arrive
          if (lane == 0) mbar_arrive(&ln_done[seq & 1]);              // the control warp publishes the job
        } else {
          asm volatile("bar.sync 5, 128;" ::: "memory");
        }
        const long long l3 = p.dbg ? clock64() : 0;
        if (!ctl && lw == 0 && lane == 0) {
          fence_proxy_async_all();                                     // consumed by TMA loads (async proxy) of other SMs
          red_release_gpu_add(L.ready + mt, 1);
        }
        if (p.dbg && lw == 0 && lane == 0) {
          long long* d = p.dbg + (blockIdx.x * CHAIN_MAX_PHASES + 2 * s) * 12;
          const long long l4 = clock64();
          d[8] += l1 - l0; d[9] += l4 - l1; d[10] += 1;
          long long* e = d + 12;                                       // breakdown of the busy part, stored under the next phase's slots 8..10
          e[8] += l2 - l1; e[9] += l3 - l2; e[10] += l4 - l3;         // own rows (loads, statistics, stores) | wait for the other warps | publish
        }
      }
    }
  }

}

}  // namespace vpb
