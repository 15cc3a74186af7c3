// qkv GEMM and attention in one launch: each item (crop b, head h) computes its own q, k and v on chip and attends over them,
// so the [batch*192, 3D] qkv activation never goes through L2 / HBM.
//
//   GEMM phase   C[192, 3 hd] = xn[192 b .. 192 b + 191, :] * [Wq_h; Wk_h; Wv_h]^T.  Warpgroup wg owns token rows 64 wg .. 64 wg
//                + 63 and issues wgmma m64n(3 hd)k16 (n96 / n192 / n240 at head_dim 32 / 64 / 80).  Operands come through a TMA
//                ring of k-blocks: a [192 x 64] box of xn and three [hd x 64] boxes of the packed qkv weight (rows h hd, D + h hd,
//                2D + h hd), 128B-swizzled, which together form the K-major [3 hd x 64] B tile.  The ring runs on across items
//                (as in gemm.cuh), so the next item's first k-blocks land while this item attends.
//   hand-off     acc + bias -> bf16 (exactly EPI_BF16's pack_bf16(acc + bias)), stored to shared memory in the byte layout the
//                attention kernel's TMA boxes have (attention.cuh: 128B swizzle at head_dim 64, 64B at 32, a 128B box of 64 dims
//                plus a 32B box of 16 at 80) for Q, K and V alike.
//   attention    attend_item (attention.cuh), the very code attention_wgmma runs.
//
// Every output element of the GEMM accumulates in k order as in the standalone GEMM, the rounding is the same and the attention
// is the same code, so the result is bit-identical to gemm_bf16_wgmma<BN, EPI_BF16> followed by attention_wgmma.
// 384 threads (the three consumer warpgroups, up to 168 registers each); thread 0 also issues the ring's loads, refilling a
// slot as soon as every warp has released it (empty barrier, one arrival per warp).
#pragma once
#include <cuda.h>

#include "attention.cuh"
#include "gemm.cuh"

namespace vpb {

template <int HD>
struct QkvAttCfg {
  using Att = AttCfg<HD>;
  static constexpr int N = 3 * HD;                            // q | k | v columns of one head
  static constexpr int A_BYTES = ATT_T * GEMM_BK * 2;         // 24576: 192 rows of xn x 64
  static constexpr int W_BYTES = HD * GEMM_BK * 2;            // one of Wq_h, Wk_h, Wv_h x 64
  static constexpr int STAGE_BYTES = A_BYTES + 3 * W_BYTES;
  static constexpr int HAND_BYTES = 3 * Att::OPER_BYTES;      // Q, K, V of the item being attended
  static constexpr int STAGES_RAW = (227 * 1024 - 1024 /*align*/ - 256 /*barriers*/ - HAND_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;   // 5 / 3 / 2 at head_dim 32 / 64 / 80
  static constexpr int SMEM = HAND_BYTES + STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(W_BYTES % 1024 == 0, "W boxes keep the 1024-byte alignment of the swizzle atoms");
  static_assert(STAGES >= 2, "ring too shallow");
};

struct QkvAttnParams {
  int batch;              // crops
  int heads;
  int dim;                // D = heads * head_dim = K of the GEMM (a multiple of 64)
  const float* bias;      // packed qkv bias [3D] (q rows carry head_dim^-0.5 like the weight)
  __nv_bfloat16* out;     // [batch*192, D]
  long long* dbg;         // debug: per CTA [8], zeroed by the caller, or nullptr.  Cycles of thread 0: 0 GEMM phase, 1 of which
                          // waiting on the ring's full barriers, 2 hand-off (both CTA barriers), 3..6 the phases of attend_item
                          // (attention.cuh); 7 items of this CTA
};

// Producer side (thread 0): load the next `count` k-blocks of the CTA's sequence (item ld_item from k-block ld_kb on, items
// blockIdx.x, + gridDim.x, ...), each into the ring slot at `lp` once every warp has released it.
template <int HD>
__device__ __forceinline__ void qkv_att_produce(int count, uint8_t* ring, uint64_t* full, uint64_t* empty, RingPos& lp, int& ld_item,
                                                int& ld_kb, int items, int num_kb, const QkvAttnParams& p, const CUtensorMap* tmap_x,
                                                const CUtensorMap* tmap_w) {
  using Cfg = QkvAttCfg<HD>;
  for (; count > 0 && ld_item < items; --count) {
    ring_wait_slot(empty, lp);
    uint8_t* st = ring + lp.stage * Cfg::STAGE_BYTES;
    const int b = ld_item / p.heads, h = ld_item % p.heads;
    mbar_expect_tx(&full[lp.stage], Cfg::STAGE_BYTES);
    tma_load_2d(st, tmap_x, &full[lp.stage], ld_kb * GEMM_BK, b * ATT_T);
#pragma unroll
    for (int o = 0; o < 3; ++o) tma_load_2d(st + Cfg::A_BYTES + o * Cfg::W_BYTES, tmap_w, &full[lp.stage], ld_kb * GEMM_BK, o * p.dim + h * HD);
    lp.next(Cfg::STAGES);
    if (++ld_kb == num_kb) { ld_kb = 0; ld_item += gridDim.x; }
  }
}

// tmap_x: xn [M, D], boxes [192 rows x 64], 128B swizzle.  tmap_w: packed qkv weight [3D, D], boxes [hd rows x 64], 128B swizzle.
template <int HD, int NPOLY = 0>
__global__ void __launch_bounds__(ATT_THREADS, 1)
qkv_attention_wgmma(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w, const QkvAttnParams p) {
  using Cfg = QkvAttCfg<HD>;
  using Att = AttCfg<HD>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem + Cfg::HAND_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31, wq = tid >> 5;
  const int items = p.batch * p.heads;
  const int num_kb = p.dim / GEMM_BK;
  PhaseClock clk(p.dbg ? p.dbg + blockIdx.x * 8 : nullptr);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], ATT_THREADS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                                                 // xn from the previous kernel is complete

  // ---- producer (thread 0): the k-blocks of this CTA's items in order; ld_item / ld_kb = the next one to load
  int ld_item = blockIdx.x, ld_kb = 0;
  RingPos lp;
  auto produce = [&](int count) {
    qkv_att_produce<HD>(count, ring, full, empty, lp, ld_item, ld_kb, items, num_kb, p, &tmap_x, &tmap_w);
  };
  if (threadIdx.x == 0) produce(STAGES);

  const uint32_t sQ = smem_u32(smem), sK = sQ + Att::OPER_BYTES, sV = sQ + 2 * Att::OPER_BYTES;
  RingPos rp;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int b = item / p.heads, h = item % p.heads;

    // ---- GEMM phase: acc = xn rows of crop b (this warpgroup's 64) x [Wq_h; Wk_h; Wv_h]^T
    // The first MMA ignores acc (scale-d = 0), but its asm operands read it: zeroing keeps the previous item's values from
    // looking live across the attention phase, where they would be spilled
    float acc[Cfg::N / 2];
#pragma unroll
    for (int i = 0; i < Cfg::N / 2; ++i) acc[i] = 0.0f;
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      const long long w0 = p.dbg ? clock64() : 0;
      mbar_wait(&full[rp.stage], rp.phase);
      if (p.dbg && threadIdx.x == 0) p.dbg[blockIdx.x * 8 + 1] += clock64() - w0;
      const uint32_t sa = smem_u32(ring + rp.stage * Cfg::STAGE_BYTES) + wg * 64 * 128;
      const uint32_t sb = smem_u32(ring + rp.stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
      const uint64_t ad = wgmma_desc<128>(sa), bd = wgmma_desc<128>(sb);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<Cfg::N>(acc, ad + 2 * k, bd + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                                        // k-block kb-1 has retired: release its slot
      if (prev >= 0) {
        if (lane == 0) mbar_arrive(&empty[prev]);
        if (threadIdx.x == 0) produce(1);
        __syncwarp();
      }
      prev = rp.stage;
      rp.next(STAGES);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (lane == 0) mbar_arrive(&empty[prev]);
    clk.mark(0);

    // every warpgroup is done with the previous item's Q, K, V and with this item's last ring slot
    __syncthreads();
    if (threadIdx.x == 0) produce(1);

    // ---- hand-off: bias, bf16, and the swizzled byte layout of the attention kernel's TMA boxes.  Column group j of the
    // accumulator (8 columns) is dims 8 (j % (hd/8)) .. + 7 of operand j / (hd/8) (q, k, v)
    {
      const int r_lo = wg * 64 + wq * 16 + (lane >> 2);      // rows r_lo and r_lo + 8 share every swizzle phase below
      const int cq = 2 * (lane & 3);
      const uint32_t main_off = r_lo * Att::MAIN_ROW + (lane & 3) * 4;
      const int main_sw = Att::MAIN_ROW == 128 ? (r_lo & 7) : ((r_lo >> 1) & 3);   // 128B / 64B swizzle of row r_lo
      const uint32_t tail_off = Att::MAIN_BYTES + r_lo * 32 + (lane & 3) * 4;
      const int tail_sw = (r_lo >> 2) & 1;                    // 32B swizzle
#pragma unroll
      for (int j = 0; j < Cfg::N / 8; ++j) {
        const int o = j / (HD / 8), c = (j % (HD / 8)) * 8;   // operand, first dim of the group
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias + o * p.dim + h * HD + c + cq));
        const uint32_t lo = pack_bf16(acc[4 * j] + b2.x, acc[4 * j + 1] + b2.y);
        const uint32_t hi = pack_bf16(acc[4 * j + 2] + b2.x, acc[4 * j + 3] + b2.y);
        uint32_t a;
        int row_bytes;
        if (c < Att::MAIN) { a = sQ + o * Att::OPER_BYTES + main_off + (((c >> 3) ^ main_sw) << 4); row_bytes = Att::MAIN_ROW; }
        else { a = sQ + o * Att::OPER_BYTES + tail_off + ((((c - Att::MAIN) >> 3) ^ tail_sw) << 4); row_bytes = 32; }
        sts_u32(a, lo);
        sts_u32(a + 8 * row_bytes, hi);
      }
    }
    fence_proxy_async_smem();                                 // the stores -> visible to wgmma's operand reads
    __syncthreads();
    clk.mark(2);

    // ---- attention over the item's Q, K, V; the barrier above the next hand-off keeps them until every warpgroup is done
    attend_item<HD, NPOLY>(sQ, sK, sV, p.out, p.dim, b, h, wg, lane, wq, clk, [] {});
  }
  if (p.dbg && threadIdx.x == 0) p.dbg[blockIdx.x * 8 + 7] = (items - 1 - blockIdx.x) / gridDim.x + 1;
}

}  // namespace vpb
