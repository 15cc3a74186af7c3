// Fused multi-head attention for ViTPose crops: T = 192 tokens, head_dim 32 / 64 / 80 (ViT-S / B,L / H), on chip.
//
// Work unit = one item (crop b, head h).  The items of a launch are handed out statically (item = blockIdx.x + i * gridDim.x,
// one CTA per SM); Q, K, V of an item arrive by TMA as [192 x hd] boxes straight out of the qkv activation [M, 3D] into one of
// two smem stages, so the loads of item i + 1 run under the math of item i.  The 192 query rows are three warpgroups of 64:
//   S = Q K^T      wgmma m64n192k16, A = Q rows and B = K from smem (both K-major), fp32 logits in registers (96 per thread);
//   softmax        in registers: row max over the thread's 48 logits and its quad (the four lanes that share a row), then
//                  P = bf16(exp2(s log2e - max log2e)) and the row sum of those rounded weights; P never touches shared memory;
//   O = P V        wgmma m64nHDk16 with A = P from registers (the accumulator layout of S is the A-fragment layout, 16 keys per
//                  step) and B = V from smem as an MN-major operand, i.e. exactly the [token][dim] box TMA delivered;
//   epilogue       O / rowsum -> bf16 -> attn_out[b*192 + t, h*hd + d].
// Operand tiles: head_dim 64 -> one 128-byte-swizzled box per operand; 32 -> one 64-byte-swizzled box; 80 -> a 128B-swizzled
// box of 64 dims plus a 32B-swizzled box of the last 16 (Q K^T: 4+1 K steps; P V: an N = 64 and an N = 16 MMA per step).
#pragma once
#include <cuda.h>

#include "ptx.cuh"
#include "wgmma.cuh"

namespace vpb {

constexpr int ATT_T = 192;
constexpr int ATT_THREADS = 3 * 128;                          // three warpgroups x 64 query rows

template <int HD>
struct AttCfg {
  static_assert(HD == 32 || HD == 64 || HD == 80, "head_dim");
  static constexpr int MAIN = HD == 32 ? 32 : 64;             // dims in the main box
  static constexpr int TAIL = HD - MAIN;                      // 0 or 16 dims in the 32B-swizzled tail box
  static constexpr int MAIN_ROW = MAIN * 2;                   // bytes per row = swizzle span (128 or 64)
  static constexpr int MAIN_BYTES = ATT_T * MAIN_ROW;         // 24576 / 12288
  static constexpr int TAIL_BYTES = TAIL ? ATT_T * 32 : 0;    // 6144
  static constexpr int OPER_BYTES = MAIN_BYTES + TAIL_BYTES;  // one of Q / K / V
  static constexpr int STAGE_BYTES = 3 * OPER_BYTES;          // Q, K, V of one item
  static constexpr int SMEM = 2 * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(OPER_BYTES % 1024 == 0 && MAIN_BYTES % 1024 == 0, "swizzled boxes keep 1024-byte alignment");
};

struct AttnParams {
  int batch;              // crops
  int heads;
  int dim;                // D = heads * head_dim
  __nv_bfloat16* out;     // [batch*192, D]
  long long* dbg;         // debug: per CTA [8], zeroed by the caller, or nullptr.  Cycles of thread 0: 0 lifetime, 1 wait for
                          // operands, 2 the rest of the item loop, 3..6 the phases of attend_item; 7 items of this CTA
};

// Per-CTA cycle counters (debug): mark(slot) adds the cycles since the previous mark to dbg[slot] (this CTA's counters), counted
// by thread 0.  Every mark is a no-op when dbg is nullptr, which is how the engine launches.
struct PhaseClock {
  long long* dbg;
  uint32_t t;                                                 // SM clock at the previous mark (phases are far below 2^32 cycles)
  __device__ __forceinline__ explicit PhaseClock(long long* d) : dbg(d), t(0) {
    if (dbg) t = clock_u32();
  }
  __device__ __forceinline__ void mark(int slot) {
    if (dbg) {
      const uint32_t now = clock_u32();
      if (threadIdx.x == 0) dbg[slot] += now - t;
      t = now;
    }
  }
  static __device__ __forceinline__ uint32_t clock_u32() {
    uint32_t c;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(c));
    return c;
  }
};

// One item's attention for warpgroup wg (query rows 64 wg .. 64 wg + 63), from Q, K, V in shared memory laid out as the TMA
// boxes above (sQ, sK, sV: shared addresses of the three operands), into out[b*192 + t, head*hd + d] (row pitch dim).
// `operands_done` runs once this warpgroup's last MMA on the operands (O = P V) has retired, before the store.  `clk` counts the
// phases in slots 3 (S = Q K^T, issue to the last wait), 4 (softmax, up to the last P V step issued), 5 (P V, to its wait, with
// operands_done) and 6 (store).  Shared by attention_wgmma and qkv_attention_wgmma (qkv_attention.cuh).
//
// Each warpgroup pipelines its own work in two key halves (keys 0..95 and 96..191), so the tensor cores run one half while the
// warpgroup's FMA / MUFU work on the other: S of both halves is issued as two commit groups and the row max of the first runs
// under the MMAs of the second; the first half's P V steps are issued before the second half's exponentials are taken.  The
// result is bit-identical to computing S, then the whole softmax, then P V:
//   - fmaxf is exact and each row's max still runs over keys j = 0..23 (groups of 8) in the same order;
//   - each row's sum still adds e0 + e1 for j = 0..23 in order, and the quad shuffles come after the last one;
//   - every weight is computed from the same logit and the same max and rounded to bf16 once, round-to-nearest-even, as before
//     (a packed convert rounds each half as the single convert does, and the old re-pack of an exact bf16 value was a no-op);
//   - O accumulates the twelve 16-key steps in issue order 0..11 into the same registers;
//   - S of either half is the same MMA sum per element as one m64n192 chain (each element is one row of Q times one of K).
template <int HD, int NPOLY, typename OperandsDone>
__device__ __forceinline__ void attend_item(uint32_t sQ, uint32_t sK, uint32_t sV, __nv_bfloat16* out, int dim, int b, int head, int wg,
                                            int lane, int wq, PhaseClock& clk, OperandsDone&& operands_done) {
  using Cfg = AttCfg<HD>;
  static_assert(NPOLY == 0 || NPOLY == 8, "NPOLY");
  constexpr float kLog2e = 1.4426950408889634f;
  constexpr int KH = ATT_T / 2;                               // keys per half
  // ---- S = Q K^T for this warpgroup's 64 rows: s[half][4j + i] = column 96 half + 8j + ..., the m64n192 layout split in two
  float s[2][KH / 2];
  wgmma_fence();
  {
    const uint64_t qd = wgmma_desc<Cfg::MAIN_ROW>(sQ + wg * 64 * Cfg::MAIN_ROW);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const uint64_t kd = wgmma_desc<Cfg::MAIN_ROW>(sK + half * KH * Cfg::MAIN_ROW);   // 96 rows in: a multiple of 1024 bytes
#pragma unroll
      for (int k = 0; k < Cfg::MAIN / 16; ++k) wgmma_ss<KH>(s[half], qd + 2 * k, kd + 2 * k, k != 0);   // +32 B per K = 16 step
      if constexpr (Cfg::TAIL > 0)
        wgmma_ss<KH>(s[half], wgmma_desc<32>(sQ + Cfg::MAIN_BYTES + wg * 64 * 32), wgmma_desc<32>(sK + Cfg::MAIN_BYTES + half * KH * 32), 1);
      wgmma_commit();
    }
  }

  // ---- row max: thread rows r_lo (h = 0: s[.][4j], s[.][4j+1]) and r_lo + 8 (h = 1: s[.][4j+2], s[.][4j+3]); a row lives in
  // one quad.  Keys 0..95 while the MMAs of 96..191 still run
  float mx[2] = {-INFINITY, -INFINITY};
  wgmma_wait<1>();
  wgmma_fence_regs(s[0]);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    if (half == 1) {
      wgmma_wait<0>();
      wgmma_fence_regs(s[1]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < KH / 8; ++j) mx[h] = fmaxf(mx[h], fmaxf(s[half][4 * j + 2 * h], s[half][4 * j + 2 * h + 1]));
  }
  clk.mark(3);
  float mscaled[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    mscaled[h] = mx[h] * kLog2e;
  }

  // ---- per half: the weights, then its six P V steps of 16 keys (P as bf16 A fragments, V MN-major).  P is rounded to bf16
  // here, and the row sum is taken over the ROUNDED weights that O = P V actually uses: the normalised weights then sum to 1 up
  // to fp32 round-off instead of carrying a per-row scale error of up to 2^-9.  Each pair of weights is rounded by one packed
  // convert (F2FP, on the ALU pipe) whose word is the A-fragment register itself, and read back for the sum by two integer ops:
  // single converts (F2F) share the MUFU's 16 / clk / SM with the exponentials and took as many slots as they did.
  // pk[2j + h] = bf16x2 of s[half][4j + 2h], s[half][4j + 2h + 1], so the A fragment of step kh is pk[4kh .. 4kh + 3]
  float sum[2] = {0.0f, 0.0f};
  float o[Cfg::MAIN / 2];
  [[maybe_unused]] float ot[8];
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    // the second half's exponentials start after the first half's P V steps are issued
    if (half == 1) wgmma_fence_regs(s[1]);
    uint32_t pk[KH / 4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int jj = 0; jj < KH / 8; ++jj) {
        const int j = half * (KH / 8) + jj;                   // key group over the whole row (the poly pattern)
        const float a1 = fmaf(s[half][4 * jj + 2 * h + 1], kLog2e, -mscaled[h]);
        const float x0 = ex2_approx(fmaf(s[half][4 * jj + 2 * h], kLog2e, -mscaled[h]));
        const float x1 = (NPOLY > 0 && (j & 1) == 0) ? ex2_poly(a1) : ex2_approx(a1);
        const uint32_t w = pack_bf16(x0, x1);
        sum[h] += __uint_as_float(w << 16) + __uint_as_float(w & 0xffff0000u);
        pk[2 * jj + h] = w;
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kh = 0; kh < KH / 16; ++kh) {
      const int kk = half * (KH / 16) + kh;                   // 16-key step over the whole row
      const uint32_t a[4] = {pk[4 * kh], pk[4 * kh + 1], pk[4 * kh + 2], pk[4 * kh + 3]};
      const uint64_t vd = wgmma_desc<Cfg::MAIN_ROW>(sV + kk * 16 * Cfg::MAIN_ROW);
      if constexpr (Cfg::MAIN == 64) wgmma_rs_n64<1>(o, a, vd, kk != 0);
      else wgmma_rs_n32<1>(o, a, vd, kk != 0);
      if constexpr (Cfg::TAIL > 0) wgmma_rs_n16<1>(ot, a, wgmma_desc<32>(sV + Cfg::MAIN_BYTES + kk * 16 * 32), kk != 0);
    }
    wgmma_commit();
  }
  clk.mark(4);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
  }
  wgmma_wait<0>();
  wgmma_fence_regs(o);
  if constexpr (Cfg::TAIL > 0) wgmma_fence_regs(ot);

  operands_done();
  clk.mark(5);

  // ---- O / rowsum -> bf16 -> attn_out
  const int r_lo = wg * 64 + wq * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float inv = 1.0f / sum[hh];
    __nv_bfloat16* orow = out + (static_cast<size_t>(b) * ATT_T + r_lo + 8 * hh) * dim + head * HD;
#pragma unroll
    for (int j = 0; j < Cfg::MAIN / 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + 8 * j + cq) = pack_bf16(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
    if constexpr (Cfg::TAIL > 0) {
#pragma unroll
      for (int j = 0; j < 2; ++j)
        *reinterpret_cast<uint32_t*>(orow + Cfg::MAIN + 8 * j + cq) = pack_bf16(ot[4 * j + 2 * hh] * inv, ot[4 * j + 2 * hh + 1] * inv);
    }
  }
  clk.mark(6);
}

// tmap_main: box [192 rows x MAIN cols] (swizzle = MAIN*2 bytes); tmap_tail: box [192 x 16] (32B swizzle), hd 80 only.
// NPOLY of every 32 exponentials go through ex2_poly (FMA pipe) instead of the MUFU: 0 (all MUFU) or 8 (every 4th)
template <int HD, int NPOLY = 0>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_wgmma(const __grid_constant__ CUtensorMap tmap_main, const __grid_constant__ CUtensorMap tmap_tail, const AttnParams p) {
  using Cfg = AttCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * Cfg::STAGE_BYTES);    // [2] Q, K, V of a stage landed

  const int wg = threadIdx.x >> 7;                            // query rows 64 wg .. 64 wg + 63
  const int tid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31, wq = tid >> 5;
  const int items = p.batch * p.heads;
  const long long t_cta0 = p.dbg ? clock64() : 0;
  PhaseClock clk(p.dbg ? p.dbg + blockIdx.x * 8 : nullptr);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_main);
    if constexpr (Cfg::TAIL > 0) tma_prefetch_desc(&tmap_tail);
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                                                 // qkv from the previous GEMM is complete

  auto oper = [&](int q, int o) { return smem + q * Cfg::STAGE_BYTES + o * Cfg::OPER_BYTES; };
  auto load_item = [&](int item, int q) {                     // thread 0 only
    const int b = item / p.heads, h = item % p.heads;
    mbar_expect_tx(&full[q], Cfg::STAGE_BYTES);
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      tma_load_2d(oper(q, o), &tmap_main, &full[q], o * p.dim + h * HD, b * ATT_T);
      if constexpr (Cfg::TAIL > 0) tma_load_2d(oper(q, o) + Cfg::MAIN_BYTES, &tmap_tail, &full[q], o * p.dim + h * HD + Cfg::MAIN, b * ATT_T);
    }
  };
  if (threadIdx.x == 0) {
    if (static_cast<int>(blockIdx.x) < items) load_item(blockIdx.x, 0);
    if (static_cast<int>(blockIdx.x + gridDim.x) < items) load_item(blockIdx.x + gridDim.x, 1);
  }

  int li = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x, ++li) {
    const int q = li & 1;
    clk.mark(2);
    mbar_wait(&full[q], (li >> 1) & 1);
    clk.mark(1);
    const uint32_t sQ = smem_u32(oper(q, 0)), sK = smem_u32(oper(q, 1)), sV = smem_u32(oper(q, 2));

    attend_item<HD, NPOLY>(sQ, sK, sV, p.out, p.dim, item / p.heads, item % p.heads, wg, lane, wq, clk, [&] {
      // every warpgroup is done with this stage's operands: thread 0 refills it with the item after next
      __syncthreads();
      if (threadIdx.x == 0 && item + 2 * static_cast<int>(gridDim.x) < items) load_item(item + 2 * gridDim.x, q);
    });
  }
  if (p.dbg && threadIdx.x == 0) { p.dbg[blockIdx.x * 8 + 0] = clock64() - t_cta0; p.dbg[blockIdx.x * 8 + 7] = li; }
}

}  // namespace vpb
