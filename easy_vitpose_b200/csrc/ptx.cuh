// Inline-PTX building blocks for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the shared-memory descriptors wgmma
// consumes (the wgmma instructions themselves are in wgmma.cuh).
// Everything here is a thin wrapper over one PTX instruction; the kernels own the protocol.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vpb {

#ifndef VPB_HANG_TRAP_SPINS
#define VPB_HANG_TRAP_SPINS (1u << 26)   // a barrier that never flips traps instead of hanging the box
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a system-dependent time)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > VPB_HANG_TRAP_SPINS) __trap();
  }
}

// ---------------------------------------------------------------- proxies / fences
// generic-proxy smem writes -> visible to the async proxy (TMA stores, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load, box lands in smem (swizzled as the tensor map says), completion on `bar`.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 4-D variant (NHWC feature maps: channel, x, y, image); coordinates may lie outside the tensor (zero fill = conv padding).
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// smem tile -> global through the tensor map (rows / columns outside the tensor are clipped).
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
// global[tile] += smem tile, element type from the tensor map (f32): the add happens in L2, the SM never reads global.
__device__ __forceinline__ void tma_reduce_add_2d(const void* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- programmatic dependent launch
// Kernels are chained on one stream with cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs
// may be scheduled (and run their prologue: barrier init, descriptor prefetch) while the previous grid is still draining.
// pdl_wait() blocks until the previous grid has completed and its writes are visible; nothing that reads or writes global
// memory may precede it.  Without the launch attribute both are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// named barrier over `count` threads (a multiple of 32) of the CTA
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// shared-memory stores through 32-bit shared addresses
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_f32x2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// ---------------------------------------------------------------- per-warpgroup register budget
// Warpgroup-wide (.sync.aligned): all four warps of the warpgroup execute it with the same N (a multiple of 8 in [24, 256]).
// dec returns registers above N to the CTA's pool; inc blocks until the pool can raise every thread of the warpgroup to N.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------- wgmma shared-memory operand descriptor (sm_90)
//   [0,14) start address >> 4     [16,30) leading byte offset >> 4     [32,46) stride byte offset >> 4
//   [49,52) base offset (0: tiles 1024-byte aligned)                     [62,64) layout: 0 none, 1 SW128, 2 SW64, 3 SW32
// Operand tiles whose rows are W bytes wide (W = 128 / 64 / 32 = the swizzle span TMA wrote them with): 8-row groups are
// 8*W bytes apart (SBO); LBO is unused for these single-atom-wide tiles.  K-major: a K = 16 step is +32 bytes of the start
// address inside the swizzle atom.  MN-major (B = V of attention): a K = 16 step is 16 whole rows further.
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  static_assert(ROW_BYTES == 128 || ROW_BYTES == 64 || ROW_BYTES == 32, "swizzle span");
  constexpr uint64_t layout = ROW_BYTES == 128 ? 1 : ROW_BYTES == 64 ? 2 : 3;
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((8 * ROW_BYTES) >> 4) << 32;
  d |= layout << 62;
  return d;
}

// ---------------------------------------------------------------- small math / packing
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// max(v, 0) as torch's relu: NaN stays NaN (fmaxf(NaN, 0) = 0 would turn a corrupt activation into a plausible one).  max.NaN
// differs from the max.f32 of fmaxf only for a NaN operand, so every other input gives fmaxf's bits.  (`v != v ? v : fmaxf(v, 0)`
// gives the same values but cost 2 % of a ViT-B 64-crop step on an H100 80GB HBM3 at 700 W; max.NaN costs nothing measurable.)
__device__ __forceinline__ float relu_keep_nan(float v) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(v), "f"(0.0f));
  return r;
}
// erf to |err| <= 1.5e-7 (Abramowitz-Stegun 7.1.26): 1 rcp + 1 ex2 + 7 fma -- the outputs that use it are rounded
// to bf16 (eps 3.9e-3), so this is exact-erf GELU for every representable result.
__device__ __forceinline__ float erf_as(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * ax * -1.4426950408889634f));
  return copysignf(fmaf(-p * t, e, 1.0f), x);
}
// GELU(x) = x * Phi(x) with erf(z) evaluated as tanh(P(z)): 0.5 x (1 + tanh(x (c0 + c1 x^2 + c2 x^4))), coefficients
// fitted to the exact erf form on [-8, 8] (max |error| 2.5e-5 with an exact tanh; tools/fit_gelu.py) -- NOT the
// 0.044715 "tanh GELU".  c2 < 0, so the polynomial would change sign near |x| = 11.1 and flip the tanh: x^2 is clamped
// to 64, beyond which P(x^2) = P(64) = 1.726 > 0 and tanh(1.726 x) is +-1 to fp32 precision, i.e. GELU(x) = x or 0 exactly
// as the erf form gives there (tests/test_gelu_fit.py bounds the formula against erf over +-40).
// tanh.approx.f32 adds <= 2^-11 relative error.  8 instructions instead of ~18, one MUFU.
// The result is rounded to bf16 (relative step 2^-8) right after, which dominates both error terms.
__device__ __forceinline__ float gelu_tanh_fit(float x) {
  const float x2 = fminf(x * x, 64.0f);
  float p = fmaf(-3.51516782e-4f, x2, 3.70056460e-2f);
  p = fmaf(p, x2, 7.97507884e-1f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x * p));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}
// One lane of a fully converged warp.  Issue loops run WARP-UNIFORM (all 32 lanes execute the control flow, descriptors and
// addresses are the same in every lane) and only the TMA instruction itself is predicated on this: inside an
// `if (lane == 0)` branch the compiler cannot prove the operands uniform and may wrap every UTMALDG in an
// ELECT + R2UR.BROADCAST + BRA.U.ANY "waterfall" loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// warp-uniform copy of a value that is the same in every lane (e.g. loaded from shared memory)
__device__ __forceinline__ uint32_t uniform_u32(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 2^x for x <= 0 on the FMA / ALU pipes (no MUFU): round-to-nearest split x = i + f with the 1.5 * 2^23 magic constant, degree-3
// minimax polynomial for 2^f on [-0.5, 0.5] (max relative error 7.5e-5, tools-free fit by weighted least squares; bf16 keeps
// 2^-9 = 2e-3), exponent added into the float's bits.  ~10 instructions; used for a fraction of the softmax exponentials so
// that the MUFU (16 ex2 / clk / SM) is not the only pipe working.
// A NaN input returns NaN: the clamp would turn it into -125 and the exponent arithmetic into a finite weight, where the MUFU path
// (and torch's softmax) propagate it.  Every other input keeps its bits.
__device__ __forceinline__ float ex2_poly(float x) {
  if (x != x) return x;
  x = fmaxf(x, -125.0f);
  const float t = x + 12582912.0f;
  const float xi = t - 12582912.0f;
  const float f = x - xi;
  float p = fmaf(0.0551716499f, f, 0.242611125f);
  p = fmaf(p, f, 0.693260968f);
  p = fmaf(p, f, 0.999928057f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}

}  // namespace vpb
