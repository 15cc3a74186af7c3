// libvitpose_b200.so: the engine object behind include/vitpose_b200.h.
// Owns the packed weights, the activation workspace and the TMA tensor maps; enqueues the kernel chain
//   patch_im2col -> GEMM(+pos) -> depth x [LN -> GEMM qkv -> attention -> GEMM proj(+res) -> LN -> GEMM fc1(GELU)
//   -> GEMM fc2(+res)] -> LN -> 2 x [phase im2col -> 4 GEMM(BN+ReLU)] -> GEMM 1x1 (NCHW heatmaps) -> decode
// on the caller's stream.  No host synchronisation on the hot path, no CPU fallback.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/vitpose_b200.h"
#include "attention.cuh"
#include "chain.cuh"
#include "decode.cuh"
#include "draw.cuh"
#include "expert_gemm.cuh"
#include "gemm.cuh"
#include "pointwise.cuh"
#include "preprocess.cuh"
#include "oks_nms.cuh"
#include "coco_eval.cuh"
#include "qkv_attention.cuh"
#include "smooth.cuh"
#include "track.cuh"

using namespace vpb;

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CU_TRY(expr)                                                                                  \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return fail(VPB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)
#define VPB_TRY(expr)            \
  do {                           \
    int _r = (expr);             \
    if (_r != VPB_OK) return _r; \
  } while (0)

extern "C" const char* vpb_last_error(void) { return g_err; }

// ------------------------------------------------------------------------------------------------ TMA maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static int load_driver_api() {
  if (g_encode) return VPB_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CU_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || fn == nullptr) return fail(VPB_ERR_CUDA, "cuTensorMapEncodeTiled not available");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return VPB_OK;
}
// Row-major [rows, cols] tensor with row pitch `ld` elements; box = [box_rows, 128 bytes of columns], 128B-swizzled.
// bf16: 64 columns per box (GEMM operands, bf16 outputs); f32: 32 columns per box (the fp32 residual stream).
// `span` = bytes of one box row = swizzle span (128 default; 64 / 32 for the narrow attention operand boxes).
static int make_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, bool f32 = false,
                    uint32_t span = 128) {
  VPB_TRY(load_driver_api());
  const uint64_t esz = f32 ? 4 : 2;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * esz};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(span / esz), box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = span == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : span == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = g_encode(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VPB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box=%u", (int)r,
                                     (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows);
  return VPB_OK;
}

// bf16 NHWC feature map [B,H,W,C] as a 4-D tensor (C, W, H, B); box = 64 channels x box_w x box_h positions x 1 image, 128B-swizzled:
// the A operand of the implicit-GEMM deconv (shifted boxes, zero fill outside the map).
static int make_map_nhwc(CUtensorMap* m, const void* base, uint64_t B, uint64_t H, uint64_t W, uint64_t C, uint32_t box_h, uint32_t box_w) {
  VPB_TRY(load_driver_api());
  cuuint64_t dims[4] = {C, W, H, B};
  cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
  cuuint32_t box[4] = {64, box_w, box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VPB_ERR_CUDA, "cuTensorMapEncodeTiled(4d) failed (%d) B=%llu H=%llu W=%llu C=%llu", (int)r,
                                     (unsigned long long)B, (unsigned long long)H, (unsigned long long)W, (unsigned long long)C);
  return VPB_OK;
}

static int g_dbg_stages = 0, g_dbg_flags = 0;      // debug knobs set by vpb_debug_gemm
static long long* g_dbg_buf = nullptr;

// Residual epilogues (patch embed, proj, fc2: x += acc + bias): 1 = load + add + TMA store (gemm.cuh: epilogue_f32_rmw), 0 = TMA
// reduce-add.  Bit-identical; process default from VPB_RESID_RMW, per engine through option "resid_rmw"; the debug flags 32 / 64
// of vpb_debug_gemm force one form for every following launch (kernel-level tests).
constexpr int kResidRmwDefault = 0;
constexpr int kLnCtlDefault = 1;      // bit-identical either way (tests/test_gpu_engine.py)
// Largest L2 access-policy window (and persisting set-aside) over the fp32 token stream x.  The H100 lets 32 MB of its 50 MB L2
// persist; with all of it held for x, the LayerNorms' bf16 outputs and the GEMMs' operands and outputs share the 18 MB left.  A
// 24 MB window keeps most of x resident and leaves them 26 MB.  bench.py on an H100 80GB HBM3 (700 W power limit), ms per step,
// window of 32 MB (the device limit) / 28 / 24 / 20 / 16 MB: b17x64 5.32 / 5.15 / 5.09-5.12 / 5.13 / 5.16; l25x64 16.30 / - /
// 15.44 / 15.53; h133x32 18.16 / - / 16.41 / 16.45; ap10k-streams (x is 18.9 MB, under the cap) 17.80 / - / 17.78 / 17.76.
// At b17x64 the LayerNorms went from 0.72 to 0.58 ms per step and fc1 from 1.50 to 1.29; qkv, proj and fc2 gave back 0.07.
// Where the window lies changes no result.
constexpr size_t kL2PersistMax = size_t(24) << 20;
static int resid_rmw_default() {
  static const int v = [] { const char* s = getenv("VPB_RESID_RMW"); return s ? (s[0] != '0') : kResidRmwDefault; }();
  return v;
}
static int resid_rmw(int engine_choice) { return (g_dbg_flags & 32) ? 1 : (g_dbg_flags & 64) ? 0 : engine_choice; }

// ------------------------------------------------------------------------------------------------ launches
// Every kernel of the chain is launched with programmatic stream serialization (see ptx.cuh: pdl_wait).
static bool g_pdl = true;
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// ------------------------------------------------------------------------------------------------ per-device state
// cudaFuncSetAttribute (dynamic smem above 48 KB) applies to the CURRENT device's context and the SM count sizes every
// persistent grid, so both are tracked per device: engines on different GPUs of one process each set their own.
constexpr int kMaxDevices = 64;
struct DeviceState {
  int sms = 0;                      // 0 = not checked yet
  bool attn_attr = false;
  unsigned gemm_attr = 0;           // bit per gemm instantiation (see gemm_slot)
  unsigned expert_attr = 0;         // bit per expert GEMM tile width (expert_launch)
};
static DeviceState g_devs[kMaxDevices];
static DeviceState* cur_dev() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= kMaxDevices) d = 0;
  return &g_devs[d];
}
static int num_sms() { return cur_dev()->sms; }

// ------------------------------------------------------------------------------------------------ GEMM dispatch

// Bit of DeviceState::gemm_attr for an instantiation: five tile widths per epilogue (EPI_BF16_GELU_ERF takes the unused index 3).
constexpr int gemm_slot(int bn, int epi) {
  return (epi == EPI_BF16_GELU_ERF ? 3 : epi) * 5 + (bn == 256 ? 0 : bn == 128 ? 1 : bn == 144 ? 2 : bn == 32 ? 3 : 4);
}
static_assert(gemm_slot(192, EPI_F32_ADD) < 32, "gemm_attr has 32 bits");

// `tout` is the output tensor map of the TMA epilogues (EPI_BF16, EPI_BF16_GELU: bf16 box 64 columns x 64 rows; EPI_F32_ADD:
// f32 box 32 x 64); direct epilogues ignore it (pass any valid map).  W maps carry boxes of BN rows.
template <int BN, int EPI>
static int gemm_launch_t(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tout, const GemmParams& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN, EPI>;
  auto kern = gemm_bf16_wgmma<BN, EPI>;
  DeviceState* ds = cur_dev();
  if (ds->sms == 0) return fail(VPB_ERR_STATE, "gemm: device not initialised (device_check)");
  constexpr unsigned slot = 1u << gemm_slot(BN, EPI);
  if (!(ds->gemm_attr & slot)) {
    CU_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    ds->gemm_attr |= slot;
  }
  const bool deconv = (EPI == EPI_BF16_RELU_UP);
  const int num_m = deconv ? p.M / (p.up_tr * p.up_tw) : (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles = num_m * (deconv ? 4 : (p.N + BN - 1) / BN);
  const int grid = tiles < ds->sms ? tiles : ds->sms;
  CU_TRY(launch_k(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, st, ta, tw, tout, p));
  return VPB_OK;
}
static int gemm_launch(int bn, int epi, const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tout, const GemmParams& p,
                       cudaStream_t st) {
  if (p.K % GEMM_BK != 0 || p.K <= 0) return fail(VPB_ERR_ARG, "gemm: K=%d must be a positive multiple of 64", p.K);
  // the fp32 epilogue stores 32 columns per TMA box (the shared columns of a ViTPose+ fc2 are D - P wide, P % 32 == 0)
  if (epi_uses_tma(epi) && (p.N % (epi == EPI_F32_ADD ? 32 : 64) != 0 || p.bias == nullptr))
    return fail(VPB_ERR_ARG, "gemm: TMA epilogue wants N %% 64 == 0 (N %% 32 == 0 for the fp32 one) and a bias");
#define VPB_CASE(BN_, EPI_) \
  if (bn == BN_ && epi == EPI_) return gemm_launch_t<BN_, EPI_>(ta, tw, tout, p, st);
  VPB_CASE(256, EPI_BF16) VPB_CASE(192, EPI_BF16) VPB_CASE(128, EPI_BF16)
  VPB_CASE(256, EPI_BF16_GELU) VPB_CASE(192, EPI_BF16_GELU) VPB_CASE(128, EPI_BF16_GELU)
  VPB_CASE(256, EPI_BF16_GELU_ERF) VPB_CASE(192, EPI_BF16_GELU_ERF) VPB_CASE(128, EPI_BF16_GELU_ERF)
  VPB_CASE(256, EPI_F32_ADD) VPB_CASE(192, EPI_F32_ADD) VPB_CASE(128, EPI_F32_ADD)
  VPB_CASE(256, EPI_BF16_RELU_UP)
  VPB_CASE(32, EPI_F32_NCHW) VPB_CASE(144, EPI_F32_NCHW)
#undef VPB_CASE
  return fail(VPB_ERR_ARG, "gemm: no kernel for BN=%d epilogue=%d", bn, epi);
}

// Grouped expert GEMM (expert_gemm.cuh).  Tile width: the widest of kExpertWidths that divides P, so no tile reads columns of
// the next expert; `tw` carries W boxes of that many rows.
constexpr int kExpertWidths[5] = {192, 128, 96, 64, 32};
static int expert_width(int P) {
  for (int w : kExpertWidths)
    if (P % w == 0) return w;
  return 0;
}
template <int BN>
static int expert_launch_t(const CUtensorMap& ta, const CUtensorMap& tw, const ExpertParams& p, cudaStream_t st) {
  using Cfg = TileCfg<BN, false>;
  auto kern = gemm_expert_segments<BN>;
  DeviceState* ds = cur_dev();
  if (ds->sms == 0) return fail(VPB_ERR_STATE, "expert gemm: device not initialised (device_check)");
  constexpr unsigned slot = 1u << (BN / 32);
  if (!(ds->expert_attr & slot)) {
    CU_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    ds->expert_attr |= slot;
  }
  const int grid = p.num_tiles < ds->sms ? p.num_tiles : ds->sms;
  CU_TRY(launch_k(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, st, ta, tw, p));
  return VPB_OK;
}
static int expert_launch(int bn, const CUtensorMap& ta, const CUtensorMap& tw, const ExpertParams& p, cudaStream_t st) {
  if (p.K % GEMM_BK != 0 || p.K <= 0 || p.num_segs < 1 || p.num_segs > EXPERT_MAX_SEGMENTS || bn <= 0 || p.P % bn != 0)
    return fail(VPB_ERR_ARG, "expert gemm: K=%d P=%d BN=%d segments=%d", p.K, p.P, bn, p.num_segs);
  switch (bn) {
    case 192: return expert_launch_t<192>(ta, tw, p, st);
    case 128: return expert_launch_t<128>(ta, tw, p, st);
    case 96: return expert_launch_t<96>(ta, tw, p, st);
    case 64: return expert_launch_t<64>(ta, tw, p, st);
    case 32: return expert_launch_t<32>(ta, tw, p, st);
  }
  return fail(VPB_ERR_ARG, "expert gemm: no kernel for BN=%d", bn);
}

// `device` must be the current device (callers cudaSetDevice / cudaGetDevice first)
static int device_check(int device) {
  if (device < 0 || device >= kMaxDevices) return fail(VPB_ERR_ARG, "device %d out of range", device);
  DeviceState* ds = &g_devs[device];
  if (ds->sms > 0 && ds->attn_attr) return VPB_OK;
  cudaDeviceProp prop;
  CU_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(VPB_ERR_ARG, "device %d is sm_%d%d; this library only runs on sm_90 (H100), no fallback", device,
                                    prop.major, prop.minor);
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<32>::SMEM));
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<64>::SMEM));
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<80>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<80>::SMEM));
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<32, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<32>::SMEM));
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<64, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<64>::SMEM));
  CU_TRY(cudaFuncSetAttribute(attention_wgmma<80, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttCfg<80>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<32>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<64>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<80>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<80>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<32, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<32>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<64, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<64>::SMEM));
  CU_TRY(cudaFuncSetAttribute(qkv_attention_wgmma<80, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, QkvAttCfg<80>::SMEM));
  ds->attn_attr = true;
  ds->sms = prop.multiProcessorCount;
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------ chained GEMM launch
template <int BN>
static int chain_launch_t(const ChainMaps& maps, const ChainParams& p, cudaStream_t st) {
  using Cfg = ChainCfg<BN>;
  auto kern = gemm_chain_wgmma<BN>;
  DeviceState* ds = cur_dev();
  if (ds->sms == 0) return fail(VPB_ERR_STATE, "chain: device not initialised (device_check)");
  constexpr unsigned slot = BN == 256 ? (1u << 30) : (1u << 31);
  if (!(ds->gemm_attr & slot)) {
    CU_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    ds->gemm_attr |= slot;
  }
  const int num_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  int tiles = 0;
  for (int i = 0; i < p.num_phases; ++i) {
    if (p.ph[i].N % BN != 0 || p.ph[i].K % GEMM_BK != 0 || p.ph[i].bias == nullptr)
      return fail(VPB_ERR_ARG, "chain: phase %d N=%d K=%d does not tile by %d x 64", i, p.ph[i].N, p.ph[i].K, BN);
    tiles += num_m * (p.ph[i].N / BN);
  }
  // every CTA of the grid must be resident at once: the in-kernel waits rely on it.  Ask the runtime how many CTAs of this
  // kernel an SM can hold instead of assuming one.
  static int max_active[kMaxDevices] = {0};
  int dev_id = 0;
  CU_TRY(cudaGetDevice(&dev_id));
  if (max_active[dev_id] == 0) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, CHAIN_THREADS, Cfg::SMEM_BYTES) != cudaSuccess || n < 1) { cudaGetLastError(); n = 1; }
    max_active[dev_id] = n * ds->sms;
  }
  const int grid = tiles < max_active[dev_id] ? tiles : max_active[dev_id];
  CU_TRY(launch_k(kern, dim3(grid), dim3(CHAIN_THREADS), Cfg::SMEM_BYTES, st, maps, p));
  return VPB_OK;
}
static int chain_launch(int bn, const ChainMaps& maps, const ChainParams& p, cudaStream_t st) {
  if (p.num_phases < 1 || p.num_phases > CHAIN_MAX_PHASES || p.num_ln < 0 || p.num_ln > CHAIN_MAX_LN) return fail(VPB_ERR_ARG, "chain: bad phase count");
  if (p.D != 384 && p.D != 768 && p.D != 1024 && p.D != 1280) return fail(VPB_ERR_ARG, "chain: LayerNorm width %d not instantiated", p.D);
  if (bn != 128) return fail(VPB_ERR_ARG, "chain: tile width %d not built (128)", bn);
  return chain_launch_t<128>(maps, p, st);
}

// ------------------------------------------------------------------------------------------------ attention dispatch
// Attention variant (process-wide switch; environment at load time, or vpb_debug_attention() for A/B runs in one process):
//   poly  every 4th softmax exponential on the FMA pipe (ex2_poly, 7.5e-5 relative error, far below P's bf16 rounding) instead
//         of the MUFU.  Default OFF; VPB_ATT_POLY=1 switches it on.
static int g_att_poly = [] { const char* e = getenv("VPB_ATT_POLY"); return (e && e[0] == '1') ? 1 : 0; }();
static const int g_att_poly_env = g_att_poly;
static int g_att_grid_cap = 0;      // tests: launch the attention kernels with at most this many CTAs (0 = one per SM)
static int g_att_form = 0;          // tests / A/B: 0 = fuse qkv + attention by the rule (fuse_qkv_attention), 1 = always, 2 = never
// flags < 0: back to the defaults (environment); else bit 0 = poly, bit 1 = force the fused qkv + attention launch, bit 2 = force
// the qkv GEMM + attention pair, bits 8.. = grid cap (how a device with fewer SMs would split the items)
extern "C" int vpb_debug_attention(int32_t flags) {
  if (flags < 0) { g_att_poly = g_att_poly_env; g_att_grid_cap = 0; g_att_form = 0; }
  else { g_att_poly = (flags & 1) ? 1 : 0; g_att_grid_cap = flags >> 8; g_att_form = (flags & 2) ? 1 : (flags & 4) ? 2 : 0; }
  return VPB_OK;
}
static int att_grid(int items) {
  const int sms = (g_att_grid_cap > 0 && g_att_grid_cap < num_sms()) ? g_att_grid_cap : num_sms();
  return items < sms ? items : sms;              // one CTA per SM (the operand stages fill the shared memory)
}

// qkv bf16 [rows, 3*D]: main operand boxes [192 x 64] (128B swizzle) or [192 x 32] (64B swizzle, head_dim 32), plus a
// [192 x 16] 32B-swizzled box for the last 16 dims of head_dim 80.
static int make_attn_maps(CUtensorMap* main, CUtensorMap* tail, const void* qkv, uint64_t rows, int D, int hd) {
  VPB_TRY(make_map(main, qkv, rows, 3 * D, 3 * D, 192, false, hd == 32 ? 64 : 128));
  if (hd == 80) VPB_TRY(make_map(tail, qkv, rows, 3 * D, 3 * D, 192, false, 32));
  else *tail = *main;
  return VPB_OK;
}
static int attention_launch(int hd, const CUtensorMap& main, const CUtensorMap& tail, const AttnParams& ap, cudaStream_t st) {
  const dim3 grid(att_grid(ap.batch * ap.heads));
  cudaError_t err;
  if (g_att_poly) {
    switch (hd) {
      case 32: err = launch_k(attention_wgmma<32, 8>, grid, dim3(ATT_THREADS), AttCfg<32>::SMEM, st, main, tail, ap); break;
      case 64: err = launch_k(attention_wgmma<64, 8>, grid, dim3(ATT_THREADS), AttCfg<64>::SMEM, st, main, tail, ap); break;
      case 80: err = launch_k(attention_wgmma<80, 8>, grid, dim3(ATT_THREADS), AttCfg<80>::SMEM, st, main, tail, ap); break;
      default: return fail(VPB_ERR_ARG, "attention: head_dim %d not built (32, 64, 80)", hd);
    }
  } else {
    switch (hd) {
      case 32: err = launch_k(attention_wgmma<32>, grid, dim3(ATT_THREADS), AttCfg<32>::SMEM, st, main, tail, ap); break;
      case 64: err = launch_k(attention_wgmma<64>, grid, dim3(ATT_THREADS), AttCfg<64>::SMEM, st, main, tail, ap); break;
      case 80: err = launch_k(attention_wgmma<80>, grid, dim3(ATT_THREADS), AttCfg<80>::SMEM, st, main, tail, ap); break;
      default: return fail(VPB_ERR_ARG, "attention: head_dim %d not built (32, 64, 80)", hd);
    }
  }
  if (err != cudaSuccess) return fail(VPB_ERR_CUDA, "attention launch: %s", cudaGetErrorString(err));
  return VPB_OK;
}
// qkv GEMM + attention as one launch (qkv_attention.cuh).  tx: xn in boxes of [192 x 64]; tw: the packed qkv weight in boxes of
// [head_dim x 64]
static int qkv_attention_launch(int hd, const CUtensorMap& tx, const CUtensorMap& tw, const QkvAttnParams& qp, cudaStream_t st) {
  const dim3 grid(att_grid(qp.batch * qp.heads));
  cudaError_t err;
  if (g_att_poly) {
    switch (hd) {
      case 32: err = launch_k(qkv_attention_wgmma<32, 8>, grid, dim3(ATT_THREADS), QkvAttCfg<32>::SMEM, st, tx, tw, qp); break;
      case 64: err = launch_k(qkv_attention_wgmma<64, 8>, grid, dim3(ATT_THREADS), QkvAttCfg<64>::SMEM, st, tx, tw, qp); break;
      case 80: err = launch_k(qkv_attention_wgmma<80, 8>, grid, dim3(ATT_THREADS), QkvAttCfg<80>::SMEM, st, tx, tw, qp); break;
      default: return fail(VPB_ERR_ARG, "qkv attention: head_dim %d not built (32, 64, 80)", hd);
    }
  } else {
    switch (hd) {
      case 32: err = launch_k(qkv_attention_wgmma<32>, grid, dim3(ATT_THREADS), QkvAttCfg<32>::SMEM, st, tx, tw, qp); break;
      case 64: err = launch_k(qkv_attention_wgmma<64>, grid, dim3(ATT_THREADS), QkvAttCfg<64>::SMEM, st, tx, tw, qp); break;
      case 80: err = launch_k(qkv_attention_wgmma<80>, grid, dim3(ATT_THREADS), QkvAttCfg<80>::SMEM, st, tx, tw, qp); break;
      default: return fail(VPB_ERR_ARG, "qkv attention: head_dim %d not built (32, 64, 80)", hd);
    }
  }
  if (err != cudaSuccess) return fail(VPB_ERR_CUDA, "qkv attention launch: %s", cudaGetErrorString(err));
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------ per-kernel timing
// Optional ("profile" option): a CUDA-event pair around every launch, on the launch stream, summed per kernel
// class by vpb_profile_collect.  bench.py uses it to report the dominant kernel's achieved FLOP/s live.
enum KClass : int { KC_PATCH_IM2COL, KC_GEMM_PATCH, KC_LN, KC_GEMM_QKV, KC_ATTN, KC_GEMM_PROJ, KC_GEMM_FC1, KC_GEMM_FC2,
                    KC_GEMM_DECONV, KC_GEMM_FINAL, KC_DECODE, KC_PREPROCESS, KC_CHAIN, KC_COUNT };
static const char* kclass_names[KC_COUNT] = {"patch_im2col", "gemm_patch_embed", "layernorm", "gemm_qkv", "attention", "gemm_proj",
                                             "gemm_fc1_gelu", "gemm_fc2", "gemm_deconv", "gemm_final_conv", "decode", "crop_preprocess", "gemm_chain"};
struct ProfRec { int cls; cudaEvent_t a, b; };
struct Profiler {
  bool on = false;
  std::vector<ProfRec> recs;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pool;
  void begin(int cls, cudaStream_t st) {
    if (!on) return;
    std::pair<cudaEvent_t, cudaEvent_t> ev;
    if (!pool.empty()) { ev = pool.back(); pool.pop_back(); }
    else { cudaEventCreate(&ev.first); cudaEventCreate(&ev.second); }
    cudaEventRecord(ev.first, st);
    recs.push_back({cls, ev.first, ev.second});
  }
  void end(cudaStream_t st) {
    if (!on) return;
    cudaEventRecord(recs.back().b, st);
  }
};

// ------------------------------------------------------------------------------------------------ engine
constexpr int kTileWidths[3] = {128, 256, 192};   // tile widths of the standalone GEMM's TMA epilogues, in pick_tile's tie order
struct LinearW {
  __nv_bfloat16* w = nullptr;   // [N,K] bf16
  float* b = nullptr;           // [N padded]
  int n = 0, k = 0;
  CUtensorMap tmap[3];          // W boxes of kTileWidths[i] rows, for each width that divides the padded N (has[i])
  bool has[3] = {false, false, false};
  CUtensorMap map_c;            // W boxes of chain_bn rows (every phase of a chained launch uses one tile width)
  const CUtensorMap* tile_map(int bn) const {
    for (int i = 0; i < 3; ++i)
      if (kTileWidths[i] == bn) return has[i] ? &tmap[i] : nullptr;
    return nullptr;
  }
};
// W maps of a [n_pad, k] weight for every tile width that divides n_pad
static int make_tile_maps(LinearW& L, const void* w, int n_pad, int k) {
  for (int i = 0; i < 3; ++i) {
    L.has[i] = (n_pad % kTileWidths[i] == 0);
    if (L.has[i]) VPB_TRY(make_map(&L.tmap[i], w, n_pad, k, k, kTileWidths[i]));
  }
  return VPB_OK;
}
struct BlockW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  // fc2 of an engine with experts (P > 0): W and bias are stacked [shared (D-P rows); expert 0 (P); ...; expert H-1], so the
  // first D rows are head 0's whole fc2 and `fc2` is exactly the single-head linear.  fc2s = the shared rows alone (maps of
  // D-P rows: TMA zero-fills the rest of a tile), m_exp = the whole stack in boxes of expert_bn rows.
  LinearW qkv, proj, fc1, fc2, fc2s;
  CUtensorMap m_exp;
  CUtensorMap m_qkv_head;       // qkv W in boxes of head_dim rows: the fused qkv + attention launch
};
// One keypoint head: TopdownHeatmapSimpleHead weights (keypoint_head.* for head 0, associate_keypoint_heads.{j-1}.* for head j)
struct HeadW {
  int K = 0, n_final = 0;           // n_final = padded channel count of the 1x1 conv GEMM
  LinearW dc1, dc2, fin;            // dc*: the 4 phase matrices stacked [4*256, 4*Cin]
  CUtensorMap m_fin_w;              // final 1x1 conv W: boxes of n_final rows (one column tile)
};
// A run of consecutive crops of one head in a multi-head call
struct Segment { int head, count; };
static bool operator==(const Segment& a, const Segment& b) { return a.head == b.head && a.count == b.count; }
struct vpb_engine {
  vpb_config cfg;
  int D, depth, heads, K, maxB;    // K = head 0's keypoints: what the single-head calls return per crop
  // keypoint heads (vpb_create_heads; vpb_create: one head, P = 0) and the expert width P of each block's fc2
  int num_kheads = 1, P = 0, Kmax = 0, expert_bn = 0;
  std::vector<HeadW> hw;
  bool finalized = false;
  int stop_after = 0;
  Profiler prof;
  // CUDA-graph replay of the kernel chain behind the patch gather: removes ~90 launches of CPU work per call, which is what
  // bounds small ragged batches (video streams).  The graph only touches engine-owned memory (the caller's crops are consumed
  // by the eagerly launched gather; org_wh / keypoints / argmax / heatmaps move by small device copies), so it is valid for
  // any caller pointers.  One graph per (mixed, segment list, affine), captured on the key's second use.  mixed = made by a
  // multi-head call (rows of K_max keypoints; at most kMaxMixedGraphs such graphs, least recently used out first), else by a
  // single-head call (the one segment {head 0, n}: one graph per batch size and decode kind, unbounded); affine = the graph
  // decodes with centre / scale instead of canvas sizes / offsets
  struct CachedGraph { bool mixed; std::vector<Segment> segs; bool affine; cudaGraphExec_t exec; unsigned long long used; };
  std::vector<CachedGraph> graph_cache;
  unsigned long long graph_clock = 0;
  bool use_graph = true;
  // L2 residency: the fp32 token stream x (37.7 MB at B=64) is read-modify-written by every residual GEMM and read by every
  // LayerNorm, but the per-layer working set (~220 MB) would evict it from the 50 MB L2 in between; an access-policy window
  // (clipped to what the device allows to persist) marks it persisting on every stream the engine launches on.  Measured on an
  // H100 80GB HBM3 (700 W power limit), ViT-B, 64 crops: 9.39 ms per call with the window, 10.52 without (tools/defaults_ab.py).
  // The window and the persisting set-aside are also capped at kL2PersistMax (see there).
  bool l2_persist = true;
  size_t l2_window_bytes = 0;
  std::vector<cudaStream_t> l2_streams;
  float* g_kpts = nullptr;      // graph-owned outputs / decode inputs: the captured chain only touches engine memory
  int32_t *g_idx = nullptr, *g_org = nullptr, *g_offs = nullptr;
  float* g_cs = nullptr;        // [max_batch,4] centre / scale the affine graphs decode with
  // affine host calls (vpb_infer_affine_host): matrices and centre / scale staged next to the slot-0 frames
  double* mat_stage = nullptr;
  float* cs_stage = nullptr;
  // frame-level entry points (crop pre-processing on the GPU): canvas sizes / frame offsets produced by frame_to_patch_rows,
  // the status word it flags empty boxes in, and per-slot frame + box staging for the host variants
  int32_t *pp_org = nullptr, *pp_offs = nullptr, *pp_status = nullptr;
  uint8_t* frame_stage[2] = {nullptr, nullptr};
  size_t frame_cap[2] = {0, 0};
  int32_t* bbox_stage[2] = {nullptr, nullptr};
  // flip test (vpb_set_flip_test): the keypoint entry points run each crop and its mirror image as one batch of 2n crops and
  // decode the averaged maps; flip_perm = the keypoint permutation of the flip pairs, flip_shift = shift_heatmap.
  // flip_heads: set by vpb_set_flip_test_heads, flip_perm then holds every head's permutation in head order (head j's at
  // perm_offset(e, j)) and the multi-head calls run the flip test too
  bool flip = false, flip_heads = false;
  int flip_shift = 0;
  int32_t* flip_perm = nullptr;
  std::map<std::string, std::pair<float*, int64_t>> staged;   // fp32 state_dict tensors on device until finalize
  std::vector<void*> allocs;
  size_t alloc_bytes = 0;          // what `allocs` holds: packed weights + workspace (vpb_device_bytes)
  // packed weights
  LinearW patch;            // bias unused (folded into pos_bias)
  float* pos_bias = nullptr;   // [192, D]
  std::vector<BlockW> blocks;
  float *lnf_g = nullptr, *lnf_b = nullptr;
  // workspace
  __nv_bfloat16 *patch_rows, *xn, *qkv, *attn, *hid, *d1, *d2;
  float *x, *heat;
  int* ln_counters = nullptr;      // one per 128-row block of x (fused LayerNorm tail of the residual GEMMs)
  // Opt-in experiment ("ln_fused"): correct and bit-identical, off by default: the CTA that finishes a row block normalises
  // its 128 rows alone, latency-bound, and the last blocks' LayerNorm sits on the kernel's critical path; a standalone
  // LayerNorm launch spreads the same rows over all SMs.
  bool ln_fused = false;
  // Chained launches (chain.cuh): patch -> LN -> qkv0, then per block proj -> LN -> fc1 -> fc2 -> LN -> qkv(next) as ONE persistent
  // kernel each; the counters that replace the kernel boundaries live in chain_counters (5 arrays of one int per 128-row
  // block per chained launch), zeroed by one memset at the start of every forward.
  // Small batches (below chain_min_batch): LayerNorm + its consumer GEMM (qkv / fc1) as ONE two-stage chained launch -- the
  // LayerNorm jobs start at once (their rows are complete), the GEMM tiles wait for their rows -- instead of a LayerNorm
  // launch followed by a GEMM launch (option "ln_in_gemm").  Bit-identical, off by default: the LayerNorm jobs then run on
  // the chain's few spare warps instead of a whole launch, and the chained kernel uses one tile width.
  bool ln_in_gemm = false;
  bool gelu_erf = false;           // option "gelu_erf": fc1 epilogue with the A&S-7.1.26 erf instead of the fitted tanh form (A/B)
  bool use_chain = false;
  // Chained launches are off by default (option "chain" / VPB_CHAIN=1 turns them on, for batches of at least "chain_min_batch" /
  // VPB_CHAIN_MIN_BATCH crops): on an H100 80GB HBM3 (700 W power limit) ViT-B ran slower chained than with one 128-wide-tile
  // kernel per GEMM at every batch size measured, 1 to 64 crops (64 crops: 9.39 vs 6.26 ms per call; 1 crop: 1.00 vs 0.77;
  // tools/defaults_ab.py).  Bit-identical either way.
  int chain_min_batch = 1;
  int resid_rmw = 0;               // residual epilogues as load + add + store instead of TMA reduce-add (see resid_rmw_default)
  int ln_job_rows = CHAIN_LN_JOB_ROWS;   // rows per LayerNorm job of the chained launches (8 or 16); option "ln_job_rows", VPB_LN_JOB_ROWS
  int ln_ctl = 0;                  // chained launches: LayerNorm polls / publishes on a control warp (chain.cuh); option "ln_ctl", VPB_LN_CTL
  int chain_bn = 128;
  int* chain_counters = nullptr;
  size_t chain_blocks = 0;         // 128-row blocks at max_batch
  // host-facing path: two staging slots (crops, org_wh in; kpts, idx out) so that slot i+1's H2D overlaps slot i's compute
  float *crops_stage[2], *kpts[2];
  int32_t *idx[2], *org_wh[2];
  cudaStream_t copy_stream = nullptr, compute_stream = nullptr;
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
  // One activation workspace per engine: calls on DIFFERENT streams are ordered against each other by an event recorded
  // after every enqueue (WsScope::end) and waited on when the stream changes (WsScope::begin); calls on one stream order themselves.
  cudaEvent_t ev_ws = nullptr;
  cudaStream_t ws_last = nullptr;
  bool ws_used = false;
  CUtensorMap m_patch_rows, m_xn, m_attn, m_hid, m_d2, m_qkv_att, m_qkv_att_tail;   // A operands / attention boxes
  CUtensorMap m_xn_att;                                                 // xn in boxes of one crop's 192 rows (fused qkv + attention)
  CUtensorMap m_feat_nhwc, m_d1_nhwc;                                 // implicit-GEMM deconv inputs (4-D)
  CUtensorMap o_qkv, o_hid, o_x;                                                             // TMA-epilogue outputs
  CUtensorMap o_xs;                             // x bounded to the shared columns [0, D-P) (multi-head fc2)
};

template <typename T>
static int dev_alloc(vpb_engine* e, T** p, size_t count) {
  void* q = nullptr;
  CU_TRY(cudaMalloc(&q, count * sizeof(T) + 256));
  e->allocs.push_back(q);
  e->alloc_bytes += count * sizeof(T) + 256;
  *p = reinterpret_cast<T*>(q);
  return VPB_OK;
}

// ViTPose+ key names: head 0 is keypoint_head, head j >= 1 is associate_keypoint_heads.{j-1} (model_split.py:97-99)
static std::string head_prefix(int j) {
  return j == 0 ? std::string("keypoint_head.") : "associate_keypoint_heads." + std::to_string(j - 1) + ".";
}
static std::vector<std::pair<std::string, int64_t>> expected_keys(const vpb_engine* e) {
  const int64_t D = e->D, P = e->P;
  std::vector<std::pair<std::string, int64_t>> v;
  v.push_back({"backbone.pos_embed", 193 * D});
  v.push_back({"backbone.patch_embed.proj.weight", D * 768});
  v.push_back({"backbone.patch_embed.proj.bias", D});
  for (int i = 0; i < e->depth; ++i) {
    const std::string p = "backbone.blocks." + std::to_string(i) + ".";
    v.push_back({p + "norm1.weight", D}); v.push_back({p + "norm1.bias", D});
    v.push_back({p + "attn.qkv.weight", 3 * D * D}); v.push_back({p + "attn.qkv.bias", 3 * D});
    v.push_back({p + "attn.proj.weight", D * D}); v.push_back({p + "attn.proj.bias", D});
    v.push_back({p + "norm2.weight", D}); v.push_back({p + "norm2.bias", D});
    v.push_back({p + "mlp.fc1.weight", 4 * D * D}); v.push_back({p + "mlp.fc1.bias", 4 * D});
    v.push_back({p + "mlp.fc2.weight", 4 * D * (D - P)}); v.push_back({p + "mlp.fc2.bias", D - P});
    for (int j = 0; P > 0 && j < e->num_kheads; ++j) {         // ViTPose+ experts: the last P output rows of head j's fc2
      v.push_back({p + "mlp.experts." + std::to_string(j) + ".weight", 4 * D * P});
      v.push_back({p + "mlp.experts." + std::to_string(j) + ".bias", P});
    }
  }
  v.push_back({"backbone.last_norm.weight", D}); v.push_back({"backbone.last_norm.bias", D});
  for (int j = 0; j < e->num_kheads; ++j) {
    const std::string hp = head_prefix(j);
    int64_t cin = D;
    for (int li : {0, 3}) {
      const std::string p = hp + "deconv_layers.";
      v.push_back({p + std::to_string(li) + ".weight", cin * 256 * 16});
      for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) v.push_back({p + std::to_string(li + 1) + s, 256});
      cin = 256;
    }
    v.push_back({hp + "final_layer.weight", static_cast<int64_t>(e->hw[j].K) * 256});
    v.push_back({hp + "final_layer.bias", e->hw[j].K});
  }
  return v;
}

extern "C" int vpb_create(const vpb_config* cfg, vpb_engine** out) {
  if (!cfg || !out) return fail(VPB_ERR_ARG, "vpb_create: null argument");
  *out = nullptr;
  if (cfg->embed_dim % 128 != 0 || cfg->num_heads <= 0 || cfg->embed_dim % cfg->num_heads != 0)
    return fail(VPB_ERR_ARG, "embed_dim=%d / num_heads=%d unsupported", cfg->embed_dim, cfg->num_heads);
  {
    const int hd = cfg->embed_dim / cfg->num_heads;
    if (hd != 32 && hd != 64 && hd != 80) return fail(VPB_ERR_ARG, "head_dim=%d: attention is built for 32, 64 and 80 (ViT-S / B,L / H)", hd);
  }
  if (cfg->embed_dim != 384 && cfg->embed_dim != 768 && cfg->embed_dim != 1024 && cfg->embed_dim != 1280)
    return fail(VPB_ERR_ARG, "embed_dim=%d has no LayerNorm instantiation", cfg->embed_dim);
  if (cfg->num_keypoints < 1 || cfg->num_keypoints > 144) return fail(VPB_ERR_ARG, "num_keypoints=%d out of range 1..144", cfg->num_keypoints);
  if (cfg->max_batch < 1 || cfg->depth < 1) return fail(VPB_ERR_ARG, "max_batch/depth must be >= 1");
  CU_TRY(cudaSetDevice(cfg->device));
  VPB_TRY(device_check(cfg->device));
  vpb_engine* e = new vpb_engine();
  e->cfg = *cfg;
  e->D = cfg->embed_dim; e->depth = cfg->depth; e->heads = cfg->num_heads; e->K = cfg->num_keypoints; e->maxB = cfg->max_batch;
  e->Kmax = e->K;
  e->hw.resize(1);
  e->hw[0].K = e->K;
  e->hw[0].n_final = e->K <= 32 ? 32 : 144;
  e->chain_bn = 128;     // D, 3D and 4D are multiples of it for every ViT; 128 accumulator columns leave the LayerNorm warps room
  {
    const char* env = getenv("VPB_CHAIN");
    if (env) e->use_chain = env[0] != '0';
    const char* ge = getenv("VPB_GELU_ERF");
    if (ge && ge[0] == '1') e->gelu_erf = true;
    const char* mb = getenv("VPB_CHAIN_MIN_BATCH");
    if (mb && atoi(mb) > 0) e->chain_min_batch = atoi(mb);
  }
  e->resid_rmw = resid_rmw_default();
  {
    const char* lc = getenv("VPB_LN_CTL");
    e->ln_ctl = lc ? (lc[0] != '0') : kLnCtlDefault;
    const char* jr = getenv("VPB_LN_JOB_ROWS");
    if (jr && (atoi(jr) == 8 || atoi(jr) == 16)) e->ln_job_rows = atoi(jr);
  }
  *out = e;
  return VPB_OK;
}

extern "C" int vpb_create_heads(const vpb_config* cfg, int32_t num_heads, const int32_t* h_keypoints, int32_t expert_rows, vpb_engine** out) {
  if (!cfg || !h_keypoints || !out) return fail(VPB_ERR_ARG, "vpb_create_heads: null argument");
  *out = nullptr;
  if (num_heads < 1 || num_heads > VPB_MAX_HEADS) return fail(VPB_ERR_ARG, "vpb_create_heads: %d heads (1..%d)", num_heads, VPB_MAX_HEADS);
  for (int j = 0; j < num_heads; ++j)
    if (h_keypoints[j] < 1 || h_keypoints[j] > 144) return fail(VPB_ERR_ARG, "vpb_create_heads: head %d has %d keypoints (1..144)", j, h_keypoints[j]);
  if (expert_rows != 0 && (expert_rows < 0 || expert_rows >= cfg->embed_dim || expert_rows % 32 != 0))
    return fail(VPB_ERR_ARG, "vpb_create_heads: expert_rows=%d must be 0 or a multiple of 32 below embed_dim=%d", expert_rows, cfg->embed_dim);
  vpb_config c = *cfg;
  c.num_keypoints = h_keypoints[0];
  VPB_TRY(vpb_create(&c, out));
  vpb_engine* e = *out;
  e->num_kheads = num_heads;
  e->P = expert_rows;
  e->expert_bn = expert_width(expert_rows);
  e->hw.resize(num_heads);
  for (int j = 0; j < num_heads; ++j) {
    e->hw[j].K = h_keypoints[j];
    e->hw[j].n_final = h_keypoints[j] <= 32 ? 32 : 144;
    e->Kmax = std::max(e->Kmax, static_cast<int>(h_keypoints[j]));
  }
  return VPB_OK;
}

extern "C" void vpb_destroy(vpb_engine* e) {
  if (!e) return;
  int prev = -1;
  if (cudaGetDevice(&prev) == cudaSuccess && prev != e->cfg.device) cudaSetDevice(e->cfg.device); else prev = -1;
  cudaDeviceSynchronize();
  for (auto& r : e->prof.recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto& ev : e->prof.pool) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  for (auto& kv : e->staged) cudaFree(kv.second.first);
  for (void* p : e->allocs) cudaFree(p);
  for (auto& g : e->graph_cache) if (g.exec) cudaGraphExecDestroy(g.exec);
  for (int s = 0; s < 2; ++s) {
    if (e->ev_h2d[s]) cudaEventDestroy(e->ev_h2d[s]);
    if (e->ev_done[s]) cudaEventDestroy(e->ev_done[s]);
  }
  if (e->ev_ws) cudaEventDestroy(e->ev_ws);
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  if (e->compute_stream) cudaStreamDestroy(e->compute_stream);
  for (int s = 0; s < 2; ++s) if (e->frame_stage[s]) cudaFree(e->frame_stage[s]);
  delete e;
  if (prev >= 0) cudaSetDevice(prev);
}

extern "C" int vpb_load_tensor(vpb_engine* e, const char* key, const float* data, int64_t numel) {
  if (!e || !key || (!data && numel > 0)) return fail(VPB_ERR_ARG, "vpb_load_tensor: null argument");
  if (e->finalized) return fail(VPB_ERR_STATE, "vpb_load_tensor after vpb_finalize");
  const std::string k(key);
  if (k.size() > 19 && k.compare(k.size() - 19, 19, "num_batches_tracked") == 0) return VPB_OK;
  bool known = false;
  for (auto& kv : expected_keys(e))
    if (kv.first == k) {
      known = true;
      if (kv.second != numel) return fail(VPB_ERR_ARG, "size mismatch for %s: got %lld elements, expected %lld", key, (long long)numel, (long long)kv.second);
    }
  if (!known) return fail(VPB_ERR_ARG, "unexpected key in state_dict: %s", key);
  if (e->staged.count(k)) return fail(VPB_ERR_ARG, "duplicate key: %s", key);
  CU_TRY(cudaSetDevice(e->cfg.device));
  float* d = nullptr;
  CU_TRY(cudaMalloc(&d, numel * sizeof(float)));
  CU_TRY(cudaMemcpy(d, data, numel * sizeof(float), cudaMemcpyHostToDevice));
  e->staged[k] = {d, numel};
  return VPB_OK;
}

static inline int cdiv(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// W and bias zero-padded to a multiple of `pad` rows
static int pack_linear(vpb_engine* e, LinearW& L, const std::string& wkey, const std::string& bkey, int n, int k, int pad,
                       int scaled_rows, float scale) {
  L.n = n; L.k = k;
  const int n_pad = cdiv(n, pad) * pad;
  VPB_TRY(dev_alloc(e, &L.w, static_cast<size_t>(n_pad) * k));
  CU_TRY(cudaMemset(L.w, 0, static_cast<size_t>(n_pad) * k * 2));
  const long long ne = static_cast<long long>(n) * k;
  pack_linear_bf16<<<cdiv(ne, 256), 256>>>(e->staged[wkey].first, L.w, ne, k, scaled_rows, scale);
  VPB_TRY(dev_alloc(e, &L.b, n_pad));
  if (!bkey.empty()) pack_bias<<<cdiv(n_pad, 256), 256>>>(e->staged[bkey].first, L.b, n, n_pad, scaled_rows, scale);
  else CU_TRY(cudaMemset(L.b, 0, n_pad * sizeof(float)));
  CU_TRY(cudaGetLastError());
  VPB_TRY(make_tile_maps(L, L.w, n_pad, k));
  if (n_pad % e->chain_bn == 0) VPB_TRY(make_map(&L.map_c, L.w, n_pad, k, k, e->chain_bn));   // else never chained (final 1x1 conv)
  return VPB_OK;
}

// The shared rows [0, S) of a stacked fc2 as a linear of S outputs (BlockW::fc2s).  A width serves when it divides S rounded up
// to 128: the W maps hold S rows, so TMA zero-fills the rows of the last column tile past S, and the output map bounds the
// stores to the S columns.
static int make_shared_maps(LinearW& Ls, __nv_bfloat16* w, float* b, int S, int K) {
  Ls.w = w; Ls.b = b; Ls.n = S; Ls.k = K;
  for (int i = 0; i < 3; ++i) {
    Ls.has[i] = (cdiv(S, 128) * 128) % kTileWidths[i] == 0;
    if (Ls.has[i]) VPB_TRY(make_map(&Ls.tmap[i], w, S, K, K, kTileWidths[i]));
  }
  return VPB_OK;
}

// ViTPose+ fc2 with experts: W / bias stacked [shared; expert 0; ...; expert H-1] (see BlockW).  The first D rows are the fc2
// that model_split.py gives head 0 (torch.cat([fc2, experts.0]), :56), packed exactly as pack_linear packs it.
static int pack_fc2_experts(vpb_engine* e, BlockW& b, const std::string& p) {
  const int D = e->D, P = e->P, K = 4 * D, S = D - P, rows = S + e->num_kheads * P;
  LinearW& L = b.fc2;
  L.n = D; L.k = K;
  VPB_TRY(dev_alloc(e, &L.w, static_cast<size_t>(rows) * K));
  VPB_TRY(dev_alloc(e, &L.b, rows));
  auto put = [&](const std::string& key, int row0, int n) -> int {
    const long long ne = static_cast<long long>(n) * K;
    pack_linear_bf16<<<cdiv(ne, 256), 256>>>(e->staged[key + ".weight"].first, L.w + static_cast<size_t>(row0) * K, ne, K, 0, 1.f);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpy(L.b + row0, e->staged[key + ".bias"].first, n * sizeof(float), cudaMemcpyDeviceToDevice));
    return VPB_OK;
  };
  VPB_TRY(put(p + "mlp.fc2", 0, S));
  for (int j = 0; j < e->num_kheads; ++j) VPB_TRY(put(p + "mlp.experts." + std::to_string(j), S + j * P, P));
  VPB_TRY(make_tile_maps(L, L.w, D, K));
  VPB_TRY(make_map(&L.map_c, L.w, D, K, K, e->chain_bn));
  VPB_TRY(make_shared_maps(b.fc2s, L.w, L.b, S, K));
  return make_map(&b.m_exp, L.w, rows, K, K, e->expert_bn);
}

static int copy_vec(vpb_engine* e, float** dst, const std::string& key) {
  auto& s = e->staged[key];
  VPB_TRY(dev_alloc(e, dst, s.second));
  CU_TRY(cudaMemcpy(*dst, s.first, s.second * sizeof(float), cudaMemcpyDeviceToDevice));
  return VPB_OK;
}

extern "C" int vpb_finalize(vpb_engine* e) {
  if (!e) return fail(VPB_ERR_ARG, "vpb_finalize: null engine");
  if (e->finalized) return fail(VPB_ERR_STATE, "vpb_finalize called twice");
  for (auto& kv : expected_keys(e))
    if (!e->staged.count(kv.first)) return fail(VPB_ERR_ARG, "missing key in state_dict: %s", kv.first.c_str());
  CU_TRY(cudaSetDevice(e->cfg.device));
  const int D = e->D;
  const float qscale = 1.0f / sqrtf(static_cast<float>(D / e->heads));

  VPB_TRY(pack_linear(e, e->patch, "backbone.patch_embed.proj.weight", "", D, 768, 128, 0, 1.f));
  VPB_TRY(dev_alloc(e, &e->pos_bias, 192 * D));
  pack_pos_bias<<<cdiv(192 * D, 256), 256>>>(e->staged["backbone.pos_embed"].first, e->staged["backbone.patch_embed.proj.bias"].first,
                                              e->pos_bias, 192, D);
  e->blocks.resize(e->depth);
  for (int i = 0; i < e->depth; ++i) {
    const std::string p = "backbone.blocks." + std::to_string(i) + ".";
    BlockW& b = e->blocks[i];
    VPB_TRY(copy_vec(e, &b.ln1_g, p + "norm1.weight")); VPB_TRY(copy_vec(e, &b.ln1_b, p + "norm1.bias"));
    VPB_TRY(copy_vec(e, &b.ln2_g, p + "norm2.weight")); VPB_TRY(copy_vec(e, &b.ln2_b, p + "norm2.bias"));
    // q rows (first D) carry head_dim^-0.5: vit.py:170 scales q before QK^T; fp32 multiply, then bf16 rounding
    VPB_TRY(pack_linear(e, b.qkv, p + "attn.qkv.weight", p + "attn.qkv.bias", 3 * D, D, 128, D, qscale));
    VPB_TRY(make_map(&b.m_qkv_head, b.qkv.w, 3 * D, D, D, D / e->heads));
    VPB_TRY(pack_linear(e, b.proj, p + "attn.proj.weight", p + "attn.proj.bias", D, D, 128, 0, 1.f));
    VPB_TRY(pack_linear(e, b.fc1, p + "mlp.fc1.weight", p + "mlp.fc1.bias", 4 * D, D, 128, 0, 1.f));
    if (e->P == 0) VPB_TRY(pack_linear(e, b.fc2, p + "mlp.fc2.weight", p + "mlp.fc2.bias", D, 4 * D, 128, 0, 1.f));
    else VPB_TRY(pack_fc2_experts(e, b, p));
  }
  VPB_TRY(copy_vec(e, &e->lnf_g, "backbone.last_norm.weight"));
  VPB_TRY(copy_vec(e, &e->lnf_b, "backbone.last_norm.bias"));
  // per head: deconv layers (4 phase matrices [256, 4*Cin] each, BN folded: eps 1e-5 = nn.BatchNorm2d default), final 1x1 conv
  for (int j = 0; j < e->num_kheads; ++j) {
    HeadW& h = e->hw[j];
    const std::string hp = head_prefix(j);
    int cin = D;
    for (int layer = 0; layer < 2; ++layer) {
      LinearW& dc = layer == 0 ? h.dc1 : h.dc2;
      const std::string wk = hp + "deconv_layers." + std::to_string(layer * 3) + ".weight";
      const std::string bnp = hp + "deconv_layers." + std::to_string(layer * 3 + 1) + ".";
      VPB_TRY(dev_alloc(e, &dc.w, static_cast<size_t>(4) * 256 * 4 * cin));
      VPB_TRY(dev_alloc(e, &dc.b, 256));
      const long long tot = 4LL * 256 * 4 * cin;
      pack_deconv<<<cdiv(tot, 256), 256>>>(e->staged[wk].first, e->staged[bnp + "weight"].first, e->staged[bnp + "bias"].first,
                                           e->staged[bnp + "running_mean"].first, e->staged[bnp + "running_var"].first, dc.w, dc.b,
                                           cin, 256, 1e-5f);
      CU_TRY(cudaGetLastError());
      dc.n = 256; dc.k = 4 * cin;
      VPB_TRY(make_tile_maps(dc, dc.w, 4 * 256, 4 * cin));
      cin = 256;
    }
    {  // final 1x1 conv: [K,256] zero-padded to the N tile
      LinearW& L = h.fin;
      VPB_TRY(pack_linear(e, L, hp + "final_layer.weight", hp + "final_layer.bias", h.K, 256, h.n_final, 0, 1.f));
      VPB_TRY(make_map(&h.m_fin_w, L.w, h.n_final, 256, 256, h.n_final));
    }
  }
  // ---- workspace for max_batch crops
  const size_t B = e->maxB, M = B * 192;
  VPB_TRY(dev_alloc(e, &e->patch_rows, M * 768));
  VPB_TRY(dev_alloc(e, &e->x, M * D));
  VPB_TRY(dev_alloc(e, &e->xn, M * D));
  VPB_TRY(dev_alloc(e, &e->qkv, M * 3 * D));
  VPB_TRY(dev_alloc(e, &e->attn, M * D));
  VPB_TRY(dev_alloc(e, &e->hid, M * 4 * D));
  VPB_TRY(dev_alloc(e, &e->d1, B * 768 * 256));
  VPB_TRY(dev_alloc(e, &e->d2, B * 3072 * 256));
  VPB_TRY(dev_alloc(e, &e->heat, B * e->Kmax * 3072));
  for (int s = 0; s < 2; ++s) {
    VPB_TRY(dev_alloc(e, &e->kpts[s], B * e->Kmax * 3));
    VPB_TRY(dev_alloc(e, &e->idx[s], B * e->Kmax));
    VPB_TRY(dev_alloc(e, &e->org_wh[s], B * 2));
    VPB_TRY(dev_alloc(e, &e->crops_stage[s], B * 3 * 256 * 192));
    CU_TRY(cudaEventCreateWithFlags(&e->ev_h2d[s], cudaEventDisableTiming));
    CU_TRY(cudaEventCreateWithFlags(&e->ev_done[s], cudaEventDisableTiming));
  }
  CU_TRY(cudaEventCreateWithFlags(&e->ev_ws, cudaEventDisableTiming));
  e->chain_blocks = (M + GEMM_BM - 1) / GEMM_BM;
  VPB_TRY(dev_alloc(e, &e->chain_counters, static_cast<size_t>(e->depth + 1) * 5 * e->chain_blocks));
  CU_TRY(cudaMemset(e->chain_counters, 0, static_cast<size_t>(e->depth + 1) * 5 * e->chain_blocks * sizeof(int)));
  VPB_TRY(dev_alloc(e, &e->ln_counters, (M + 127) / 128 + 1));
  CU_TRY(cudaMemset(e->ln_counters, 0, ((M + 127) / 128 + 1) * sizeof(int)));
  VPB_TRY(dev_alloc(e, &e->g_kpts, B * e->Kmax * 3));
  VPB_TRY(dev_alloc(e, &e->g_idx, B * e->Kmax));
  VPB_TRY(dev_alloc(e, &e->g_org, B * 2));
  VPB_TRY(dev_alloc(e, &e->g_offs, B * 2));
  VPB_TRY(dev_alloc(e, &e->g_cs, B * 4));
  VPB_TRY(dev_alloc(e, &e->mat_stage, B * 6));
  VPB_TRY(dev_alloc(e, &e->cs_stage, B * 4));
  VPB_TRY(dev_alloc(e, &e->pp_org, B * 2));
  VPB_TRY(dev_alloc(e, &e->pp_offs, B * 2));
  VPB_TRY(dev_alloc(e, &e->pp_status, 1));
  CU_TRY(cudaMemset(e->pp_status, 0, sizeof(int32_t)));
  for (int s = 0; s < 2; ++s) VPB_TRY(dev_alloc(e, &e->bbox_stage[s], B * 4));
  {
    int ksum = 0;
    for (const HeadW& h : e->hw) ksum += h.K;
    VPB_TRY(dev_alloc(e, &e->flip_perm, ksum));        // every head's permutation (vpb_set_flip_test_heads)
  }
  CU_TRY(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
  CU_TRY(cudaStreamCreateWithFlags(&e->compute_stream, cudaStreamNonBlocking));
  VPB_TRY(make_map(&e->m_patch_rows, e->patch_rows, M, 768, 768, 128));
  VPB_TRY(make_map(&e->m_xn, e->xn, M, D, D, 128));
  VPB_TRY(make_map(&e->m_xn_att, e->xn, M, D, D, 192));
  VPB_TRY(make_map(&e->m_attn, e->attn, M, D, D, 128));
  VPB_TRY(make_map(&e->m_hid, e->hid, M, 4 * D, 4 * D, 128));
  VPB_TRY(make_map_nhwc(&e->m_feat_nhwc, e->xn, B, 16, 12, D, 8, 12));   // 8 x 12 = 96 positions per M tile (12 is not a multiple of 8)
  VPB_TRY(make_map_nhwc(&e->m_d1_nhwc, e->d1, B, 32, 24, 256, 16, 8));  // 16 x 8 = 128 positions per M tile: full tiles
  VPB_TRY(make_map(&e->m_d2, e->d2, B * 3072, 256, 256, 128));
  VPB_TRY(make_attn_maps(&e->m_qkv_att, &e->m_qkv_att_tail, e->qkv, M, D, D / e->heads));
  VPB_TRY(make_map(&e->o_qkv, e->qkv, M, 3 * D, 3 * D, 64));
  VPB_TRY(make_map(&e->o_hid, e->hid, M, 4 * D, 4 * D, 64));
  VPB_TRY(make_map(&e->o_x, e->x, M, D, D, 64, /*f32=*/true));
  if (e->P > 0) VPB_TRY(make_map(&e->o_xs, e->x, M, D - e->P, D, 64, /*f32=*/true));
  {
    const char* env = getenv("VPB_L2_PERSIST");
    if (env && env[0] == '0') e->l2_persist = false;
    cudaDeviceProp prop;
    CU_TRY(cudaGetDeviceProperties(&prop, e->cfg.device));
    size_t want = M * D * sizeof(float);
    if (want > static_cast<size_t>(prop.accessPolicyMaxWindowSize)) want = prop.accessPolicyMaxWindowSize;
    if (want > static_cast<size_t>(prop.persistingL2CacheMaxSize)) want = prop.persistingL2CacheMaxSize;
    if (want > kL2PersistMax) want = kL2PersistMax;
    if (e->l2_persist && want > 0) {
      CU_TRY(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
      e->l2_window_bytes = want;
    }
  }
  CU_TRY(cudaDeviceSynchronize());
  for (auto& kv : e->staged) cudaFree(kv.second.first);
  e->staged.clear();
  e->finalized = true;
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------ forward
template <int D>
static void ln_launch(const float* x, const float* g, const float* b, __nv_bfloat16* y, int rows, float eps, cudaStream_t st) {
  const int want = cdiv(rows, 4), cap = num_sms() * 4;     // 4 warps per CTA, at most 4 CTAs per SM (persistent, row stride)
  launch_k(layernorm_f32_to_bf16<D>, dim3(want < cap ? want : cap), dim3(128), 0, st, x, g, b, y, rows, eps);
}
static int layernorm(const float* x, const float* g, const float* b, __nv_bfloat16* y, int rows, int D, float eps, cudaStream_t st) {
  switch (D) {
    case 384: ln_launch<384>(x, g, b, y, rows, eps, st); break;
    case 768: ln_launch<768>(x, g, b, y, rows, eps, st); break;
    case 1024: ln_launch<1024>(x, g, b, y, rows, eps, st); break;
    case 1280: ln_launch<1280>(x, g, b, y, rows, eps, st); break;
    default: return fail(VPB_ERR_ARG, "layernorm: dim %d not instantiated", D);
  }
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vpb_debug_gemm(int32_t stages_limit, void* d_counters) {   // counters: int64 [grid*8], see GemmParams::dbg
  // one stage cannot serve two k-blocks: a slot is released only once the MMAs of the next k-block have been issued
  if ((stages_limit & 0xff) == 1) return fail(VPB_ERR_ARG, "vpb_debug_gemm: a ring of 1 stage (0 = the compiled depth, else >= 2)");
  g_dbg_flags = stages_limit >> 8;       // bits 8.. carry GemmParams::dbg_flags
  g_dbg_stages = stages_limit & 0xff;
  g_dbg_buf = reinterpret_cast<long long*>(d_counters);
  return VPB_OK;
}
static GemmParams gp(int M, int N, int K, const float* bias, void* out, int ldc) {
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.stages_limit = g_dbg_stages; p.dbg = g_dbg_buf; p.dbg_flags = g_dbg_flags;
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.out = out; p.ldc = ldc;
  p.rmw = resid_rmw(resid_rmw_default());
  return p;
}

// stop_after stages (debug): 1 patch rows, 2 patch embed, 3 first LN, 4 first qkv, 5 first attention, 6 first proj,
// 7 first fc1, 8 first block, 9 all blocks, 10 last norm, 11 deconv1, 12 deconv2
// B crops of patch rows from n_src source crops: n_src == B, or B == 2 n_src for the flip test (crops n_src.. mirrored)
static int patch_gather(vpb_engine* e, const float* d_crops, int n_src, int B, cudaStream_t st) {
  e->prof.begin(KC_PATCH_IM2COL, st);
  CU_TRY(launch_k(patch_im2col, dim3(cdiv(static_cast<long long>(B) * 3 * 256 * 24, 256)), dim3(256), 0, st, d_crops, e->patch_rows, B,
                  n_src, reinterpret_cast<const float4*>(e->pos_bias), reinterpret_cast<float4*>(e->x), e->D));
  e->prof.end(st);
  return VPB_OK;
}
// Where a batch of patch rows comes from: normalised f32 crops (patch_im2col) or a table of uint8 frames + boxes
// (frame_to_patch_rows: crop pre-processing fused with the im2col; it also fills pp_org / pp_offs for the decode).
// Affine crops (frame_to_patch_rows_affine) take a matrix per box instead of a box, and their keypoints are decoded with
// centre / scale (decode mode 4) instead of canvas sizes and offsets.
// YUV frames (every layout, NV12 included) come as a YuvEntry table instead (each entry carries the call's matrix and
// range); the gathers then launch the YUV instantiation of the same kernels, outside the captured graph, so the graph cache
// needs no YUV key.
struct Source {
  const float* crops = nullptr;
  const FrameEntry* frames = nullptr;       // num_frames entries, only frames that have boxes
  const YuvEntry* yuv = nullptr;            // instead of frames: YUV frames
  int num_frames = 0;
  const int32_t* bboxes = nullptr;
  const double* mats = nullptr;             // [n,6] affine matrices (then bboxes is unused)
  const float* cs = nullptr;                // [n,4] centre / scale of the affine decode
};
static void set_table(Source& s, const FrameEntry* tab) { s.frames = tab; }
static void set_table(Source& s, const YuvEntry* tab) { s.yuv = tab; }
template <class Entry>
static AffineParamsT<Entry> affine_params(const Entry* frames, int num_frames, const double* mats, const float* cs, int n, int* status) {
  AffineParamsT<Entry> q;
  memset(&q, 0, sizeof(q));
  q.mats = mats; q.cs = cs; q.n = n; q.status = status; q.num_frames = num_frames;
  memcpy(q.frames, frames, static_cast<size_t>(num_frames) * sizeof(Entry));
  return q;
}
template <class Entry>
static int affine_gather(vpb_engine* e, const Source& src, const Entry* tab, int n_src, int B, cudaStream_t st) {
  AffineParamsT<Entry> q = affine_params(tab, src.num_frames, src.mats, src.cs, n_src, e->pp_status);
  q.rows = e->patch_rows; q.pos_bias = reinterpret_cast<const float4*>(e->pos_bias); q.stream = reinterpret_cast<float4*>(e->x); q.D = e->D;
  e->prof.begin(KC_PREPROCESS, st);
  CU_TRY(launch_k(frame_to_patch_rows_affine<Entry>, dim3(B, 16), dim3(384), 0, st, q));
  e->prof.end(st);
  return VPB_OK;
}
template <class Entry>
static int frame_gather(vpb_engine* e, const Source& src, const Entry* tab, int n_src, int B, cudaStream_t st) {
  FramePatchParamsT<Entry> q;
  memset(&q, 0, sizeof(q));
  q.pp.bboxes = src.bboxes;
  q.pp.n = n_src; q.pp.pad = 10; q.pp.crops = nullptr; q.pp.org_wh = e->pp_org; q.pp.offs_yx = e->pp_offs; q.pp.status = e->pp_status;
  q.rows = e->patch_rows; q.pos_bias = reinterpret_cast<const float4*>(e->pos_bias); q.stream = reinterpret_cast<float4*>(e->x); q.D = e->D;
  q.num_frames = src.num_frames;
  memcpy(q.frames, tab, static_cast<size_t>(src.num_frames) * sizeof(Entry));
  e->prof.begin(KC_PREPROCESS, st);
  CU_TRY(launch_k(frame_to_patch_rows<Entry>, dim3(B, 16), dim3(384), 0, st, q));
  e->prof.end(st);
  return VPB_OK;
}
template <class Entry>
static int table_gather(vpb_engine* e, const Source& src, const Entry* tab, int n_src, int B, cudaStream_t st) {
  return src.mats ? affine_gather(e, src, tab, n_src, B, st) : frame_gather(e, src, tab, n_src, B, st);
}
static int gather(vpb_engine* e, const Source& src, int n_src, int B, cudaStream_t st) {
  if (src.crops) return patch_gather(e, src.crops, n_src, B, st);
  return src.yuv ? table_gather(e, src, src.yuv, n_src, B, st) : table_gather(e, src, src.frames, n_src, B, st);
}
// Chained form of the backbone (chain.cuh): 1 + depth persistent GEMM launches + depth attention launches.
//   launch 0:        patch embed (+= x) -> LN(norm1 of block 0) -> qkv of block 0
//   launch i+1:      proj_i (+= x) -> LN(norm2_i) -> fc1_i + GELU -> fc2_i (+= x) -> LN(norm1_{i+1} | last_norm) [-> qkv_{i+1}]
static int backbone_chained(vpb_engine* e, int B, cudaStream_t st) {
  const int D = e->D, M = B * 192, bn = e->chain_bn;
  const size_t nb = e->chain_blocks;
  CU_TRY(cudaMemsetAsync(e->chain_counters, 0, static_cast<size_t>(e->depth + 1) * 5 * nb * sizeof(int), st));
  auto counters = [&](int launch, int which) { return e->chain_counters + (static_cast<size_t>(launch) * 5 + which) * nb; };
  auto phase = [&](ChainParams& p, ChainMaps& m, int i, const CUtensorMap& a, const LinearW& L, const CUtensorMap& out, int epi, const int* a_ready,
                   int a_target, int* out_done) {
    m.a[i] = a; m.w[i] = L.map_c; m.out[i] = out;
    p.ph[i].N = L.n; p.ph[i].K = L.k; p.ph[i].epi = epi; p.ph[i].bias = L.b; p.ph[i].a_ready = a_ready; p.ph[i].a_target = a_target;
    p.ph[i].out_done = out_done;
  };
  auto base = [&](ChainParams& p) {
    memset(&p, 0, sizeof(p));
    p.M = M; p.D = D; p.x = e->x; p.xn = e->xn; p.eps = 1e-6f;
    static const int nowait = [] { const char* v = getenv("VPB_CHAIN_NOWAIT"); return (v && v[0] == '1') ? 1 : 0; }();
    p.dbg_nowait = nowait;
    p.rmw = resid_rmw(e->resid_rmw);
    p.ln_ctl = e->ln_ctl; p.ln_job_rows = e->ln_job_rows;
    // tile order inside a chained launch: phase-major by default (lag >= number of row blocks).  Interleaving the reduce-add
    // phases with their consumers (VPB_CHAIN_LAG0/1 = lag in 128-row blocks) is an experiment: a consumer tile needs the
    // producer's tile, its epilogue and a LayerNorm job behind it, and CTAs stalled on that delay the very producer tiles the
    // next consumers wait for.
    static const int lag0 = [] { const char* v = getenv("VPB_CHAIN_LAG0"); return v ? atoi(v) : (1 << 20); }();
    static const int lag1 = [] { const char* v = getenv("VPB_CHAIN_LAG1"); return v ? atoi(v) : (1 << 20); }();
    p.wave_lag[0] = lag0; p.wave_lag[1] = lag1;
    p.dbg = g_dbg_buf;                      // vpb_debug_gemm(0, counters): [grid CTAs][4 phases][12] int64, accumulated over launches
  };
  const int nD = D / bn, n4D = 4 * D / bn;                    // column tiles of the D-wide and 4D-wide phases
  {
    ChainParams p; ChainMaps m;
    base(p);
    // patch.b is a zero vector: the conv bias and pos_embed were folded into the stream seed by the gather
    phase(p, m, 0, e->m_patch_rows, e->patch, e->o_x, EPI_F32_ADD, nullptr, 0, counters(0, 0));
    p.ln[0] = {counters(0, 0), nD, e->blocks[0].ln1_g, e->blocks[0].ln1_b, counters(0, 1)};
    phase(p, m, 1, e->m_xn, e->blocks[0].qkv, e->o_qkv, EPI_BF16, counters(0, 1), 0, nullptr);
    p.num_phases = 2; p.num_ln = 1;
    for (int i = 2; i < CHAIN_MAX_PHASES; ++i) { m.a[i] = m.a[0]; m.w[i] = m.w[0]; m.out[i] = m.out[0]; }
    e->prof.begin(KC_CHAIN, st);
    VPB_TRY(chain_launch(bn, m, p, st));
    e->prof.end(st);
  }
  for (int i = 0; i < e->depth; ++i) {
    BlockW& b = e->blocks[i];
    {
      AttnParams ap;
      ap.batch = B; ap.heads = e->heads; ap.dim = D; ap.out = e->attn; ap.dbg = nullptr;
      e->prof.begin(KC_ATTN, st);
      VPB_TRY(attention_launch(D / e->heads, e->m_qkv_att, e->m_qkv_att_tail, ap, st));
      e->prof.end(st);
    }
    const bool last = (i + 1 == e->depth);
    const int L = i + 1;
    ChainParams p; ChainMaps m;
    base(p);
    phase(p, m, 0, e->m_attn, b.proj, e->o_x, EPI_F32_ADD, nullptr, 0, counters(L, 0));
    p.ln[0] = {counters(L, 0), nD, b.ln2_g, b.ln2_b, counters(L, 1)};
    phase(p, m, 1, e->m_xn, b.fc1, e->o_hid, e->gelu_erf ? EPI_BF16_GELU_ERF : EPI_BF16_GELU, counters(L, 1), 0, counters(L, 2));
    phase(p, m, 2, e->m_hid, b.fc2, e->o_x, EPI_F32_ADD, counters(L, 2), n4D, counters(L, 3));
    p.ln[1] = {counters(L, 3), nD, last ? e->lnf_g : e->blocks[i + 1].ln1_g, last ? e->lnf_b : e->blocks[i + 1].ln1_b, counters(L, 4)};
    p.num_ln = 2;
    if (!last) {
      phase(p, m, 3, e->m_xn, e->blocks[i + 1].qkv, e->o_qkv, EPI_BF16, counters(L, 4), 0, nullptr);
      p.num_phases = 4;
    } else {
      m.a[3] = m.a[0]; m.w[3] = m.w[0]; m.out[3] = m.out[0];
      p.num_phases = 3;
    }
    e->prof.begin(KC_CHAIN, st);
    VPB_TRY(chain_launch(bn, m, p, st));
    e->prof.end(st);
  }
  return VPB_OK;
}

// Tile width of a standalone GEMM launch with a TMA epilogue, from the widths in kTileWidths that divide N.  A persistent launch
// of T tiles on S SMs runs ceil(T / S) waves, and a tile costs about its width, so the rule takes the width with the least
// ceil(num_m * N / BN / S) * BN.  At 1 crop (2 row blocks) that is 128: the narrow tile gives the most CTAs.  Ties go to the
// later entry of kTileWidths: 192, then 256, then 128.  Measured on an H100 80GB HBM3 (700 W power limit), us per launch
// (tools/gemm_width_ab.py), the three-way ties: ViT-B fc1 at 64 crops 101.1 / 100.4 / 104.0 (128 / 192 / 256), ViT-L qkv at
// 64 crops 123.9 / 118.7 / 119.2; 128 against 256: ViT-B qkv at 8 crops 13.0 / 12.2, ViT-L fc2 at 64 crops 176.6 / 159.6,
// ViT-H fc2 at 32 crops 147.9 / 125.3, ViT-H proj at 32 crops 52.1 / 52.0, ViT-L proj at 64 crops 69.3 / 75.7 (the one tie
// the narrow tile wins).  Debug overrides (vpb_debug_gemm): flag 8 forces 128-wide tiles, flag 16 the widest width N allows,
// and flags >> 8 = W forces width W.  The accumulation order of an output element does not depend on the tile width: every
// choice is bit-identical.
static int pick_tile(const LinearW& L, int M, int* bn, const CUtensorMap** wm) {
  const int num_m = cdiv(M, GEMM_BM), sms = num_sms();
  const int forced = (g_dbg_flags & 8) ? 128 : (g_dbg_flags >> 8);
  *bn = 0;
  long long best = 0;
  for (int i = 0; i < 3; ++i) {
    const int w = kTileWidths[i];
    if (!L.has[i] || (forced && w != forced)) continue;
    const long long cost = static_cast<long long>(cdiv(static_cast<long long>(num_m) * cdiv(L.n, w), sms)) * w;
    if ((g_dbg_flags & 16) ? w > *bn : (*bn == 0 || cost <= best)) { *bn = w; best = cost; }
  }
  if (*bn == 0) return fail(VPB_ERR_ARG, "gemm: no tile width for N=%d (forced width %d)", L.n, forced);
  *wm = L.tile_map(*bn);
  return VPB_OK;
}

// fc2 of a multi-head call on an engine with experts: the shared columns [0, D-P) for all rows (the standalone GEMM, its
// output map bounded to those columns), then the expert columns of every segment in one grouped launch (expert_gemm.cuh)
// The shared columns: x[:, :S] += A Ws^T + bias over all M rows, `o_xs` = x [M, S] with the row pitch of x (D).
static int fc2_shared_launch(const LinearW& Ls, int M, int D, float* x, const CUtensorMap& ta, const CUtensorMap& o_xs, cudaStream_t st) {
  GemmParams p = gp(M, Ls.n, Ls.k, Ls.b, x, D);
  p.rmw = 0;                          // TMA reduce-add: the rmw epilogue bounds columns by ldc, not N (bit-identical either way)
  int bn;
  const CUtensorMap* wm;
  VPB_TRY(pick_tile(Ls, M, &bn, &wm));
  return gemm_launch(bn, EPI_F32_ADD, ta, *wm, o_xs, p, st);
}
// The grouped expert launch's parameters without segments (add_expert_segment appends them): K = 4D, the P expert columns
// [D-P, D) of x, W and bias stacked as [shared (D-P rows); expert 0 (P); ...].
static ExpertParams expert_params(int D, int P, const float* bias, float* x) {
  ExpertParams q;
  memset(&q, 0, sizeof(q));
  q.K = 4 * D; q.P = P; q.col0 = D - P; q.ldx = D; q.w_row0 = D - P; q.n_tiles = P / expert_width(P);
  q.bias = bias; q.x = x; q.stages = g_dbg_stages;
  return q;
}
// rows [row_begin, row_end) use `expert`; first_tile = the prefix sum of the earlier segments' tile counts
static void add_expert_segment(ExpertParams& q, int row_begin, int row_end, int expert) {
  ExpertSegment& t = q.seg[q.num_segs++];
  t.row_begin = row_begin; t.row_end = row_end; t.expert = expert; t.first_tile = q.num_tiles;
  q.num_tiles += cdiv(row_end - row_begin, GEMM_BM) * q.n_tiles;
}
static int fc2_experts(vpb_engine* e, const BlockW& b, int M, const std::vector<Segment>& segs, cudaStream_t st) {
  const int D = e->D, P = e->P;
  e->prof.begin(KC_GEMM_FC2, st);
  VPB_TRY(fc2_shared_launch(b.fc2s, M, D, e->x, e->m_hid, e->o_xs, st));
  e->prof.end(st);
  ExpertParams q = expert_params(D, P, b.fc2.b, e->x);
  int row = 0;
  for (const Segment& sg : segs) {
    add_expert_segment(q, row, row + sg.count * 192, sg.head);
    row += sg.count * 192;
  }
  e->prof.begin(KC_GEMM_FC2, st);
  VPB_TRY(expert_launch(e->expert_bn, e->m_hid, b.m_exp, q, st));
  e->prof.end(st);
  return VPB_OK;
}

// Whether the unchained backbone runs each block's qkv GEMM and attention as ONE launch (qkv_attention.cuh) at B model crops:
// head_dim 64 (ViT-B, ViT-L) with at least two items (crop, head) per SM.  The fused launch has B * heads items, one CTA per SM
// at most, where the standalone qkv GEMM spreads 128 x BN tiles over every SM, so small batches stay with the two launches.
// Measured on an H100 80GB HBM3 (700 W power limit), ms per keypoint call with its CUDA graph, separate / fused
// (tools/qkv_attention_ab.py, median of 3):
//   ViT-B   1 crop 0.85 / 0.91, 2: 0.85 / 0.90, 4: 1.02 / 0.98, 8: 1.46 / 1.31, 11: 1.74 / 1.52, 16: 2.19 / 2.01, 32: 4.06 / 3.50,
//           64: 6.09 / 5.76
//   ViT-L   1 crop 1.77 / 1.95, 2: 1.85 / 2.01, 4: 2.39 / 2.22, 8: 3.46 / 2.99, 16: 5.58 / 5.20, 32: 10.11 / 9.65, 64: 18.21 / 17.31
//   ViT-S   0.96 to 1.04 of the separate time from 1 to 64 crops, within the run-to-run spread: no gain, so head_dim 32 stays unfused
//   ViT-H   slower fused at every batch (1 crop 2.78 / 3.67, 16: 9.80 / 9.85, 64: 36.2 / 37.7): at head_dim 80 the shared memory
//           leaves two ring stages, too few to keep the MMAs fed, so head_dim 80 stays unfused
// With the threshold at one item per SM (ViT-B 11 crops), bench.py --config ap10k-streams (16 calls of Poisson(10) ViT-B crops per
// step) ran 18.16 ms per step against 17.92 with every call unfused (two runs each, alternating), although the calls timed alone
// favour fusing from 4 crops up; at two items per SM (ViT-B 22 crops, ViT-L 17) those ragged calls keep the two launches and
// b17x64 / l25x64 fuse.  The ln_in_gemm mini-chains and stop_after keep the two launches.  Bit-identical either way
// (tests/test_gpu_qkv_attention.py); vpb_debug_attention can force either form.
static bool fuse_qkv_attention(const vpb_engine* e, int B) {
  if ((e->ln_in_gemm && !e->ln_fused) || e->stop_after) return false;
  if (g_att_form) return g_att_form == 1;
  return e->D / e->heads == 64 && B * e->heads >= 2 * num_sms();
}

// everything after the patch gather, up to last_norm.  `segs` (a multi-head call): the heads of the crops, in runs
static int backbone(vpb_engine* e, int B, cudaStream_t st, const std::vector<Segment>* segs = nullptr) {
  const int D = e->D, M = B * 192;
  const int stop = e->stop_after;
  if (stop == 1) return VPB_OK;
  // multi-head calls run unchained (bit-identical to the chained form); with experts the LayerNorm after fc2 cannot ride in the
  // fc2 tail (two launches write x) and runs standalone, bit-identical to the fused tail
  const bool experts = segs != nullptr && e->P > 0;
  const bool ln_fused = e->ln_fused;
  if (e->use_chain && B >= e->chain_min_batch && !stop && !e->ln_fused && !segs) return backbone_chained(e, B, st);
  // LayerNorm i is produced either by its own kernel or (ln_fused) by the tail of the GEMM that completes x
  auto fuse_ln = [&](GemmParams& p, const float* g, const float* b) {
    if (!ln_fused) return;
    p.ln_gamma = g; p.ln_beta = b; p.ln_out = e->xn; p.ln_counters = e->ln_counters; p.ln_eps = 1e-6f;
  };
  auto standalone_ln = [&](const float* g, const float* b) -> int {
    if (ln_fused) return VPB_OK;
    e->prof.begin(KC_LN, st);
    VPB_TRY(layernorm(e->x, g, b, e->xn, M, D, 1e-6f, st));
    e->prof.end(st);
    return VPB_OK;
  };
  // LayerNorm(x; g, b) -> xn followed by xn * W^T + bias (epilogue epi) as one chained launch: one LayerNorm stage whose source
  // rows are already complete (target 0) and one GEMM phase that waits for the normalised rows of its tile
  const bool mini = e->ln_in_gemm && !ln_fused && !stop;
  const bool fused = fuse_qkv_attention(e, B);
  const size_t nblk = e->chain_blocks;
  if (mini) CU_TRY(cudaMemsetAsync(e->chain_counters, 0, static_cast<size_t>(e->depth + 1) * 5 * nblk * sizeof(int), st));
  auto ln_gemm = [&](const float* g, const float* b, const LinearW& L, const CUtensorMap& out, int epi, int slot, int kclass) -> int {
    ChainParams p; ChainMaps m;
    memset(&p, 0, sizeof(p));
    p.M = M; p.D = D; p.x = e->x; p.xn = e->xn; p.eps = 1e-6f; p.wave_lag[0] = p.wave_lag[1] = 1 << 20; p.dbg = nullptr;
    p.ln_ctl = e->ln_ctl; p.ln_job_rows = e->ln_job_rows;
    int* ready = e->chain_counters + static_cast<size_t>(slot) * nblk;
    p.ln[0] = {ready, 0, g, b, ready};                      // source counter: any valid address, target 0 = "already complete"
    p.num_ln = 1; p.num_phases = 1;
    for (int i = 0; i < CHAIN_MAX_PHASES; ++i) { m.a[i] = e->m_xn; m.w[i] = L.map_c; m.out[i] = out; }
    p.ph[0].N = L.n; p.ph[0].K = L.k; p.ph[0].epi = epi; p.ph[0].bias = L.b; p.ph[0].a_ready = ready; p.ph[0].a_target = 0; p.ph[0].out_done = nullptr;
    e->prof.begin(kclass, st);
    VPB_TRY(chain_launch(e->chain_bn, m, p, st));
    e->prof.end(st);
    return VPB_OK;
  };
  {  // tokens += rows * Wpatch^T; the stream was seeded with pos_embed[1+t] + pos_embed[0] + conv bias by the gather
    GemmParams p = gp(M, D, 768, e->patch.b, e->x, D);   // patch.b is a zero vector (the conv bias lives in pos_bias)
    fuse_ln(p, e->blocks[0].ln1_g, e->blocks[0].ln1_b);
    e->prof.begin(KC_GEMM_PATCH, st);
    int bn;
    const CUtensorMap* wm;
    VPB_TRY(pick_tile(e->patch, M, &bn, &wm));
    p.rmw = resid_rmw(e->resid_rmw);
    VPB_TRY(gemm_launch(bn, EPI_F32_ADD, e->m_patch_rows, *wm, e->o_x, p, st));
    e->prof.end(st);
  }
  if (stop == 2) return VPB_OK;
  for (int i = 0; i < e->depth; ++i) {
    BlockW& b = e->blocks[i];
    if (mini) {
      VPB_TRY(ln_gemm(b.ln1_g, b.ln1_b, b.qkv, e->o_qkv, EPI_BF16, i * 5 + 4, KC_GEMM_QKV));
    } else {
    VPB_TRY(standalone_ln(b.ln1_g, b.ln1_b));
    if (stop == 3) return VPB_OK;
    e->prof.begin(KC_GEMM_QKV, st);
    if (fused) {                                        // qkv + attention: the profile's gemm_qkv then includes the attention
      QkvAttnParams qp;
      qp.batch = B; qp.heads = e->heads; qp.dim = D; qp.bias = b.qkv.b; qp.out = e->attn; qp.dbg = nullptr;
      VPB_TRY(qkv_attention_launch(D / e->heads, e->m_xn_att, b.m_qkv_head, qp, st));
    } else {
      int bn;
      const CUtensorMap* wm;
      VPB_TRY(pick_tile(b.qkv, M, &bn, &wm));
      VPB_TRY(gemm_launch(bn, EPI_BF16, e->m_xn, *wm, e->o_qkv, gp(M, 3 * D, D, b.qkv.b, e->qkv, 3 * D), st));
    }
    e->prof.end(st);
    }
    if (stop == 4) return VPB_OK;
    if (!fused) {
      AttnParams ap;
      ap.batch = B; ap.heads = e->heads; ap.dim = D; ap.out = e->attn; ap.dbg = nullptr;
      e->prof.begin(KC_ATTN, st);
      VPB_TRY(attention_launch(D / e->heads, e->m_qkv_att, e->m_qkv_att_tail, ap, st));
      e->prof.end(st);
    }
    if (stop == 5) return VPB_OK;
    {
      GemmParams p = gp(M, D, D, b.proj.b, e->x, D);     // x += attn * Wproj^T + b   (TMA reduce-add into the fp32 stream) [+ norm2]
      fuse_ln(p, b.ln2_g, b.ln2_b);
      e->prof.begin(KC_GEMM_PROJ, st);
      int bn;
      const CUtensorMap* wm;
      VPB_TRY(pick_tile(b.proj, M, &bn, &wm));
      p.rmw = resid_rmw(e->resid_rmw);
      VPB_TRY(gemm_launch(bn, EPI_F32_ADD, e->m_attn, *wm, e->o_x, p, st));
      e->prof.end(st);
    }
    if (stop == 6) return VPB_OK;
    if (mini) {
      VPB_TRY(ln_gemm(b.ln2_g, b.ln2_b, b.fc1, e->o_hid, e->gelu_erf ? EPI_BF16_GELU_ERF : EPI_BF16_GELU, (i + 1) * 5 + 1, KC_GEMM_FC1));
    } else {
    VPB_TRY(standalone_ln(b.ln2_g, b.ln2_b));
    e->prof.begin(KC_GEMM_FC1, st);
    {
      int bn;
      const CUtensorMap* wm;
      VPB_TRY(pick_tile(b.fc1, M, &bn, &wm));
      VPB_TRY(gemm_launch(bn, e->gelu_erf ? EPI_BF16_GELU_ERF : EPI_BF16_GELU, e->m_xn, *wm, e->o_hid, gp(M, 4 * D, D, b.fc1.b, e->hid, 4 * D), st));
    }
    e->prof.end(st);
    }
    if (stop == 7) return VPB_OK;
    if (experts) {
      VPB_TRY(fc2_experts(e, b, M, *segs, st));
      if (ln_fused) {
        const bool last = i + 1 == e->depth;
        e->prof.begin(KC_LN, st);
        VPB_TRY(layernorm(e->x, last ? e->lnf_g : e->blocks[i + 1].ln1_g, last ? e->lnf_b : e->blocks[i + 1].ln1_b, e->xn, M, D, 1e-6f, st));
        e->prof.end(st);
      }
    } else {
      GemmParams p = gp(M, D, 4 * D, b.fc2.b, e->x, D);  // [+ norm1 of the next block, or last_norm]
      if (i + 1 < e->depth) fuse_ln(p, e->blocks[i + 1].ln1_g, e->blocks[i + 1].ln1_b);
      else fuse_ln(p, e->lnf_g, e->lnf_b);
      e->prof.begin(KC_GEMM_FC2, st);
      int bn;
      const CUtensorMap* wm;
      VPB_TRY(pick_tile(b.fc2, M, &bn, &wm));
      p.rmw = resid_rmw(e->resid_rmw);
      VPB_TRY(gemm_launch(bn, EPI_F32_ADD, e->m_hid, *wm, e->o_x, p, st));
      e->prof.end(st);
    }
    if (stop == 8) return VPB_OK;
  }
  if (stop == 9) return VPB_OK;
  return standalone_ln(e->lnf_g, e->lnf_b);
}

// Head j on crops c0 .. c0+B-1 of the workspace -> heatmaps of crop c at d_heat + c * ch_stride maps (ch_stride = the head's K
// for the single-head calls, K_max for a multi-head call).  A deconv tile never straddles a crop, so a segment of crops is the
// same launches on A maps and outputs that start at crop c0; the crop-0 maps are the engine's own.
static int head(vpb_engine* e, int B, float* d_heat, cudaStream_t st, int j = 0, int c0 = 0, int ch_stride = 0) {
  const int D = e->D;
  const int stop = e->stop_after;
  const HeadW& h = e->hw[j];
  CUtensorMap feat = e->m_feat_nhwc, d1 = e->m_d1_nhwc, d2 = e->m_d2;
  if (c0 > 0) {
    VPB_TRY(make_map_nhwc(&feat, e->xn + static_cast<size_t>(c0) * 192 * D, B, 16, 12, D, 8, 12));
    VPB_TRY(make_map_nhwc(&d1, e->d1 + static_cast<size_t>(c0) * 768 * 256, B, 32, 24, 256, 16, 8));
    VPB_TRY(make_map(&d2, e->d2 + static_cast<size_t>(c0) * 3072 * 256, static_cast<uint64_t>(B) * 3072, 256, 256, 128));
  }
  {  // deconv 1: tokens as NHWC 16x12xD -> d1 NHWC 32x24x256, all four sub-pixel phases in one implicit-GEMM launch
    GemmParams p = gp(B * 192, 256, 4 * D, h.dc1.b, e->d1 + static_cast<size_t>(c0) * 768 * 256, 256);
    p.up_h = 16; p.up_w = 12; p.up_tr = 8; p.up_tw = 12; p.up_c = D;
    e->prof.begin(KC_GEMM_DECONV, st);
    VPB_TRY(gemm_launch(256, EPI_BF16_RELU_UP, feat, *h.dc1.tile_map(256), e->m_xn, p, st));
    e->prof.end(st);
  }
  if (stop == 11) return VPB_OK;
  {  // deconv 2: d1 -> d2 NHWC 64x48x256
    GemmParams p = gp(B * 768, 256, 1024, h.dc2.b, e->d2 + static_cast<size_t>(c0) * 3072 * 256, 256);
    p.up_h = 32; p.up_w = 24; p.up_tr = 16; p.up_tw = 8; p.up_c = 256;
    e->prof.begin(KC_GEMM_DECONV, st);
    VPB_TRY(gemm_launch(256, EPI_BF16_RELU_UP, d1, *h.dc2.tile_map(256), e->m_xn, p, st));
    e->prof.end(st);
  }
  if (stop == 12) return VPB_OK;
  {
    GemmParams p = gp(B * 3072, h.n_final, 256, h.fin.b, d_heat, 0);
    p.n_valid = h.K; p.pix = 3072; p.ch_stride = ch_stride;
    e->prof.begin(KC_GEMM_FINAL, st);
    VPB_TRY(gemm_launch(h.n_final, EPI_F32_NCHW, d2, h.m_fin_w, d2, p, st));
    e->prof.end(st);
  }
  return VPB_OK;
}

static int apply_l2_policy(vpb_engine* e, cudaStream_t st) {
  if (!e->l2_persist || e->l2_window_bytes == 0) return VPB_OK;
  for (cudaStream_t s : e->l2_streams) if (s == st) return VPB_OK;
  cudaStreamAttrValue v;
  memset(&v, 0, sizeof(v));
  v.accessPolicyWindow.base_ptr = e->x;
  v.accessPolicyWindow.num_bytes = e->l2_window_bytes;
  v.accessPolicyWindow.hitRatio = 1.0f;
  v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  CU_TRY(cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v));
  e->l2_streams.push_back(st);
  return VPB_OK;
}

static bool stream_is_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (st == nullptr) return false;                              // the legacy default stream cannot be captured
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); return false; }
  return cs != cudaStreamCaptureStatusNone;
}
// Workspace hand-over between streams (see vpb_engine::ev_ws).  Inside a caller-side stream capture the events are left
// alone (a wait on an event recorded outside the capture would be a cross-capture dependency): the caller then owns the
// ordering of that graph against the engine's other users.
//
// Chained launches add a per-DEVICE rule.  A chained kernel (chain.cuh) spins on counters that other clusters of the same
// launch advance, so every cluster of its grid has to become resident; two chained kernels of two engines sharing one GPU on
// two streams could each hold part of the SMs and wait for the rest forever.  Calls that may launch chained kernels are
// therefore serialised per device: the enqueue runs under the device's gate mutex (engines driven from different host
// threads) and waits for the event the previous chained call on that device recorded when it came from another engine or
// stream.  Other processes on the same GPU (MPS) are outside this gate: run chained engines with the GPU to themselves, or
// switch the chain off (option "chain" = 0).
struct ChainGate {
  std::mutex mu;
  cudaEvent_t ev = nullptr;
  const vpb_engine* owner = nullptr;
  cudaStream_t st = nullptr;
};
static ChainGate g_gates[kMaxDevices];

struct WsScope {
  vpb_engine* e;
  cudaStream_t st;
  bool capturing = false;
  ChainGate* gate = nullptr;
  std::unique_lock<std::mutex> lk;
  WsScope(vpb_engine* e_, cudaStream_t st_) : e(e_), st(st_) {}
  int begin(int batch) {
    capturing = stream_is_capturing(st);
    if (e->ws_used && e->ws_last != st && !capturing) CU_TRY(cudaStreamWaitEvent(st, e->ev_ws, 0));
    if (!e->ln_fused && !e->stop_after && ((e->use_chain && batch >= e->chain_min_batch) || e->ln_in_gemm)) {   // any chained kernel ahead
      const int dev = e->cfg.device;
      gate = &g_gates[dev >= 0 && dev < kMaxDevices ? dev : 0];
      lk = std::unique_lock<std::mutex>(gate->mu);
      if (!capturing && gate->ev && (gate->owner != e || gate->st != st)) CU_TRY(cudaStreamWaitEvent(st, gate->ev, 0));
    }
    return VPB_OK;
  }
  int end() {
    if (capturing) return VPB_OK;
    CU_TRY(cudaEventRecord(e->ev_ws, st));
    e->ws_last = st; e->ws_used = true;
    if (gate) {
      if (!gate->ev) CU_TRY(cudaEventCreateWithFlags(&gate->ev, cudaEventDisableTiming));
      CU_TRY(cudaEventRecord(gate->ev, st));
      gate->owner = e; gate->st = st;
    }
    return VPB_OK;
  }
};

// Makes the engine's device current for the scope of an entry point and restores the caller's afterwards, so engines on
// different GPUs can be driven from one thread (the stream argument must belong to the engine's device).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(const vpb_engine* e) {
    int cur = -1;
    if (e && cudaGetDevice(&cur) == cudaSuccess && cur != e->cfg.device && cudaSetDevice(e->cfg.device) == cudaSuccess) prev = cur;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int check_ready(vpb_engine* e, int batch) {
  if (!e) return fail(VPB_ERR_ARG, "null engine");
  if (!e->finalized) return fail(VPB_ERR_STATE, "weights not finalized: call vpb_finalize first");
  if (batch < 1 || batch > e->maxB) return fail(VPB_ERR_ARG, "batch %d outside 1..max_batch=%d", batch, e->maxB);
  return VPB_OK;
}
// the keypoint entry points: with flip test on, the batch and its mirror images share the max_batch workspace
static int check_ready_keypoints(vpb_engine* e, int batch) {
  VPB_TRY(check_ready(e, batch));
  if (e->flip && 2 * batch > e->maxB)
    return fail(VPB_ERR_ARG, "batch %d: with flip test on a call takes at most max_batch / 2 = %d crops (max_batch=%d)", batch, e->maxB / 2, e->maxB);
  return VPB_OK;
}

extern "C" int vpb_forward(vpb_engine* e, const float* d_crops, int32_t batch, float* d_heatmaps, void* stream) {
  VPB_TRY(check_ready(e, batch));
  DeviceGuard dev_guard(e);
  if (!d_crops || !d_heatmaps) return fail(VPB_ERR_ARG, "vpb_forward: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  VPB_TRY(apply_l2_policy(e, st));
  WsScope ws(e, st);
  VPB_TRY(ws.begin(batch));
  VPB_TRY(patch_gather(e, d_crops, batch, batch, st));
  VPB_TRY(backbone(e, batch, st));
  if (!(e->stop_after && e->stop_after <= 10)) VPB_TRY(head(e, batch, d_heatmaps, st));
  return ws.end();
}

extern "C" int vpb_forward_features(vpb_engine* e, const float* d_crops, int32_t batch, float* d_features, void* stream) {
  VPB_TRY(check_ready(e, batch));
  DeviceGuard dev_guard(e);
  if (!d_crops || !d_features) return fail(VPB_ERR_ARG, "vpb_forward_features: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  WsScope ws(e, st);
  VPB_TRY(ws.begin(batch));
  VPB_TRY(patch_gather(e, d_crops, batch, batch, st));
  VPB_TRY(backbone(e, batch, st));
  const long long tot = static_cast<long long>(batch) * e->D * 192;
  tokens_to_nchw<<<cdiv(tot, 256), 256, 0, st>>>(e->xn, d_features, batch, e->D);
  CU_TRY(cudaGetLastError());
  return ws.end();
}

static int decode_launch(const float* d_heatmaps, int32_t n, int32_t k, const int32_t* d_org_wh, const int32_t* d_offs_yx, float* d_kpts,
                         int32_t* d_idx, int32_t wrap_batch, void* stream) {
  if (!d_heatmaps || !d_org_wh || !d_kpts) return fail(VPB_ERR_ARG, "vpb_decode: null pointer");
  if (n < 0 || k < 1) return fail(VPB_ERR_ARG, "vpb_decode: n=%d k=%d", n, k);
  if (n == 0) return VPB_OK;
  DecodeParams p;
  p.heatmaps = d_heatmaps; p.org_wh = d_org_wh; p.kpts = d_kpts; p.idx = d_idx; p.n = n; p.k = k; p.wrap_batch = wrap_batch;
  p.offs_yx = d_offs_yx;
  launch_k(decode_heatmaps<false>, dim3(cdiv(static_cast<long long>(n) * k, DECODE_WARPS)), dim3(DECODE_WARPS * 32), 0, static_cast<cudaStream_t>(stream), p);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_decode(const float* d_heatmaps, int32_t n, int32_t k, const int32_t* d_org_wh, float* d_kpts, int32_t* d_idx,
                          int32_t wrap_batch, void* stream) {
  return decode_launch(d_heatmaps, n, k, d_org_wh, nullptr, d_kpts, d_idx, wrap_batch, stream);
}
// keypoint_head(features): TopdownHeatmapSimpleHead.forward (head/topdown_heatmap_simple_head.py:188-193) on backbone features
extern "C" int vpb_head(vpb_engine* e, const float* d_features, int32_t batch, float* d_heatmaps, void* stream) {
  VPB_TRY(check_ready(e, batch));
  DeviceGuard dev_guard(e);
  if (!d_features || !d_heatmaps) return fail(VPB_ERR_ARG, "vpb_head: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long tot = static_cast<long long>(batch) * e->D * 192;
  WsScope ws(e, st);
  VPB_TRY(ws.begin(0));                                     // the head launches no chained kernel
  nchw_to_tokens<<<cdiv(tot, 256), 256, 0, st>>>(d_features, e->xn, batch, e->D);
  CU_TRY(cudaGetLastError());
  VPB_TRY(head(e, batch, d_heatmaps, st));
  return ws.end();
}
extern "C" int vpb_flip_back(const float* d_in, int32_t n, int32_t k, const int32_t* d_perm, int32_t shift, float* d_out, void* stream) {
  if (!d_in || !d_out || !d_perm || d_in == d_out) return fail(VPB_ERR_ARG, "vpb_flip_back: null or aliased pointers");
  if (n < 0 || k < 1) return fail(VPB_ERR_ARG, "vpb_flip_back: n=%d k=%d", n, k);
  if (n == 0) return VPB_OK;
  const long long tot = static_cast<long long>(n) * k * 3072;
  flip_back_heatmaps<<<cdiv(tot, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d_in, d_out, d_perm, n, k, shift);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}
// cv2.getGaussianKernel(ksize, sigma <= 0) for a CV_32F image: sigma = 0.3 * ((ksize - 1) * 0.5 - 1) + 0.8, exp(-d^2 / (2 sigma^2))
// normalised to sum 1 in double, stored as float; indexed by the distance from the centre.  ksize odd, 1..35; for 9 taps and
// fewer cv2 returns fixed tables instead (small_gaussian_tab; pinned against cv2 in oracle/make_golden_modes_small.py).
static bool gauss_taps(int ksize, GaussTaps& tp) {
  if (ksize < 1 || ksize > 2 * MAX_RADIUS + 1 || ksize % 2 == 0) return false;
  const int r = ksize / 2;
  if (ksize <= 9) {
    static const float small[5][5] = {{1.0f},
                                      {0.5f, 0.25f},
                                      {0.375f, 0.25f, 0.0625f},
                                      {0.28125f, 0.21875f, 0.109375f, 0.03125f},
                                      {60.0f / 256, 51.0f / 256, 30.0f / 256, 13.0f / 256, 4.0f / 256}};
    tp.radius = r;
    for (int d = 0; d <= r; ++d) tp.t[d] = small[r][d];
    return true;
  }
  const double sigma = 0.3 * ((ksize - 1) * 0.5 - 1.0) + 0.8;
  double v[2 * MAX_RADIUS + 1], sum = 0.0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) / 2.0;
    v[i] = std::exp(-(x * x) / (2.0 * sigma * sigma));
    sum += v[i];
  }
  tp.radius = r;
  for (int d = 0; d <= r; ++d) tp.t[d] = static_cast<float>(v[r + d] / sum);
  return true;
}

extern "C" int vpb_decode_modes_ex(const float* d_heatmaps, int32_t n, int32_t k, int32_t mode, int32_t kernel, float valid_radius,
                                   const float* d_cs32, const double* d_cs64, float* d_kpts, int32_t* d_idx, void* stream) {
  if (!d_heatmaps || !d_kpts || (d_cs32 == nullptr) == (d_cs64 == nullptr))
    return fail(VPB_ERR_ARG, "vpb_decode_modes: null pointer, or not exactly one of d_cs32 / d_cs64");
  if (n < 0 || k < 1 || mode < DECODE_NONE || mode > DECODE_COMBINED) return fail(VPB_ERR_ARG, "vpb_decode_modes: n=%d k=%d mode=%d", n, k, mode);
  const bool blurs = mode >= DECODE_UNBIASED;
  GaussTaps taps, wide;
  if (blurs && !gauss_taps(kernel, taps)) return fail(VPB_ERR_ARG, "vpb_decode_modes: kernel=%d (odd, 1..%d)", kernel, 2 * MAX_RADIUS + 1);
  if (kernel == 1 && (mode == DECODE_UNBIASED || mode == DECODE_MEGVII))     // the reference's _gaussian_blur raises (border = 0)
    return fail(VPB_ERR_ARG, "vpb_decode_modes: kernel=1 has no zero-bordered blur (top_down_eval.py:443-455 raises)");
  if (mode == DECODE_COMBINED && !gauss_taps(2 * kernel + 1, wide))
    return fail(VPB_ERR_ARG, "vpb_decode_modes: CombinedTarget blurs with 2*kernel+1 = %d (limit %d)", 2 * kernel + 1, 2 * MAX_RADIUS + 1);
  if (n == 0) return VPB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (mode == DECODE_DARK_UDP) {                            // one reference call on the whole array: wrap_batch = 1
    DecodeParams p;
    p.heatmaps = d_heatmaps; p.org_wh = nullptr; p.kpts = d_kpts; p.idx = d_idx; p.n = n; p.k = k; p.wrap_batch = 1; p.offs_yx = nullptr;
    p.cs32 = d_cs32; p.cs64 = d_cs64; p.taps = taps;
    const dim3 grid(cdiv(static_cast<long long>(n) * k, DECODE_WARPS)), block(DECODE_WARPS * 32);
    if (kernel == 11) { CU_TRY(launch_k(decode_heatmaps<false>, grid, block, 0, st, p)); }
    else              { CU_TRY(launch_k(decode_heatmaps<true>, grid, block, 0, st, p)); }
  } else {
    DecodeModesParams p;
    p.heatmaps = d_heatmaps; p.cs32 = d_cs32; p.cs64 = d_cs64; p.kpts = d_kpts; p.idx = d_idx; p.n = n; p.k = k; p.mode = mode;
    p.taps = taps; p.taps_wide = wide; p.valid_radius = valid_radius;
    CU_TRY(launch_k(decode_modes, dim3(n * k), dim3(256), 0, st, p));
  }
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_decode_modes(const float* d_heatmaps, int32_t n, int32_t k, int32_t mode, const float* d_cs32, const double* d_cs64,
                                float* d_kpts, int32_t* d_idx, void* stream) {
  if (mode == DECODE_COMBINED) return fail(VPB_ERR_ARG, "vpb_decode_modes: CombinedTarget needs vpb_decode_modes_ex (valid_radius)");
  return vpb_decode_modes_ex(d_heatmaps, n, k, mode, 11, 0.0f, d_cs32, d_cs64, d_kpts, d_idx, stream);
}
extern "C" int vpb_decode_frame(const float* d_heatmaps, int32_t n, int32_t k, const int32_t* d_org_wh, const int32_t* d_offs_yx,
                                float* d_kpts, int32_t* d_idx, int32_t wrap_batch, void* stream) {
  return decode_launch(d_heatmaps, n, k, d_org_wh, d_offs_yx, d_kpts, d_idx, wrap_batch, stream);
}

// Crops one keypoint call runs through the model: the batch, and with flip test on its mirror images as well.
static int model_crops(const vpb_engine* e, int batch) { return e->flip ? 2 * batch : batch; }

// Flip test: `raw` holds the raw maps of one forward, crop c at raw + c * kstride maps and its mirror image `mirror` crops
// later; `out` (same layout; may be `raw`) gets the flip-back average of the first `batch` crops, with head permutation `perm`
// of k keypoints.
static int flip_average(vpb_engine* e, const float* raw, int batch, int k, const int* perm, int kstride, int mirror, float* out,
                        cudaStream_t st) {
  const long long tot = static_cast<long long>(batch) * k * 3072;
  e->prof.begin(KC_DECODE, st);
  CU_TRY(launch_k(flip_average_heatmaps, dim3(cdiv(tot, 256)), dim3(256), 0, st, raw, out, perm, batch, k, e->flip_shift, kstride, mirror));
  e->prof.end(st);
  return VPB_OK;
}

// first entry of head j's permutation in flip_perm (the heads' permutations concatenated in head order)
static int perm_offset(const vpb_engine* e, int j) {
  int off = 0;
  for (int i = 0; i < j; ++i) off += e->hw[i].K;
  return off;
}

// The segments the model runs for a call: `segs`, and with flip test on `segs` again for the mirror images (the gathers
// mirror crop b - n into model crop b >= n), runs of one head merged across the seam.
static std::vector<Segment> model_segments(const vpb_engine* e, const std::vector<Segment>& segs) {
  std::vector<Segment> out = segs;
  if (!e->flip) return out;
  for (const Segment& sg : segs) {
    if (out.back().head == sg.head) out.back().count += sg.count;
    else out.push_back(sg);
  }
  return out;
}

// Keypoint rows per crop in a call's outputs: head 0's K for the single-head calls, K_max for the multi-head calls.
static int row_stride(const vpb_engine* e, bool mixed) { return mixed ? e->Kmax : e->K; }

// The keypoint pipeline of every call; a single-head call is the one segment {head 0, n} with kstride = head 0's K.
// Gather (unless done), backbone with the experts of the model segments, then per model segment the head's deconvs + 1x1 conv
// (crop c at c * kstride maps), and per segment the flip-back average (flip test: raw maps in e->heat, average into `heat`)
// and the decode of its K_head maps into kpts [n, kstride, 3] / idx [n, kstride].  d_cs (affine calls): centre / scale,
// decode mode 4 as one reference call per segment; else canvas sizes + offsets, one reference call per crop.  A call whose
// model crops all use head 0 runs the single-head backbone launches.
static int heads_enqueue(vpb_engine* e, const Source* src, const std::vector<Segment>& segs, int n, int kstride, const int32_t* d_org_wh,
                         const int32_t* d_offs_yx, const float* d_cs, float* d_kpts, int32_t* d_idx, float* heat, cudaStream_t st) {
  const std::vector<Segment> msegs = model_segments(e, segs);
  const int nb = model_crops(e, n);
  if (src) VPB_TRY(gather(e, *src, n, nb, st));
  VPB_TRY(backbone(e, nb, st, (msegs.size() == 1 && msegs[0].head == 0) ? nullptr : &msegs));
  if (e->stop_after && e->stop_after <= 10) return VPB_OK;
  float* raw = e->flip ? e->heat : heat;
  int c0 = 0;
  for (const Segment& sg : msegs) {
    VPB_TRY(head(e, sg.count, raw + static_cast<size_t>(c0) * kstride * 3072, st, sg.head, c0, kstride));
    c0 += sg.count;
  }
  if (e->stop_after) return VPB_OK;
  c0 = 0;
  for (const Segment& sg : segs) {
    const size_t m0 = static_cast<size_t>(c0) * kstride * 3072;
    const int K = e->hw[sg.head].K;
    if (e->flip) VPB_TRY(flip_average(e, raw + m0, sg.count, K, e->flip_perm + perm_offset(e, sg.head), kstride, n, heat + m0, st));
    DecodeParams p;
    p.heatmaps = heat + m0; p.org_wh = d_cs ? nullptr : d_org_wh + 2 * c0; p.offs_yx = (d_offs_yx && !d_cs) ? d_offs_yx + 2 * c0 : nullptr;
    p.kpts = d_kpts + static_cast<size_t>(c0) * kstride * 3; p.idx = d_idx ? d_idx + static_cast<size_t>(c0) * kstride : nullptr;
    p.n = sg.count; p.k = K; p.kstride = kstride;
    p.wrap_batch = d_cs ? 1 : 0;                            // mode 4: keypoints_from_heatmaps on the segment's array
    p.cs32 = d_cs ? d_cs + 4 * c0 : nullptr;
    e->prof.begin(KC_DECODE, st);
    CU_TRY(launch_k(decode_heatmaps<false>, dim3(cdiv(static_cast<long long>(p.n) * p.k, DECODE_WARPS)), dim3(DECODE_WARPS * 32), 0, st, p));
    e->prof.end(st);
    c0 += sg.count;
  }
  return VPB_OK;
}

// rows 0 .. K_head-1 of every crop of every segment: [n, kstride, row] -> [n, kstride, row] (rows past K_head are left alone);
// one contiguous copy for a segment whose head's K is the stride, as in every single-head call
static int copy_head_rows(const vpb_engine* e, const std::vector<Segment>& segs, int kstride, void* dst, const void* src, size_t row_bytes,
                          cudaMemcpyKind kind, cudaStream_t st) {
  const size_t pitch = static_cast<size_t>(kstride) * row_bytes;
  size_t off = 0;
  for (const Segment& sg : segs) {
    char* d = static_cast<char*>(dst) + off;
    const char* s = static_cast<const char*>(src) + off;
    const size_t width = e->hw[sg.head].K * row_bytes;
    if (width == pitch) CU_TRY(cudaMemcpyAsync(d, s, sg.count * pitch, kind, st));
    else CU_TRY(cudaMemcpy2DAsync(d, pitch, s, pitch, width, sg.count, kind, st));
    off += sg.count * pitch;
  }
  return VPB_OK;
}

static_assert(2 * VPB_MAX_SEGMENTS <= EXPERT_MAX_SEGMENTS, "a flip-test call's crops and mirror images fit the expert GEMM's table");
constexpr size_t kMaxMixedGraphs = 16;

static void drop_graphs(vpb_engine* e) {
  for (auto& g : e->graph_cache) if (g.exec) cudaGraphExecDestroy(g.exec);
  e->graph_cache.clear();
}

// Graph replay of everything behind the gather (see vpb_engine::graph_cache): eager on a key's first use, captured on its
// second.  The gather runs eagerly in front of the replay; the decode inputs move to g_org / g_offs, or for the affine calls
// the centre / scale to g_cs, and the outputs come back from g_kpts / g_idx / heat.  mixed: a multi-head entry point.
static int heads_core_locked(vpb_engine* e, const Source& src, const std::vector<Segment>& segs, bool mixed, int n, const int32_t* d_org_wh,
                             const int32_t* d_offs_yx, float* d_kpts, int32_t* d_idx, float* d_heatmaps, cudaStream_t st) {
  float* heat = d_heatmaps ? d_heatmaps : e->heat;
  const int ks = row_stride(e, mixed);
  // eager launches on the legacy default stream (cannot be captured) and when the CALLER is already capturing `st`
  // (a nested cudaStreamBeginCapture would fail): the engine's kernels then simply become nodes of the caller's graph
  if (!e->use_graph || e->prof.on || e->stop_after || st == nullptr || stream_is_capturing(st))
    return heads_enqueue(e, &src, segs, n, ks, d_org_wh, d_offs_yx, src.cs, d_kpts, d_idx, heat, st);
  const bool affine = src.cs != nullptr;
  vpb_engine::CachedGraph* g = nullptr;
  for (auto& c : e->graph_cache)
    if (c.mixed == mixed && c.segs == segs && c.affine == affine) g = &c;
  if (!g) {                                                               // first use of this key: run eagerly
    if (mixed) {
      auto lru = e->graph_cache.end();
      size_t count = 0;
      for (auto it = e->graph_cache.begin(); it != e->graph_cache.end(); ++it)
        if (it->mixed) {
          ++count;
          if (lru == e->graph_cache.end() || it->used < lru->used) lru = it;
        }
      if (count == kMaxMixedGraphs) {
        if (lru->exec) cudaGraphExecDestroy(lru->exec);
        e->graph_cache.erase(lru);
      }
    }
    e->graph_cache.push_back({mixed, segs, affine, nullptr, ++e->graph_clock});
    return heads_enqueue(e, &src, segs, n, ks, d_org_wh, d_offs_yx, src.cs, d_kpts, d_idx, heat, st);
  }
  g->used = ++e->graph_clock;
  VPB_TRY(gather(e, src, n, model_crops(e, n), st));
  if (affine) {
    CU_TRY(cudaMemcpyAsync(e->g_cs, src.cs, static_cast<size_t>(n) * 4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  } else {
    CU_TRY(cudaMemcpyAsync(e->g_org, d_org_wh, static_cast<size_t>(n) * 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (d_offs_yx) CU_TRY(cudaMemcpyAsync(e->g_offs, d_offs_yx, static_cast<size_t>(n) * 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    else CU_TRY(cudaMemsetAsync(e->g_offs, 0, static_cast<size_t>(n) * 2 * sizeof(int32_t), st));
  }
  if (!g->exec) {                                                         // second use: capture, instantiate
    cudaGraph_t graph = nullptr;
    CU_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = heads_enqueue(e, nullptr, segs, n, ks, e->g_org, e->g_offs, affine ? e->g_cs : nullptr, e->g_kpts, e->g_idx, e->heat, st);
    const cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != VPB_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) return fail(VPB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
    const cudaError_t ie = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { g->exec = nullptr; return fail(VPB_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(ie)); }
  }
  CU_TRY(cudaGraphLaunch(g->exec, st));
  VPB_TRY(copy_head_rows(e, segs, ks, d_kpts, e->g_kpts, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (d_idx) VPB_TRY(copy_head_rows(e, segs, ks, d_idx, e->g_idx, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (d_heatmaps) VPB_TRY(copy_head_rows(e, segs, ks, d_heatmaps, e->heat, 3072 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return VPB_OK;
}
// crops (or frames + boxes, or affine crops: `src`) -> keypoints; d_offs_yx (nullable) moves the keypoints from crop to frame
// coordinates inside the decode kernel
static int heads_core(vpb_engine* e, const Source& src, const std::vector<Segment>& segs, bool mixed, int n, const int32_t* d_org_wh,
                      const int32_t* d_offs_yx, float* d_kpts, int32_t* d_idx, float* d_heatmaps, cudaStream_t st) {
  VPB_TRY(apply_l2_policy(e, st));
  WsScope ws(e, st);
  VPB_TRY(ws.begin(model_crops(e, n)));
  VPB_TRY(heads_core_locked(e, src, segs, mixed, n, d_org_wh, d_offs_yx, d_kpts, d_idx, d_heatmaps, st));
  return ws.end();
}

// The end of every host call: D2H of the keypoint and argmax rows of staging slot `slot` on `st`, the stream that computed
// them, then ev_done[slot] for the slot's next user; the synchronous forms (sync) wait for it all.
static int host_tail(vpb_engine* e, const std::vector<Segment>& segs, bool mixed, int slot, float* h_kpts, int32_t* h_idx, cudaStream_t st,
                     bool sync) {
  const int ks = row_stride(e, mixed);
  VPB_TRY(copy_head_rows(e, segs, ks, h_kpts, e->kpts[slot], 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (h_idx) VPB_TRY(copy_head_rows(e, segs, ks, h_idx, e->idx[slot], sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU_TRY(cudaEventRecord(e->ev_done[slot], st));
  if (sync) CU_TRY(cudaStreamSynchronize(st));
  return VPB_OK;
}

extern "C" int vpb_infer(vpb_engine* e, const float* d_crops, const int32_t* d_org_wh, int32_t batch, float* d_kpts, int32_t* d_idx,
                         float* d_heatmaps, void* stream) {
  VPB_TRY(check_ready_keypoints(e, batch));
  DeviceGuard dev_guard(e);
  if (!d_crops || !d_org_wh || !d_kpts) return fail(VPB_ERR_ARG, "vpb_infer: null pointer");
  Source src;
  src.crops = d_crops;
  return heads_core(e, src, {{0, batch}}, false, batch, d_org_wh, nullptr, d_kpts, d_idx, d_heatmaps, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ frame-level entry points
extern "C" int vpb_preprocess(const uint8_t* d_frame, int32_t frame_h, int32_t frame_w, int64_t pitch_bytes, const int32_t* d_bboxes,
                              int32_t n, int32_t pad_bbox, float* d_crops, int32_t* d_org_wh, int32_t* d_offs_yx, int32_t* d_status,
                              void* stream) {
  if (!d_frame || !d_bboxes || !d_crops || !d_org_wh || !d_offs_yx) return fail(VPB_ERR_ARG, "vpb_preprocess: null pointer");
  if (frame_h < 1 || frame_w < 1 || n < 0 || pad_bbox < 0) return fail(VPB_ERR_ARG, "vpb_preprocess: frame %dx%d n=%d pad=%d", frame_h, frame_w, n, pad_bbox);
  if (pitch_bytes == 0) pitch_bytes = static_cast<int64_t>(frame_w) * 3;
  if (pitch_bytes < static_cast<int64_t>(frame_w) * 3) return fail(VPB_ERR_ARG, "vpb_preprocess: pitch %lld < 3 * width", static_cast<long long>(pitch_bytes));
  if (n == 0) return VPB_OK;
  PreprocParams p;
  p.frame = d_frame; p.pitch = pitch_bytes; p.fh = frame_h; p.fw = frame_w; p.bboxes = d_bboxes; p.n = n; p.pad = pad_bbox;
  p.crops = d_crops; p.org_wh = d_org_wh; p.offs_yx = d_offs_yx; p.status = d_status;
  crop_resize_normalise<<<dim3(n, PP_H / PP_ROWS), PP_W, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

static_assert(VPB_MAX_FRAMES == FP_MAX_FRAMES, "the header's frame limit is the gather's table size");
// `rotation` sits in what was the structs' tail padding: sizes and the other offsets are those of the structs without it
static_assert(sizeof(vpb_frame) == 32 && offsetof(vpb_frame, num_boxes) == 24 && offsetof(vpb_frame, rotation) == 28,
              "vpb_frame layout");
static_assert(sizeof(vpb_frame_nv12) == 48 && offsetof(vpb_frame_nv12, num_boxes) == 40 && offsetof(vpb_frame_nv12, rotation) == 44,
              "vpb_frame_nv12 layout");
static_assert(sizeof(vpb_frame_yuv) == 56 && offsetof(vpb_frame_yuv, num_boxes) == 48 && offsetof(vpb_frame_yuv, rotation) == 52,
              "vpb_frame_yuv layout");

// Keypoints of the boxes d_bboxes of a frame table, or with d_mats of its affine crops (centre / scale d_cs for the decode;
// the canvas sizes and offsets are then unused).  The crops are never materialised: the gathers write the bf16 patch rows
// directly.  `tab`: num_frames frames with boxes, first_box ascending; the n boxes are in frame order.
template <class Entry>
static int frames_core(vpb_engine* e, const Entry* tab, int num_frames, const int32_t* d_bboxes, const double* d_mats, const float* d_cs,
                       const std::vector<Segment>& segs, bool mixed, int32_t n, float* d_kpts, int32_t* d_idx, cudaStream_t st) {
  Source src;
  set_table(src, tab); src.num_frames = num_frames; src.bboxes = d_bboxes; src.mats = d_mats; src.cs = d_cs;
  return heads_core(e, src, segs, mixed, n, e->pp_org, e->pp_offs, d_kpts, d_idx, nullptr, st);
}

// one packed frame that owns every box of the call
static FrameEntry single_frame(const uint8_t* data, int32_t fh, int32_t fw) {
  FrameEntry f;
  memset(&f, 0, sizeof(f));
  f.data = data; f.pitch = static_cast<long long>(fw) * 3; f.fh = fh; f.fw = fw; f.first_box = 0;
  return f;
}

// The caller's frame array -> the gather's table.  Frames without boxes are left out (they do not count towards
// VPB_MAX_FRAMES).  *n = the total number of boxes, checked against the batch limit.  build_frame_table is the engine-free
// part (vpb_preprocess_affine): at most `limit` boxes.  Per frame type, check_call checks what applies to the whole call and
// table_entry one frame with boxes and its entry (first_box is filled by the caller):
//   vpb_frame        pitch_bytes 0 (packed rows) or >= 3 * width; `fmt` is unused
//   vpb_frame_yuv    the layout's size rules (even width; even height for 4:2:0), pitches 0 (packed) or >= the row's bytes,
//                    the planes the layout uses non-NULL, and a known layout, matrix and range, written into every entry
//   vpb_frame_nv12   the NV12, limited-range vpb_frame_yuv
// and every frame's rotation is 0, 90, 180 or 270 (the entry's rot code); the entry keeps the stored size.
static_assert(VPB_YUV_BT601 == YUV_BT601 && VPB_YUV_BT709 == YUV_BT709 && VPB_YUV_LIMITED == YUV_LIMITED && VPB_YUV_FULL == YUV_FULL,
              "the header's conversion constants are the gather's");
struct YuvFormat { int32_t layout = VPB_YUV_NV12, matrix = VPB_YUV_BT601, range = VPB_YUV_LIMITED; };
static YuvFormat yuv_format(int32_t layout, int32_t matrix, int32_t range) {
  YuvFormat f;
  f.layout = layout; f.matrix = matrix; f.range = range;
  return f;
}
static YuvFormat nv12_format(int32_t matrix) { return yuv_format(VPB_YUV_NV12, matrix, VPB_YUV_LIMITED); }
// vpb_frame*.rotation (degrees counter-clockwise) -> the entries' rot code 0..3, or -1
static int rotation_code(int32_t degrees) {
  switch (degrees) {
    case 0: return 0;
    case 90: return 1;
    case 180: return 2;
    case 270: return 3;
    default: return -1;
  }
}
// the size of a frame's view: stored (height, width), swapped for 90 and 270 degrees
template <class Frame>
static void view_size(const Frame& f, int32_t* h, int32_t* w) {
  const bool swap = rotation_code(f.rotation) & 1;
  *h = swap ? f.width : f.height;
  *w = swap ? f.height : f.width;
}
static int check_call(const char*, const vpb_frame*, const YuvFormat&) { return VPB_OK; }
static int check_call(const char* fn, const vpb_frame_yuv*, const YuvFormat& c) {
  if (c.layout < VPB_YUV_NV12 || c.layout > VPB_YUV_UYVY)
    return fail(VPB_ERR_ARG, "%s: unknown YUV layout %d (VPB_YUV_NV12 .. VPB_YUV_UYVY expected)", fn, c.layout);
  if (c.range != VPB_YUV_LIMITED && c.range != VPB_YUV_FULL)
    return fail(VPB_ERR_ARG, "%s: unknown YUV range %d (VPB_YUV_LIMITED or VPB_YUV_FULL expected)", fn, c.range);
  if (c.matrix != VPB_YUV_BT601 && c.matrix != VPB_YUV_BT709)
    return fail(VPB_ERR_ARG, "%s: unknown YUV matrix %d (VPB_YUV_BT601 or VPB_YUV_BT709 expected)", fn, c.matrix);
  return VPB_OK;
}
static int check_call(const char* fn, const vpb_frame_nv12*, const YuvFormat& c) {
  return check_call(fn, static_cast<const vpb_frame_yuv*>(nullptr), c);
}
static int table_entry(const char* fn, int j, const vpb_frame& f, const YuvFormat&, FrameEntry* t) {
  const long long pitch = f.pitch_bytes ? f.pitch_bytes : 3LL * f.width;
  if (!f.data || f.height < 1 || f.width < 1 || pitch < 3LL * f.width)
    return fail(VPB_ERR_ARG, "%s: frame %d: data %p, %dx%d (w x h), pitch %lld bytes (0 or >= 3 * width expected)", fn, j,
                static_cast<const void*>(f.data), f.width, f.height, static_cast<long long>(f.pitch_bytes));
  memset(t, 0, sizeof(*t));
  t->data = f.data; t->pitch = pitch; t->fh = f.height; t->fw = f.width; t->rot = rotation_code(f.rotation);
  return VPB_OK;
}
// the pointers and steps of preprocess.cuh's YuvEntry for each layout (the table above YuvEntry)
static int table_entry(const char* fn, int j, const vpb_frame_yuv& f, const YuvFormat& c, YuvEntry* t) {
  static const char* const names[] = {"NV12", "NV21", "I420", "YV12", "YUYV", "UYVY"};
  const bool packed = c.layout == VPB_YUV_YUYV || c.layout == VPB_YUV_UYVY, planar = c.layout == VPB_YUV_I420 || c.layout == VPB_YUV_YV12;
  const long long yrow = packed ? 2LL * f.width : f.width, crow = planar ? f.width / 2 : f.width;
  const long long yp = f.y_pitch ? f.y_pitch : yrow, cp = packed ? yp : (f.c_pitch ? f.c_pitch : crow);
  const int planes = packed ? 1 : planar ? 3 : 2;
  bool ok = f.height >= 1 && f.width >= 2 && !(f.width & 1) && (packed || !(f.height & 1)) && yp >= yrow && cp >= crow;
  for (int i = 0; i < planes; ++i) ok = ok && f.plane[i];
  if (!ok)
    return fail(VPB_ERR_ARG, "%s: frame %d: %s %dx%d (w x h, even width%s expected), planes %p %p %p (%d used), pitches %lld / %lld "
                "bytes (0 or >= %lld / %lld expected)", fn, j, names[c.layout], f.width, f.height, packed ? "" : " and height",
                static_cast<const void*>(f.plane[0]), static_cast<const void*>(f.plane[1]), static_cast<const void*>(f.plane[2]), planes,
                static_cast<long long>(f.y_pitch), static_cast<long long>(f.c_pitch), yrow, crow);
  memset(t, 0, sizeof(*t));
  const uint8_t *p0 = f.plane[0], *p1 = f.plane[1], *p2 = f.plane[2];
  switch (c.layout) {
    case VPB_YUV_NV12: t->y = p0; t->u = p1; t->v = p1 + 1; break;
    case VPB_YUV_NV21: t->y = p0; t->u = p1 + 1; t->v = p1; break;
    case VPB_YUV_I420: t->y = p0; t->u = p1; t->v = p2; break;
    case VPB_YUV_YV12: t->y = p0; t->u = p2; t->v = p1; break;
    case VPB_YUV_YUYV: t->y = p0; t->u = p0 + 1; t->v = p0 + 3; break;
    default:           t->y = p0 + 1; t->u = p0; t->v = p0 + 2; break;       // UYVY
  }
  t->y_step = packed ? 2 : 1;
  t->c_step = packed ? 4 : planar ? 1 : 2;
  t->c_vshift = packed ? 0 : 1;
  t->y_pitch = yp; t->c_pitch = cp; t->fh = f.height; t->fw = f.width;
  t->conv = static_cast<uint8_t>(c.matrix | c.range << 1);
  t->rot = static_cast<uint8_t>(rotation_code(f.rotation));
  return VPB_OK;
}
static int table_entry(const char* fn, int j, const vpb_frame_nv12& f, const YuvFormat& c, YuvEntry* t) {
  vpb_frame_yuv g;
  memset(&g, 0, sizeof(g));
  g.plane[0] = f.y; g.plane[1] = f.uv; g.y_pitch = f.y_pitch; g.c_pitch = f.uv_pitch;
  g.height = f.height; g.width = f.width; g.num_boxes = f.num_boxes; g.rotation = f.rotation;
  return table_entry(fn, j, g, c, t);
}
template <class Frame, class Entry>
static int build_frame_table(const char* fn, const Frame* fr, int32_t num_frames, const YuvFormat& fmt, int limit, Entry* tab, int* num_tab,
                             int32_t* n) {
  if (num_frames < 0 || (num_frames > 0 && !fr)) return fail(VPB_ERR_ARG, "%s: %d frames, frame array %p", fn, num_frames, fr);
  VPB_TRY(check_call(fn, fr, fmt));
  long long boxes = 0;
  int used = 0;
  for (int j = 0; j < num_frames; ++j) {
    const Frame& f = fr[j];
    if (f.num_boxes < 0) return fail(VPB_ERR_ARG, "%s: frame %d has num_boxes = %d", fn, j, f.num_boxes);
    if (rotation_code(f.rotation) < 0)
      return fail(VPB_ERR_ARG, "%s: frame %d has rotation %d (0, 90, 180 or 270 expected)", fn, j, f.rotation);
    if (f.num_boxes == 0) continue;
    Entry t;
    VPB_TRY(table_entry(fn, j, f, fmt, &t));
    if (used == VPB_MAX_FRAMES) return fail(VPB_ERR_ARG, "%s: more than VPB_MAX_FRAMES = %d frames with boxes", fn, VPB_MAX_FRAMES);
    if (boxes + f.num_boxes > limit)
      return fail(VPB_ERR_ARG, "%s: more than max_batch = %d boxes (frames 0..%d)", fn, limit, j);
    t.first_box = static_cast<int>(boxes);
    tab[used++] = t;
    boxes += f.num_boxes;
  }
  *num_tab = used;
  *n = static_cast<int32_t>(boxes);
  return VPB_OK;
}
template <class Frame, class Entry>
static int frame_table(const char* fn, vpb_engine* e, const Frame* fr, int32_t num_frames, const YuvFormat& fmt, Entry* tab, int* num_tab,
                       int32_t* n) {
  if (!e) return fail(VPB_ERR_ARG, "null engine");
  if (!e->finalized) return fail(VPB_ERR_STATE, "weights not finalized: call vpb_finalize first");
  VPB_TRY(build_frame_table(fn, fr, num_frames, fmt, e->maxB, tab, num_tab, n));
  return *n ? check_ready_keypoints(e, *n) : VPB_OK;
}

// Status word of the device-side frame path (bit 0: a box was empty after padding + clipping; such a box is decoded from
// a black crop with scale 0 where the reference raises).  Synchronous: waits for the device, copies the word, clears it.
extern "C" int vpb_frame_status(vpb_engine* e, int32_t* h_status) {
  if (!e || !h_status) return fail(VPB_ERR_ARG, "vpb_frame_status: null argument");
  if (!e->finalized) return fail(VPB_ERR_STATE, "not finalized");
  DeviceGuard dev_guard(e);
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(h_status, e->pp_status, sizeof(int32_t), cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemset(e->pp_status, 0, sizeof(int32_t)));
  return VPB_OK;
}

// host boxes are checked here, where the reference raises (ZeroDivisionError in pad_image / cv2.resize on an empty crop)
// (frame >= 0: the multi-frame calls, whose message names the frame and the box's index within it)
static int check_boxes_host(const int32_t* bb, int32_t n, int32_t fh, int32_t fw, int frame = -1) {
  for (int i = 0; i < n; ++i) {
    const int x0 = std::min(std::max(bb[4 * i] - 10, 0), fw), x1 = std::min(std::max(bb[4 * i + 2] + 10, 0), fw);
    const int y0 = std::min(std::max(bb[4 * i + 1] - 10, 0), fh), y1 = std::min(std::max(bb[4 * i + 3] + 10, 0), fh);
    if (x1 - x0 <= 0 || y1 - y0 <= 0) {
      if (frame >= 0)
        return fail(VPB_ERR_ARG, "frame %d box %d (%d,%d,%d,%d) is empty after padding and clipping to the %dx%d frame", frame, i,
                    bb[4 * i], bb[4 * i + 1], bb[4 * i + 2], bb[4 * i + 3], fw, fh);
      return fail(VPB_ERR_ARG, "box %d (%d,%d,%d,%d) is empty after padding and clipping to the %dx%d frame", i, bb[4 * i], bb[4 * i + 1],
                  bb[4 * i + 2], bb[4 * i + 3], fw, fh);
    }
  }
  return VPB_OK;
}
template <class Frame>            // vpb_frame | vpb_frame_yuv | vpb_frame_nv12, after build_frame_table checked the rotations
static int check_frames_boxes_host(const Frame* fr, int32_t num_frames, const int32_t* bb) {
  for (int j = 0, first = 0; j < num_frames; first += fr[j].num_boxes, ++j) {
    int32_t h = 0, w = 0;
    view_size(fr[j], &h, &w);
    VPB_TRY(check_boxes_host(bb + 4 * static_cast<size_t>(first), fr[j].num_boxes, h, w, j));
  }
  return VPB_OK;
}
// host matrices / centre-scale: what the device forms can only flag in the status word is an argument error here
static int check_affine_host(const double* mats, const float* cs, int32_t n) {
  for (int i = 0; i < n; ++i) {
    for (int j = 0; j < 6; ++j)
      if (!std::isfinite(mats[6 * i + j])) return fail(VPB_ERR_ARG, "box %d: matrix entry %d is %g (finite expected)", i, j, mats[6 * i + j]);
    if (!cs) continue;
    const float* c = cs + 4 * i;
    if (!std::isfinite(c[0]) || !std::isfinite(c[1]) || !(c[2] > 0.f) || !(c[3] > 0.f) || !std::isfinite(c[2]) || !std::isfinite(c[3]))
      return fail(VPB_ERR_ARG, "box %d: centre (%g, %g), scale (%g, %g): finite centre and scale > 0 expected", i, c[0], c[1], c[2], c[3]);
  }
  return VPB_OK;
}
static int frame_stage_reserve(vpb_engine* e, int slot, size_t bytes) {
  if (e->frame_cap[slot] >= bytes) return VPB_OK;
  if (e->frame_stage[slot]) { CU_TRY(cudaDeviceSynchronize()); CU_TRY(cudaFree(e->frame_stage[slot])); e->frame_stage[slot] = nullptr; e->frame_cap[slot] = 0; }
  void* q = nullptr;
  CU_TRY(cudaMalloc(&q, bytes + 256));
  e->frame_stage[slot] = static_cast<uint8_t*>(q);
  e->frame_cap[slot] = bytes;
  return VPB_OK;
}

// one plane of `rows` rows of `row` bytes, host pitch `pitch` -> packed at dst
static int stage_plane(uint8_t* dst, const uint8_t* src, long long pitch, size_t row, int rows, cudaStream_t st) {
  if (static_cast<size_t>(pitch) == row) CU_TRY(cudaMemcpyAsync(dst, src, row * rows, cudaMemcpyHostToDevice, st));
  else CU_TRY(cudaMemcpy2DAsync(dst, row, src, static_cast<size_t>(pitch), row, rows, cudaMemcpyHostToDevice, st));
  return VPB_OK;
}
static size_t staged_bytes(const FrameEntry& t) { return static_cast<size_t>(t.fh) * t.fw * 3; }
static size_t staged_bytes(const YuvEntry& t) {        // 4:2:2: 2 B per pixel; 4:2:0: Y, then the chroma plane(s), 1.5 B per pixel
  return static_cast<size_t>(t.fh) * t.fw * (t.c_step == 4 ? 4 : 3) / 2;
}
static int stage_entry(FrameEntry& t, uint8_t* dst, cudaStream_t st) {
  const size_t row = static_cast<size_t>(t.fw) * 3;
  VPB_TRY(stage_plane(dst, t.data, t.pitch, row, t.fh, st));
  t.data = dst; t.pitch = static_cast<long long>(row);
  return VPB_OK;
}
// The layout family follows from c_step (table_entry): 4 = packed 4:2:2, 2 = semi-planar (NV12 / NV21), 1 = planar (I420 / YV12).
// Packed and semi-planar planes are staged whole from their first byte, and y / u / v keep their offsets into them.
static int stage_entry(YuvEntry& t, uint8_t* dst, cudaStream_t st) {
  const size_t w = static_cast<size_t>(t.fw), h = static_cast<size_t>(t.fh);
  if (t.c_step == 4) {
    const uint8_t* base = std::min({t.y, t.u, t.v});
    VPB_TRY(stage_plane(dst, base, t.y_pitch, 2 * w, t.fh, st));
    t.y = dst + (t.y - base); t.u = dst + (t.u - base); t.v = dst + (t.v - base);
    t.y_pitch = t.c_pitch = static_cast<long long>(2 * w);
    return VPB_OK;
  }
  VPB_TRY(stage_plane(dst, t.y, t.y_pitch, w, t.fh, st));
  uint8_t* c = dst + w * h;
  if (t.c_step == 2) {
    const uint8_t* base = std::min(t.u, t.v);
    VPB_TRY(stage_plane(c, base, t.c_pitch, w, t.fh / 2, st));
    t.u = c + (t.u - base); t.v = c + (t.v - base);
    t.c_pitch = static_cast<long long>(w);
  } else {
    VPB_TRY(stage_plane(c, t.u, t.c_pitch, w / 2, t.fh / 2, st));
    VPB_TRY(stage_plane(c + (w / 2) * (h / 2), t.v, t.c_pitch, w / 2, t.fh / 2, st));
    t.u = c; t.v = c + (w / 2) * (h / 2);
    t.c_pitch = static_cast<long long>(w / 2);
  }
  t.y = dst; t.y_pitch = static_cast<long long>(w);
  return VPB_OK;
}
// Host frames -> staging slot `slot`, enqueued on `st` after the slot's last user: each frame packed (a 2D copy from its pitch;
// YUV: stage_entry), then the boxes of all frames in one copy, or for the affine calls
// (h_mats) the matrices and the centre / scale (slot 0: the affine calls have no pipelined form).  Repoints `tab` at the
// staged frames.
template <class Entry>
static int stage_frames_host(vpb_engine* e, int slot, Entry* tab, int nt, const int32_t* h_bboxes, const double* h_mats, const float* h_cs,
                             int32_t n, cudaStream_t st) {
  size_t total = 0;
  for (int j = 0; j < nt; ++j) total += staged_bytes(tab[j]);
  VPB_TRY(frame_stage_reserve(e, slot, total));
  CU_TRY(cudaStreamWaitEvent(st, e->ev_done[slot], 0));   // slot 0 is shared with the pipelined path: its last user is done
  size_t off = 0;
  for (int j = 0; j < nt; ++j) {
    const size_t bytes = staged_bytes(tab[j]);
    VPB_TRY(stage_entry(tab[j], e->frame_stage[slot] + off, st));
    off += bytes;
  }
  if (h_mats) {
    CU_TRY(cudaMemcpyAsync(e->mat_stage, h_mats, static_cast<size_t>(n) * 6 * sizeof(double), cudaMemcpyHostToDevice, st));
    CU_TRY(cudaMemcpyAsync(e->cs_stage, h_cs, static_cast<size_t>(n) * 4 * sizeof(float), cudaMemcpyHostToDevice, st));
  } else {
    CU_TRY(cudaMemcpyAsync(e->bbox_stage[slot], h_bboxes, static_cast<size_t>(n) * 4 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  return VPB_OK;
}
// synchronous host form on slot 0 and the caller's stream: the frames with their boxes (or affine matrices) staged, the call,
// the host tail
template <class Entry>
static int frames_host_sync(vpb_engine* e, Entry* tab, int nt, const int32_t* h_bboxes, const double* h_mats, const float* h_cs,
                            const std::vector<Segment>& segs, bool mixed, int32_t n, float* h_kpts, int32_t* h_idx, cudaStream_t st) {
  VPB_TRY(stage_frames_host(e, 0, tab, nt, h_bboxes, h_mats, h_cs, n, st));
  VPB_TRY(frames_core(e, tab, nt, e->bbox_stage[0], h_mats ? e->mat_stage : nullptr, h_mats ? e->cs_stage : nullptr, segs, mixed, n,
                      e->kpts[0], e->idx[0], st));
  return host_tail(e, segs, mixed, 0, h_kpts, h_idx, st, true);
}
// Pipelined frames (video): same slots, events and vpb_wait_host as vpb_submit_host; the H2D per step is the uint8 frames and
// 16 B per box instead of 589 824 B per crop.
template <class Entry>
static int frames_host_submit(vpb_engine* e, Entry* tab, int nt, const int32_t* h_bboxes, int32_t n, float* h_kpts, int32_t* h_idx,
                              int slot) {
  VPB_TRY(stage_frames_host(e, slot, tab, nt, h_bboxes, nullptr, nullptr, n, e->copy_stream));
  CU_TRY(cudaEventRecord(e->ev_h2d[slot], e->copy_stream));
  CU_TRY(cudaStreamWaitEvent(e->compute_stream, e->ev_h2d[slot], 0));
  const std::vector<Segment> segs{{0, n}};
  VPB_TRY(frames_core(e, tab, nt, e->bbox_stage[slot], nullptr, nullptr, segs, false, n, e->kpts[slot], e->idx[slot], e->compute_stream));
  return host_tail(e, segs, false, slot, h_kpts, h_idx, e->compute_stream, false);
}

extern "C" int vpb_infer_frame(vpb_engine* e, const uint8_t* d_frame, int32_t frame_h, int32_t frame_w, const int32_t* d_bboxes,
                               int32_t n, float* d_kpts, int32_t* d_idx, void* stream) {
  VPB_TRY(check_ready_keypoints(e, n));
  DeviceGuard dev_guard(e);
  if (!d_frame || !d_bboxes || !d_kpts || frame_h < 1 || frame_w < 1) return fail(VPB_ERR_ARG, "vpb_infer_frame: bad argument");
  const FrameEntry f = single_frame(d_frame, frame_h, frame_w);
  return frames_core(e, &f, 1, d_bboxes, nullptr, nullptr, {{0, n}}, false, n, d_kpts, d_idx, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_infer_frame_host(vpb_engine* e, const uint8_t* h_frame, int32_t frame_h, int32_t frame_w, const int32_t* h_bboxes,
                                    int32_t n, float* h_kpts, int32_t* h_idx, void* stream) {
  VPB_TRY(check_ready_keypoints(e, n));
  DeviceGuard dev_guard(e);
  if (!h_frame || !h_bboxes || !h_kpts || frame_h < 1 || frame_w < 1) return fail(VPB_ERR_ARG, "vpb_infer_frame_host: bad argument");
  VPB_TRY(check_boxes_host(h_bboxes, n, frame_h, frame_w));
  FrameEntry f = single_frame(h_frame, frame_h, frame_w);
  return frames_host_sync(e, &f, 1, h_bboxes, nullptr, nullptr, {{0, n}}, false, n, h_kpts, h_idx, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_submit_frame_host(vpb_engine* e, const uint8_t* h_frame, int32_t frame_h, int32_t frame_w, const int32_t* h_bboxes,
                                     int32_t n, float* h_kpts, int32_t* h_idx, int32_t slot) {
  VPB_TRY(check_ready_keypoints(e, n));
  DeviceGuard dev_guard(e);
  if (!h_frame || !h_bboxes || !h_kpts || frame_h < 1 || frame_w < 1 || slot < 0 || slot > 1)
    return fail(VPB_ERR_ARG, "vpb_submit_frame_host: bad argument");
  VPB_TRY(check_boxes_host(h_bboxes, n, frame_h, frame_w));
  FrameEntry f = single_frame(h_frame, frame_h, frame_w);
  return frames_host_submit(e, &f, 1, h_bboxes, n, h_kpts, h_idx, slot);
}

// ---- the multi-frame calls: one body per call kind, for RGB frames (vpb_frame -> FrameEntry; `fmt` unused) and YUV frames
// (vpb_frame_yuv, vpb_frame_nv12 -> YuvEntry); `fn` names the entry point in the messages
template <class Entry, class Frame>
static int infer_frames_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt, const int32_t* d_bboxes,
                          float* d_kpts, int32_t* d_idx, void* stream) {
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!d_bboxes || !d_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  return frames_core(e, tab, nt, d_bboxes, nullptr, nullptr, {{0, n}}, false, n, d_kpts, d_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int infer_frames_host_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                               const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream) {
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!h_bboxes || !h_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  VPB_TRY(check_frames_boxes_host(h_frames, num_frames, h_bboxes));
  return frames_host_sync(e, tab, nt, h_bboxes, nullptr, nullptr, {{0, n}}, false, n, h_kpts, h_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int submit_frames_host_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                                const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, int32_t slot) {
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  if (slot < 0 || slot > 1) return fail(VPB_ERR_ARG, "%s: slot %d", fn, slot);
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!h_bboxes || !h_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  VPB_TRY(check_frames_boxes_host(h_frames, num_frames, h_bboxes));
  return frames_host_submit(e, tab, nt, h_bboxes, n, h_kpts, h_idx, slot);
}

extern "C" int vpb_infer_frames(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* d_bboxes,
                                float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_frames_t<FrameEntry>("vpb_infer_frames", e, h_frames, num_frames, YuvFormat{}, d_bboxes, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_frames_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_bboxes,
                                     float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_frames_host_t<FrameEntry>("vpb_infer_frames_host", e, h_frames, num_frames, YuvFormat{}, h_bboxes, h_kpts, h_idx, stream);
}
extern "C" int vpb_submit_frames_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_bboxes,
                                      float* h_kpts, int32_t* h_idx, int32_t slot) {
  return submit_frames_host_t<FrameEntry>("vpb_submit_frames_host", e, h_frames, num_frames, YuvFormat{}, h_bboxes, h_kpts, h_idx, slot);
}
extern "C" int vpb_infer_frames_nv12(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                     const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_frames_t<YuvEntry>("vpb_infer_frames_nv12", e, h_frames, num_frames, nv12_format(matrix), d_bboxes, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_frames_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                          const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_frames_host_t<YuvEntry>("vpb_infer_frames_nv12_host", e, h_frames, num_frames, nv12_format(matrix), h_bboxes, h_kpts, h_idx, stream);
}
extern "C" int vpb_submit_frames_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                           const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, int32_t slot) {
  return submit_frames_host_t<YuvEntry>("vpb_submit_frames_nv12_host", e, h_frames, num_frames, nv12_format(matrix), h_bboxes, h_kpts, h_idx, slot);
}
extern "C" int vpb_infer_frames_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                    int32_t range, const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_frames_t<YuvEntry>("vpb_infer_frames_yuv", e, h_frames, num_frames, yuv_format(layout, matrix, range), d_bboxes, d_kpts,
                                  d_idx, stream);
}
extern "C" int vpb_infer_frames_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                         int32_t range, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_frames_host_t<YuvEntry>("vpb_infer_frames_yuv_host", e, h_frames, num_frames, yuv_format(layout, matrix, range), h_bboxes,
                                       h_kpts, h_idx, stream);
}
extern "C" int vpb_submit_frames_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                          int32_t range, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, int32_t slot) {
  return submit_frames_host_t<YuvEntry>("vpb_submit_frames_yuv_host", e, h_frames, num_frames, yuv_format(layout, matrix, range), h_bboxes,
                                        h_kpts, h_idx, slot);
}

// ------------------------------------------------------------------------------------------------ affine top-down crops
extern "C" int vpb_preprocess_affine(const vpb_frame* h_frames, int32_t num_frames, const double* d_mats, float* d_crops, void* stream) {
  FrameEntry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(build_frame_table("vpb_preprocess_affine", h_frames, num_frames, YuvFormat{}, 1 << 30, tab, &nt, &n));
  if (n == 0) return VPB_OK;
  if (!d_mats || !d_crops) return fail(VPB_ERR_ARG, "vpb_preprocess_affine: null pointer");
  AffineParams q = affine_params(tab, nt, d_mats, nullptr, n, nullptr);
  q.crops = d_crops;
  crop_warp_normalise<<<dim3(n, PP_H / PP_ROWS), PP_W, 0, static_cast<cudaStream_t>(stream)>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------------------ pose overlay
static long long draw_records(long long n, long long k, long long num_limbs) { return n * (num_limbs + k); }
extern "C" int64_t vpb_draw_workspace_bytes(int32_t n, int32_t k, int32_t num_limbs) {
  if (n < 0 || k < 1 || num_limbs < 0) return -1;
  return draw_records(n, k, num_limbs) * (long long)(sizeof(DrawRec) + sizeof(int4));
}
extern "C" int vpb_draw_poses(const vpb_canvas* h_frames, int32_t num_frames, int32_t channel_order, const float* d_kpts, int32_t k,
                              const int32_t* d_person_index, const int32_t* h_limbs, int32_t num_limbs, const uint8_t* h_point_bgr,
                              int32_t num_point_colors, const uint8_t* h_limb_bgr, int32_t num_limb_colors, int32_t radius,
                              float threshold, void* d_workspace, void* stream) {
  const char* fn = "vpb_draw_poses";
  if (channel_order != VPB_DRAW_RGB && channel_order != VPB_DRAW_BGR) return fail(VPB_ERR_ARG, "%s: unknown channel order %d", fn, channel_order);
  if (k < 1) return fail(VPB_ERR_ARG, "%s: k=%d", fn, k);
  if (num_limbs < 0 || num_limbs > DRAW_MAX_LIMBS || (num_limbs > 0 && !h_limbs))
    return fail(VPB_ERR_ARG, "%s: %d limbs (0..%d and a table)", fn, num_limbs, DRAW_MAX_LIMBS);
  if (num_point_colors < 1 || num_point_colors > DRAW_MAX_COLORS || num_limb_colors < 1 || num_limb_colors > DRAW_MAX_COLORS ||
      !h_point_bgr || !h_limb_bgr)
    return fail(VPB_ERR_ARG, "%s: colour tables of %d and %d entries (1..%d each)", fn, num_point_colors, num_limb_colors, DRAW_MAX_COLORS);
  if (radius > DRAW_MAX_RADIUS) return fail(VPB_ERR_ARG, "%s: radius %d above %d", fn, radius, DRAW_MAX_RADIUS);
  if (num_frames < 0 || (num_frames > 0 && !h_frames)) return fail(VPB_ERR_ARG, "%s: %d frames", fn, num_frames);
  DrawParams q;
  memset(&q, 0, sizeof(q));
  for (int e = 0; e < num_limbs; ++e)
    for (int j = 0; j < 2; ++j) {
      const int32_t v = h_limbs[2 * e + j];
      if (v < 0 || v >= k) return fail(VPB_ERR_ARG, "%s: limb %d joins keypoint %d, outside [0, %d)", fn, e, v, k);
      q.limbs[e][j] = static_cast<uint16_t>(v);
    }
  const bool rgb = channel_order == VPB_DRAW_RGB;
  for (int c = 0; c < 3; ++c) {
    const int src = rgb ? 2 - c : c;                         // BGR tables, written reversed into RGB frames
    for (int i = 0; i < num_point_colors; ++i) q.point_rgb[i][c] = h_point_bgr[3 * i + src];
    for (int i = 0; i < num_limb_colors; ++i) q.limb_rgb[i][c] = h_limb_bgr[3 * i + src];
  }
  long long n = 0, tiles = 0;
  int nt = 0;
  for (int j = 0; j < num_frames; ++j) {
    const vpb_canvas& c = h_frames[j];
    if (c.num_people < 0) return fail(VPB_ERR_ARG, "%s: frame %d has %d people", fn, j, c.num_people);
    if (c.num_people == 0) continue;
    if (nt == DRAW_MAX_FRAMES) return fail(VPB_ERR_ARG, "%s: more than %d frames with people", fn, VPB_MAX_FRAMES);
    if (!c.data) return fail(VPB_ERR_ARG, "%s: frame %d has people and no data", fn, j);
    if (c.height < 1 || c.width < 1) return fail(VPB_ERR_ARG, "%s: frame %d is %d x %d", fn, j, c.height, c.width);
    const long long pitch = c.pitch_bytes == 0 ? 3LL * c.width : c.pitch_bytes;
    if (pitch < 3LL * c.width) return fail(VPB_ERR_ARG, "%s: frame %d pitch %lld below 3 * width %d", fn, j, (long long)c.pitch_bytes, c.width);
    const int r = radius > 0 ? radius : std::max(1, std::min(c.height, c.width) / 150);
    if (r > DRAW_MAX_RADIUS) return fail(VPB_ERR_ARG, "%s: frame %d radius %d above %d", fn, j, r, DRAW_MAX_RADIUS);
    DrawFrame& f = q.frames[nt++];
    f.data = c.data; f.pitch = pitch; f.h = c.height; f.w = c.width;
    f.first_person = static_cast<int>(n); f.num_people = c.num_people; f.radius = r; f.first_tile = static_cast<int>(tiles);
    n += c.num_people;
    tiles += (long long)((c.width + DRAW_TILE_W - 1) / DRAW_TILE_W) * ((c.height + DRAW_TILE_H - 1) / DRAW_TILE_H);
    if (draw_records(n, k, num_limbs) > 0x7fffffffLL || tiles > 0x7fffffffLL) return fail(VPB_ERR_ARG, "%s: call too large", fn);
  }
  if (n == 0) return VPB_OK;
  if (!d_kpts || !d_workspace) return fail(VPB_ERR_ARG, "%s: null keypoints or workspace", fn);
  if (reinterpret_cast<uintptr_t>(d_workspace) % 16 != 0) return fail(VPB_ERR_ARG, "%s: workspace not 16-byte aligned", fn);
  const long long recs = draw_records(n, k, num_limbs);
  q.kpts = d_kpts; q.person_index = d_person_index;
  q.recs = static_cast<DrawRec*>(d_workspace);
  q.boxes = reinterpret_cast<int4*>(static_cast<char*>(d_workspace) + recs * sizeof(DrawRec));
  q.n = static_cast<int>(n); q.k = k; q.num_limbs = num_limbs; q.num_point_colors = num_point_colors; q.num_limb_colors = num_limb_colors;
  q.num_frames = nt; q.total_tiles = static_cast<int>(tiles); q.threshold = threshold;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  draw_setup<<<static_cast<unsigned>(cdiv(recs, DRAW_SETUP_THREADS)), DRAW_SETUP_THREADS, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  draw_raster<<<static_cast<unsigned>(tiles), DRAW_TILE_W * DRAW_TILE_H, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------------------ SORT tracker
struct vpb_tracker {
  int device = 0;
  void* mem = nullptr;          // one allocation; TrackParams points into it
  TrackParams q{};
};

struct TrackerDevice {          // makes the tracker's device current for one call
  int prev = -1;
  explicit TrackerDevice(const vpb_tracker* t) {
    int cur = -1;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != t->device && cudaSetDevice(t->device) == cudaSuccess) prev = cur;
  }
  ~TrackerDevice() { if (prev >= 0) cudaSetDevice(prev); }
};

extern "C" int vpb_tracker_create(int32_t num_streams, int32_t max_age, int32_t min_hits, double iou_threshold, int32_t device,
                                  vpb_tracker** out) {
  const char* fn = "vpb_tracker_create";
  if (!out) return fail(VPB_ERR_ARG, "%s: null output", fn);
  *out = nullptr;
  if (num_streams < 1 || num_streams > 65535) return fail(VPB_ERR_ARG, "%s: %d streams (1..65535)", fn, num_streams);
  if (max_age < 0 || min_hits < 0) return fail(VPB_ERR_ARG, "%s: max_age %d and min_hits %d must be >= 0", fn, max_age, min_hits);
  if (!std::isfinite(iou_threshold)) return fail(VPB_ERR_ARG, "%s: iou_threshold is not finite", fn);
  int ndev = 0;
  CU_TRY(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(VPB_ERR_ARG, "%s: device %d of %d", fn, device, ndev);
  vpb_tracker* t = new vpb_tracker();
  t->device = device;
  TrackerDevice guard(t);
  const size_t S = static_cast<size_t>(num_streams), M = TRACK_MAX;
  const size_t bytes_state = S * TRACK_FIELDS * M * sizeof(double), bytes_ids = S * M * sizeof(long long);
  const size_t bytes_i32 = (3 * S * M + 4 * S + 2) * sizeof(int32_t);
  const size_t total = bytes_state + bytes_ids + 2 * sizeof(long long) + bytes_i32;
  cudaError_t err = cudaMalloc(&t->mem, total);
  if (err == cudaSuccess) err = cudaMemset(t->mem, 0, total);
  if (err == cudaSuccess)
    err = cudaFuncSetAttribute(track_associate, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(TrackSmem)));
  if (err != cudaSuccess) {
    if (t->mem) cudaFree(t->mem);
    delete t;
    return fail(VPB_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(err));
  }
  char* p = static_cast<char*>(t->mem);
  TrackParams& q = t->q;
  q.state = reinterpret_cast<double*>(p); p += bytes_state;
  q.ids = reinterpret_cast<long long*>(p); p += bytes_ids;
  q.next_id = reinterpret_cast<long long*>(p); p += sizeof(long long);
  q.id_base = reinterpret_cast<long long*>(p); p += sizeof(long long);
  int32_t* ip = reinterpret_cast<int32_t*>(p);
  q.tsu = ip; ip += S * M;
  q.hits = ip; ip += S * M;
  q.new_det = ip; ip += S * M;
  q.num_tracks = ip; ip += S;
  q.frame_count = ip; ip += S;
  q.num_new = ip; ip += S;
  q.status = ip;
  q.num_streams = num_streams; q.max_age = max_age; q.min_hits = min_hits; q.iou_threshold = iou_threshold;
  *out = t;
  return VPB_OK;
}

extern "C" void vpb_tracker_destroy(vpb_tracker* t) {
  if (!t) return;
  TrackerDevice guard(t);
  cudaDeviceSynchronize();
  cudaFree(t->mem);
  delete t;
}

extern "C" int vpb_tracker_update(vpb_tracker* t, const double* d_dets, const int32_t* d_counts, double* d_rows, int32_t* d_boxes,
                                  int32_t* d_out_counts, void* stream) {
  if (!t) return fail(VPB_ERR_ARG, "vpb_tracker_update: null tracker");
  if (!d_dets || !d_counts || !d_rows || !d_boxes || !d_out_counts) return fail(VPB_ERR_ARG, "vpb_tracker_update: null buffer");
  TrackerDevice guard(t);
  TrackParams q = t->q;
  q.dets = d_dets; q.counts = d_counts; q.rows = d_rows; q.boxes = d_boxes; q.out_counts = d_out_counts;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  track_associate<<<q.num_streams, TRACK_THREADS, sizeof(TrackSmem), st>>>(q);
  CU_TRY(cudaGetLastError());
  track_emit<<<q.num_streams, TRACK_THREADS, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vpb_tracker_reset(vpb_tracker* t, int32_t stream_index, void* stream) {
  if (!t) return fail(VPB_ERR_ARG, "vpb_tracker_reset: null tracker");
  const int S = t->q.num_streams;
  if (stream_index < -1 || stream_index >= S) return fail(VPB_ERR_ARG, "vpb_tracker_reset: stream %d of %d", stream_index, S);
  TrackerDevice guard(t);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int first = stream_index < 0 ? 0 : stream_index, count = stream_index < 0 ? S : 1;
  CU_TRY(cudaMemsetAsync(t->q.num_tracks + first, 0, count * sizeof(int32_t), st));
  CU_TRY(cudaMemsetAsync(t->q.frame_count + first, 0, count * sizeof(int32_t), st));
  return VPB_OK;
}

extern "C" int vpb_tracker_next_id(vpb_tracker* t, int64_t* out) {
  if (!t || !out) return fail(VPB_ERR_ARG, "vpb_tracker_next_id: null argument");
  TrackerDevice guard(t);
  long long v = 0;
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(&v, t->q.next_id, sizeof(v), cudaMemcpyDeviceToHost));
  *out = v;
  return VPB_OK;
}

extern "C" int vpb_tracker_set_next_id(vpb_tracker* t, int64_t next_id) {
  if (!t) return fail(VPB_ERR_ARG, "vpb_tracker_set_next_id: null tracker");
  if (next_id < 0) return fail(VPB_ERR_ARG, "vpb_tracker_set_next_id: negative id %lld", (long long)next_id);
  TrackerDevice guard(t);
  const long long v = next_id;
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(t->q.next_id, &v, sizeof(v), cudaMemcpyHostToDevice));
  return VPB_OK;
}

extern "C" int vpb_tracker_status(vpb_tracker* t, int32_t* h_status) {
  if (!t || !h_status) return fail(VPB_ERR_ARG, "vpb_tracker_status: null argument");
  TrackerDevice guard(t);
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(h_status, t->q.status, sizeof(int32_t), cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemset(t->q.status, 0, sizeof(int32_t)));
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------------ One Euro smoother
struct vpb_smoother {
  int device = 0;
  void* mem = nullptr;          // one allocation; SmoothParams points into it
  SmoothParams q{};
};

struct SmootherDevice {         // makes the smoother's device current for one call
  int prev = -1;
  explicit SmootherDevice(const vpb_smoother* s) {
    int cur = -1;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != s->device && cudaSetDevice(s->device) == cudaSuccess) prev = cur;
  }
  ~SmootherDevice() { if (prev >= 0) cudaSetDevice(prev); }
};

extern "C" int vpb_smoother_create(int32_t num_streams, int32_t k, double min_cutoff, double beta, double d_cutoff, double fps,
                                   double dx0, int32_t max_gap, int32_t device, vpb_smoother** out) {
  const char* fn = "vpb_smoother_create";
  if (!out) return fail(VPB_ERR_ARG, "%s: null output", fn);
  *out = nullptr;
  if (num_streams < 1 || num_streams > 65535) return fail(VPB_ERR_ARG, "%s: %d streams (1..65535)", fn, num_streams);
  if (k < 1 || k > SMOOTH_MAX_K) return fail(VPB_ERR_ARG, "%s: %d keypoints (1..%d)", fn, k, SMOOTH_MAX_K);
  if (!std::isfinite(min_cutoff) || !std::isfinite(beta) || !std::isfinite(d_cutoff) || !std::isfinite(fps) || !std::isfinite(dx0))
    return fail(VPB_ERR_ARG, "%s: a filter parameter is not finite", fn);
  if (max_gap < 0) return fail(VPB_ERR_ARG, "%s: max_gap %d must be >= 0", fn, max_gap);
  int ndev = 0;
  CU_TRY(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(VPB_ERR_ARG, "%s: device %d of %d", fn, device, ndev);
  vpb_smoother* s = new vpb_smoother();
  s->device = device;
  SmootherDevice guard(s);
  const size_t S = static_cast<size_t>(num_streams), M = SMOOTH_MAX;
  const size_t bytes_state = 2 * S * M * k * 2 * sizeof(double), bytes_f64 = 2 * S * M * sizeof(double);
  const size_t bytes_i32 = (5 * S * M + 3 * S + 1) * sizeof(int32_t);
  const size_t total = bytes_state + bytes_f64 + bytes_i32;
  cudaError_t err = cudaMalloc(&s->mem, total);
  if (err == cudaSuccess) err = cudaMemset(s->mem, 0, total);
  SmoothParams& q = s->q;
  char* p = static_cast<char*>(s->mem);
  q.x_prev = reinterpret_cast<double*>(p); p += bytes_state / 2;
  q.dx_prev = reinterpret_cast<double*>(p); p += bytes_state / 2;
  q.c_last = reinterpret_cast<double*>(p); p += S * M * sizeof(double);
  q.row_te = reinterpret_cast<double*>(p); p += S * M * sizeof(double);
  int32_t* ip = reinterpret_cast<int32_t*>(p);
  q.slot_id = ip; ip += S * M;
  q.slot_u = ip; ip += S * M;
  q.slot_first = ip; ip += S * M;
  q.row_slot = ip; ip += S * M;
  q.row_mode = ip; ip += S * M;
  q.updates = ip; ip += S;
  q.rows = ip; ip += S;
  q.row0 = ip; ip += S;
  q.status = ip;
  if (err == cudaSuccess) err = cudaMemset(q.slot_u, 0xFF, S * M * sizeof(int32_t));      // every slot free (-1)
  if (err != cudaSuccess) {
    if (s->mem) cudaFree(s->mem);
    delete s;
    return fail(VPB_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(err));
  }
  q.num_streams = num_streams; q.k = k; q.max_gap = max_gap; q.realtime = fps <= 0.0;
  q.min_cutoff = min_cutoff; q.beta = beta; q.d_cutoff = d_cutoff; q.dx0 = dx0;
  q.deriv_cutoff = fps <= 0.0 ? d_cutoff : fps;
  *out = s;
  return VPB_OK;
}

extern "C" void vpb_smoother_destroy(vpb_smoother* s) {
  if (!s) return;
  SmootherDevice guard(s);
  cudaDeviceSynchronize();
  cudaFree(s->mem);
  delete s;
}

extern "C" int vpb_smoother_update(vpb_smoother* s, float* d_kpts, int32_t n, const int32_t* d_counts, const int32_t* d_ids,
                                   const double* d_clock, double* d_out, void* stream) {
  const char* fn = "vpb_smoother_update";
  if (!s) return fail(VPB_ERR_ARG, "%s: null smoother", fn);
  if (n < 0) return fail(VPB_ERR_ARG, "%s: %d rows", fn, n);
  if (!d_counts || (n > 0 && (!d_kpts || !d_ids))) return fail(VPB_ERR_ARG, "%s: null buffer", fn);
  if (s->q.realtime && !d_clock) return fail(VPB_ERR_ARG, "%s: realtime mode (fps <= 0) needs d_clock", fn);
  SmootherDevice guard(s);
  SmoothParams q = s->q;
  q.kpts = d_kpts; q.n = n; q.counts = d_counts; q.ids = d_ids; q.clock = d_clock; q.out = d_out;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  smooth_assign<<<q.num_streams, SMOOTH_THREADS, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  const dim3 grid(static_cast<unsigned>(cdiv(SMOOTH_MAX * q.k, SMOOTH_APPLY_THREADS)), static_cast<unsigned>(q.num_streams));
  smooth_apply<<<grid, SMOOTH_APPLY_THREADS, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vpb_smoother_reset(vpb_smoother* s, int32_t stream_index, void* stream) {
  if (!s) return fail(VPB_ERR_ARG, "vpb_smoother_reset: null smoother");
  const int S = s->q.num_streams;
  if (stream_index < -1 || stream_index >= S) return fail(VPB_ERR_ARG, "vpb_smoother_reset: stream %d of %d", stream_index, S);
  SmootherDevice guard(s);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t first = stream_index < 0 ? 0 : stream_index, count = stream_index < 0 ? S : 1;
  CU_TRY(cudaMemsetAsync(s->q.slot_u + first * SMOOTH_MAX, 0xFF, count * SMOOTH_MAX * sizeof(int32_t), st));
  CU_TRY(cudaMemsetAsync(s->q.updates + first, 0, count * sizeof(int32_t), st));
  return VPB_OK;
}

extern "C" int vpb_smoother_status(vpb_smoother* s, int32_t* h_status) {
  if (!s || !h_status) return fail(VPB_ERR_ARG, "vpb_smoother_status: null argument");
  SmootherDevice guard(s);
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(h_status, s->q.status, sizeof(int32_t), cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemset(s->q.status, 0, sizeof(int32_t)));
  return VPB_OK;
}

// ---------------------------------------------------------------------------------------------------------------- OKS NMS
// easy_ViTPose/vit_utils/post_processing/nms.py:66-70: the COCO-17 sigmas oks_iou uses when it is given none
static const double kCocoSigmas[17] = {.26 / 10.0, .25 / 10.0, .25 / 10.0, .35 / 10.0, .35 / 10.0, .79 / 10.0, .79 / 10.0, .72 / 10.0,
                                       .72 / 10.0, .62 / 10.0, .62 / 10.0, 1.07 / 10.0, 1.07 / 10.0, .87 / 10.0, .87 / 10.0, .89 / 10.0,
                                       .89 / 10.0};

// the checks and the parameters vpb_oks_nms and vpb_oks_iou share
static int oks_params(const char* fn, const float* d_kpts, int32_t n_rows, int32_t k, const int32_t* d_counts, int32_t num_frames,
                      const double* d_areas, const double* h_sigmas, double vis_thr, int32_t* d_status, OksNmsParams* q) {
  if (k < 1 || k > NMS_MAX_K) return fail(VPB_ERR_ARG, "%s: %d keypoints (1..%d)", fn, k, NMS_MAX_K);
  if (n_rows < 0) return fail(VPB_ERR_ARG, "%s: %d rows", fn, n_rows);
  if (num_frames < 0 || num_frames > 65535) return fail(VPB_ERR_ARG, "%s: %d frames (0..65535)", fn, num_frames);
  if (!d_status || (num_frames > 0 && !d_counts) || (n_rows > 0 && (!d_kpts || !d_areas)))
    return fail(VPB_ERR_ARG, "%s: null buffer", fn);
  if (!h_sigmas && k != 17) return fail(VPB_ERR_ARG, "%s: %d keypoints need sigmas (the default table has 17)", fn, k);
  const double* sig = h_sigmas ? h_sigmas : kCocoSigmas;
  memset(q, 0, sizeof(*q));
  for (int j = 0; j < k; ++j) {
    if (!std::isfinite(sig[j])) return fail(VPB_ERR_ARG, "%s: sigma %d is not finite", fn, j);
    const double v = sig[j] * 2.0;
    q->vars[j] = v * v;
  }
  q->kpts = d_kpts; q->counts = d_counts; q->areas = d_areas; q->status = d_status;
  q->n_rows = n_rows; q->k = k; q->num_frames = num_frames;
  q->use_vis = !std::isnan(vis_thr);
  q->vis_thr = static_cast<float>(vis_thr);
  return VPB_OK;
}

extern "C" int vpb_oks_nms(const float* d_kpts, int32_t n_rows, int32_t k, const int32_t* d_counts, int32_t num_frames,
                           const double* d_areas, const double* d_scores, const double* h_sigmas, const vpb_oks_nms_params* params,
                           int32_t* d_keep, int32_t* d_keep_counts, double* d_scores_out, int32_t* d_status, void* stream) {
  const char* fn = "vpb_oks_nms";
  if (!params) return fail(VPB_ERR_ARG, "%s: null params", fn);
  OksNmsParams q;
  VPB_TRY(oks_params(fn, d_kpts, n_rows, k, d_counts, num_frames, d_areas, h_sigmas, params->vis_thr, d_status, &q));
  if (!std::isfinite(params->thr)) return fail(VPB_ERR_ARG, "%s: thr %g is not finite", fn, params->thr);
  if (params->soft != 0 && params->soft != 1) return fail(VPB_ERR_ARG, "%s: soft %d (0 or 1)", fn, params->soft);
  if (params->soft && (params->max_dets < 0 || params->max_dets > NMS_MAX_DETS))
    return fail(VPB_ERR_ARG, "%s: max_dets %d (0..%d)", fn, params->max_dets, NMS_MAX_DETS);
  if ((num_frames > 0 && !d_keep_counts) || (n_rows > 0 && (!d_scores || !d_keep))) return fail(VPB_ERR_ARG, "%s: null buffer", fn);
  if (num_frames == 0) return VPB_OK;
  q.scores = d_scores; q.keep = d_keep; q.keep_counts = d_keep_counts; q.scores_out = d_scores_out;
  q.soft = params->soft; q.max_dets = params->max_dets; q.thr = static_cast<float>(params->thr);
  q.rescore = !std::isnan(params->rescore_vis_thr);
  q.rescore_vis_thr = static_cast<float>(params->rescore_vis_thr);
  oks_nms_kernel<<<num_frames, NMS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vpb_oks_iou(const float* d_kpts, int32_t n_rows, int32_t k, const int32_t* d_counts, int32_t num_frames,
                           const double* d_areas, const double* h_sigmas, double vis_thr, float* d_oks, int32_t* d_status, void* stream) {
  const char* fn = "vpb_oks_iou";
  OksNmsParams q;
  VPB_TRY(oks_params(fn, d_kpts, n_rows, k, d_counts, num_frames, d_areas, h_sigmas, vis_thr, d_status, &q));
  if (n_rows > 0 && !d_oks) return fail(VPB_ERR_ARG, "%s: null buffer", fn);
  if (num_frames == 0) return VPB_OK;
  q.oks = d_oks;
  oks_iou_kernel<<<num_frames, NMS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

// ---------------------------------------------------------------------------------------------------------------- COCO eval
// the workspace vpb_coco_eval carves, in this order, each piece aligned to 256 bytes
struct CocoWorkspace {
  size_t frame_row0, key0, key1, slot0, slot1, bits, num_dets, npig, summary, total;
};
static CocoWorkspace coco_workspace(int64_t num_images, int64_t num_frames) {
  CocoWorkspace w;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) / 256 * 256; return at; };
  const int64_t slots = num_images * COCO_MAX_DETS;
  w.frame_row0 = take(num_frames * sizeof(int32_t));
  w.key0 = take(slots * sizeof(double));
  w.key1 = take(slots * sizeof(double));
  w.slot0 = take(slots * sizeof(int32_t));
  w.slot1 = take(slots * sizeof(int32_t));
  w.bits = take(slots * sizeof(unsigned long long));
  w.num_dets = take(num_images * sizeof(int32_t));
  w.npig = take(COCO_A * num_images * sizeof(int32_t));
  w.summary = take(10 * COCO_SUMMARY_TERMS * sizeof(double));
  w.total = off;
  return w;
}

extern "C" int64_t vpb_coco_eval_workspace_bytes(int32_t num_images, int32_t num_frames) {
  if (num_images < 1 || num_images > VPB_COCO_MAX_IMAGES || num_frames < 0) return -1;
  return static_cast<int64_t>(coco_workspace(num_images, num_frames).total);
}

extern "C" int vpb_coco_eval(int32_t k, const double* h_sigmas, const vpb_coco_gts* gts, const vpb_coco_dets* dets, void* d_workspace,
                             int64_t workspace_bytes, double* d_stats, double* d_precision, double* d_recall, int32_t* d_status,
                             void* stream) {
  const char* fn = "vpb_coco_eval";
  if (!gts || !dets) return fail(VPB_ERR_ARG, "%s: null gts or dets", fn);
  if (k < 1 || k > COCO_MAX_K) return fail(VPB_ERR_ARG, "%s: %d keypoints (1..%d)", fn, k, COCO_MAX_K);
  const int32_t I = gts->num_images, G = gts->num_gts, F = dets->num_frames, n = dets->n_rows;
  if (I < 1 || I > VPB_COCO_MAX_IMAGES) return fail(VPB_ERR_ARG, "%s: %d images (1..%d)", fn, I, VPB_COCO_MAX_IMAGES);
  if (G < 0 || F < 0 || n < 0) return fail(VPB_ERR_ARG, "%s: %d ground truths, %d frames, %d rows", fn, G, F, n);
  if (!gts->offsets || (G > 0 && (!gts->kpts || !gts->area || !gts->bbox || !gts->iscrowd || !gts->num_keypoints)))
    return fail(VPB_ERR_ARG, "%s: null ground-truth buffer", fn);
  if ((F > 0 && (!dets->counts || !dets->frame_image)) || (n > 0 && (!dets->kpts || !dets->scores)))
    return fail(VPB_ERR_ARG, "%s: null detection buffer", fn);
  if (dets->keep && F > 0 && !dets->keep_counts) return fail(VPB_ERR_ARG, "%s: a keep list needs keep counts", fn);
  if (!d_workspace || !d_stats || !d_precision || !d_recall || !d_status) return fail(VPB_ERR_ARG, "%s: null output buffer", fn);
  const CocoWorkspace w = coco_workspace(I, F);
  if (workspace_bytes < static_cast<int64_t>(w.total))
    return fail(VPB_ERR_ARG, "%s: workspace of %lld bytes (%lld needed)", fn, static_cast<long long>(workspace_bytes),
                static_cast<long long>(w.total));
  if (!h_sigmas && k != 17) return fail(VPB_ERR_ARG, "%s: %d keypoints need sigmas (the default table has 17)", fn, k);
  CocoEvalParams q;
  memset(&q, 0, sizeof(q));
  const double* sig = h_sigmas ? h_sigmas : kCocoSigmas;
  for (int j = 0; j < k; ++j) {
    if (!std::isfinite(sig[j])) return fail(VPB_ERR_ARG, "%s: sigma %d is not finite", fn, j);
    const double v = sig[j] * 2.0;
    q.vars[j] = v * v;
  }
  char* ws = static_cast<char*>(d_workspace);
  q.gt_offsets = gts->offsets; q.gt_kpts = gts->kpts; q.gt_area = gts->area; q.gt_bbox = gts->bbox;
  q.gt_iscrowd = gts->iscrowd; q.gt_num_kpts = gts->num_keypoints;
  q.dt_kpts = dets->kpts; q.dt_scores = dets->scores; q.counts = dets->counts; q.frame_image = dets->frame_image;
  q.keep = dets->keep; q.keep_counts = dets->keep_counts;
  q.frame_row0 = reinterpret_cast<int32_t*>(ws + w.frame_row0);
  q.key[0] = reinterpret_cast<double*>(ws + w.key0); q.key[1] = reinterpret_cast<double*>(ws + w.key1);
  q.slot[0] = reinterpret_cast<int32_t*>(ws + w.slot0); q.slot[1] = reinterpret_cast<int32_t*>(ws + w.slot1);
  q.bits = reinterpret_cast<unsigned long long*>(ws + w.bits);
  q.num_dets = reinterpret_cast<int32_t*>(ws + w.num_dets);
  q.npig = reinterpret_cast<int32_t*>(ws + w.npig);
  q.summary = reinterpret_cast<double*>(ws + w.summary);
  q.stats = d_stats; q.precision = d_precision; q.recall = d_recall; q.status = d_status;
  q.k = k; q.num_images = I; q.num_gts = G; q.num_frames = F; q.n_rows = n;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int smem = static_cast<int>(sizeof(CocoImageShared));
  CU_TRY(cudaFuncSetAttribute(coco_image_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (F > 0) coco_frames_kernel<<<1, 1024, 0, st>>>(q);
  coco_image_kernel<<<I, COCO_THREADS, smem, st>>>(q);
  const long long slots = static_cast<long long>(I) * COCO_MAX_DETS;
  int src = 0;
  for (long long width = COCO_MAX_DETS; width < slots; width *= 2, src ^= 1)
    coco_merge_kernel<<<static_cast<unsigned>((slots + COCO_THREADS - 1) / COCO_THREADS), COCO_THREADS, 0, st>>>(q, src, width);
  coco_accumulate_kernel<<<COCO_A * COCO_T, COCO_ACC_THREADS, 0, st>>>(q, src);
  coco_summarize_kernel<<<1, 32, 0, st>>>(q);
  CU_TRY(cudaGetLastError());
  return VPB_OK;
}

// RGB and NV12 as the multi-frame calls
template <class Entry, class Frame>
static int infer_affine_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt, const double* d_mats,
                          const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream) {
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!d_mats || !d_cs || !d_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  return frames_core(e, tab, nt, nullptr, d_mats, d_cs, {{0, n}}, false, n, d_kpts, d_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int infer_affine_host_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                               const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream) {
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!h_mats || !h_cs || !h_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  VPB_TRY(check_affine_host(h_mats, h_cs, n));
  return frames_host_sync(e, tab, nt, nullptr, h_mats, h_cs, {{0, n}}, false, n, h_kpts, h_idx, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_infer_affine(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const double* d_mats, const float* d_cs,
                                float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_affine_t<FrameEntry>("vpb_infer_affine", e, h_frames, num_frames, YuvFormat{}, d_mats, d_cs, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_affine_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const double* h_mats, const float* h_cs,
                                     float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_affine_host_t<FrameEntry>("vpb_infer_affine_host", e, h_frames, num_frames, YuvFormat{}, h_mats, h_cs, h_kpts, h_idx, stream);
}
extern "C" int vpb_infer_affine_nv12(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                     const double* d_mats, const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_affine_t<YuvEntry>("vpb_infer_affine_nv12", e, h_frames, num_frames, nv12_format(matrix), d_mats, d_cs, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_affine_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                          const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_affine_host_t<YuvEntry>("vpb_infer_affine_nv12_host", e, h_frames, num_frames, nv12_format(matrix), h_mats, h_cs, h_kpts, h_idx, stream);
}
extern "C" int vpb_infer_affine_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                    int32_t range, const double* d_mats, const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_affine_t<YuvEntry>("vpb_infer_affine_yuv", e, h_frames, num_frames, yuv_format(layout, matrix, range), d_mats, d_cs, d_kpts,
                                  d_idx, stream);
}
extern "C" int vpb_infer_affine_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                         int32_t range, const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_affine_host_t<YuvEntry>("vpb_infer_affine_yuv_host", e, h_frames, num_frames, yuv_format(layout, matrix, range), h_mats, h_cs,
                                       h_kpts, h_idx, stream);
}

// ------------------------------------------------------------------------------------------------ multi-head calls
static int check_ready_heads(vpb_engine* e, const char* fn) {
  if (!e) return fail(VPB_ERR_ARG, "%s: null engine", fn);
  if (!e->finalized) return fail(VPB_ERR_STATE, "weights not finalized: call vpb_finalize first");
  if (e->flip && !e->flip_heads)
    return fail(VPB_ERR_STATE, "%s: flip test was set by vpb_set_flip_test; the multi-head calls take vpb_set_flip_test_heads", fn);
  return VPB_OK;
}
// appends `count` crops of `head` to the runs (runs of one head merge; empty ones vanish)
static int add_segment(vpb_engine* e, const char* fn, std::vector<Segment>& segs, int item, int head, int count) {
  if (head < 0 || head >= e->num_kheads) return fail(VPB_ERR_ARG, "%s: entry %d names head %d (the engine has %d)", fn, item, head, e->num_kheads);
  if (count < 0) return fail(VPB_ERR_ARG, "%s: entry %d has count %d", fn, item, count);
  if (count == 0) return VPB_OK;
  if (!segs.empty() && segs.back().head == head) segs.back().count += count;
  else segs.push_back({head, count});
  return VPB_OK;
}

extern "C" int vpb_infer_heads(vpb_engine* e, const float* d_crops, const int32_t* d_org_wh, const vpb_segment* h_segs, int32_t num_segs,
                               float* d_kpts, int32_t* d_idx, float* d_heatmaps, void* stream) {
  VPB_TRY(check_ready_heads(e, "vpb_infer_heads"));
  if (num_segs < 0 || num_segs > VPB_MAX_SEGMENTS || (num_segs > 0 && !h_segs))
    return fail(VPB_ERR_ARG, "vpb_infer_heads: %d segments (0..%d), segment array %p", num_segs, VPB_MAX_SEGMENTS, static_cast<const void*>(h_segs));
  std::vector<Segment> segs;
  long long n = 0;
  for (int i = 0; i < num_segs; ++i) {
    VPB_TRY(add_segment(e, "vpb_infer_heads", segs, i, h_segs[i].head, h_segs[i].count));
    n += h_segs[i].count;
  }
  if (n > e->maxB) return fail(VPB_ERR_ARG, "vpb_infer_heads: %lld crops exceed max_batch = %d", n, e->maxB);
  if (e->flip && 2 * n > e->maxB)
    return fail(VPB_ERR_ARG, "vpb_infer_heads: %lld crops: with flip test on a call takes at most max_batch / 2 = %d", n, e->maxB / 2);
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!d_crops || !d_org_wh || !d_kpts) return fail(VPB_ERR_ARG, "vpb_infer_heads: null pointer");
  Source src;
  src.crops = d_crops;
  return heads_core(e, src, segs, true, static_cast<int>(n), d_org_wh, nullptr, d_kpts, d_idx, d_heatmaps, static_cast<cudaStream_t>(stream));
}

// the runs of equal head over the frames that have boxes (frame j's boxes all belong to head h_heads[j])
template <class Frame>
static int frame_segments(vpb_engine* e, const char* fn, const Frame* fr, int32_t num_frames, const int32_t* h_heads,
                          std::vector<Segment>* segs) {
  if (num_frames > 0 && !h_heads) return fail(VPB_ERR_ARG, "%s: null head array", fn);
  for (int j = 0; j < num_frames; ++j)
    if (fr[j].num_boxes > 0) VPB_TRY(add_segment(e, fn, *segs, j, h_heads[j], fr[j].num_boxes));
  return VPB_OK;
}

// one body per multi-head call kind, for RGB frames (FrameEntry) and YUV frames (YuvEntry), as the multi-frame calls
template <class Entry, class Frame>
static int infer_frames_heads_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                                const int32_t* h_heads, const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream) {
  VPB_TRY(check_ready_heads(e, fn));
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  std::vector<Segment> segs;
  VPB_TRY(frame_segments(e, fn, h_frames, num_frames, h_heads, &segs));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!d_bboxes || !d_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  return frames_core(e, tab, nt, d_bboxes, nullptr, nullptr, segs, true, n, d_kpts, d_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int infer_frames_heads_host_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                                     const int32_t* h_heads, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream) {
  VPB_TRY(check_ready_heads(e, fn));
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  std::vector<Segment> segs;
  VPB_TRY(frame_segments(e, fn, h_frames, num_frames, h_heads, &segs));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!h_bboxes || !h_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  VPB_TRY(check_frames_boxes_host(h_frames, num_frames, h_bboxes));
  return frames_host_sync(e, tab, nt, h_bboxes, nullptr, nullptr, segs, true, n, h_kpts, h_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int infer_affine_heads_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                                const int32_t* h_heads, const double* d_mats, const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream) {
  VPB_TRY(check_ready_heads(e, fn));
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  std::vector<Segment> segs;
  VPB_TRY(frame_segments(e, fn, h_frames, num_frames, h_heads, &segs));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!d_mats || !d_cs || !d_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  return frames_core(e, tab, nt, nullptr, d_mats, d_cs, segs, true, n, d_kpts, d_idx, static_cast<cudaStream_t>(stream));
}
template <class Entry, class Frame>
static int infer_affine_heads_host_t(const char* fn, vpb_engine* e, const Frame* h_frames, int32_t num_frames, const YuvFormat& fmt,
                                     const int32_t* h_heads, const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx,
                                     void* stream) {
  VPB_TRY(check_ready_heads(e, fn));
  Entry tab[VPB_MAX_FRAMES];
  int nt = 0;
  int32_t n = 0;
  VPB_TRY(frame_table(fn, e, h_frames, num_frames, fmt, tab, &nt, &n));
  std::vector<Segment> segs;
  VPB_TRY(frame_segments(e, fn, h_frames, num_frames, h_heads, &segs));
  if (n == 0) return VPB_OK;
  DeviceGuard dev_guard(e);
  if (!h_mats || !h_cs || !h_kpts) return fail(VPB_ERR_ARG, "%s: null pointer", fn);
  VPB_TRY(check_affine_host(h_mats, h_cs, n));
  return frames_host_sync(e, tab, nt, nullptr, h_mats, h_cs, segs, true, n, h_kpts, h_idx, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_infer_frames_heads(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                      const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_frames_heads_t<FrameEntry>("vpb_infer_frames_heads", e, h_frames, num_frames, YuvFormat{}, h_heads, d_bboxes, d_kpts, d_idx,
                                          stream);
}
extern "C" int vpb_infer_frames_heads_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                           const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_frames_heads_host_t<FrameEntry>("vpb_infer_frames_heads_host", e, h_frames, num_frames, YuvFormat{}, h_heads, h_bboxes,
                                               h_kpts, h_idx, stream);
}
extern "C" int vpb_infer_affine_heads(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                      const double* d_mats, const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_affine_heads_t<FrameEntry>("vpb_infer_affine_heads", e, h_frames, num_frames, YuvFormat{}, h_heads, d_mats, d_cs, d_kpts,
                                          d_idx, stream);
}
extern "C" int vpb_infer_affine_heads_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                           const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_affine_heads_host_t<FrameEntry>("vpb_infer_affine_heads_host", e, h_frames, num_frames, YuvFormat{}, h_heads, h_mats, h_cs,
                                               h_kpts, h_idx, stream);
}
extern "C" int vpb_infer_frames_heads_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout,
                                          int32_t matrix, int32_t range, const int32_t* h_heads, const int32_t* d_bboxes, float* d_kpts,
                                          int32_t* d_idx, void* stream) {
  return infer_frames_heads_t<YuvEntry>("vpb_infer_frames_heads_yuv", e, h_frames, num_frames, yuv_format(layout, matrix, range), h_heads,
                                        d_bboxes, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_frames_heads_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout,
                                               int32_t matrix, int32_t range, const int32_t* h_heads, const int32_t* h_bboxes,
                                               float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_frames_heads_host_t<YuvEntry>("vpb_infer_frames_heads_yuv_host", e, h_frames, num_frames, yuv_format(layout, matrix, range),
                                             h_heads, h_bboxes, h_kpts, h_idx, stream);
}
extern "C" int vpb_infer_affine_heads_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout,
                                          int32_t matrix, int32_t range, const int32_t* h_heads, const double* d_mats, const float* d_cs,
                                          float* d_kpts, int32_t* d_idx, void* stream) {
  return infer_affine_heads_t<YuvEntry>("vpb_infer_affine_heads_yuv", e, h_frames, num_frames, yuv_format(layout, matrix, range), h_heads,
                                        d_mats, d_cs, d_kpts, d_idx, stream);
}
extern "C" int vpb_infer_affine_heads_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout,
                                               int32_t matrix, int32_t range, const int32_t* h_heads, const double* h_mats,
                                               const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream) {
  return infer_affine_heads_host_t<YuvEntry>("vpb_infer_affine_heads_yuv_host", e, h_frames, num_frames, yuv_format(layout, matrix, range),
                                             h_heads, h_mats, h_cs, h_kpts, h_idx, stream);
}

// ------------------------------------------------------------------------------------------------ host crops
extern "C" int vpb_infer_host(vpb_engine* e, const float* h_crops, const int32_t* h_org_wh, int32_t batch, float* h_kpts,
                              int32_t* h_idx, void* stream) {
  VPB_TRY(check_ready_keypoints(e, batch));
  DeviceGuard dev_guard(e);
  if (!h_crops || !h_org_wh || !h_kpts) return fail(VPB_ERR_ARG, "vpb_infer_host: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CU_TRY(cudaStreamWaitEvent(st, e->ev_done[0], 0));      // slot 0 is shared with the pipelined path: its last user is done
  CU_TRY(cudaMemcpyAsync(e->crops_stage[0], h_crops, static_cast<size_t>(batch) * 3 * 256 * 192 * sizeof(float), cudaMemcpyHostToDevice, st));
  CU_TRY(cudaMemcpyAsync(e->org_wh[0], h_org_wh, static_cast<size_t>(batch) * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  VPB_TRY(vpb_infer(e, e->crops_stage[0], e->org_wh[0], batch, e->kpts[0], e->idx[0], nullptr, st));
  return host_tail(e, {{0, batch}}, false, 0, h_kpts, h_idx, st, true);
}

// Pipelined form of vpb_infer_host: submit(slot) enqueues H2D on the engine's copy stream and the path + D2H on its compute
// stream and returns; wait(slot) blocks until that slot's keypoints are in the caller's buffer.  With two slots in flight
// the H2D of batch i+1 runs under the compute of batch i.  Host buffers must stay valid (and should be pinned) until wait().
extern "C" int vpb_submit_host(vpb_engine* e, const float* h_crops, const int32_t* h_org_wh, int32_t batch, float* h_kpts,
                               int32_t* h_idx, int32_t slot) {
  VPB_TRY(check_ready_keypoints(e, batch));
  DeviceGuard dev_guard(e);
  if (!h_crops || !h_org_wh || !h_kpts || slot < 0 || slot > 1) return fail(VPB_ERR_ARG, "vpb_submit_host: bad argument");
  // the slot's previous use must have finished with its staging buffers before they are overwritten
  CU_TRY(cudaStreamWaitEvent(e->copy_stream, e->ev_done[slot], 0));
  CU_TRY(cudaMemcpyAsync(e->crops_stage[slot], h_crops, static_cast<size_t>(batch) * 3 * 256 * 192 * sizeof(float), cudaMemcpyHostToDevice,
                         e->copy_stream));
  CU_TRY(cudaMemcpyAsync(e->org_wh[slot], h_org_wh, static_cast<size_t>(batch) * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, e->copy_stream));
  CU_TRY(cudaEventRecord(e->ev_h2d[slot], e->copy_stream));
  CU_TRY(cudaStreamWaitEvent(e->compute_stream, e->ev_h2d[slot], 0));
  VPB_TRY(vpb_infer(e, e->crops_stage[slot], e->org_wh[slot], batch, e->kpts[slot], e->idx[slot], nullptr, e->compute_stream));
  return host_tail(e, {{0, batch}}, false, slot, h_kpts, h_idx, e->compute_stream, false);
}
extern "C" int vpb_wait_host(vpb_engine* e, int32_t slot) {
  if (!e || slot < 0 || slot > 1) return fail(VPB_ERR_ARG, "vpb_wait_host: bad argument");
  CU_TRY(cudaEventSynchronize(e->ev_done[slot]));
  return VPB_OK;
}

extern "C" void* vpb_host_alloc(int64_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, static_cast<size_t>(bytes), cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
extern "C" void vpb_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

extern "C" int vpb_cached_graphs(const vpb_engine* e, int32_t mixed, int32_t* entries, int32_t* captured) {
  if (!e || !entries || !captured) return fail(VPB_ERR_ARG, "vpb_cached_graphs: null argument");
  *entries = *captured = 0;
  for (const auto& g : e->graph_cache)
    if (g.mixed == (mixed != 0)) { ++*entries; *captured += g.exec != nullptr; }
  return VPB_OK;
}
extern "C" int64_t vpb_device_bytes(const vpb_engine* e) {
  if (!e) return -1;
  size_t b = e->alloc_bytes;
  for (int s = 0; s < 2; ++s) b += e->frame_cap[s] ? e->frame_cap[s] + 256 : 0;
  return static_cast<int64_t>(b);
}

extern "C" int vpb_kernel_launches(const vpb_engine* e, int32_t batch) {
  if (!e) return -1;
  // patch im2col + patch GEMM + depth*(qkv, attention, proj, fc1, fc2) + 2 deconv GEMMs + 1x1 GEMM + decode; the 2*depth+1
  // LayerNorms ride in the tails of the patch / proj / fc2 GEMMs unless ln_fused is switched off
  // flip test adds the flip-back average in front of the decode; the chains then see 2 * batch crops
  if (e->use_chain && model_crops(e, batch) >= e->chain_min_batch && !e->ln_fused)
    return 1 + (1 + e->depth) + e->depth + 2 + 1 + 1 + (e->flip ? 1 : 0);   // gather, chains, attention, deconvs, 1x1, decode
  // one kernel per GEMM: gather, patch GEMM, depth x (qkv, attention, proj, fc1, fc2), 2 deconvs, 1x1, decode; the LayerNorms are
  // launches of their own (2 * depth + 1), or ride in front of qkv / fc1 (ln_in_gemm: only last_norm is left), or in the tails.
  // qkv and attention are one launch per block where fuse_qkv_attention says so (large batches)
  return 2 + e->depth * (fuse_qkv_attention(e, model_crops(e, batch)) ? 4 : 5) + 2 + 1 + 1 +
         (e->ln_fused ? 0 : e->ln_in_gemm ? 1 : 2 * e->depth + 1) + (e->flip ? 1 : 0);
}

// Debug option "poison": every float and bf16 activation and staging buffer filled with 0xFF bytes (NaN in both types), so a test
// can tell whether a call uses a value it did not write itself (padding rows of a ragged row block, the unused rows of the 96-position
// deconv tiles, the maps past a smaller head's K, what an earlier and larger call left behind).  Integer and double buffers,
// counters and status words (idx, org_wh, g_org, g_offs, pp_*, bbox_stage, mat_stage, flip_perm, chain_counters, ln_counters)
// are left alone: garbage there would change addressing or the chained-launch protocol, not values.  The cached graphs stay.
static int poison_workspace(vpb_engine* e) {
  if (!e->finalized) return fail(VPB_ERR_STATE, "poison: not finalized");
  DeviceGuard dev_guard(e);
  CU_TRY(cudaDeviceSynchronize());              // pending calls (submit slots included) finish on the memory they started with
  const size_t B = e->maxB, M = B * 192, D = e->D, K = e->Kmax, bf = sizeof(__nv_bfloat16), f = sizeof(float);
  const std::pair<void*, size_t> bufs[] = {
      {e->patch_rows, M * 768 * bf}, {e->x, M * D * f}, {e->xn, M * D * bf}, {e->qkv, M * 3 * D * bf}, {e->attn, M * D * bf},
      {e->hid, M * 4 * D * bf}, {e->d1, B * 768 * 256 * bf}, {e->d2, B * 3072 * 256 * bf}, {e->heat, B * K * 3072 * f},
      {e->g_kpts, B * K * 3 * f}, {e->kpts[0], B * K * 3 * f}, {e->kpts[1], B * K * 3 * f},
      {e->crops_stage[0], B * 3 * 256 * 192 * f}, {e->crops_stage[1], B * 3 * 256 * 192 * f}, {e->g_cs, B * 4 * f}, {e->cs_stage, B * 4 * f}};
  for (const auto& b : bufs) CU_TRY(cudaMemset(b.first, 0xFF, b.second));
  CU_TRY(cudaDeviceSynchronize());
  return VPB_OK;
}

extern "C" int vpb_set_option(vpb_engine* e, const char* name, int32_t value) {
  if (!e || !name) return fail(VPB_ERR_ARG, "vpb_set_option: null argument");
  if (!strcmp(name, "stop_after")) e->stop_after = value;
  else if (!strcmp(name, "poison")) { if (value) VPB_TRY(poison_workspace(e)); }
  else if (!strcmp(name, "profile")) e->prof.on = value != 0;
  else if (!strcmp(name, "pdl")) g_pdl = value != 0;
  else if (!strcmp(name, "graph")) e->use_graph = value != 0;
  else if (!strcmp(name, "chain") || !strcmp(name, "chain_min_batch") || !strcmp(name, "gelu_erf") || !strcmp(name, "ln_in_gemm") ||
           !strcmp(name, "resid_rmw") || !strcmp(name, "ln_ctl") || !strcmp(name, "ln_job_rows")) {
    if (!strcmp(name, "ln_job_rows") && value != 8 && value != 16) return fail(VPB_ERR_ARG, "ln_job_rows must be 8 or 16");
    if (!strcmp(name, "gelu_erf")) e->gelu_erf = value != 0;
    else if (!strcmp(name, "resid_rmw")) e->resid_rmw = value != 0;
    else if (!strcmp(name, "ln_ctl")) e->ln_ctl = value != 0;
    else if (!strcmp(name, "ln_job_rows")) e->ln_job_rows = value;
    else if (!strcmp(name, "ln_in_gemm")) e->ln_in_gemm = value != 0;
    else if (!strcmp(name, "chain")) e->use_chain = value != 0;
    else e->chain_min_batch = value;
    drop_graphs(e);                   // captured chains embed the choice
  }
  else if (!strcmp(name, "ln_fused")) {
    e->ln_fused = value != 0;
    drop_graphs(e);                   // captured chains embed the choice
  }
  else return fail(VPB_ERR_ARG, "unknown option %s", name);
  return VPB_OK;
}

extern "C" int vpb_set_flip_test(vpb_engine* e, const int32_t* h_perm, int32_t k, int32_t shift) {
  if (!e) return fail(VPB_ERR_ARG, "vpb_set_flip_test: null engine");
  if (!e->finalized) return fail(VPB_ERR_STATE, "not finalized");
  if (e->num_kheads > 1) return fail(VPB_ERR_STATE, "vpb_set_flip_test: not supported on an engine with %d heads", e->num_kheads);
  if (h_perm) {
    if (k != e->K) return fail(VPB_ERR_ARG, "vpb_set_flip_test: permutation of %d keypoints, the engine has %d", k, e->K);
    for (int i = 0; i < k; ++i)
      if (h_perm[i] < 0 || h_perm[i] >= k) return fail(VPB_ERR_ARG, "vpb_set_flip_test: perm[%d] = %d outside 0..%d", i, h_perm[i], k - 1);
  }
  DeviceGuard dev_guard(e);
  // calls already enqueued (submit slots in flight included) read the old permutation: let them finish first
  if (e->ws_used) CU_TRY(cudaEventSynchronize(e->ev_ws));
  if (h_perm) CU_TRY(cudaMemcpy(e->flip_perm, h_perm, static_cast<size_t>(k) * sizeof(int32_t), cudaMemcpyHostToDevice));
  e->flip = h_perm != nullptr;
  e->flip_heads = false;
  e->flip_shift = shift ? 1 : 0;
  drop_graphs(e);                     // captured chains embed the batch and the average
  return VPB_OK;
}

extern "C" int vpb_set_flip_test_heads(vpb_engine* e, const int32_t* h_perms, int32_t total, int32_t shift) {
  if (!e) return fail(VPB_ERR_ARG, "vpb_set_flip_test_heads: null engine");
  if (!e->finalized) return fail(VPB_ERR_STATE, "not finalized");
  if (h_perms) {
    const int want = perm_offset(e, e->num_kheads);
    if (total != want) return fail(VPB_ERR_ARG, "vpb_set_flip_test_heads: %d permutation entries, the heads have %d keypoints in all", total, want);
    for (int j = 0; j < e->num_kheads; ++j) {
      const int32_t* p = h_perms + perm_offset(e, j);
      for (int i = 0; i < e->hw[j].K; ++i)
        if (p[i] < 0 || p[i] >= e->hw[j].K)
          return fail(VPB_ERR_ARG, "vpb_set_flip_test_heads: head %d: perm[%d] = %d outside 0..%d", j, i, p[i], e->hw[j].K - 1);
    }
  }
  DeviceGuard dev_guard(e);
  if (e->ws_used) CU_TRY(cudaEventSynchronize(e->ev_ws));     // pending calls read the old permutations
  if (h_perms) CU_TRY(cudaMemcpy(e->flip_perm, h_perms, static_cast<size_t>(total) * sizeof(int32_t), cudaMemcpyHostToDevice));
  e->flip = e->flip_heads = h_perms != nullptr;
  e->flip_shift = shift ? 1 : 0;
  drop_graphs(e);
  return VPB_OK;
}

extern "C" int vpb_profile_classes(void) { return KC_COUNT; }
extern "C" const char* vpb_profile_class_name(int32_t cls) { return (cls >= 0 && cls < KC_COUNT) ? kclass_names[cls] : ""; }
extern "C" int vpb_profile_collect(vpb_engine* e, float* ms_per_class, int32_t* launches_per_class) {
  if (!e || !ms_per_class || !launches_per_class) return fail(VPB_ERR_ARG, "vpb_profile_collect: null argument");
  CU_TRY(cudaDeviceSynchronize());
  for (int i = 0; i < KC_COUNT; ++i) { ms_per_class[i] = 0.f; launches_per_class[i] = 0; }
  for (auto& r : e->prof.recs) {
    float ms = 0.f;
    CU_TRY(cudaEventElapsedTime(&ms, r.a, r.b));
    ms_per_class[r.cls] += ms;
    launches_per_class[r.cls] += 1;
    e->prof.pool.push_back({r.a, r.b});
  }
  e->prof.recs.clear();
  return VPB_OK;
}

extern "C" int vpb_read_buffer(vpb_engine* e, const char* name, void* host_dst, int64_t bytes) {
  if (!e || !name || !host_dst) return fail(VPB_ERR_ARG, "vpb_read_buffer: null argument");
  if (!e->finalized) return fail(VPB_ERR_STATE, "not finalized");
  const void* src = nullptr;
  const std::string n(name);
  if (n == "patch_rows") src = e->patch_rows;
  else if (n == "x") src = e->x;
  else if (n == "xn") src = e->xn;
  else if (n == "qkv") src = e->qkv;
  else if (n == "attn") src = e->attn;
  else if (n == "hid") src = e->hid;
  else if (n == "d1") src = e->d1;
  else if (n == "d2") src = e->d2;
  else if (n == "heat") src = e->heat;
  else return fail(VPB_ERR_ARG, "unknown buffer %s", name);
  CU_TRY(cudaDeviceSynchronize());
  CU_TRY(cudaMemcpy(host_dst, src, bytes, cudaMemcpyDeviceToHost));
  return VPB_OK;
}

// ------------------------------------------------------------------------------------------------ kernel-level entry points
extern "C" int vpb_gemm(const void* d_a, const void* d_w, const float* d_bias, void* d_out, int32_t m, int32_t n, int32_t k,
                        int32_t epilogue, const float* d_resid, int32_t resid_mod, int32_t aux0, int32_t aux1, int32_t aux2,
                        int32_t aux3, void* stream) {
  if (!d_a || !d_w || !d_out) return fail(VPB_ERR_ARG, "vpb_gemm: null pointer");
  if (m < 1 || n < 1) return fail(VPB_ERR_ARG, "vpb_gemm: M=%d N=%d must be positive", m, n);
  if (!d_bias && epilogue != EPI_F32_NCHW) return fail(VPB_ERR_ARG, "vpb_gemm: epilogue %d reads a bias", epilogue);
  if (epilogue == EPI_F32_NCHW && (aux0 < 1 || aux0 > n || aux1 < 1))
    return fail(VPB_ERR_ARG, "vpb_gemm: NCHW epilogue with %d channels of %d, %d pixels", aux0, n, aux1);
  if (epilogue == EPI_BF16_RELU_UP && (aux0 < 1 || aux1 < 1)) return fail(VPB_ERR_ARG, "vpb_gemm: deconv input %d x %d", aux0, aux1);
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  VPB_TRY(device_check(dev));
  int bn;
  CUtensorMap ta, tw, tout;
  if (epi_uses_tma(epilogue)) {                  // the engine's width rule and debug overrides (pick_tile)
    LinearW L;
    L.n = n; L.k = k;
    VPB_TRY(make_tile_maps(L, d_w, n, k));
    const CUtensorMap* wm;
    VPB_TRY(pick_tile(L, m, &bn, &wm));
  } else {
    bn = epilogue == EPI_F32_NCHW ? (n <= 32 ? 32 : 144) : 256;
  }
  if (epilogue == EPI_BF16_RELU_UP && n % bn != 0) return fail(VPB_ERR_ARG, "vpb_gemm: N=%d must be a multiple of %d", n, bn);
  if (epilogue == EPI_F32_NCHW && n != bn) return fail(VPB_ERR_ARG, "vpb_gemm: NCHW epilogue wants W padded to %d rows", bn);
  if (epilogue == EPI_BF16_RELU_UP) {
    // d_a: NHWC input [m / (H*W), H, W, C] with H = aux0, W = aux1, tile = aux2 rows x (aux3 >> 16) columns (96 or 128
    // positions), C = aux3 & 0xffff = k / 4; d_w: the four phase matrices stacked [4*256, 4*C]
    const int tile_w = aux3 >> 16, cin = aux3 & 0xffff;
    if ((tile_w * aux2 != 96 && tile_w * aux2 != 128) || cin * 4 != k || aux0 % aux2 != 0 || aux1 % tile_w != 0 || m % (aux0 * aux1) != 0)
      return fail(VPB_ERR_ARG, "vpb_gemm: bad deconv geometry");
    VPB_TRY(make_map_nhwc(&ta, d_a, m / (aux0 * aux1), aux0, aux1, cin, aux2, tile_w));
    VPB_TRY(make_map(&tw, d_w, 4 * n, k, k, bn));
  } else {
    VPB_TRY(make_map(&ta, d_a, m, k, k, 128));
    VPB_TRY(make_map(&tw, d_w, n, k, k, bn));
  }
  VPB_TRY(make_map(&tout, d_w, n, k, k, bn));   // placeholder for direct epilogues
  if (epilogue == EPI_BF16 || epilogue == EPI_BF16_GELU || epilogue == EPI_BF16_GELU_ERF) VPB_TRY(make_map(&tout, d_out, m, n, n, 64));
  if (epilogue == EPI_F32_ADD) VPB_TRY(make_map(&tout, d_out, m, n, n, 64, /*f32=*/true));
  GemmParams p = gp(m, n, k, d_bias, d_out, n);
  (void)d_resid; (void)resid_mod;
  if (epilogue == EPI_F32_NCHW) { p.n_valid = aux0; p.pix = aux1; }
  if (epilogue == EPI_BF16_RELU_UP) { p.up_h = aux0; p.up_w = aux1; p.up_tr = aux2; p.up_tw = aux3 >> 16; p.up_c = aux3 & 0xffff; }
  return gemm_launch(bn, epilogue, ta, tw, tout, p, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_expert_gemm(const void* d_a, const void* d_w, const float* d_bias, float* d_x, int32_t m, int32_t d, int32_t p,
                               int32_t num_experts, const int32_t* h_segs, int32_t num_segs, int32_t shared, void* stream) {
  if (!d_a || !d_w || !d_bias || !d_x || !h_segs) return fail(VPB_ERR_ARG, "vpb_expert_gemm: null pointer");
  if (m < 1 || d < 64 || d % 32 != 0 || p < 32 || p >= d || p % 32 != 0 || num_experts < 1 || num_segs < 1 || num_segs > EXPERT_MAX_SEGMENTS)
    return fail(VPB_ERR_ARG, "vpb_expert_gemm: M=%d D=%d P=%d experts=%d segments=%d", m, d, p, num_experts, num_segs);
  ExpertParams q = expert_params(d, p, d_bias, d_x);
  for (int i = 0, prev_end = 0; i < num_segs; ++i) {
    const int32_t* sg = h_segs + 3 * i;
    if (sg[0] < prev_end || sg[1] <= sg[0] || sg[1] > m || sg[2] < 0 || sg[2] >= num_experts)
      return fail(VPB_ERR_ARG, "vpb_expert_gemm: segment %d = rows [%d, %d) expert %d", i, sg[0], sg[1], sg[2]);
    add_expert_segment(q, sg[0], sg[1], sg[2]);
    prev_end = sg[1];
  }
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  VPB_TRY(device_check(dev));
  const int S = d - p, K = 4 * d;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap ta, tw;
  VPB_TRY(make_map(&ta, d_a, m, K, K, 128));
  if (shared) {
    LinearW Ls;
    CUtensorMap o_xs;
    VPB_TRY(make_shared_maps(Ls, static_cast<__nv_bfloat16*>(const_cast<void*>(d_w)), const_cast<float*>(d_bias), S, K));
    VPB_TRY(make_map(&o_xs, d_x, m, S, d, 64, /*f32=*/true));
    VPB_TRY(fc2_shared_launch(Ls, m, d, d_x, ta, o_xs, st));
  }
  VPB_TRY(make_map(&tw, d_w, S + static_cast<uint64_t>(num_experts) * p, K, K, expert_width(p)));
  return expert_launch(expert_width(p), ta, tw, q, st);
}

// The attention entry points' shape checks, before any device work: a built head_dim, positive counts, and no int overflow of
// the qkv row width 3 D, the item count batch * heads or the row count batch * 192 (all int in the kernels and TMA coordinates)
static int attention_shape_check(const char* fn, int32_t batch, int32_t heads, int32_t head_dim) {
  if (head_dim != 32 && head_dim != 64 && head_dim != 80) return fail(VPB_ERR_ARG, "%s: head_dim %d not built (32, 64, 80)", fn, head_dim);
  if (batch < 1 || heads < 1) return fail(VPB_ERR_ARG, "%s: batch %d, heads %d must be positive", fn, batch, heads);
  constexpr int64_t kMax = INT32_MAX;
  if (3 * static_cast<int64_t>(heads) * head_dim > kMax || static_cast<int64_t>(batch) * heads > kMax || static_cast<int64_t>(batch) * ATT_T > kMax)
    return fail(VPB_ERR_ARG, "%s: batch %d x heads %d x head_dim %d overflows int", fn, batch, heads, head_dim);
  return VPB_OK;
}

extern "C" int vpb_attention(const void* d_qkv, int32_t batch, int32_t heads, int32_t head_dim, void* d_out, void* stream) {
  if (!d_qkv || !d_out) return fail(VPB_ERR_ARG, "vpb_attention: null pointer");
  VPB_TRY(attention_shape_check("vpb_attention", batch, heads, head_dim));
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  VPB_TRY(device_check(dev));
  const int D = heads * head_dim;
  CUtensorMap tm, tt;
  VPB_TRY(make_attn_maps(&tm, &tt, d_qkv, static_cast<uint64_t>(batch) * 192, D, head_dim));
  AttnParams ap;
  ap.batch = batch; ap.heads = heads; ap.dim = D; ap.out = reinterpret_cast<__nv_bfloat16*>(d_out); ap.dbg = g_dbg_buf;
  return attention_launch(head_dim, tm, tt, ap, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_qkv_attention(const void* d_xn, const void* d_w, const float* d_bias, int32_t batch, int32_t heads, int32_t head_dim,
                                 void* d_out, void* stream) {
  if (!d_xn || !d_w || !d_bias || !d_out) return fail(VPB_ERR_ARG, "vpb_qkv_attention: null pointer");
  VPB_TRY(attention_shape_check("vpb_qkv_attention", batch, heads, head_dim));
  const int D = heads * head_dim;
  if (D % 64 != 0) return fail(VPB_ERR_ARG, "vpb_qkv_attention: D = %d is not a whole number of 64-wide k-blocks", D);
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  VPB_TRY(device_check(dev));
  CUtensorMap tx, tw;
  VPB_TRY(make_map(&tx, d_xn, static_cast<uint64_t>(batch) * 192, D, D, 192));
  VPB_TRY(make_map(&tw, d_w, 3 * static_cast<uint64_t>(D), D, D, head_dim));
  QkvAttnParams qp;
  qp.batch = batch; qp.heads = heads; qp.dim = D; qp.bias = d_bias; qp.out = reinterpret_cast<__nv_bfloat16*>(d_out); qp.dbg = g_dbg_buf;
  return qkv_attention_launch(head_dim, tx, tw, qp, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, void* d_y, int32_t rows, int32_t dim, float eps,
                             void* stream) {
  if (!d_x || !d_gamma || !d_beta || !d_y) return fail(VPB_ERR_ARG, "vpb_layernorm: null pointer");
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  VPB_TRY(device_check(dev));
  return layernorm(d_x, d_gamma, d_beta, reinterpret_cast<__nv_bfloat16*>(d_y), rows, dim, eps, static_cast<cudaStream_t>(stream));
}
