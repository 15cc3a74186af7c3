// HBM/L2-bound helper kernels around the tensor-core GEMMs: LayerNorm, the patch-embedding im2col gather
// and the one-time weight packing (the deconvs need no gather: gemm.cuh reads shifted NHWC boxes by 4-D TMA).  All of them move
// 16 bytes per thread per access and keep a warp on consecutive addresses.
#pragma once
#include "ptx.cuh"

namespace vpb {

// ------------------------------------------------------------------------------------------------
// LayerNorm(eps) over the last dim of x f32 [rows, D] -> bf16 [rows, D].  Persistent warps (grid = a few CTAs per SM)
// walk rows with stride; a row lives in registers (D/128 float4 per lane) and the NEXT row's loads are already in flight
// while the current row is reduced (fp32 mean and biased variance by warp shuffles) and written.
// Reference: nn.LayerNorm(eps=1e-6) at backbone/vit.py:190,198,304.
template <int D>
__global__ void __launch_bounds__(128) layernorm_f32_to_bf16(const float* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                                                             int rows, float eps) {
  static_assert(D % 128 == 0, "row must split into float4 per lane");
  constexpr int V = D / 128;
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  pdl_launch_dependents();
  pdl_wait();
  if (row >= rows) return;
  float4 nxt[V];
  {
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
#pragma unroll
    for (int i = 0; i < V; ++i) nxt[i] = xr[i * 32 + lane];
  }
  for (; row < rows; row += warps_total) {
    float4 v[V];
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = nxt[i];
    const int nrow = row + warps_total;
    if (nrow < rows) {
      const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(nrow) * D);
#pragma unroll
      for (int i = 0; i < V; ++i) nxt[i] = xr[i * 32 + lane];
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    // a correctly rounded division, not s * fl(1/D): fl(1/D) is off by up to 2^-24 for D = 384, 768, 1280, which made the
    // mean of a constant row differ from its value by an ulp; at variance 0 rstd = eps^-1/2 = 1000 turned that into an
    // output of beta - 0.12 gamma instead of beta (a row of 1024.0 at D = 384).  ln_row_l2 and chain.cuh's LnRow match it.
    const float mean = s / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * (1.0f / D) + eps);
    uint2* yr = reinterpret_cast<uint2*>(y + static_cast<size_t>(row) * D);
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
}

// ------------------------------------------------------------------------------------------------
// Patch-embedding im2col: crops f32 [B,3,256,192] -> rows bf16 [B*192, 768],
//   row (b, py, px), col c*256 + ky*16 + kx  =  x[b, c, 16py-2+ky, 16px-2+kx]   (0 outside the image)
// Conv2d(k16,s16,p2) geometry from backbone/vit.py:222.  One thread = 8 consecutive kx of one patch
// row: reads 32 B of the image (8-byte aligned: columns start at -2), writes 16 B.
// The same launch seeds the fp32 token stream with  pos_embed[1+t] + pos_embed[0] + conv bias  (vit.py:382), so that the
// patch GEMM can add its product into it with the TMA reduce-add epilogue like every other residual GEMM.
// Flip test: with n_src < batch (batch = 2 n_src) the rows of crop b >= n_src are the im2col of flip(x[b - n_src], dims=[3]):
// image column xx reads source column 191 - xx, so the float2 pair (xx, xx + 1) is the source pair at 190 - xx (still
// 8-byte aligned) with its halves swapped.  The mirrored crops are never written to memory.
__global__ void __launch_bounds__(256) patch_im2col(const float* __restrict__ x, __nv_bfloat16* __restrict__ a, int batch, int n_src,
                                                    const float4* __restrict__ pos_bias, float4* __restrict__ stream, int D) {
  const int total = batch * 3 * 256 * 24;                  // (b, c, y', xchunk)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();            // the previous step may still be reading patch rows / the stream
  const int per_crop4 = 192 * D / 4;                       // float4 per crop in the stream
  for (long long j = i; j < static_cast<long long>(batch) * per_crop4; j += static_cast<long long>(gridDim.x) * blockDim.x)
    stream[j] = __ldg(pos_bias + j % per_crop4);
  if (i >= total) return;
  const int xc = i % 24;
  const int yp = (i / 24) % 256;                           // y' = 16*py + ky
  const int c = (i / (24 * 256)) % 3;
  const int b = i / (24 * 256 * 3);
  const int y = yp - 2, x0 = xc * 8 - 2;
  const bool mirror = b >= n_src;
  float v[8];
  if (y >= 0) {                                            // y' < 256 -> y <= 253 < 256 always
    const float* src = x + ((static_cast<size_t>(mirror ? b - n_src : b) * 3 + c) * 256 + y) * 192;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      const int xx = x0 + j;                               // even offset from -2: pairs never straddle the border
      if (xx >= 0 && xx < 192) {
        if (mirror) {
          const float2 f = *reinterpret_cast<const float2*>(src + 190 - xx);
          v[j] = f.y; v[j + 1] = f.x;
        } else {
          const float2 f = *reinterpret_cast<const float2*>(src + xx);
          v[j] = f.x; v[j + 1] = f.y;
        }
      } else {
        v[j] = 0.f; v[j + 1] = 0.f;
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
  }
  const int py = yp >> 4, ky = yp & 15, px = xc >> 1, kx0 = (xc & 1) * 8;
  const size_t row = (static_cast<size_t>(b) * 16 + py) * 12 + px;
  uint4 o;
  o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]); o.z = pack_bf16(v[4], v[5]); o.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(a + row * 768 + c * 256 + ky * 16 + kx0) = o;
}

// ------------------------------------------------------------------------------------------------
// One-time weight packing (fp32 state_dict tensors already on the device -> bf16 / folded fp32).
// Linear weight [N,K] f32 -> bf16, rows < scaled_rows multiplied by `scale` in fp32 first
// (the q rows of attn.qkv get head_dim^-0.5: vit.py:170 scales q before QK^T).
__global__ void pack_linear_bf16(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, long long n_elem, int K,
                                 int scaled_rows, float scale) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_elem) return;
  const int row = static_cast<int>(i / K);
  const float v = w[i] * (row < scaled_rows ? scale : 1.0f);
  out[i] = __float2bfloat16_rn(v);
}
__global__ void pack_bias(const float* __restrict__ b, float* __restrict__ out, int n, int n_padded, int scaled, float scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_padded) return;
  out[i] = i < n ? b[i] * (i < scaled ? scale : 1.0f) : 0.0f;
}
// pos_bias[t, d] = pos_embed[1+t, d] + pos_embed[0, d] + patch_bias[d]     (vit.py:382 + conv bias)
__global__ void pack_pos_bias(const float* __restrict__ pos, const float* __restrict__ pbias, float* __restrict__ out, int T, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * D) return;
  const int t = i / D, d = i % D;
  out[i] = pos[(1 + t) * D + d] + pos[d] + pbias[d];
}
// ConvTranspose2d(k4,s2,p1) = 4 sub-pixel phases (py,px); output (2m+py, 2n+px) sums 2x2 taps of the input
// (head/topdown_heatmap_simple_head.py:305-313, SURVEY.md 9.4):
//   T(0) = {(ky=1,dy=0),(ky=3,dy=-1)}   T(1) = {(ky=0,dy=+1),(ky=2,dy=0)}        (same along x)
// weight [Cin,Cout,4,4] + eval BatchNorm -> 4 phase matrices bf16 [Cout, 4*Cin] (tap-major K) with the
// BN scale folded into the rows, and the BN shift as bias.
//   Wp[phase][co][(iy*2+ix)*Cin + ci] = W[ci][co][ky(py,iy)][kx(px,ix)] * gamma[co]/sqrt(var[co]+eps)
__global__ void pack_deconv(const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ mean, const float* __restrict__ var, __nv_bfloat16* __restrict__ wp,
                            float* __restrict__ shift, int Cin, int Cout, float eps) {
  const long long total = 4LL * Cout * 4 * Cin;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ci = static_cast<int>(i % Cin);
  const int tap = static_cast<int>((i / Cin) % 4);
  const int co = static_cast<int>((i / (4LL * Cin)) % Cout);
  const int phase = static_cast<int>(i / (4LL * Cin * Cout));
  const int py = phase >> 1, px = phase & 1, iy = tap >> 1, ix = tap & 1;
  const int ky = py ? (iy ? 2 : 0) : (iy ? 3 : 1);
  const int kx = px ? (ix ? 2 : 0) : (ix ? 3 : 1);
  const float s = gamma[co] / sqrtf(var[co] + eps);
  wp[i] = __float2bfloat16_rn(w[((static_cast<size_t>(ci) * Cout + co) * 4 + ky) * 4 + kx] * s);
  if (phase == 0 && tap == 0 && ci == 0) shift[co] = beta[co] - mean[co] * s;
}
// token-major bf16 [B*192, D] -> f32 NCHW [B, D, 16, 12]   (ViT.forward's final permute, vit.py:388)
__global__ void tokens_to_nchw(const __nv_bfloat16* __restrict__ tok, float* __restrict__ out, int batch, int D) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(batch) * D * 192) return;
  const int t = static_cast<int>(i % 192);
  const int d = static_cast<int>((i / 192) % D);
  const int b = static_cast<int>(i / (192LL * D));
  out[i] = __bfloat162float(tok[(static_cast<size_t>(b) * 192 + t) * D + d]);
}

// f32 NCHW [B, D, 16, 12] -> token-major bf16 [B*192, D]: the way back, for callers that hand backbone features to the head
// (TopdownHeatmapSimpleHead.forward / inference_model, head/topdown_heatmap_simple_head.py:188-218).  Features produced by
// tokens_to_nchw are bf16 values, so the round trip is exact.
__global__ void nchw_to_tokens(const float* __restrict__ in, __nv_bfloat16* __restrict__ tok, int batch, int D) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;      // output index: coalesced bf16 writes
  if (i >= static_cast<long long>(batch) * D * 192) return;
  const int d = static_cast<int>(i % D);
  const int t = static_cast<int>((i / D) % 192);
  const int b = static_cast<int>(i / (192LL * D));
  tok[i] = __float2bfloat16_rn(__ldg(in + (static_cast<size_t>(b) * D + d) * 192 + t));
}

// flip_back (vit_utils/post_processing/post_transforms.py:110-147, GaussianHeatmap) + the optional one-pixel shift of
// inference_model (head/topdown_heatmap_simple_head.py:210-212):  out[n,k,y,x] = in[n, perm[k], y, W-1-x'] with x' = x, or
// x' = max(x - 1, 0) when shift is set (numpy's overlapping `a[..., 1:] = a[..., :-1]` copies first).  perm is the
// keypoint permutation the left/right pairs induce.  Pure data movement: bit-exact.
__global__ void flip_back_heatmaps(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ perm, int n, int k,
                                   int shift) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * k * 3072) return;
  const int x = static_cast<int>(i % 48), y = static_cast<int>((i / 48) % 64);
  const int kk = static_cast<int>((i / 3072) % k), nn = static_cast<int>(i / (3072LL * k));
  const int xs = shift ? max(x - 1, 0) : x;
  out[i] = __ldg(in + ((static_cast<size_t>(nn) * k + perm[kk]) * 64 + y) * 48 + (47 - xs));
}

// Flip-test average over the maps of one forward (maps of crop i < n from the crops, those of crop mirror + i from their mirror
// images):
//   out[i,k,y,x] = (heat[i,k,y,x] + heat[mirror+i, perm[k], y, 47 - x']) * 0.5f      (i < n, x' as in flip_back_heatmaps)
// mmpose's (output + output_flipped) * 0.5 with output_flipped = flip_back_heatmaps of the mirror maps, in the same fp32
// operations, so bit-identical to that composition.  kstride = maps between consecutive crops in heat and out (0 = k).  The
// single-head calls pass mirror = n and kstride = 0; a multi-head call launches once per segment, with heat / out at the
// segment's first crop, its head's k and permutation, kstride = K_max and mirror = the call's crop count.  `out` may be
// `heat` itself: each output element reads its own position and a mirror position, which is never written.
__global__ void flip_average_heatmaps(const float* heat, float* out, const int* __restrict__ perm, int n, int k, int shift, int kstride,
                                      int mirror) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();                                               // the 1x1-conv GEMM writes `heat`
  if (i >= static_cast<long long>(n) * k * 3072) return;
  const int x = static_cast<int>(i % 48), y = static_cast<int>((i / 48) % 64);
  const int kk = static_cast<int>((i / 3072) % k), nn = static_cast<int>(i / (3072LL * k));
  const int ks = kstride ? kstride : k;
  const int xs = shift ? max(x - 1, 0) : x;
  const size_t o = (static_cast<size_t>(nn) * ks + kk) * 3072 + y * 48 + x;
  const float m = heat[((static_cast<size_t>(mirror + nn) * ks + perm[kk]) * 64 + y) * 48 + (47 - xs)];
  out[o] = __fmul_rn(__fadd_rn(heat[o], m), 0.5f);
}

}  // namespace vpb
