"""Single-stage fp64 references of the engine's forward, with element-wise error bounds  --  TEST INFRASTRUCTURE ONLY.

Each function restates one stage of the engine (csrc/engine.cu: backbone() and head(), the stop_after stages) in float64
torch on whatever device its inputs live on.  It takes the PREVIOUS stage's buffer as the engine left it (teacher forcing:
no error accumulates from stage to stage) and the state dict, and returns (ref, bound): the exact result of the stage on
those inputs, and a bound on |engine - ref| per element.

The references reproduce the engine's deliberate roundings, and only those:
  * weights are bf16 after packing (pack_linear_bf16); the q rows of attn.qkv are multiplied by the engine's fp32 q scale
    1.0f / sqrtf(head_dim) before the rounding, and the q bias by the same scale in fp32 (pack_bias);
  * the token stream is seeded with pos[1+t] + pos[0] + patch_bias, added in that order in fp32 (pack_pos_bias);
  * a deconv weight is bf16(w * s) with the fp32 BatchNorm scale s = gamma / sqrtf(var + 1e-5f); its shift is
    beta - mean * s (pack_deconv);
  * xn, qkv, attn, hid, d1 and d2 are bf16; x and the heatmaps stay fp32;
  * the LayerNorm eps is the fp32 value the kernels receive.
Everything else -- fp32 accumulation, the fitted GELU, ex2.approx / ex2_poly, the bf16 softmax weights -- is error the
bound has to cover.

How the bounds are derived (u = 2^-24, the fp32 unit round-off):
  GEMM      The bf16 x bf16 products are exact in fp32.  The tensor cores accumulate in fp32 but round-to-nearest is not
            guaranteed, so each addition may cost one fp32 ulp, 2^-23 relative: a K-term dot product is off by at most
            K * 2^-23 * sum|a*w| (UACC below).  Adding the bias rounds once more (u |z|).
            bf16 outputs: the fp32 value z is rounded to bf16, at most half a bf16 ulp of |z| <= |ref| + delta.
            fp32 residual outputs (x += ...): one more rounding of the sum, u |x|.
  GELU      fc1 evaluates gelu_tanh_fit: |fit - erf GELU| <= 3e-5 (tests/test_gelu_fit.py pins it on [-8, 8]; outside it
            the clamp makes the fit exact to 1e-6 relative), tanh.approx.f32 adds <= 2^-10.9 relative to tanh, i.e.
            <= 2^-10.9 * |x/2| on the result, and four fp32 operations <= 4u |x|.  The input error passes through
            with the GELU's largest slope, 1.13.
  LayerNorm The kernel sums a row as a tree of depth D/128 + 7 (per lane D/128 float4 partial sums of two pairs, then
            five xor-shuffle levels): mean off by (D/128 + 7) u mean|x| + 2u|mean|, each centred value by that plus
            u |x - mean|.  The variance carries those errors squared and linearly, the same tree error and two more
            roundings; rstd = rsqrtf(var + eps) adds 2 ulp.  The normalise-scale-shift adds three roundings.
  Attention Logits are hd-term GEMMs (above).  Each softmax weight exp(s - max) is computed as ex2 of an fp32 argument
            (rounding of log2e, of max*log2e and of the fma: u (2|s - max| + |max|)), ex2.approx or ex2_poly (relative
            7.5e-5, flush to zero below 2^-126 / clamp at 2^-125), then rounded to bf16 (2^-9).  If every weight p_j
            carries a relative error |e_j| <= eps, the normalised weights shift by w_j (e_j - mean e) / (1 + mean e),
            so the output moves by at most 2 eps / (1 - eps) * sum_j w_j |v_j - o|.  P V is a 192-term fp32 GEMM, the
            row sum a 192-term fp32 sum, and 1 / sum and the product round twice.  Keys more than 1000 below their
            row's max (masked keys) have weight 0 or 2^-125 p(0) whatever their logit's error, so they stay out of eps.
  Deconv    An implicit GEMM of K = 4 Cin (each output phase reads 2 x 2 taps); the shift beta - mean * s in fp32 adds
            two roundings; ReLU is 1-Lipschitz.
No constant here was adjusted to make a test pass.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import vitpose_oracle as O

U = 2.0 ** -24                    # fp32 unit round-off
UACC = 2.0 ** -23                 # per-addition error of an fp32 tensor-core accumulation (no round-to-nearest promise)
GELU_FIT = 3e-5                   # |gelu_tanh_fit - erf GELU|, tests/test_gelu_fit.py
TANH_APPROX = 2.0 ** -10.9        # tanh.approx.f32 relative error
GELU_SLOPE = 1.13                 # max |d GELU / dx| = 1.1289
EX2 = 7.5e-5                      # ex2.approx.ftz.f32 and ex2_poly, relative
P_BF16 = 2.0 ** -9                # rounding of a softmax weight to bf16
RSQRT = 2.0 ** -22                # rsqrtf: 2 ulp
LN_EPS = float(np.float32(1e-6))  # what the LayerNorm launches receive
BN_EPS = np.float32(1e-5)
F64 = torch.float64


# ------------------------------------------------------------------------------------------------ rounding helpers
def bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 values -> bf16 (round to nearest even, __float2bfloat16_rn) -> fp64.  The input must already be fp32 values:
    rounding fp64 straight to bf16 could round twice differently."""
    return t.to(torch.float32).to(torch.bfloat16).to(F64)


def half_ulp_bf16(m: torch.Tensor) -> torch.Tensor:
    """Half a bf16 ulp (8 significant bits) of a value of magnitude m >= 0: 2^(floor(log2 m) - 8), normal range."""
    _, e = torch.frexp(m.clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(m), (e - 9).to(torch.int32))


def bf16_bound(ref: torch.Tensor, delta: torch.Tensor) -> torch.Tensor:
    """Bound on |bf16(z) - ref| when the fp32 value z lies within delta of ref."""
    return delta + half_ulp_bf16(ref.abs() + delta)


def t64(v, device=None) -> torch.Tensor:
    return torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).to(device=device, dtype=F64)


def t32(v, device=None) -> torch.Tensor:
    return torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).to(device=device, dtype=torch.float32)


def worst_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - ref| / bound over all elements (<= 1: within the bound).  NaN anywhere counts as infinitely far."""
    r = (got.to(F64) - ref).abs() / bound
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return float(r.max())


# ------------------------------------------------------------------------------------------------ packed weights
def q_scale(head_dim: int) -> np.float32:
    """The engine's q scale: 1.0f / sqrtf(head_dim) in fp32 (vpb_finalize), which is head_dim^-0.5 up to fp32 rounding."""
    return np.float32(1.0) / np.sqrt(np.float32(head_dim))


def linear_weights(sd: dict, key: str, device, scaled_rows: int = 0, scale=np.float32(1.0)):
    """(W, b) of a linear layer as the engine packs them: W bf16 of fp32 w * scale on rows < scaled_rows, b fp32."""
    w = t32(sd[key + ".weight"], device)
    w = w.reshape(w.shape[0], -1)
    b = t32(sd[key + ".bias"], device)
    if scaled_rows:
        s = torch.ones(w.shape[0], 1, dtype=torch.float32, device=device)
        s[:scaled_rows] = torch.tensor(float(scale), dtype=torch.float32)
        w = w * s
        b = b * s[:, 0]
    return bf16(w), b.to(F64)


def pos_bias(sd: dict, device) -> torch.Tensor:
    """[192, D] fp32 stream seed pos[1+t] + pos[0] + patch bias, in that order (pack_pos_bias)."""
    pos = t32(sd["backbone.pos_embed"], device)[0]
    return ((pos[1:] + pos[:1]) + t32(sd["backbone.patch_embed.proj.bias"], device)[None]).to(F64)


def deconv_weights(sd: dict, prefix: str, layer: int, device):
    """(W [Cin, 256, 4, 4] of bf16(w * s), shift [256], |mean * s| [256]) for deconv `layer` (0 or 1) of the head at
    `prefix` (pack_deconv).  The scale is fp32 arithmetic (IEEE sqrt and division, as the packing kernel compiles them); the
    shift is returned in fp64 from that fp32 scale, and |mean * s| sizes the two fp32 roundings of the kernel's
    beta - mean * s in deconv()'s bound."""
    li = 3 * layer
    bn = f"{prefix}deconv_layers.{li + 1}."
    g, be, mu, var = (np.asarray(sd[bn + n], np.float32) for n in ("weight", "bias", "running_mean", "running_var"))
    s = g / np.sqrt(var + BN_EPS)
    w = np.asarray(sd[f"{prefix}deconv_layers.{li}.weight"], np.float32) * s[None, :, None, None]
    shift = be.astype(np.float64) - mu.astype(np.float64) * s.astype(np.float64)
    return bf16(torch.from_numpy(w).to(device)), torch.from_numpy(shift).to(device), torch.from_numpy(mu.astype(np.float64) * s).to(device).abs()


# ------------------------------------------------------------------------------------------------ GEMM core
def _gemm(a: torch.Tensor, w: torch.Tensor, b: torch.Tensor):
    """z = a w^T + b (fp64) and the bound of the fp32 accumulation plus the bias add."""
    z = a @ w.T + b
    delta = a.shape[-1] * UACC * (a.abs() @ w.abs().T) + U * z.abs()
    return z, delta


def gelu_erf(z: torch.Tensor) -> torch.Tensor:
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def gelu_bound(z: torch.Tensor, d_z: torch.Tensor):
    """The fc1 epilogue on a pre-activation z known to within d_z: the exact erf GELU of z and the bound of the bf16 output."""
    ref = gelu_erf(z)
    delta = GELU_SLOPE * d_z + GELU_FIT + (TANH_APPROX + 8 * U) * 0.5 * (z.abs() + d_z)
    return ref, bf16_bound(ref, delta)


def residual(x: torch.Tensor, z: torch.Tensor, delta: torch.Tensor):
    """The fp32 stream after x += z, z known to within delta: the sum and its bound (one more rounding of the sum)."""
    ref = x.to(F64) + z
    return ref, delta + U * ref.abs()


def conv_transpose_bound(feat: torch.Tensor, w: torch.Tensor, shift: torch.Tensor, ms: torch.Tensor):
    """relu(ConvTranspose2d(k4,s2,p1)(feat) + shift) of NHWC feat [B,H,W,Cin] and bf16 w [Cin,Cout,4,4] as one implicit GEMM of
    K = 4 Cin, NHWC out, and its bound; |ms| = |mean * s| sizes the fp32 roundings of a folded BatchNorm's shift (0: none)."""
    cin = w.shape[0]
    a = feat.to(F64).permute(0, 3, 1, 2)
    z = F.conv_transpose2d(a, w, stride=2, padding=1) + shift[None, :, None, None]
    s = F.conv_transpose2d(a.abs(), w.abs(), stride=2, padding=1)
    delta = 4 * cin * UACC * s + U * z.abs() + 2 * U * (shift.abs() + ms)[None, :, None, None]
    ref = torch.relu(z)
    return ref.permute(0, 2, 3, 1), bf16_bound(ref, delta).permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ stages
def patch_rows(crops) -> torch.Tensor:
    """Stage 1: the bf16 im2col of the crops [B,3,256,192] -> [B*192, 768]; bit-exact, no bound."""
    c = np.asarray(crops.cpu() if isinstance(crops, torch.Tensor) else crops, np.float32)
    r = torch.from_numpy(O.patch_rows(c).reshape(-1, 768))
    return bf16(r)


def patch_embed(rows: torch.Tensor, sd: dict):
    """Stage 2: x = pos_bias + rows Wpatch^T ([B*192, 768] bf16 -> [B*192, D] fp32).  The conv bias lives in pos_bias; the
    GEMM's bias is a zero vector, so its add is exact."""
    dev = rows.device
    a = rows.to(F64)
    w = bf16(t32(sd["backbone.patch_embed.proj.weight"], dev).reshape(-1, 768))
    acc = a @ w.T
    seed = pos_bias(sd, dev).repeat(a.shape[0] // 192, 1)
    ref = seed + acc
    bound = 768 * UACC * (a.abs() @ w.abs().T) + U * ref.abs()
    return ref, bound


def layernorm(x: torch.Tensor, gamma, beta, eps: float = LN_EPS):
    """LayerNorm over the last dim, fp32 x -> bf16 (stages 3, LN2 and 10; eps 1e-6 in fp32)."""
    dev = x.device
    x = x.to(F64)
    D = x.shape[-1]
    g, b = t64(t32(gamma, dev), dev), t64(t32(beta, dev), dev)
    depth = D // 128 + 7
    mu = x.mean(-1, keepdim=True)
    c = x - mu
    var = (c * c).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xh = c * rstd
    ref = xh * g + b
    d_mu = depth * U * x.abs().mean(-1, keepdim=True) + 2 * U * mu.abs()
    e_c = d_mu + U * c.abs()
    E = e_c.amax(-1, keepdim=True)
    d_var = 2 * E * c.abs().mean(-1, keepdim=True) + E * E + (depth + 3) * U * (var + eps)
    d_rstd = 0.5 * rstd ** 3 * d_var * (1 + d_var * rstd ** 2) + RSQRT * rstd
    delta = g.abs() * (e_c * rstd + c.abs() * d_rstd) + 3 * U * ((xh * g).abs() + ref.abs())
    return ref, bf16_bound(ref, delta)


def block_norm(x: torch.Tensor, sd: dict, i: int, which: int, eps: float = LN_EPS):
    """norm1 (which=1) or norm2 (which=2) of block i."""
    p = f"backbone.blocks.{i}.norm{which}."
    return layernorm(x, sd[p + "weight"], sd[p + "bias"], eps)


def last_norm(x: torch.Tensor, sd: dict, eps: float = LN_EPS):
    """Stage 10: backbone.last_norm of the stream after the last block."""
    return layernorm(x, sd["backbone.last_norm.weight"], sd["backbone.last_norm.bias"], eps)


def qkv(xn: torch.Tensor, sd: dict, i: int, heads: int):
    """Stage 4: qkv = xn Wqkv^T + b with the q rows (first D) pre-scaled, -> bf16 [M, 3D]."""
    D = xn.shape[-1]
    w, b = linear_weights(sd, f"backbone.blocks.{i}.attn.qkv", xn.device, D, q_scale(D // heads))
    z, delta = _gemm(xn.to(F64), w, b)
    return z, bf16_bound(z, delta)


MASKED = 1000.0                   # a key this far below its row's max logit is masked: exp(s - max) < e^-1000 is 0 in fp64


def attention_items(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, guard: bool = True):
    """softmax(q k^T) v of items [..., 192, hd] (fp64 of bf16 values, q pre-scaled) and the bound of the fp32 value before
    the bf16 rounding of the output (the Attention paragraph above).

    With `guard`, masked keys (s < max - MASKED) are left out of eps and of the logit error of the max (d_s.amax): the kernel
    computes their weight as ex2 of an fp32 argument below -1000 log2e, which is 0 (MUFU) or 2^-125 p(0) (ex2_poly's clamp)
    whatever that argument's error, and the `tiny` term already covers such weights.  Without the guard one key of logit
    -1e30 (or -inf) makes d_s, and so the bound of its whole row, infinite: a test would pass that row unchecked."""
    hd = q.shape[-1]
    s = q @ k.transpose(-1, -2)
    d_s = hd * UACC * (q.abs() @ k.abs().transpose(-1, -2))
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    w = p / p.sum(-1, keepdim=True)
    o = w @ v
    if guard:
        masked = s < m - MASKED
        d_s = d_s.masked_fill(masked, 0.0)
    arg = d_s + d_s.amax(-1, keepdim=True) + U * (2 * (s - m).abs() + m.abs())
    if guard:
        arg = arg.masked_fill(masked, -math.inf)
    eps = (torch.exp(arg + math.log1p(P_BF16) + math.log1p(EX2)) - 1).amax(-1, keepdim=True)
    vo = (v.unsqueeze(-3) - o.unsqueeze(-2)).abs()                              # [..., query, key, hd] = |v_j - o|
    dev_v = (w.unsqueeze(-1) * vo).sum(-2)
    tiny = 192 * 2.0 ** -124 * vo.amax(-2)                 # weights flushed to zero or clamped at 2^-125 (sum of p >= 1)
    delta = (2 * eps / (1 - eps)) * dev_v + 2 * tiny + 192 * UACC * (1 + 2 * eps) * (w @ v.abs()) \
        + (192 * U + 2 * U) * (o.abs() + dev_v)
    return o, delta


def attention(qkv_buf: torch.Tensor, heads: int):
    """Stage 5: softmax(q k^T) v per (crop, head) from the qkv buffer [B*192, 3D] (q pre-scaled) -> bf16 [B*192, D]."""
    M, D3 = qkv_buf.shape
    D, B = D3 // 3, M // 192
    hd = D // heads
    t = qkv_buf.to(F64).reshape(B, 192, 3, heads, hd).permute(2, 0, 3, 1, 4)      # [3, B, H, 192, hd]
    refs, deltas = [], []
    for c in range(B):                                     # one crop at a time: sum_j w_j |v_j - o| is [H, 192, 192, hd]
        o, delta = attention_items(t[0, c], t[1, c], t[2, c])
        refs.append(o.permute(1, 0, 2).reshape(192, D))
        deltas.append(delta.permute(1, 0, 2).reshape(192, D))
    ref, delta = torch.cat(refs), torch.cat(deltas)
    return ref, bf16_bound(ref, delta)


def proj(attn: torch.Tensor, x: torch.Tensor, sd: dict, i: int):
    """Stage 6: x += attn Wproj^T + b (fp32 stream, TMA reduce-add)."""
    w, b = linear_weights(sd, f"backbone.blocks.{i}.attn.proj", attn.device)
    return residual(x, *_gemm(attn.to(F64), w, b))


def fc1(xn: torch.Tensor, sd: dict, i: int):
    """Stage 7: hid = GELU(xn W1^T + b1) -> bf16 [M, 4D], against the exact erf GELU."""
    w, b = linear_weights(sd, f"backbone.blocks.{i}.mlp.fc1", xn.device)
    return gelu_bound(*_gemm(xn.to(F64), w, b))


def fc2(hid: torch.Tensor, x: torch.Tensor, sd: dict, i: int):
    """Stage 8: x += hid W2^T + b2 (fp32 stream).  For an engine with experts pass the head's split state dict
    (split_vitpose_plus), whose fc2 holds the shared rows followed by the head's expert rows."""
    w, b = linear_weights(sd, f"backbone.blocks.{i}.mlp.fc2", hid.device)
    return residual(x, *_gemm(hid.to(F64), w, b))


def deconv(feat: torch.Tensor, sd: dict, layer: int, prefix: str = "keypoint_head."):
    """Deconv `layer` (0: tokens xn [B*192, D] or [B,16,12,D] -> d1 [B,32,24,256]; 1: d1 -> d2 [B,64,48,256]), NHWC in
    and out: ConvTranspose2d(k4,s2,p1) with the BatchNorm folded, + shift, ReLU, -> bf16."""
    dev = feat.device
    w, shift, ms = deconv_weights(sd, prefix, layer, dev)
    if layer == 0:
        feat = feat.reshape(-1, 16, 12, w.shape[0])
    return conv_transpose_bound(feat, w, shift, ms)


def final_layer(d2: torch.Tensor, sd: dict, prefix: str = "keypoint_head."):
    """The 1x1 conv: d2 [B,64,48,256] bf16 -> heatmaps [B,K,64,48] fp32."""
    w, b = linear_weights(sd, prefix + "final_layer", d2.device)
    z, delta = _gemm(d2.to(F64).reshape(-1, 256), w, b)
    B = d2.shape[0]
    return (z.reshape(B, 64, 48, -1).permute(0, 3, 1, 2), delta.reshape(B, 64, 48, -1).permute(0, 3, 1, 2))


# ------------------------------------------------------------------------------------------------ whole forward
def chained_forward(crops, sd: dict, depth: int, heads: int):
    """The stages chained on their own outputs, each rounded as the engine rounds its buffer (bf16 where the engine stores
    bf16, fp32 for the stream): what the engine computes, minus its accumulated round-off.  Returns the heatmaps."""
    r = patch_rows(crops)
    x = patch_embed(r, sd)[0].float().double()
    for i in range(depth):
        xn = bf16(block_norm(x, sd, i, 1)[0].float())
        a = bf16(attention(bf16(qkv(xn, sd, i, heads)[0].float()), heads)[0].float())
        x = proj(a, x, sd, i)[0].float().double()
        h = bf16(fc1(bf16(block_norm(x, sd, i, 2)[0].float()), sd, i)[0].float())
        x = fc2(h, x, sd, i)[0].float().double()
    xn = bf16(last_norm(x, sd)[0].float())
    d1 = bf16(deconv(xn, sd, 0)[0].float())
    d2 = bf16(deconv(d1, sd, 1)[0].float())
    return final_layer(d2, sd)[0]
