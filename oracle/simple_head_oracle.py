"""fp64 references of the simple decoder (relu -> 4x bilinear upsample -> 3x3 conv) and its error bound  --  TEST
INFRASTRUCTURE ONLY.

The ReLU comes BEFORE the upsample.  That is the upstream ViTPose head's order: its
TopdownHeatmapSimpleHead._transform_inputs returns
    resize(input=F.relu(inputs), scale_factor=self.upsample, mode='bilinear', align_corners=self.align_corners)
for a tensor input with upsample > 0, and the published simple-decoder checkpoints were trained with that code (the paper's
prose puts the ReLU after the upsample; the two differ, relu does not commute with interpolation).  The reference here
raises NotImplementedError at that point (vit_models/head/topdown_heatmap_simple_head.py:269-271) and its `resize` helper
is a stub (vit_utils/util.py:231-249), so oracle/make_golden_simple.py puts the upstream line back on the instance.

Two forms: `direct` is the definition (F.interpolate, then F.conv2d with zero padding of the UPSAMPLED map); `taps` is what
simple_head.cuh computes, Y_t = relu(tokens) W_t^T at token resolution and the separable stencil of the bilinear weights.
`mutant` gives the usual ways to get it wrong, for the bound's teeth.

Bound of the engine (csrc/simple_head.cuh) against `taps` on the engine's own bf16 inputs and bf16-rounded weights:
  Y         a D-term fp32 tensor-core accumulation of exact bf16 products: |dY| <= D * 2^-23 * sum_c |a_c w_c|
  stencil   the dyadic weights are exact; out = bias + sum over <= 3 row taps of 2 terms, each a sum over <= 3 column taps of
            2 terms, started from the bias: at most 6 + 7 fp32 additions on the path of each product, so <= 16 u of the
            absolute stencil plus |bias|;
  and the stencil carries |dY| with its (non-negative) weights.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import vitpose_oracle as O

U = 2.0 ** -24
UACC = 2.0 ** -23
F64 = torch.float64
UP = 4


def bilinear_matrix(n_out: int, n_in: int, align_corners: bool = False, clamp: bool = True) -> np.ndarray:
    """[n_out, n_in] weights of F.interpolate(mode='bilinear') along one axis for a scale of n_out / n_in.  clamp=False
    drops the out-of-range source instead of clamping it to the edge (a mutant)."""
    R = np.zeros((n_out, n_in))
    for o in range(n_out):
        if align_corners:
            src = o * (n_in - 1) / (n_out - 1)
        else:
            src = (o + 0.5) * n_in / n_out - 0.5
            if clamp:
                src = max(src, 0.0)
        i0 = int(np.floor(src))
        lam = src - i0
        for i, w in ((i0, 1.0 - lam), (i0 + 1, lam)):
            if 0 <= i < n_in:
                R[o, i] += w
            elif clamp:
                R[o, min(max(i, 0), n_in - 1)] += w
    return R


def tap_table(n_out: int, n_in: int) -> "list[tuple[int, int, float, float]]":
    """(i0, i1, w0, w1) of every output row as the kernel's sh_taps computes them: weights (3/8, 5/8), (1/8, 7/8), (7/8, 1/8),
    (5/8, 3/8) for row % 4 = 0..3, source indices clamped to [0, n_in - 1]."""
    out = []
    for y in range(n_out):
        q, s = y >> 2, y & 3
        i0 = (max(q - 1, 0) if s < 2 else q)
        i1 = (q if s < 2 else min(q + 1, n_in - 1))
        w0 = (0.375, 0.125, 0.875, 0.625)[s]
        out.append((i0, i1, w0, 1.0 - w0))
    return out


def _shifted(R: np.ndarray, d: int) -> np.ndarray:
    """Rows y of R read at y + d, zero where y + d leaves the map (the conv's zero padding of the upsampled map)."""
    S = np.zeros_like(R)
    n = R.shape[0]
    for y in range(n):
        if 0 <= y + d < n:
            S[y] = R[y + d]
    return S


def direct(feat: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The definition in fp64: feat [B, D, 16, 12], w [K, D, 3, 3], b [K] -> [B, K, 64, 48]."""
    u = F.interpolate(torch.relu(feat.to(F64)), scale_factor=UP, mode="bilinear", align_corners=False)
    return F.conv2d(u, w.to(F64), b.to(F64), padding=1)


def tap_outputs(feat: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Y [B, 9, K, 16, 12] = relu(feat) contracted with each tap W_t[k, c] = w[k, c, t // 3, t % 3], in fp64."""
    r = torch.relu(feat.to(F64))
    return torch.einsum("bchw,kct->btkhw", r, w.to(F64).flatten(2))


def stencil(Y: torch.Tensor, b: "torch.Tensor | None") -> torch.Tensor:
    """out[b, k] = bias + sum_t Ry(dy) Y_t Rx(dx)^T with the shifted bilinear matrices (Y may be |Y| / |dY| for bounds)."""
    Ry, Rx = bilinear_matrix(64, 16), bilinear_matrix(48, 12)
    out = None
    for t in range(9):
        dy, dx = t // 3 - 1, t % 3 - 1
        ry = torch.as_tensor(_shifted(Ry, dy), dtype=F64, device=Y.device)
        rx = torch.as_tensor(_shifted(Rx, dx), dtype=F64, device=Y.device)
        o = torch.einsum("yi,bkij,xj->bkyx", ry, Y[:, t].to(F64), rx)
        out = o if out is None else out + o
    if b is not None:
        out = out + b.to(F64).view(1, -1, 1, 1)
    return out


def taps(feat: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The tap form of the kernel, fp64: equal to direct() to round-off."""
    return stencil(tap_outputs(feat, w), b)


def bound(feat: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> "tuple[torch.Tensor, torch.Tensor]":
    """(ref, per-element bound on |engine - ref|) for bf16 features and bf16 weights (the engine's rounded operands)."""
    D = feat.shape[1]
    Y = tap_outputs(feat, w)
    absY = torch.einsum("bchw,kct->btkhw", torch.relu(feat.to(F64)), w.to(F64).abs().flatten(2))
    ref = stencil(Y, b)
    dY = D * UACC * absY
    return ref, stencil(dY, None) + 16 * U * (stencil(Y.abs() + dY, None) + b.to(F64).abs().view(1, -1, 1, 1))


MUTANTS = ("align_corners", "relu_after", "no_relu", "lowres_conv", "swap_taps", "no_clamp")


def mutant(name: str, feat: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """A wrong simple head, fp64: align_corners=True; relu after the upsample; no relu; the 3x3 conv (and its padding) on the
    16 x 12 map, upsampled after; dy and dx of the taps swapped; the edge clamp of the bilinear sources dropped."""
    f, w, b = feat.to(F64), w.to(F64), b.to(F64)
    if name == "align_corners":
        return F.conv2d(F.interpolate(torch.relu(f), scale_factor=UP, mode="bilinear", align_corners=True), w, b, padding=1)
    if name == "relu_after":
        return F.conv2d(torch.relu(F.interpolate(f, scale_factor=UP, mode="bilinear", align_corners=False)), w, b, padding=1)
    if name == "no_relu":
        return F.conv2d(F.interpolate(f, scale_factor=UP, mode="bilinear", align_corners=False), w, b, padding=1)
    if name == "lowres_conv":
        return F.interpolate(F.conv2d(torch.relu(f), w, b, padding=1), scale_factor=UP, mode="bilinear", align_corners=False)
    if name == "swap_taps":
        return direct(f, w.transpose(2, 3), b)
    if name == "no_clamp":
        Ry, Rx = (torch.as_tensor(bilinear_matrix(n, m, clamp=False), dtype=F64, device=f.device) for n, m in ((64, 16), (48, 12)))
        u = torch.einsum("yi,bcij,xj->bcyx", Ry, torch.relu(f), Rx)
        return F.conv2d(u, w, b, padding=1)
    raise KeyError(name)


def make_state_dict(embed_dim: int, depth: int, num_keypoints: int, seed: int, peaky: float = 1.0,
                    bumps: bool = False) -> "dict[str, np.ndarray]":
    """Seeded float32 weights of a simple-decoder ViTPose under the reference key names: the backbone is exactly
    vitpose_oracle.make_state_dict's (same seed, same draws), the head is final_layer [K, D, 3, 3] + bias drawn next from the
    same stream.  bumps=True adds the simple form of vitpose_oracle's bump pathway: keypoint k owns token t_k and channel
    c_k = k % D, pos_embed makes c_k hot at t_k, and the conv reads c_k into heatmap k through its centre tap, so the
    upsampled hot token is the one clear peak of map k."""
    D, K = embed_dim, num_keypoints
    sd = {k: v for k, v in O.make_state_dict(D, depth, K, seed).items() if k.startswith("backbone.")}
    rs = np.random.RandomState(seed)
    rs.standard_normal(sum(v.size for v in sd.values()))              # the backbone's draws (every one is a standard normal)

    def nrm(*shape, std=1.0):
        return (rs.standard_normal(shape) * std).astype(np.float32)

    sd["keypoint_head.final_layer.weight"] = nrm(K, D, 3, 3, std=0.02 * peaky / math.sqrt(9 * D / 256))
    sd["keypoint_head.final_layer.bias"] = nrm(K, std=0.01)
    if bumps:
        amp = 12.0 * depth / 12.0
        for k in range(K):
            c = k % D
            t = int(rs.randint(0, O.TOKENS))
            sd["backbone.pos_embed"][0, 1 + t, c] += np.float32(amp)
            sd["keypoint_head.final_layer.weight"][k, c, 1, 1] += np.float32(0.2)
    return sd


def engine_weights(w: np.ndarray) -> torch.Tensor:
    """final_layer.weight as the engine packs it: fp32 -> bf16 (pack_simple_head), as fp64."""
    return torch.as_tensor(np.asarray(w, np.float32)).to(torch.bfloat16).to(F64)
