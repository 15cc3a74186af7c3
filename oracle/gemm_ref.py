"""Operands, fp64 references and element-wise bounds of bare GEMM launches  --  TEST INFRASTRUCTURE ONLY.

The kernel-level GEMM tests (tests/test_gpu_gemm_conformance.py) and the CPU check that their bounds catch typical schedule
faults (tests/test_gemm_bound_teeth_cpu.py) share these.  The bounds are oracle/stage_ref.py's, applied to a bare GEMM:
_gemm for the fp32 accumulation and the bias, bf16_bound for bf16 outputs, gelu_bound for the GELU epilogues and residual for
the fp32 stream.  Nothing is re-derived here.
"""
from __future__ import annotations

import torch

from oracle import stage_ref as S

EPI_BF16, EPI_BF16_GELU, EPI_F32_ADD, EPI_BF16_GELU_ERF = 0, 1, 5, 6
F64 = torch.float64


def operands(M: int, N: int, K: int, seed: int, device="cpu"):
    """(a [M,K] bf16, w [N,K] bf16, bias [N] f32, x0 [M,N] f32).  Every row of A, every k of A, every row of W has its own
    non-zero scale and every column its own bias, so a swapped tile, row block or k-block cannot cancel out; z = a w^T is
    O(1).  Drawn on the CPU from `seed`, then moved: the same operands on every device."""
    g = torch.Generator().manual_seed(seed)
    r_a = 0.5 + torch.rand(M, 1, generator=g)
    k_a = 0.5 + torch.rand(1, K, generator=g)
    r_w = 0.5 + torch.rand(N, 1, generator=g)
    a = (torch.randn(M, K, generator=g) * r_a * k_a).bfloat16()
    w = (torch.randn(N, K, generator=g) * r_w * (K ** -0.5)).bfloat16()
    bias = torch.randn(N, generator=g) * 0.5
    x0 = torch.randn(M, N, generator=g)
    return a.to(device), w.to(device), bias.to(device), x0.to(device)


def reference(a, w, bias, epi: int, x0=None):
    """(ref, bound) of the launch's output: bf16 [M,N] for EPI_BF16 / EPI_BF16_GELU / EPI_BF16_GELU_ERF, the fp32 stream
    x0 + (a w^T + bias) for EPI_F32_ADD.  The GELU epilogues are held to the exact erf GELU with fc1's allowance (the fitted
    tanh form's and tanh.approx's error cover the A&S erf of EPI_BF16_GELU_ERF, |err| <= 1.5e-7)."""
    z, delta = S._gemm(a.to(F64), w.to(F64), bias.to(F64))
    if epi == EPI_BF16:
        return z, S.bf16_bound(z, delta)
    if epi in (EPI_BF16_GELU, EPI_BF16_GELU_ERF):
        return S.gelu_bound(z, delta)
    if epi == EPI_F32_ADD:
        return S.residual(x0, z, delta)
    raise ValueError(f"no reference for epilogue {epi}")


def expert_reference(a, w, bias, x0, D: int, P: int, segs, shared: bool):
    """The fp32 stream after vpb_expert_gemm, and its bound: for every segment (row_begin, row_end, expert) the expert columns
    [D-P, D) of its rows += a W_e^T + bias_e, W_e the P rows of expert e after the D-P shared rows of the stacked w; with
    `shared`, the columns [0, D-P) of every row += a W_s^T + bias_s.  Elements no launch writes keep x0 with a zero bound."""
    S_ = D - P
    a64, w64, b64 = a.to(F64), w.to(F64), bias.to(F64)
    ref = x0.to(F64).clone()
    bound = torch.zeros_like(ref)
    if shared:
        ref[:, :S_], bound[:, :S_] = S.residual(x0[:, :S_], *S._gemm(a64, w64[:S_], b64[:S_]))
    for rb, re, e in segs:
        rows = slice(S_ + e * P, S_ + (e + 1) * P)
        ref[rb:re, S_:], bound[rb:re, S_:] = S.residual(x0[rb:re, S_:], *S._gemm(a64[rb:re], w64[rows], b64[rows]))
    return ref, bound


def first_offender(got, ref, bound, bn: int, a=None, w=None) -> str:
    """Where the worst violation of a bound sits: the first element over its bound, its 128-row block, its column tile of
    width `bn` and, given the operands, the 64-wide k-block whose contribution (taken once more or dropped) the error matches
    best."""
    r = (got.to(F64) - ref).abs() / bound
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    bad = (r > 1).nonzero()
    if len(bad) == 0:
        return "no element over its bound"
    row, col = (int(v) for v in bad[0])
    msg = (f"{len(bad)} elements over the bound, first at (row {row}, col {col}): got {float(got[row, col])}, ref {float(ref[row, col])}, "
           f"bound {float(bound[row, col]):.3g}; row block {row // 128} (rows {row // 128 * 128}..{row // 128 * 128 + 127}), "
           f"column tile {col // bn} (cols {col // bn * bn}..{col // bn * bn + bn - 1})")
    if a is not None and w is not None:
        parts = (a[row].to(F64) * w[col].to(F64)).reshape(-1, 64).sum(-1)
        err = float(got[row, col]) - float(ref[row, col])
        j = int((parts.abs() - abs(err)).abs().argmin())
        msg += f", k range 0..{a.shape[1] - 1}: the error {err:.4g} is closest to k-block {j} (k {64 * j}..{64 * j + 63}: {float(parts[j]):.4g})"
    return msg
