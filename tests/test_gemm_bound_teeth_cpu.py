"""CPU: the element-wise GEMM bounds of oracle/gemm_ref.py (stage_ref's GEMM, bf16, GELU and residual bounds) reject the
results a broken GEMM schedule typically produces, and accept an honest fp32-accumulated GEMM of the same operands.  The
faults are simulated on the fp64 reference of the shapes tests/test_gpu_gemm_conformance.py runs, in one 128 x 128 tile.

What the bounds can and cannot see: a misplaced k-block, bias column, row half or residual moves an element by O(|z|) and is
caught at every K.  A rounding fault (truncation instead of round-to-nearest-even, the bias added after the bf16 rounding)
moves an element by at most one bf16 ulp; the accumulation allowance K * 2^-23 * sum|a w| grows with K and passes half a bf16
ulp near K = 3072, so these are caught at K <= 768 only.  The fc1 GELU allowance (tanh.approx's 2^-10.9 relative and the fit's
3e-5) is larger than what an error of 1e-3 in the fitted tanh form's leading constant (0.7975) does to any element after the
bf16 rounding; errors from 3e-3 up are caught at K <= 320, from 1e-2 up at K <= 768."""
import pytest
import torch

from oracle import gemm_ref as G
from oracle import stage_ref as S

F64 = torch.float64
BN = 128
SHAPES = [(128, 128, 64), (129, 576, 192), (193, 384, 320), (65, 768, 768), (256, 640, 3072), (64, 384, 5120)]
EPIS = [G.EPI_BF16, G.EPI_BF16_GELU, G.EPI_F32_ADD]


def _trunc_bf16(t):
    """fp32 -> bf16 by dropping the low 16 bits (round toward zero) instead of round-to-nearest-even"""
    return (t.to(torch.float32).view(torch.int32) & ~0xFFFF).view(torch.float32).to(F64)


def _gelu_fit(z, dc0=0.0):
    """the fc1 epilogue's fitted tanh form (csrc/ptx.cuh: gelu_tanh_fit) with an exact tanh, leading constant + dc0"""
    x2 = (z * z).clamp_max(64.0)
    p = (-3.51516782e-4 * x2 + 3.70056460e-2) * x2 + 7.97507884e-1 + dc0
    return 0.5 * z * (1.0 + torch.tanh(z * p))


def _out(z, epi, x0):
    """what an epilogue stores for a pre-activation z computed in fp64 (the fault, if any, is already in z)"""
    if epi == G.EPI_BF16:
        return S.bf16(z)
    if epi == G.EPI_BF16_GELU:
        return S.bf16(_gelu_fit(z))
    return (x0 + z.to(torch.float32)).to(F64)


def _case(M, N, K):
    a, w, bias, x0 = G.operands(M, N, K, seed=M * 7 + N + K)
    a64, w64, b64 = a.to(F64), w.to(F64), bias.to(F64)
    acc = a64 @ w64.T
    rows = slice(0, min(BN, M))
    cols = slice(BN * min(1, N // BN - 1), BN * min(1, N // BN - 1) + BN)         # the second column tile where there is one
    return a, w, bias, x0, a64, w64, b64, acc, rows, cols


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bound_rejects_misplaced_data(M, N, K, epi):
    a, w, bias, x0, a64, w64, b64, acc, rows, cols = _case(M, N, K)
    ref, bound = G.reference(a, w, bias, epi, x0)
    z = acc + b64
    kb = slice(64 * (K // 128), 64 * (K // 128) + 64)                               # a middle k-block
    part = a64[rows, kb] @ w64[cols, kb].T
    faults = {}
    zz = z.clone(); zz[rows, cols] -= part; faults["k-block dropped"] = _out(zz, epi, x0)
    zz = z.clone(); zz[rows, cols] += part; faults["k-block counted twice"] = _out(zz, epi, x0)
    zz = z.clone(); zz[:, cols] += b64[cols].roll(-8) - b64[cols]; faults["bias shifted by 8 columns"] = _out(zz, epi, x0)
    if M >= 128:
        o = _out(z, epi, x0).clone()
        o[0:64, cols], o[64:128, cols] = o[64:128, cols].clone(), o[0:64, cols].clone()
        faults["64-row halves swapped"] = o
    if epi == G.EPI_F32_ADD:
        faults["residual added twice"] = (x0 + x0 + z.to(torch.float32)).to(F64)
    for name, got in faults.items():
        r = S.worst_ratio(got, ref, bound)
        print(f"{name}: worst ratio {r:.3g}")
        assert r > 1, f"{name} at M={M} N={N} K={K} epilogue {epi} passes the bound (worst ratio {r:.3g})"


@pytest.mark.parametrize("M,N,K", [s for s in SHAPES if s[2] <= 768])
def test_bound_rejects_rounding_faults_at_short_k(M, N, K):
    a, w, bias, x0, a64, w64, b64, acc, rows, cols = _case(M, N, K)
    z = acc + b64
    ref, bound = G.reference(a, w, bias, G.EPI_BF16)
    faults = {"bf16 truncation": _trunc_bf16(z), "bias added after the bf16 rounding": S.bf16(S.bf16(acc) + b64)}
    ref1, bound1 = G.reference(a, w, bias, G.EPI_BF16_GELU)
    for name, got in faults.items():
        r = S.worst_ratio(got, ref, bound)
        print(f"{name}: worst ratio {r:.3g}")
        assert r > 1, f"{name} at M={M} N={N} K={K} passes the bound (worst ratio {r:.3g})"
    r = S.worst_ratio(_trunc_bf16(_gelu_fit(z)), ref1, bound1)
    assert r > 1, f"GELU output truncated to bf16 passes the bound (worst ratio {r:.3g})"
    dc0 = 3e-3 if K <= 320 else 1e-2
    r = S.worst_ratio(S.bf16(_gelu_fit(z, dc0)), ref1, bound1)
    print(f"GELU leading constant off by {dc0}: worst ratio {r:.3g}")
    assert r > 1, f"GELU with its leading constant off by {dc0} passes the bound (worst ratio {r:.3g})"


@pytest.mark.parametrize("epi", EPIS + [G.EPI_BF16_GELU_ERF])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bound_accepts_an_fp32_accumulated_gemm(M, N, K, epi):
    """torch's fp32 GEMM of the same bf16 operands, + bias in fp32, then the epilogue's rounding: within the bound."""
    a, w, bias, x0 = G.operands(M, N, K, seed=M * 7 + N + K)
    ref, bound = G.reference(a, w, bias, epi, x0)
    z32 = a.float() @ w.float().T + bias
    if epi == G.EPI_BF16:
        got = S.bf16(z32)
    elif epi == G.EPI_F32_ADD:
        got = (x0 + z32).to(F64)
    else:
        got = S.bf16(_gelu_fit(z32.to(F64)).to(torch.float32))
    r = S.worst_ratio(got, ref, bound)
    print(f"fp32 GEMM, epilogue {epi}: worst ratio {r:.3g}")
    assert r <= 1
