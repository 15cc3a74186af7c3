"""-m gpu: the GEMM kernels element by element against fp64, with stage_ref's bounds (oracle/gemm_ref.py).

The standalone GEMM (vpb_gemm) runs every tile width N allows (128, 192, 256), every ring depth from 3 up to the compiled depth
of that width, and both tile orders (n fastest, the default, and m fastest), at ragged M from 1 row to many waves of tiles per
CTA, and at K whose k-block counts leave every remainder modulo every depth, so that the ring's (stage, phase) position
wraps inside tiles and across tile boundaries.  Every launch must
  * hold every output element within its fp64 bound,
  * leave the padding around the [M, N] output untouched (a sentinel before and after it),
  * give the same bits as every other launch of the case: the k order of an element is fixed, so neither the tile width, the
    ring depth, the tile order nor the residual form (TMA reduce-add or load + add + store) may change a bit.
The head's GEMMs (implicit deconv, 1x1 conv) and the grouped expert GEMM (vpb_expert_gemm) are held to the same standard at
their own geometries.  On a failure the message names the first element over its bound, its 128-row block, its column tile and
the k-block its error matches."""
import ctypes as C

import pytest
import torch

from easy_vitpose_b200 import _lib
from gpu_util import bits, gemm, ptr, sentinel_buffer, stream, untouched
from oracle import gemm_ref as G
from oracle import stage_ref as S

pytestmark = pytest.mark.gpu

FRONT = 64                                   # sentinel elements before an output (keeps the TMA base 128-byte aligned)


def _stages(bn: int, staged: bool) -> int:
    """The compiled ring depth of a 128 x bn tile (csrc/gemm.cuh: TileCfg): 6 at 128 and 4 at 192 / 256 with the TMA
    epilogues' staging, 5 / 7 / 8 / 8 / 8 at 192 / 128 / 96 / 64 / 32 without (the expert GEMM)."""
    stage = 128 * 64 * 2 + bn * 64 * 2
    return min(8, (227 * 1024 - 2048 - (4 * 8192 if staged else 0)) // stage)


def _debug(depth=0, m_fastest=False, width=0, rmw=None):
    """vpb_debug_gemm: ring depth in bits 0..7; dbg_flags in bits 8..: 4 = m-fastest tile order, 32 / 64 = load + add + store /
    TMA reduce-add residual, the forced tile width from bit 8 of the flags on"""
    flags = (4 if m_fastest else 0) | {None: 0, True: 32, False: 64}[rmw] | (width << 8)
    _lib.check(_lib.lib().vpb_debug_gemm(depth | (flags << 8), None))


@pytest.fixture
def debug_reset():
    yield
    _lib.lib().vpb_debug_gemm(0, None)


# ------------------------------------------------------------------------------------------------ standalone GEMM
M_MANY = 8257        # 65 row blocks: 390 to 1560 tiles, 3 to 12 per CTA on 132 SMs, the last row block ragged
# (M, N, K): every M, N and K of the sweep; K = 64, 128, 192, 256, 320, 768, 3072, 5120 give 1, 2, 3, 4, 5, 12, 48, 80 k-blocks,
# every remainder modulo the depths 3, 4, 5 and 6
SHAPES = [
    (1, 128, 64), (63, 384, 128), (64, 576, 192), (65, 640, 256), (127, 768, 320), (128, 2304, 768), (129, 3072, 64),
    (191, 128, 3072), (192, 384, 5120), (193, 576, 768), (1, 3072, 320), (65, 2304, 5120), (129, 640, 3072), (191, 768, 128),
    (193, 2304, 256), (M_MANY, 768, 768), (M_MANY, 3072, 320), (M_MANY, 576, 256),
]
EPIS = [G.EPI_BF16, G.EPI_BF16_GELU, G.EPI_BF16_GELU_ERF, G.EPI_F32_ADD]


def _variants(N, epi):
    """(width, depth, m_fastest, rmw) of every launch of a case: each width that divides N (vpb_gemm's tile maps), each ring
    depth 3 .. compiled - 1 and 0 (= the compiled depth), both tile orders; the residual epilogue in both forms"""
    out = []
    for width in (128, 192, 256):
        if N % width:
            continue
        for depth in [0] + list(range(3, _stages(width, True))):
            for m_fastest in (False, True):
                for rmw in ((False, True) if epi == G.EPI_F32_ADD else (None,)):
                    out.append((width, depth, m_fastest, rmw))
    return out


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_conformance(debug_reset, M, N, K, epi):
    a, w, bias, x0 = G.operands(M, N, K, seed=M * 7 + N * 3 + K + epi, device="cuda")
    ref, bound = G.reference(a, w, bias, epi, x0)
    f32 = epi == G.EPI_F32_ADD
    dtype = torch.float32 if f32 else torch.bfloat16
    back = 2 * N + FRONT
    first = None
    worst = 0.0
    for width, depth, m_fastest, rmw in _variants(N, epi):
        what = f"M={M} N={N} K={K} epilogue {epi}, width {width}, ring depth {depth or 'compiled'}, " \
               f"{'m' if m_fastest else 'n'}-fastest tiles" + ("" if rmw is None else (", load + add + store" if rmw else ", TMA reduce-add"))
        buf, sentinel = sentinel_buffer(FRONT + M * N + back, dtype)
        out = buf[FRONT:FRONT + M * N].view(M, N)
        if f32:
            out.copy_(x0)
        _debug(depth, m_fastest, width, rmw)
        gemm(a, w, bias, out, epi)
        assert untouched(buf, FRONT, FRONT + M * N, sentinel), f"{what}: stores outside the [M, N] output"
        if first is None:
            worst = S.worst_ratio(out, ref, bound)
            assert worst <= 1, f"{what}: " + G.first_offender(out, ref, bound, width, a, w)
            first = (out.clone(), what)
        else:
            same = bits(out) == bits(first[0])
            assert bool(same.all()), (f"{what} differs from {first[1]} in {int((~same).sum())} elements; "
                                      + G.first_offender(out, ref, bound, width, a, w))
    print(f"GEMM conformance epilogue {epi} M={M} N={N} K={K}: {len(_variants(N, epi))} launches bit-identical, "
          f"worst |err| / bound {worst:.3g}")


# ------------------------------------------------------------------------------------------------ grouped expert GEMM
def _segments(kind, M):
    """(row_begin, row_end, expert) tables"""
    if kind == "one":
        return [(0, M, 1)]
    if kind == "crops":            # one crop each: 128-row tiles straddle two segments; equal and different neighbours
        return [(0, 192, 0), (192, 384, 0), (384, 576, 2), (576, 768, 1), (768, 960, 1), (960, M, 2)]
    if kind == "gaps":             # rows outside every segment must keep their bits; odd sizes; the last one ends at M
        return [(5, 70, 2), (70, 71, 0), (200, 455, 1), (455, 600, 1), (700, M, 0)]
    if kind == "max":              # EXPERT_MAX_SEGMENTS segments of 1 .. 150 rows, a few gaps
        g = torch.Generator().manual_seed(3)
        segs, row = [], 0
        for i in range(128):
            row += int(torch.randint(0, 3, (1,), generator=g)) * (i % 5 == 0)
            n = 1 + int(torch.randint(0, 150, (1,), generator=g))
            segs.append((row, row + n, i % 3))
            row += n
        return segs
    raise ValueError(kind)


def _expert_rows(kind):
    return {"one": 576, "crops": 1152, "gaps": 811, "max": None}[kind]


# (D, P): every tile width of the expert GEMM (P = 32, 64, 96, 128, 192 -> widths 32, 64, 96, 128, 192) and shared parts
# D - P whose last column tile runs past D - P
EXPERT_DP = [(384, 32), (384, 64), (384, 96), (768, 128), (384, 192)]


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("kind", ["one", "crops", "gaps", "max"])
@pytest.mark.parametrize("D,P", EXPERT_DP)
def test_expert_gemm_conformance(debug_reset, D, P, kind, shared):
    segs = _segments(kind, _expert_rows(kind) or 0)
    M = _expert_rows(kind) or segs[-1][1]
    H, K = 3, 4 * D
    g = torch.Generator().manual_seed(D + P + M + shared)
    a = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g))).bfloat16().cuda()
    w = (torch.randn(D - P + H * P, K, generator=g) * (0.5 + torch.rand(D - P + H * P, 1, generator=g)) * K ** -0.5).bfloat16().cuda()
    bias = (torch.randn(D - P + H * P, generator=g) * 0.5).cuda()
    x0 = torch.randn(M, D, generator=g).cuda()
    ref, bound = G.expert_reference(a, w, bias, x0, D, P, segs, bool(shared))
    written = bound > 0
    table = (C.c_int32 * (3 * len(segs)))(*[v for s in segs for v in s])
    bn = next(b for b in (192, 128, 96, 64, 32) if P % b == 0)
    first = None
    for depth in [0] + list(range(3, _stages(bn, False))):
        _debug(depth)
        x = x0.clone()
        _lib.check(_lib.lib().vpb_expert_gemm(ptr(a), ptr(w), ptr(bias), ptr(x), M, D, P, H, table, len(segs), shared, stream()))
        torch.cuda.synchronize()
        what = f"D={D} P={P} (width {bn}) {kind} segments, shared columns {'on' if shared else 'off'}, ring depth {depth or 'compiled'}"
        kept = bits(x)[~written] == bits(x0)[~written]
        assert bool(kept.all()), f"{what}: {int((~kept).sum())} elements outside the segments' columns were written"
        if first is None:
            r = S.worst_ratio(x[written], ref[written], bound[written])
            assert r <= 1, f"{what}: " + G.first_offender(torch.where(written, x.double(), ref), ref, bound.clamp_min(1e-30), bn)
            first = x
        else:
            assert torch.equal(bits(x), bits(first)), f"{what} differs from the compiled depth"
    print(f"expert GEMM {what}: worst |err| / bound {r:.3g}")
