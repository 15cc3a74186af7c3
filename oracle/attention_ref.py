"""Operands, fp64 references and element-wise bounds of bare attention launches  --  TEST INFRASTRUCTURE ONLY.

The kernel-level attention tests (tests/test_gpu_attention_conformance.py) and the CPU check that the bound catches typical
faults of attend_item (tests/test_attention_bound_teeth_cpu.py) share these.  The bound is stage_ref.attention_items', with
masked keys kept out of eps; nothing is re-derived here.

Every item (crop b, head h; item = b * heads + h, the order the kernels hand items out in) takes the logit shape MENU[item %
13].  13 divides none of the grids the tests launch (1, 2, 3, 7, 131, 132 CTAs), so neighbouring items of a CTA, and so its
operand stages and ring slots, always hold different shapes.  Dim 0 of q and k carries the shape: q[t, 0] = rho_t, a per-row
scale that differs between the three warpgroups' 64-row blocks and between the rows r and r + 8 of a quad, and k[j, 0] = o_j,
a per-key logit offset, so logit[t, j] = rho_t o_j + (the random part of the other dims).
"""
from __future__ import annotations

import torch

from oracle import stage_ref as S

F64 = torch.float64
T = 192
KH = 96                                            # keys per half in attend_item
MENU = ["std1", "std10", "std30", "dominant_first", "dominant_second", "spike_second", "max_at_95", "max_at_96", "equal",
        "v_offset", "masked", "nan_q_v", "nan_k"]
NAN_Q_ROW, NAN_V_KEY, NAN_K_KEY = 77, 150, 40


def row_scale(device=None) -> torch.Tensor:
    """rho_t: 0.5 on rows r (t % 16 < 8) and 1.5 on rows r + 8 of a quad, times 1, 1.25, 1.5 on the three warpgroups, plus
    a small per-row ramp.  A spike of 200 then sits 100 to 340 above its row's other keys, and the maxima of rows r and
    r + 8 differ by more than fp32's exp range."""
    t = torch.arange(T, dtype=F64, device=device)
    return (0.5 + ((t % 16) >= 8).to(F64)) * (1 + 0.25 * (t // 64)) * (1 + 0.01 * (t % 8))


def _offsets(shape: str, g: torch.Generator, device) -> torch.Tensor:
    """o_j of one item"""
    o = torch.zeros(T, dtype=F64, device=device)
    if shape in ("std10", "std30"):
        o = torch.randn(T, generator=g, device=device, dtype=F64) * float(shape[3:])
    elif shape == "dominant_first":
        o[int(torch.randint(0, KH, (1,), generator=g, device=device))] = 12.0
    elif shape == "dominant_second":
        o[int(torch.randint(KH, T, (1,), generator=g, device=device))] = 12.0
    elif shape == "spike_second":
        o[int(torch.randint(KH, T, (1,), generator=g, device=device))] = 200.0
    elif shape == "max_at_95":
        o[95] = 12.0
    elif shape == "max_at_96":
        o[96] = 12.0
    elif shape == "masked":                        # every third key 1e4 below the others, the rest std 3
        o = torch.randn(T, generator=g, device=device, dtype=F64) * 3.0
        o[1::3] = -1e4
    return o


def operands(batch: int, heads: int, hd: int, seed: int, device="cpu", fused: bool = False):
    """Standalone (fused=False): qkv [B*192, 3D] bf16, q pre-scaled, in the layout the qkv GEMM writes.

    Fused: (xn [B*192, D] bf16, w [3D, D] bf16, bias [3D] f32), the packed qkv weight with the q rows pre-scaled.  Every xn row
    and every W row has its own scale, so a swapped k-block or head cannot cancel out.  Three xn columns per head carry the
    item's shape through single unit weights: c1 (k[:, 0] = o), c2 (q[:, 0] = rho) and c3 (v += 100 for v_offset); no other
    W row reads them.  The GEMM's random part of the other dims stays in every item, so "equal" keys only have a zero offset
    here.  A NaN in xn spoils its token in every head of the crop, so the NaN shapes are not drawn per item either: with 3 or
    more crops, one NaN in the last crop's xn turns that whole crop NaN."""
    D = heads * hd
    g = torch.Generator(device=device).manual_seed(seed)
    rho = row_scale(device)
    qs = float(S.q_scale(hd))
    if not fused:
        q = torch.randn(batch, heads, T, hd, generator=g, device=device, dtype=F64) * qs
        k = torch.randn(batch, heads, T, hd, generator=g, device=device, dtype=F64)
        v = torch.randn(batch, heads, T, hd, generator=g, device=device, dtype=F64)
        q[..., 0] = rho
        for item in range(batch * heads):
            b, h = divmod(item, heads)
            shape = MENU[item % len(MENU)]
            k[b, h, :, 0] = _offsets(shape, g, device)
            if shape == "equal":
                k[b, h] = k[b, h, :1].clone()
            elif shape == "v_offset":
                v[b, h] += 100.0
            elif shape == "nan_q_v":
                q[b, h, NAN_Q_ROW, 1] = float("nan")
                v[b, h, NAN_V_KEY, hd - 1] = float("nan")
            elif shape == "nan_k":
                k[b, h, NAN_K_KEY, 2] = float("nan")
        qkv = torch.stack([q, k, v], 2).permute(0, 3, 2, 1, 4).reshape(batch * T, 3 * D)
        return qkv.float().bfloat16()
    assert 3 * heads <= D
    c1, c2, c3 = (torch.arange(heads, device=device) + i * heads for i in range(3))
    free = torch.ones(D, dtype=torch.bool, device=device)
    free[:3 * heads] = False
    r_x = 0.5 + torch.rand(batch * T, 1, generator=g, device=device, dtype=F64)
    xn = torch.randn(batch * T, D, generator=g, device=device, dtype=F64) * r_x
    r_w = 0.5 + torch.rand(3 * D, 1, generator=g, device=device, dtype=F64)
    w = torch.randn(3 * D, D, generator=g, device=device, dtype=F64) * r_w * (D - 3 * heads) ** -0.5
    w[:D] *= qs
    w[:, ~free] = 0.0
    bias = torch.randn(3 * D, generator=g, device=device, dtype=F64) * 0.1
    bias[:D] *= qs
    xv = xn.view(batch, T, D)
    for h in range(heads):
        w[h * hd, :] = 0.0                         # q[:, 0] = xn[:, c2]
        w[h * hd, c2[h]] = 1.0
        w[D + h * hd, :] = 0.0                     # k[:, 0] = xn[:, c1]
        w[D + h * hd, c1[h]] = 1.0
        w[2 * D + h * hd:2 * D + (h + 1) * hd, c3[h]] = 1.0
        bias[h * hd] = bias[D + h * hd] = 0.0
        xv[:, :, c2[h]] = rho
        for b in range(batch):
            shape = MENU[(b * heads + h) % len(MENU)]
            xv[b, :, c1[h]] = _offsets(shape, g, device)
            xv[b, :, c3[h]] = 100.0 if shape == "v_offset" else 0.0
    if batch >= 3:
        xv[batch - 1, 100, -1] = float("nan")
    return xn.float().bfloat16(), w.float().bfloat16(), bias.float()


def _items(qkv: torch.Tensor, heads: int):
    """q, k, v [B*heads, 192, hd] fp64 in item order"""
    M, D3 = qkv.shape
    D, B = D3 // 3, M // T
    t = qkv.to(F64).reshape(B, T, 3, heads, D // heads).permute(2, 0, 3, 1, 4)
    return [t[i].reshape(B * heads, T, D // heads) for i in range(3)]


def _untangle(x: torch.Tensor, batch: int, heads: int) -> torch.Tensor:
    """[B*heads, 192, hd] -> [B*192, D]"""
    hd = x.shape[-1]
    return x.reshape(batch, heads, T, hd).permute(0, 2, 1, 3).reshape(batch * T, heads * hd)


def reference(qkv: torch.Tensor, heads: int, chunk_bytes: float = 1.5e9):
    """(ref, bound, nan_mask) [B*192, D] of vpb_attention on qkv [B*192, 3D] (q pre-scaled), in fp64 on qkv's device.

    ref and bound are stage_ref's (attention_items with masked keys guarded, then bf16_bound).  nan_mask is where the output
    must be NaN: every row whose q holds a NaN, every item whose k holds one, and column d of every item whose v[:, d] holds
    one.  Elsewhere the NaNs are replaced by 0 for the reference, so the other elements keep a finite reference and bound;
    the function asserts that the bound is finite wherever the reference is."""
    M, D3 = qkv.shape
    D, B = D3 // 3, M // T
    hd = D // heads
    q, k, v = _items(qkv, heads)
    nan = q.isnan().any(-1, keepdim=True) | k.isnan().any(-1).any(-1)[:, None, None] | v.isnan().any(-2, keepdim=True)
    q, k, v = (x.nan_to_num(nan=0.0) for x in (q, k, v))
    n = max(1, int(chunk_bytes // (T * T * hd * 8)))   # items per chunk: sum_j w_j |v_j - o| is [n, 192, 192, hd]
    o, delta = torch.empty_like(q[..., :hd]), torch.empty_like(q[..., :hd])
    for i in range(0, q.shape[0], n):
        o[i:i + n], delta[i:i + n] = S.attention_items(q[i:i + n], k[i:i + n], v[i:i + n])
    nan = nan.expand_as(o)
    ref, delta = _untangle(o, B, heads), _untangle(delta, B, heads)
    nan_mask = _untangle(nan.to(F64), B, heads) > 0
    bound = S.bf16_bound(ref, delta)
    finite = ref.isfinite() & ~nan_mask
    assert bool(bound[finite].isfinite().all()), "the bound is infinite on a finite reference element"
    ref = ref.masked_fill(nan_mask, float("nan"))
    return ref, bound, nan_mask


def worst_ratio(got, ref, bound, nan_mask) -> float:
    """max |got - ref| / bound over the elements off nan_mask (NaN there counts as infinitely far); inf if any element of
    nan_mask is not NaN"""
    if not bool(got[nan_mask].isnan().all()):
        return float("inf")
    keep = ~nan_mask
    return S.worst_ratio(got[keep], ref[keep], bound[keep]) if bool(keep.any()) else 0.0


def fused_stages(hd: int) -> int:
    """The fused kernel's ring depth (qkv_attention.cuh: QkvAttCfg): 5 / 3 / 2 at head_dim 32 / 64 / 80"""
    oper = T * (64 if hd == 32 else 128) + (T * 32 if hd == 80 else 0)
    stage = T * 64 * 2 + 3 * hd * 64 * 2
    return min(6, (227 * 1024 - 1024 - 256 - 3 * oper) // stage)


def first_offender(got, ref, bound, nan_mask, qkv, heads: int, grid: int, fused: bool = False) -> str:
    """Where the first violation sits: the element, its crop, head and item with the item's shape, the CTA (item % grid) and
    the item's ordinal there, hence its operand stage (standalone) or the ring slots of its k-blocks (fused), the query row's
    warpgroup, warp and quad, whether the dim is in the main or the tail box, and the key half that holds the row's argmax."""
    r = (got.to(F64) - ref).abs() / bound
    bad = torch.where(nan_mask, ~got.isnan(), r.isnan() | (r > 1))
    idx = bad.nonzero()
    if len(idx) == 0:
        return "no element outside its bound"
    row, col = (int(x) for x in idx[0])
    D = ref.shape[1]
    hd = D // heads
    b, t, h, d = row // T, row % T, col // hd, col % hd
    item = b * heads + h
    cta, nth = item % grid, item // grid
    msg = (f"{len(idx)} elements wrong, first at (row {row}, col {col}): got {float(got[row, col])}, ref {float(ref[row, col])}, "
           f"bound {float(bound[row, col]):.3g}{' (must be NaN)' if bool(nan_mask[row, col]) else ''}; crop {b}, head {h}, item {item} "
           f"({MENU[item % len(MENU)] if not fused else 'fused shape ' + MENU[item % len(MENU)]}), CTA {cta} of {grid}, its item {nth}")
    if fused:
        nkb, st = D // 64, fused_stages(hd)
        msg += f" (k-blocks in ring slots {', '.join(str((nth * nkb + i) % st) for i in range(nkb))} of {st})"
    else:
        msg += f" (operand stage {nth % 2}, phase {(nth // 2) % 2})"
    main = 32 if hd == 32 else 64
    msg += (f"; query row {t}: warpgroup {t // 64}, warp {(t % 64) // 16}, quad {t % 8} ({'r + 8' if t % 16 >= 8 else 'r'}); "
            f"dim {d} in the {'main' if d < main else 'tail'} box")
    q, k, _ = _items(qkv, heads)
    s = (q[item, t] @ k[item].T).nan_to_num(nan=-float("inf"))
    j = int(s.argmax())
    return msg + f"; the row's max logit is at key {j}, key half {j // KH}"
