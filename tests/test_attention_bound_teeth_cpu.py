"""CPU: the attention bound (oracle/stage_ref.py attention_items, applied by oracle/attention_ref.py) accepts an fp32
restatement of attend_item (csrc/attention.cuh) and rejects the results typical faults of it produce, on the logit shapes of
attention_ref's menu at head_dim 32, 64 and 80; and ex2_poly (csrc/ptx.cuh) stays within the relative error EX2 the bound
assumes.

What the bound can and cannot see: softmax does not change when a row's logits all shift by the same amount, so a wrong row
max (taken over one key half, or the other row of a quad's) shows only where a weight overflows or every weight underflows:
on the spike 100+ above a row's other keys, which the menu puts in the second key half, and on rows whose maxima differ by
more than fp32's exp range.  A row sum over the unrounded weights instead of the bf16 ones P V uses moves an output by a few
parts in 1e4 of the weighted spread of V, which only shows against the bf16 rounding of a large output (V offset by +100),
and even there only marginally.  Misplaced data (a dropped or repeated P V step, V rows of the wrong key half, a missing
tail box, another warpgroup's Q rows) is caught on every shape whose rows are not uniform."""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import attention_ref as A
from oracle import stage_ref as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = torch.float32
LOG2E = float(np.float32(1.4426950408889634))


# ------------------------------------------------------------------------------------------------ attend_item in fp32
def _bf16(t):
    return t.to(torch.bfloat16).to(F32)


def _fma(a, b, c):
    """fmaf: the fp32 product is exact in fp64; the sum rounds in fp64 and then to fp32 (a double rounding that can differ
    from fmaf by one ulp in rare ties, far below anything the bound resolves)"""
    return (a.double() * b + c.double()).to(F32)


def attend(qkv, heads, fault=None, poly=False):
    """attend_item's arithmetic on every item: fp32 logits, the row max, the fma argument, ex2 (MUFU: flushed below 2^-126;
    every 4th by ex2_poly with `poly`), bf16 weights, the row sum of the rounded weights, fp32 P V in twelve 16-key steps,
    O * (1 / sum), bf16.  `fault` names a deliberate error.  Returns [B*192, D] as fp64."""
    q, k, v = (x.to(F32) for x in A._items(qkv, heads))
    n, T, hd = q.shape
    if fault == "warpgroup 1 reads warpgroup 0's Q rows":
        q = q.clone()
        q[:, 64:128] = q[:, 0:64]
    kk = k[..., :64] if fault == "tail dims dropped from S" else k
    s = q[..., :kk.shape[-1]] @ kk.transpose(-1, -2)
    mx = (s[..., :A.KH] if fault == "row max over keys 0..95" else s).amax(-1, keepdim=True)
    swap = torch.arange(T).view(-1, 2, 8).flip(1).reshape(-1)                 # row r <-> r + 8 inside each 16-row group
    if fault == "rows r and r + 8 swapped in the max":
        mx = mx[:, swap]
    arg = _fma(s, LOG2E, -(mx * LOG2E))
    e = torch.exp2(arg)
    e = torch.where(e < 2.0 ** -126, torch.zeros_like(e), e)                  # ex2.approx.ftz
    if poly:
        col = torch.arange(T)
        use = ((col % 2) == 1) & (((col // 8) % 2) == 0)                      # x1 of the even key groups: every 4th
        e[..., use] = torch.from_numpy(ex2_poly(arg[..., use].numpy()))
    p = _bf16(e)
    total = (e if fault == "row sum over the unrounded weights" else p).sum(-1, keepdim=True)
    if fault == "rows r and r + 8 swapped in the sum":
        total = total[:, swap]
    o = torch.zeros(n, T, hd, dtype=F32)
    for step in range(T // 16):
        rows = slice(16 * step, 16 * step + 16)
        vrows = slice(16 * step - A.KH, 16 * step - A.KH + 16) if fault == "V rows of the second half from the first" and step >= 6 else rows
        part = p[..., rows] @ v[:, vrows]
        if fault == "P V step 7 dropped" and step == 7:
            continue
        o = o + part
        if fault == "P V step 7 taken twice" and step == 7:
            o = o + part
    if fault == "tail dims dropped from O":
        o[..., 64:] = 0.0
    out = _bf16(o * (1.0 / total))
    B = qkv.shape[0] // T
    return A._untangle(out.double(), B, heads)


# ------------------------------------------------------------------------------------------------ the menu at each head_dim
@pytest.fixture(scope="module", params=[32, 64, 80])
def menu(request):
    """one crop with one item of every shape (13 heads), its reference, bound and NaN mask"""
    hd = request.param
    heads = len(A.MENU)
    qkv = A.operands(1, heads, hd, seed=hd)
    return hd, heads, qkv, A.reference(qkv, heads)


def _per_shape(got, heads, ref, bound, nan_mask):
    """{shape: worst ratio} over each item's elements"""
    hd = ref.shape[1] // heads
    out = {}
    for h, shape in enumerate(A.MENU):
        c = slice(h * hd, (h + 1) * hd)
        out[shape] = A.worst_ratio(got[:, c], ref[:, c], bound[:, c], nan_mask[:, c])
    return out


@pytest.mark.parametrize("poly", [False, True])
def test_restatement_is_within_the_bound(menu, poly):
    hd, heads, qkv, (ref, bound, nan_mask) = menu
    r = _per_shape(attend(qkv, heads, poly=poly), heads, ref, bound, nan_mask)
    print(f"hd {hd} {'ex2_poly' if poly else 'MUFU'}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    assert max(r.values()) <= 1, r
    assert bool(nan_mask.any()) and not bool(nan_mask.all())


# fault -> the shapes on which it must be caught
FAULTS = {
    "P V step 7 dropped": ["std1", "std10", "masked", "v_offset"],
    "P V step 7 taken twice": ["std1", "std10", "masked", "v_offset"],
    "V rows of the second half from the first": ["std1", "dominant_second", "max_at_96", "spike_second"],
    "tail dims dropped from S": ["std1", "std10"],
    "tail dims dropped from O": ["std1", "dominant_first", "v_offset"],
    "rows r and r + 8 swapped in the max": ["spike_second"],
    "rows r and r + 8 swapped in the sum": ["std1", "std10", "v_offset"],
    "warpgroup 1 reads warpgroup 0's Q rows": ["std1", "std10", "std30", "dominant_first"],
    "row max over keys 0..95": ["spike_second"],
    "row sum over the unrounded weights": ["v_offset"],
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_faults_leave_the_bound(menu, fault):
    hd, heads, qkv, (ref, bound, nan_mask) = menu
    if "tail" in fault and hd != 80:
        pytest.skip("only head_dim 80 has a tail box")
    r = _per_shape(attend(qkv, heads, fault), heads, ref, bound, nan_mask)
    print(f"hd {hd}, {fault}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    missed = [s for s in FAULTS[fault] if not r[s] > 1]
    assert not missed, f"{fault} at hd {hd} passes the bound on {missed}: {r}"


def test_masked_keys_keep_the_bound_finite():
    """One key of logit -1e30 (and the menu's keys 1e4 below their row max): with the guard every row keeps a finite bound
    that still catches a dropped P V step; stage_ref's derivation without it gives those rows an infinite bound."""
    hd, heads = 64, len(A.MENU)
    qkv = A.operands(1, heads, hd, seed=5)
    D = heads * hd
    qkv[:, D + A.MENU.index("std1") * hd] = 0.0
    qkv[3, D + A.MENU.index("std1") * hd] = -1e30                            # k[3, 0] of the std1 item: logits -5e29 .. -3e30
    ref, bound, nan_mask = A.reference(qkv, heads)                            # asserts a finite bound on finite elements
    q, k, v = A._items(qkv, heads)
    largest = {}
    for shape in ("std1", "masked"):
        i = A.MENU.index(shape)
        largest[shape] = [float(S.attention_items(q[i], k[i], v[i], guard=g)[1].max()) for g in (True, False)]
        print(f"{shape}: largest bound with the guard {largest[shape][0]:.3g}, without {largest[shape][1]:.3g}")
    assert not math.isfinite(largest["std1"][1]) and math.isfinite(largest["std1"][0])     # inf (or inf * 0 = NaN) unguarded
    assert largest["masked"][1] > 10 * largest["masked"][0]
    r = _per_shape(attend(qkv, heads, "P V step 7 dropped"), heads, ref, bound, nan_mask)
    assert r["std1"] > 1 and r["masked"] > 1, r


# ------------------------------------------------------------------------------------------------ ex2_poly
def _ex2_poly_constants():
    src = open(os.path.join(ROOT, "easy_vitpose_b200", "csrc", "ptx.cuh")).read()
    body = src[src.index("float ex2_poly(float x)"):]
    body = body[:body.index("}")]
    lo = float(re.search(r"fmaxf\(x, (-?\d+\.\d+)f\)", body).group(1))
    magic = float(re.search(r"x \+ (\d+\.\d+)f", body).group(1))
    c = [float(v) for v in re.findall(r"fmaf\(p?[^,]*, f, (-?\d\.\d+)f\)", body)]
    c3 = float(re.search(r"fmaf\((\d\.\d+)f, f,", body).group(1))
    assert len(c) == 3, body
    return lo, magic, [c3] + c


def _fma32(a, b, c):
    """fmaf on float32 arrays with one rounding: the fp64 sum of the exact product, corrected where rounding it to fp32
    would round a second time at a tie"""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                                           # s + err = p + c exactly
    r = s.astype(np.float32)
    diff = s - r.astype(np.float64)                                           # s lies this far past r ...
    other = np.nextafter(r, np.where(diff > 0, np.float32(np.inf), np.float32(-np.inf)))
    tie = (diff != 0) & (2 * np.abs(diff) == np.abs(other.astype(np.float64) - r))   # ... halfway to the next float
    return np.where(tie & (err != 0) & (np.sign(err) == np.sign(diff)), other, r).astype(np.float32)


def ex2_poly(x: np.ndarray) -> np.ndarray:
    """ex2_poly in float32, one rounding per operation as the device computes it"""
    lo, magic, (c3, c2, c1, c0) = _ex2_poly_constants()
    f32 = np.float32
    x = np.asarray(x, np.float32)
    nan = np.isnan(x)
    with np.errstate(invalid="ignore"):
        x = np.maximum(x, f32(lo))
    t = (x + f32(magic)).astype(np.float32)
    xi = (t - f32(magic)).astype(np.float32)
    f = (x - xi).astype(np.float32)
    p = _fma32(np.full_like(f, c3), f, np.full_like(f, c2))
    p = _fma32(p, f, np.full_like(f, c1))
    p = _fma32(p, f, np.full_like(f, c0))
    bits = (p.view(np.int32).astype(np.int64) + (t.view(np.int32).astype(np.int64) << 23)) & 0xFFFFFFFF
    out = bits.astype(np.uint32).view(np.float32)
    return np.where(nan, x, out)


def test_ex2_poly_relative_error():
    """[-125, 0] densely, finely around the maximum near -0.5, and the small positive arguments fmaf(s, log2e, -m log2e)
    gives at s = m (the rounding error of m log2e)"""
    rs = np.random.RandomState(0)
    m = np.concatenate([rs.uniform(-2e4, 2e4, 200000), np.exp(rs.uniform(-8, 10, 100000))]).astype(np.float32)
    at_max = _fma32(m, np.full_like(m, LOG2E), -(m * np.float32(LOG2E)).astype(np.float32))
    x = np.concatenate([np.linspace(-125, 0, 2000001, dtype=np.float64).astype(np.float32),
                        np.arange(-0.55, -0.45, 2e-7).astype(np.float32), at_max])
    assert (at_max > 0).sum() > 1000 and at_max.max() > 1e-4
    y = ex2_poly(x).astype(np.float64)
    rel = np.abs(y / np.exp2(x.astype(np.float64)) - 1)
    i = int(rel.argmax())
    print(f"ex2_poly: max relative error {rel.max():.4g} at x = {x[i]:.6g} (EX2 = {S.EX2}); largest positive argument {at_max.max():.3g}")
    assert rel.max() <= S.EX2


def test_ex2_poly_edges():
    lo, _, (_, _, _, c0) = _ex2_poly_constants()
    clamp = np.float32(c0) * np.float32(2.0 ** lo)
    y = ex2_poly(np.array([-125.0, -125.5, -126.0, -200.0, -1e30, -np.inf, np.nan], np.float32))
    assert np.all(y[1:6] == clamp) and y[0] == clamp, y
    assert 0.9999 * 2.0 ** -125 < clamp < 2.0 ** -125                       # 0.99993 * 2^-125, not 0
    assert clamp <= 2.0 ** -124                                              # each such weight is within `tiny`'s allowance
    assert np.isnan(y[-1])
    assert ex2_poly(np.array([0.0], np.float32))[0] == np.float32(c0)        # p(0) is the constant term
