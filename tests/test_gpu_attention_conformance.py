"""-m gpu: the attention kernels element by element against fp64, with stage_ref's bound (oracle/attention_ref.py).

The standalone kernel (vpb_attention) and the fused qkv + attention kernel (vpb_qkv_attention) run at every head_dim (32, 64,
80), at head counts whose k-block counts D / 64 leave every remainder modulo the fused ring's depth (5 / 3 / 2), and at item
counts (crops x heads) below, at and just over one item per SM (132) and at 1024 or more (about 8 per CTA).  Each case runs
the grid caps none, 1, 2, 3, 7 and 131 (vpb_debug_attention bits 8..), so a CTA attends odd and even numbers of items and its
two operand stages, or the fused ring, wrap many times.  Every item takes a logit shape from attention_ref's menu by its
index, so neighbouring items of a CTA differ.  Every launch must
  * hold every element within its fp64 bound and be NaN exactly where the inputs make the result NaN,
  * leave a sentinel before and after the [B*192, D] output untouched and no sentinel inside it,
  * give the same bits at every grid cap and on a repeated launch, separately with the MUFU exponentials and with every 4th
    one by ex2_poly (vpb_debug_attention bit 0; within the same bound, not the MUFU's bits);
and the fused form must give the same bits as the qkv GEMM followed by the standalone kernel.  On a failure the message names
the element's crop, head, item, CTA, operand stage or ring slots, warpgroup, quad, dim box and argmax key half."""
import pytest
import torch

from easy_vitpose_b200 import _lib
from gpu_util import EPI_BF16, bits, gemm, ptr, sentinel_buffer, stream, untouched
from oracle import attention_ref as A

pytestmark = pytest.mark.gpu

SMS = 132
FRONT = BACK = 64                                 # sentinel elements before and after an output
CAPS = [0, 1, 2, 3, 7, 131]                        # 0: one CTA per SM


def _batches(heads):
    """crop counts whose items (crops x heads) fall below, on (where heads divides 132) and just over one item per SM, and
    at 1024 or more"""
    out = {1, 131 // heads, -(-133 // heads), -(-1024 // heads)}
    if SMS % heads == 0:
        out.add(SMS // heads)
    return sorted(b for b in out if b >= 1)


STANDALONE = {32: [1, 2, 6, 12], 64: [1, 3, 12, 16], 80: [1, 4, 16]}
FUSED = {32: [2, 4, 6, 8, 10, 12], 64: [1, 2, 3, 4, 12, 16], 80: [4, 8, 12, 16]}
STANDALONE_CASES = [(hd, h, b) for hd, hs in STANDALONE.items() for h in hs for b in _batches(h)]
FUSED_CASES = [(hd, h, b) for hd, hs in FUSED.items() for h in hs for b in _batches(h)]


def _grid(items, cap):
    return min(items, cap if 0 < cap < SMS else SMS)


def test_the_sweep_reaches_what_it_claims():
    """From the grids and item counts alone: some CTA attends 3 or more items on each of its two operand stages at every
    head_dim, and the fused ring wraps in the middle of an item at every head_dim; the fused k-block counts take every
    remainder modulo the ring depth; every case has counts on both sides of one item per SM."""
    for hd in (32, 64, 80):
        per_cta = [-(-h * b // _grid(h * b, cap)) for _, h, b in (c for c in STANDALONE_CASES if c[0] == hd) for cap in CAPS]
        assert max(per_cta) >= 6, f"hd {hd}: no CTA takes three items on each operand stage"
        st = A.fused_stages(hd)
        assert {(h * hd // 64) % st for h in FUSED[hd]} == set(range(st)), f"hd {hd}: k-block counts miss a remainder of {st}"
        wraps = False
        for _, h, b in (c for c in FUSED_CASES if c[0] == hd):
            nkb = h * hd // 64
            for cap in CAPS:
                n = -(-h * b // _grid(h * b, cap))                            # items of CTA 0
                # item i of a CTA starts at ring position i * nkb; it wraps mid-item if a slot-(st-1) -> slot-0 step falls inside it
                wraps |= any((i * nkb + j) % st == st - 1 for i in range(n) for j in range(nkb - 1))
        assert wraps, f"hd {hd}: the fused ring never wraps inside an item"
    for cases in (STANDALONE_CASES, FUSED_CASES):
        for hd, h in {(c[0], c[1]) for c in cases}:
            items = [c[1] * c[2] for c in cases if c[:2] == (hd, h)]
            assert min(items) < SMS < max(items) and max(items) >= 1024, (hd, h, items)


@pytest.fixture
def debug_reset():
    yield
    _lib.lib().vpb_debug_attention(-1)


def _launch(fn, M, D):
    """run fn(out) on an output inside a sentinel buffer; returns the output after checking the sentinels"""
    buf, sentinel = sentinel_buffer(FRONT + M * D + BACK, torch.bfloat16)
    out = buf[FRONT:FRONT + M * D].view(M, D)
    fn(out)
    torch.cuda.synchronize()
    assert untouched(buf, FRONT, FRONT + M * D, sentinel), "stores outside the [B*192, D] output"
    assert not bool((bits(out) == sentinel).any()), f"{int((bits(out) == sentinel).sum())} output elements never written"
    return out


def _sweep(launchers, ref, bound, nan_mask, qkv, heads, fused, what):
    """launchers: [(name, fn(out))] run at every cap, MUFU and ex2_poly.  Returns the worst ratio per exponential."""
    M, D = ref.shape
    items = heads * (M // 192)
    worst = {}
    for poly in (0, 1):
        first = None
        for cap in CAPS:
            for name, fn in launchers:
                for repeat in ((0, 1) if cap == 0 and name == launchers[0][0] else (0,)):
                    _lib.lib().vpb_debug_attention(poly | (cap << 8))
                    tag = f"{what}, {name}, {'ex2_poly' if poly else 'MUFU'}, grid {_grid(items, cap)}{' (repeated)' if repeat else ''}"
                    try:
                        out = _launch(fn, M, D)
                    except AssertionError as e:
                        raise AssertionError(f"{tag}: {e}") from None
                    if first is None:
                        worst[poly] = A.worst_ratio(out, ref, bound, nan_mask)
                        assert worst[poly] <= 1, f"{tag}: " + A.first_offender(out, ref, bound, nan_mask, qkv, heads, _grid(items, cap), fused)
                        first = (out, tag)
                    else:
                        same = bits(out) == bits(first[0])
                        assert bool(same.all()), (f"{tag} differs from {first[1]} in {int((~same).sum())} elements; "
                                                  + A.first_offender(out, ref, bound, nan_mask, qkv, heads, _grid(items, cap), fused))
    return worst


@pytest.mark.parametrize("hd,heads,batch", STANDALONE_CASES)
def test_attention_conformance(debug_reset, hd, heads, batch):
    qkv = A.operands(batch, heads, hd, seed=1000 * hd + 10 * heads + batch, device="cuda")
    ref, bound, nan_mask = A.reference(qkv, heads)

    def standalone(out):
        _lib.check(_lib.lib().vpb_attention(ptr(qkv), batch, heads, hd, ptr(out), stream()))

    worst = _sweep([("vpb_attention", standalone)], ref, bound, nan_mask, qkv, heads, False, f"hd {hd}, {heads} heads, {batch} crops")
    print(f"attention conformance hd {hd} heads {heads} crops {batch}: worst |err| / bound MUFU {worst[0]:.3g}, ex2_poly {worst[1]:.3g}")


@pytest.mark.parametrize("hd,heads,batch", FUSED_CASES)
def test_qkv_attention_conformance(debug_reset, hd, heads, batch):
    D = heads * hd
    xn, w, bias = A.operands(batch, heads, hd, seed=2000 * hd + 10 * heads + batch, device="cuda", fused=True)
    qkv = torch.empty(batch * 192, 3 * D, dtype=torch.bfloat16, device="cuda")
    gemm(xn, w, bias, qkv, EPI_BF16)                         # the separate form's qkv: the fused kernel's rounding of q, k, v
    ref, bound, nan_mask = A.reference(qkv, heads)

    def fused(out):
        _lib.check(_lib.lib().vpb_qkv_attention(ptr(xn), ptr(w), ptr(bias), batch, heads, hd, ptr(out), stream()))

    def separate(out):
        q = torch.empty_like(qkv)
        gemm(xn, w, bias, q, EPI_BF16)
        _lib.check(_lib.lib().vpb_attention(ptr(q), batch, heads, hd, ptr(out), stream()))

    worst = _sweep([("vpb_qkv_attention", fused), ("qkv GEMM + vpb_attention", separate)], ref, bound, nan_mask, qkv, heads, True,
                   f"hd {hd}, {heads} heads, {batch} crops")
    print(f"qkv attention conformance hd {hd} heads {heads} crops {batch}: worst |err| / bound MUFU {worst[0]:.3g}, ex2_poly {worst[1]:.3g}")
