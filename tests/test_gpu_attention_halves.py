"""-m gpu: attention over the two key halves (attend_item in csrc/attention.cuh takes S = Q K^T, the softmax and P V in halves of
96 keys) on inputs that put each row's maximum in either half, and on rows that are entirely -inf or NaN.  The fused qkv +
attention launch (vpb_qkv_attention) must equal the qkv GEMM followed by the standalone attention kernel bit for bit, at every
head_dim, with every exponential on the MUFU and with every 4th one by the polynomial."""
import pytest
import torch

from easy_vitpose_b200 import _lib
from gpu_util import EPI_BF16, attention, gemm, ptr, stream

pytestmark = pytest.mark.gpu

T = 192
BATCH = 6


def _inputs(heads, hd, seed):
    """xn, the packed qkv weight and its bias.  Crop 0 as drawn; crops 1 and 2 scale the xn rows of keys 96..191 (1) or 0..95 (2)
    by 8, so that most rows take their maximum logit in that half; crop 3 has one NaN in xn (its keys, and so all its rows, turn
    NaN); in the last head, the q bias of dim 0 is -inf and the k weight of dim 0 gives every key a positive value there, so
    every logit of that head is -inf."""
    D = heads * hd
    g = torch.Generator().manual_seed(seed)
    xn = torch.randn(BATCH * T, D, generator=g) * 0.5
    xn = xn.view(BATCH, T, D)
    xn[1, 96:] *= 8
    xn[2, :96] *= 8
    xn[3, 17, 5] = float("nan")
    xn[:, :, 0] = 1.0 + xn[:, :, 0].abs()                     # column 0 > 0 in every row but the NaN crop's
    w = torch.randn(3 * D, D, generator=g) * D ** -0.5
    bias = torch.randn(3 * D, generator=g) * 0.1
    last = (heads - 1) * hd
    w[D + last, :] = 0.0
    w[D + last, 0] = 1.0                                      # k[dim 0] = xn[:, 0] > 0
    w[last, 0] = 0.0
    bias[last] = float("-inf")                                # q[dim 0] = -inf
    return (xn.view(BATCH * T, D).bfloat16().cuda(), w.bfloat16().cuda(), bias.float().cuda())


def _two_launches(xn, w, bias, heads, hd):
    qkv = torch.empty((xn.shape[0], w.shape[0]), dtype=torch.bfloat16, device=xn.device)
    gemm(xn, w, bias, qkv, EPI_BF16)
    return attention(qkv, BATCH, heads, hd)


def _fused(xn, w, bias, heads, hd):
    out = torch.empty((xn.shape[0], heads * hd), dtype=torch.bfloat16, device=xn.device)
    _lib.check(_lib.lib().vpb_qkv_attention(ptr(xn), ptr(w), ptr(bias), BATCH, heads, hd, ptr(out), stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("heads,hd", [(6, 32), (12, 64), (16, 80)])
def test_fused_equals_two_launches_on_split_inputs(heads, hd, poly):
    xn, w, bias = _inputs(heads, hd, 10 * hd + poly)
    try:
        _lib.lib().vpb_debug_attention(poly)
        ref = _two_launches(xn, w, bias, heads, hd)
        out = _fused(xn, w, bias, heads, hd)
    finally:
        _lib.lib().vpb_debug_attention(-1)
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), f"hd {hd}, poly {poly}: fused != qkv GEMM + attention"

    # the inputs do what they are for: maxima in the first and in the second key half, -inf and NaN rows
    qkv = torch.empty((xn.shape[0], 3 * heads * hd), dtype=torch.bfloat16, device=xn.device)
    gemm(xn, w, bias, qkv, EPI_BF16)
    D = heads * hd
    q = qkv[:, :D].float().view(BATCH, T, heads, hd).transpose(1, 2)
    k = qkv[:, D:2 * D].float().view(BATCH, T, heads, hd).transpose(1, 2)
    s = q[:, :-1] @ k[:, :-1].transpose(-1, -2)               # [B, heads - 1, T, T] logits of the finite heads
    second = s.argmax(-1) >= 96
    assert second[1].float().mean() > 0.9 and second[2].float().mean() < 0.1 and 0 < second[0].float().mean() < 1
    out = out.float().view(BATCH, T, heads, hd)
    assert out[3].isnan().all(), "a NaN key spoils every row of its crop"
    assert out[:, :, -1].isnan().all(), "rows whose logits are all -inf"
    assert out[[0, 1, 2, 4, 5], :, :-1].isfinite().all()
