"""-m gpu: each hand-written kernel through the C ABI against a plain fp32 torch restatement of the same op
(floating-point kernels) or the oracle / golden vectors (decode: integer argmax bit-exact)."""
import os

import numpy as np
import pytest
import torch

from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need an H100"
    return torch.device("cuda", 0)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("name,wrap", [("decode_crop", False), ("decode_batch", True)])
def test_decode_matches_reference_golden(golden_dir, name, wrap):
    from easy_vitpose_b200 import decode_heatmaps
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    N, K, seed = (int(v) for v in g["meta"])
    maps = O.make_decode_maps(N, K, seed)
    kp, idx = decode_heatmaps(torch.from_numpy(maps).to(_dev()), torch.from_numpy(g["org_wh"]), wrap_batch=wrap)
    kp, idx = kp.cpu().numpy(), idx.cpu().numpy()
    assert np.array_equal(idx, g["idx"])                              # integer argmax indices: bit-exact
    assert np.array_equal(kp[..., 2], g["kpts"][..., 2])              # score = raw max: bit-exact
    ref = g["kpts"][..., :2]
    err = np.abs(kp[..., :2] - ref)
    kinds = (np.arange(N * K) % 10).reshape(N, K)
    well = np.isin(kinds, [0, 1, 2, 3, 5, 7])
    print("decode err well-conditioned max", err[well].max(), "other max", err[~well].max())
    assert err[well].max() < 2e-3                                    # px; blur bit-exact, logf vs np.log differ by ulps
    assert np.all(err[~well] <= 2e-3 + 2e-3 * np.abs(ref[~well]))


def test_decode_matches_oracle_random_maps():
    from easy_vitpose_b200 import decode_heatmaps
    maps = O.make_decode_maps(8, 17, 4242)
    org = np.stack([np.arange(8) * 37 + 64, np.arange(8) * 29 + 80], 1).astype(np.int32)
    kp, idx = decode_heatmaps(torch.from_numpy(maps).to(_dev()), torch.from_numpy(org), wrap_batch=False)
    okp, oidx = O.decode_maps(maps, org, wrap="crop")
    assert np.array_equal(idx.cpu().numpy(), oidx)
    kp = kp.cpu().numpy()
    assert np.array_equal(kp[..., 2], okp[..., 2])
    kinds = (np.arange(8 * 17) % 10).reshape(8, 17)
    well = np.isin(kinds, [0, 1, 2, 3, 5, 7])
    assert np.abs(kp[..., :2] - okp[..., :2])[well].max() < 2e-3


def test_decode_nan_and_ties_first_index():
    from easy_vitpose_b200 import decode_heatmaps
    m = np.zeros((1, 3, 64, 48), np.float32)
    m[0, 0].reshape(-1)[[100, 2000]] = 1.0                 # tie -> 100
    m[0, 1].reshape(-1)[[77, 78]] = [np.nan, 5.0]          # np.argmax: first NaN wins
    m[0, 2] = -1.0                                         # all equal negative -> index 0, sentinel
    _, idx = decode_heatmaps(torch.from_numpy(m).to(_dev()), torch.tensor([[192, 256]], dtype=torch.int32))
    assert idx.cpu().numpy().tolist() == [[100, 77, 0]]
    assert np.argmax(m.reshape(3, -1), -1).tolist() == [100, 77, 0]
    # the lane-local scan (one lane owns elements 4l..4l+3 of every 128): same-lane and cross-lane orderings of NaN, +-inf, +-0
    rs = np.random.RandomState(5)
    cases = []
    for trial in range(40):
        h = rs.standard_normal(3072).astype(np.float32)
        kind = trial % 8
        a, b = sorted(rs.choice(3072, 2, replace=False))
        if kind == 0: h[a] = h[b] = np.nan                           # two NaNs: the first
        elif kind == 1: h[b] = np.nan; h[a] = 100.0                  # number first, NaN later: the NaN
        elif kind == 2: h[:] = -np.inf                               # all -inf: index 0
        elif kind == 3: h[:] = -np.inf; h[b] = -1e30
        elif kind == 4: h[0] = np.nan                                # NaN in the very first element
        elif kind == 5: h[:] = -0.0; h[b] = 0.0                      # +0 == -0: index 0
        elif kind == 6: h[a] = h[a + 128 if a + 128 < 3072 else a] = 50.0   # tie inside one lane (stride 128)
        else: h[a] = np.inf; h[b] = np.inf
        cases.append(h.reshape(64, 48))
    mm = np.stack(cases)[None]
    _, idx = decode_heatmaps(torch.from_numpy(mm).to(_dev()), torch.tensor([[192, 256]], dtype=torch.int32))
    assert np.array_equal(idx.cpu().numpy()[0], np.argmax(mm.reshape(40, -1), -1))


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("D", [384, 768, 1024, 1280])
def test_layernorm(D):
    from gpu_util import layernorm
    torch.manual_seed(D)
    x = torch.randn(1000, D, device=_dev()) * 3 + 0.5
    g = torch.randn(D, device=_dev()) * 0.1 + 1
    b = torch.randn(D, device=_dev()) * 0.1
    y = layernorm(x, g, b).float()
    ref = torch.nn.functional.layer_norm(x, (D,), g, b, 1e-6)
    assert (y - ref).abs().max() < 0.03                    # bf16 output rounding of values up to ~|5|
    assert (y - ref.bfloat16().float()).abs().max() < 0.035


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (384, 768, 768), (1000, 2304, 768), (12288, 768, 3072), (200, 384, 384)])
def test_gemm_bias_bf16(M, N, K):
    from gpu_util import EPI_BF16, gemm
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    bias = torch.randn(N, device=_dev())
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=_dev())
    gemm(a, w, bias, out, EPI_BF16)
    ref = a.float() @ w.float().T + bias
    r = _rel(out.float(), ref)
    print("gemm bf16 rel err", r)
    assert r < 1e-2


def test_gemm_gelu():
    from gpu_util import EPI_BF16_GELU, gemm
    torch.manual_seed(1)
    M, N, K = 640, 3072, 768
    a = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    bias = torch.randn(N, device=_dev()) * 0.1
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=_dev())
    gemm(a, w, bias, out, EPI_BF16_GELU)
    ref = torch.nn.functional.gelu(a.float() @ w.float().T + bias)
    assert _rel(out.float(), ref) < 1e-2


def test_gemm_gelu_fit_against_the_erf_epilogue():
    """The fitted tanh-form GELU (default fc1 epilogue) against the A&S-erf epilogue (EPI 6, |erf error| <= 1.5e-7) on the same
    GEMM: after bf16 rounding the two may differ by at most one bf16 step, and on few elements."""
    from gpu_util import EPI_BF16_GELU, EPI_BF16_GELU_ERF, gemm
    torch.manual_seed(7)
    M, N, K = 512, 3072, 768
    a = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.08).bfloat16()              # pre-activations ~ N(0, 1.1): the range trained models use
    bias = torch.randn(N, device=_dev()) * 0.5
    o_fit = torch.zeros(M, N, dtype=torch.bfloat16, device=_dev())
    o_erf = torch.zeros(M, N, dtype=torch.bfloat16, device=_dev())
    gemm(a, w, bias, o_fit, EPI_BF16_GELU)
    gemm(a, w, bias, o_erf, EPI_BF16_GELU_ERF)
    ref = torch.nn.functional.gelu(a.float() @ w.float().T + bias)
    d = (o_fit.float() - o_erf.float()).abs()
    step = 2.0 ** -7 * o_erf.float().abs() + 6e-5                 # one bf16 step of the result (8-bit significand) + the fit's own 2.6e-5
    differ = float((d > 0).float().mean())
    print("fit vs erf epilogue: elements that differ", differ, "| max |fit - erf|", float(d.max()), "| erf epilogue vs exact gelu rel", _rel(o_erf.float(), ref))
    assert bool((d <= step).all())
    assert differ < 0.05
    assert _rel(o_erf.float(), ref) < 5e-3


def test_gemm_gelu_wide_range():
    """Pre-activations from -40 to +40 (bias sweep; the product term is small): the fc1 epilogue's GELU must follow the
    exact erf form everywhere, in particular beyond |x| ~ 11 where the unclamped fit flipped sign (ADVICE r1, high)."""
    from gpu_util import EPI_BF16_GELU, gemm
    torch.manual_seed(5)
    M, N, K = 256, 1024, 64
    a = (torch.randn(M, K, device=_dev()) * 0.1).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    bias = torch.linspace(-40.0, 40.0, N, device=_dev())
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=_dev())
    gemm(a, w, bias, out, EPI_BF16_GELU)
    pre = a.float() @ w.float().T + bias
    ref = torch.nn.functional.gelu(pre)                       # exact erf GELU (vit.py:127,132)
    err = (out.float() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 4e-5                        # bf16 output rounding + the fit's 2.6e-5 + tanh.approx
    worst = float((err / tol).max())
    print("gelu wide range: max err / tol", worst, "| max abs err", float(err.max()), "at pre =", float(pre.flatten()[err.argmax()]))
    assert worst < 1.0
    big = pre.abs() > 11
    pos, neg = big & (pre > 0), big & (pre < 0)
    assert float(((out.float() - pre).abs() / pre.abs())[pos].max()) <= 2.0 ** -8                 # GELU(x) = x there (bf16 step)
    assert float(out[neg].float().abs().max()) < 1e-5                                             # and 0 on the other side


def test_gemm_reduce_add_into_fp32_stream():
    from gpu_util import EPI_F32_ADD, gemm
    torch.manual_seed(2)
    M, N, K = 576, 768, 768
    a = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    bias = torch.randn(N, device=_dev())
    x = torch.randn(M, N, device=_dev())
    ref = x + a.float() @ w.float().T + bias
    gemm(a, w, bias, x, EPI_F32_ADD)                                 # x += ..., like patch embed / proj / fc2 (TMA reduce-add)
    assert _rel(x, ref) < 2e-3


@pytest.mark.parametrize("M,N,K", [(576, 768, 768), (12288, 768, 768), (1000, 384, 1536), (200, 1280, 320), (129, 1024, 4096)])
def test_gemm_residual_rmw_equals_reduce_add(M, N, K):
    """The residual epilogue as load + add + TMA store (gemm.cuh: epilogue_f32_rmw) against the TMA reduce-add form: every
    element has one writer per launch and both forms round fl(x + fl(acc + bias)) -> bit-identical, ragged row blocks, the
    128-wide tiles (N = 384) and subnormal / zero / huge stream values included."""
    from gpu_util import EPI_F32_ADD, gemm
    from easy_vitpose_b200 import _lib
    torch.manual_seed(M + N)
    a = (torch.randn(M, K, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    bias = torch.randn(N, device=_dev())
    x0 = torch.randn(M, N, device=_dev())
    x0[::7, ::5] = 0.0
    x0[3::11, 1::9] *= 1e30
    x0[5::13, 2::3] *= 1e-30
    x0[6::17, 4::7] = 1e-40                                          # subnormal stream values
    outs = []
    L = _lib.lib()
    try:
        for flag in (64, 32, 64, 32):                                # 64 = force reduce-add, 32 = force load + add + store
            L.vpb_debug_gemm(flag << 8, None)
            x = x0.clone()
            gemm(a, w, bias, x, EPI_F32_ADD)
            outs.append(x)
    finally:
        L.vpb_debug_gemm(0, None)
    ref = x0 + a.float() @ w.float().T + bias
    ok = torch.isfinite(ref) & (ref.abs() < 1e20)
    assert _rel(outs[0][ok], ref[ok]) < 2e-3
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), \
        f"{int((outs[0].view(torch.int32) != outs[1].view(torch.int32)).sum())} of {M * N} elements differ"


def _deconv_operands(B, H, W, C, seed):
    """x NHWC bf16, the four phase matrices [4*256, 4*C] bf16 as the engine packs them, the same weights as a
    ConvTranspose2d kernel [C, 256, 4, 4] (fp64 of bf16 values) and a per-channel shift"""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, W, C, generator=g) * (0.5 + torch.rand(1, 1, 1, C, generator=g))).bfloat16()
    w = (torch.randn(C, 256, 4, 4, generator=g) * (0.5 + torch.rand(1, 256, 1, 1, generator=g)) / C ** 0.5).bfloat16().double()
    shift = torch.randn(256, generator=g) * 0.2
    wp = torch.empty(4, 256, 4, C, dtype=torch.float64)                             # [phase, co, tap, ci]
    for py in (0, 1):
        for px in (0, 1):
            for iy in (0, 1):
                for ix in (0, 1):
                    ky = (2 if iy else 0) if py else (3 if iy else 1)
                    kx = (2 if ix else 0) if px else (3 if ix else 1)
                    wp[py * 2 + px, :, iy * 2 + ix, :] = w[:, :, ky, kx].T
    return x.to(_dev()), wp.reshape(4 * 256, 4 * C).bfloat16().contiguous().to(_dev()), w.to(_dev()), shift.to(_dev())


# The engine's two geometries, deconv 1 on the 16 x 12 token grid in 8 x 12 = 96-position tiles and deconv 2 on 32 x 24 in
# 16 x 8 = 128-position tiles, at 1, 2 and many crops (40 and 12 crops: 320 and 288 tiles, more than the SMs), and the other
# geometry vpb_gemm accepts (4 x 24 = 96 positions on 32 x 24)
@pytest.mark.parametrize("B,H,W,C,TR,TW", [(3, 16, 12, 768, 8, 12), (2, 32, 24, 256, 16, 8), (5, 16, 12, 384, 8, 12), (3, 32, 24, 256, 4, 24),
                                          (1, 16, 12, 768, 8, 12), (2, 16, 12, 1024, 8, 12), (40, 16, 12, 384, 8, 12),
                                          (1, 32, 24, 256, 16, 8), (12, 32, 24, 256, 16, 8)])
def test_gemm_implicit_deconv_bn_relu(B, H, W, C, TR, TW):
    """ConvTranspose2d(k4,s2,p1) + eval BatchNorm + ReLU as ONE implicit-GEMM launch (4 phases, shifted 4-D TMA boxes)
    against fp64 on the same bf16-rounded operands, element by element within stage_ref's deconv bound.  Every element of the
    B output crops, their borders included, is written; the crop after them is not."""
    from easy_vitpose_b200 import _lib
    from gpu_util import BF16_SENTINEL, EPI_BF16_RELU_UP, ptr, sentinel_buffer, stream
    from oracle import stage_ref as S
    x, wp, w, shift = _deconv_operands(B, H, W, C, B * H + C + TR)
    ref, bound = S.conv_transpose_bound(x, w, shift.double(), torch.zeros(256, dtype=torch.float64, device=_dev()))
    buf, _ = sentinel_buffer((B + 1) * 4 * H * W * 256, torch.bfloat16)
    out = buf.view(B + 1, 2 * H, 2 * W, 256)
    _lib.check(_lib.lib().vpb_gemm(ptr(x), ptr(wp), ptr(shift), ptr(out), B * H * W, 256, 4 * C, EPI_BF16_RELU_UP, None, 0,
                                   H, W, TR, (TW << 16) | C, stream()))
    torch.cuda.synchronize()
    assert bool((out[B].view(torch.int16) == BF16_SENTINEL).all()), "stores past the last crop"
    got = out[:B]
    unwritten = got.view(torch.int16) == BF16_SENTINEL
    for name, edge in (("top", unwritten[:, 0]), ("bottom", unwritten[:, -1]), ("left", unwritten[:, :, 0]), ("right", unwritten[:, :, -1])):
        assert not bool(edge.any()), f"{name} border of the {2 * H} x {2 * W} output not written"
    r = S.worst_ratio(got, ref, bound)
    print("implicit deconv worst |err| / bound", r)
    if r > 1:
        bad = ((got.double() - ref).abs() / bound).nan_to_num(float("inf")) > 1
        b, y, xx, c = (int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{int(bad.sum())} elements over the bound, first at crop {b} (y {y}, x {xx}) channel {c}: "
                             f"got {float(got[b, y, xx, c])} ref {float(ref[b, y, xx, c])} bound {float(bound[b, y, xx, c]):.3g}; "
                             f"phase {(y % 2) * 2 + xx % 2}, input tile ({(y // 2) // TR}, {(xx // 2) // TW})")


@pytest.mark.parametrize("Kk,Npad", [(17, 32), (25, 32), (133, 144), (1, 32), (32, 32), (33, 144), (144, 144)])
def test_gemm_heatmap_nchw(Kk, Npad):
    """The final 1x1 conv (epilogue 4): fp32 NCHW heatmaps of Kk channels from W padded to Npad rows, its rows and bias past
    Kk non-zero, against fp64 within the GEMM bound; the padded channels [Kk, Npad) are never stored (nothing past the output)."""
    from easy_vitpose_b200 import _lib
    from gpu_util import EPI_F32_NCHW, ptr, sentinel_buffer, stream, untouched
    from oracle import gemm_ref as G
    from oracle import stage_ref as S
    B, pix, K = 2, 3072, 256
    a, w, bias, _ = G.operands(B * pix, Npad, K, seed=Kk, device=_dev())
    z, delta = S._gemm(a.double(), w.double(), bias.double())
    ref = z[:, :Kk].reshape(B, pix, Kk).permute(0, 2, 1)
    bound = delta[:, :Kk].reshape(B, pix, Kk).permute(0, 2, 1)
    buf, sentinel = sentinel_buffer(B * Kk * pix + Npad * pix, torch.float32)
    out = buf[:B * Kk * pix].view(B, Kk, pix)
    _lib.check(_lib.lib().vpb_gemm(ptr(a), ptr(w), ptr(bias), ptr(out), B * pix, Npad, K, EPI_F32_NCHW, None, 0, Kk, pix, 0, 0, stream()))
    torch.cuda.synchronize()
    assert untouched(buf, 0, B * Kk * pix, sentinel), f"channels {Kk}..{Npad - 1} stored past the output"
    r = S.worst_ratio(out, ref, bound)
    print("1x1 conv worst |err| / bound", r)
    assert r <= 1
