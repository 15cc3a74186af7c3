"""-m gpu: crop isolation.  A crop's result must depend on that crop alone: not on the other crops of the call, not on its row
position in the 128-row GEMM blocks, not on what an earlier (larger) call left in the workspace.  Clean inputs cannot show a
break -- a kernel that masks a padding row by multiplying it by zero, or folds a row it should not use into a reduction, gives
the same bits whenever that row holds ordinary numbers -- so these tests put NaN and +-Inf where a leak would carry them:

* kernels through the C ABI: non-finite elements in chosen places; the output must be non-finite exactly on the mask the op's
  dependency structure gives (derived on the CPU) and bit-identical to the clean run everywhere else;
* the engine on a poisoned workspace (option "poison": every float / bf16 activation and staging buffer NaN before each call)
  against a clean engine, bit for bit, over the entry points, the backbone options and ragged batch sizes, each graph key run
  eagerly, captured and replayed;
* hostile crops (NaN, +-Inf, 1e30, 3.4e38, zeros, one NaN pixel) next to clean crops that share a row block, a mirror image or
  an expert segment with them: every clean crop bit-identical to an all-clean call;
* a non-finite crop's own result: NaN heatmaps everywhere (as oracle/torch_ref.py gives on the CPU), decoded as
  O.decode_maps decodes them, NaN scores -- not a finite pose."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
FUSED, SEPARATE = 2, 4                      # vpb_debug_attention: force the fused qkv + attention launch / the two launches
MAX_BATCH = 16


def _ints(t):
    """bit pattern of a tensor / array (NaN payloads included) for exact comparison"""
    if isinstance(t, torch.Tensor):
        t = t.detach().contiguous()
        t = t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32) if t.dtype == torch.float32 else t
        return t.cpu().numpy()
    a = np.ascontiguousarray(t)
    return a.view(np.int32) if a.dtype == np.float32 else a


def _nonfinite(t):
    return ~np.isfinite(t.detach().float().cpu().numpy())


def _check_mask(got, clean, mask, what):
    """got is non-finite exactly on `mask` and bit-identical to `clean` everywhere else"""
    bad = _nonfinite(got)
    assert np.array_equal(bad, mask), \
        f"{what}: {int((bad & ~mask).sum())} non-finite outside the mask, {int((mask & ~bad).sum())} finite inside it (mask {int(mask.sum())})"
    g, c = _ints(got), _ints(clean)
    assert np.array_equal(g[~mask], c[~mask]), f"{what}: {int((g != c)[~mask].sum())} elements outside the mask differ from the clean run"


def _debug_gemm(width=0, flags=0):
    """vpb_debug_gemm: bits 8.. of the GEMM debug flags force the tile width, 32 / 64 the residual epilogue's load + add +
    store / TMA reduce-add form"""
    from easy_vitpose_b200 import _lib
    _lib.lib().vpb_debug_gemm(((width << 8) | flags) << 8, None)


@pytest.fixture
def debug_reset():
    from easy_vitpose_b200 import _lib
    yield
    _lib.lib().vpb_debug_gemm(0, None)
    _lib.lib().vpb_debug_attention(-1)


# ================================================================================================ kernels through the C ABI
BAD_VALUES = (NAN, INF, -INF)


def _gemm_operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, generator=g, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, generator=g, device="cuda")
    return a, w, bias


# (row, column of A, value): rows at both ends of the first and the last (ragged) 128-row block and in between
GEMM_BAD = ((0, 5, NAN), (127, 700, INF), (128, 0, -INF), (200, 767, NAN), (255, 64, -INF), (256, 300, INF), (330, 767, NAN))


@pytest.mark.parametrize("width", [128, 192, 256])
@pytest.mark.parametrize("epi,flags", [(0, 0), (1, 0), (6, 0), (5, 64), (5, 32)],
                         ids=["bf16", "gelu", "gelu_erf", "f32_reduce_add", "f32_load_add_store"])
def test_gemm_bad_row_of_a_spoils_that_row(debug_reset, epi, flags, width):
    """vpb_gemm with the TMA epilogues at every forced tile width: a non-finite A[r, k] spoils output row r and nothing else
    (the other 127 rows of its block, the ragged last block's padding rows and every other block keep their clean bits)."""
    from gpu_util import EPI_F32_ADD, gemm
    M, N, K = 331, 768, 768
    a, w, bias = _gemm_operands(M, N, K, 17 * width + epi)
    x0 = torch.randn(M, N, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    bad = a.clone()
    for r, k, v in GEMM_BAD:
        bad[r, k] = v
    mask = np.zeros((M, N), bool)
    mask[[r for r, _, _ in GEMM_BAD]] = True
    _debug_gemm(width, flags)
    outs = []
    for src in (a, bad):
        out = x0.clone() if epi == EPI_F32_ADD else torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        gemm(src, w, bias, out, epi)
        outs.append(out)
    assert not _nonfinite(outs[0]).any()
    _check_mask(outs[1], outs[0], mask, f"epilogue {epi}, flags {flags}, width {width}")


@pytest.mark.parametrize("Kk,Npad", [(17, 32), (133, 144)])
def test_gemm_heatmap_nchw_bad_pixel_row(Kk, Npad):
    """The 1x1-conv epilogue (NCHW heatmaps, N padded to 32 / 144): a non-finite input pixel spoils that pixel of every real
    channel, nothing else; the padded weight rows never reach the output."""
    from gpu_util import EPI_F32_NCHW, gemm
    B, pix, K = 3, 3072, 256
    a, w, bias = _gemm_operands(B * pix, Npad, K, Kk)
    w[Kk:] = 0
    bias[Kk:] = 0
    rows = ((0, 0, NAN), (3071, 255, INF), (3072, 17, -INF), (2 * 3072 + 1500, 100, NAN), (B * pix - 1, 3, INF))
    bad = a.clone()
    mask = np.zeros((B, Kk, pix), bool)
    for r, k, v in rows:
        bad[r, k] = v
        mask[r // pix, :, r % pix] = True
    outs = []
    for src in (a, bad):
        out = torch.zeros(B, Kk, pix, device="cuda")
        gemm(src, w, bias, out, EPI_F32_NCHW, aux=(Kk, pix, 0, 0))
        outs.append(out)
    _check_mask(outs[1], outs[0], mask, f"NCHW K={Kk}")


def _deconv_weights(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn(4 * 256, 4 * C, generator=g, device="cuda") / (C ** 0.5)        # [phase * 256 + co, tap * C + ci]
    shift = torch.randn(256, generator=g, device="cuda") * 0.2
    return w.bfloat16().contiguous(), shift


def _deconv(x, wp, shift, TR, TW):
    from easy_vitpose_b200 import _lib
    from gpu_util import EPI_BF16_RELU_UP, ptr, stream
    B, H, W, Cin = x.shape
    out = torch.full((B, 2 * H, 2 * W, 256), -7.0, dtype=torch.bfloat16, device="cuda")
    _lib.check(_lib.lib().vpb_gemm(ptr(x), ptr(wp), ptr(shift), ptr(out), B * H * W, 256, 4 * Cin, EPI_BF16_RELU_UP, None, 0,
                                   H, W, TR, (TW << 16) | Cin, stream()))
    torch.cuda.synchronize()
    return out


def _deconv_bad_sum(bad, wp, B, H, W, Cin):
    """float64 sum of the non-finite inputs' contributions to every output of ConvTranspose2d(k4, s2, p1) in the engine's
    phase form: output (2y + py, 2x + px) reads input (y + dy, x + dx) through tap (iy, ix) of phase (py, px) (gemm.cuh, the
    deconv producer).  NaN / +-Inf where a bad input reaches, 0 elsewhere."""
    wf = wp.float().cpu().numpy().astype(np.float64).reshape(4, 256, 4, Cin)
    s = np.zeros((B, 2 * H, 2 * W, 256))
    with np.errstate(invalid="ignore"):
        for b, yi, xi, c, v in bad:
            for py in (0, 1):
                for px in (0, 1):
                    for iy in (0, 1):
                        for ix in (0, 1):
                            dy = (0 if iy else 1) if py else (-1 if iy else 0)
                            dx = (0 if ix else 1) if px else (-1 if ix else 0)
                            y, x = yi - dy, xi - dx
                            if 0 <= y < H and 0 <= x < W:
                                s[b, 2 * y + py, 2 * x + px] += v * wf[2 * py + px, :, 2 * iy + ix, c]
    return s


@pytest.mark.parametrize("B,H,W,Cin,TR,TW", [(3, 16, 12, 768, 8, 12), (2, 32, 24, 256, 16, 8)], ids=["8x12", "16x8"])
def test_deconv_bad_input_spoils_its_footprint(B, H, W, Cin, TR, TW):
    """The implicit-GEMM deconv + BN + ReLU with both tile shapes (96 positions: rows 96..127 of every A tile hold stale shared
    memory; 128 positions).  A NaN input spoils exactly its transposed-conv footprint -- the indicator convolved with an
    all-ones 4x4 stride-2 kernel, all 256 channels -- and ReLU must keep it NaN, as torch's relu does.  +-Inf inputs: where
    the contributions sum to +Inf or NaN the output is non-finite, where they sum to -Inf ReLU gives exactly 0."""
    g = torch.Generator(device="cuda").manual_seed(B * H + Cin)
    x = (torch.randn(B, H, W, Cin, generator=g, device="cuda") * 0.5).bfloat16()
    wp, shift = _deconv_weights(Cin, Cin + TR)
    clean = _deconv(x, wp, shift, TR, TW)
    assert not _nonfinite(clean).any()
    cases = {
        "nan": [(0, 0, 0, 5, NAN), (0, H - 1, W - 1, Cin - 1, NAN), (1, TR - 1, W // 2, 64, NAN), (B - 1, H // 2, 3, 0, NAN)],
        "inf": [(0, 0, W - 1, 7, INF), (1, TR, TW - 1, 100, -INF), (B - 1, H - 1, 0, Cin - 2, INF), (B - 1, 5, 6, 1, -INF)],
    }
    for kind, bad in cases.items():
        xb = x.clone()
        for b, y, xx, c, v in bad:
            xb[b, y, xx, c] = v
        got = _deconv(xb, wp, shift, TR, TW)
        s = _deconv_bad_sum(bad, wp, B, H, W, Cin)
        if kind == "nan":
            ind = torch.zeros(B, 1, H, W, dtype=torch.float64)
            for b, y, xx, _, _ in bad:
                ind[b, 0, y, xx] = 1
            foot = torch.nn.functional.conv_transpose2d(ind, torch.ones(1, 1, 4, 4, dtype=torch.float64), stride=2, padding=1)[:, 0] > 0
            assert np.array_equal(np.isnan(s).any(-1), foot.numpy())                      # the derivation is the footprint
        mask = np.isnan(s) | (s == np.inf)
        zero = s == -np.inf
        assert np.array_equal(_ints(got)[zero], np.zeros(int(zero.sum()), np.int16)), f"{kind}: relu(-inf) must be +0"
        _check_mask(got, torch.where(torch.from_numpy(zero).cuda(), torch.zeros_like(clean), clean), mask, f"deconv {TR}x{TW}, {kind}")


def _qkv(B, heads, hd, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = heads * hd
    qkv = torch.randn(B * 192, 3 * D, generator=g, device="cuda")
    qkv[:, :D] *= (hd ** -0.5) * 2.0
    return qkv.bfloat16()


# key / value rows in a column the polynomial exponential serves (j % 16 in {1, 3, 5, 7}) and in MUFU columns
POLY_KEYS, MUFU_KEYS = (1, 23, 191 - 8), (0, 8, 191)


@pytest.mark.parametrize("hd", [32, 64, 80])
@pytest.mark.parametrize("poly", [0, 1])
def test_attention_bad_query_key_value(debug_reset, hd, poly):
    """vpb_attention, every exponential on the MUFU or every 4th by ex2_poly.  A non-finite element of a key row spoils the whole
    (crop, head); of a value row, that column of the (crop, head); of a query row, that row of the head.  Each key / value row
    is tried in a column the polynomial serves and in a MUFU column: a polynomial that turns a NaN logit into a finite weight
    leaves the head finite."""
    from easy_vitpose_b200 import _lib
    from gpu_util import attention
    B, heads = 3, (4 if hd == 80 else 6)
    D = heads * hd
    qkv = _qkv(B, heads, hd, 31 * hd + poly)
    _lib.lib().vpb_debug_attention(poly)
    clean = attention(qkv, B, heads, hd)
    assert not _nonfinite(clean).any()

    def run(cells, what):
        bad = qkv.clone()
        mask = np.zeros((B * 192, D), bool)
        for part, b, t, h, d, v, rows, cols in cells:
            bad[b * 192 + t, part * D + h * hd + d] = v
            mask[b * 192 + rows[0]: b * 192 + rows[1], h * hd + cols[0]: h * hd + cols[1]] = True
        _check_mask(attention(bad, B, heads, hd), clean, mask, f"hd {hd}, poly {poly}: {what}")

    for keys, col in ((POLY_KEYS, "polynomial"), (MUFU_KEYS, "MUFU")):
        # key rows: NaN (an infinite key gives -inf logits in some rows, which softmax legitimately zeroes)
        run([(1, 0, keys[0], 0, 3, NAN, (0, 192), (0, hd)), (1, B - 1, keys[2], heads - 1, hd - 1, NAN, (0, 192), (0, hd))],
            f"NaN keys in {col} columns")
        # value rows: the column of that element, every query row of the crop
        run([(2, 0, keys[1], 1, 0, NAN, (0, 192), (0, 1)), (2, 1, keys[0], 0, hd - 1, INF, (0, 192), (hd - 1, hd)),
             (2, B - 1, keys[2], heads - 1, 17, -INF, (0, 192), (17, 18))], f"bad values in {col} rows")
    for v in BAD_VALUES:
        run([(0, 0, 0, 0, 0, v, (0, 1), (0, hd)), (0, 1, 100, heads - 1, hd - 1, v, (100, 101), (0, hd)),
             (0, B - 1, 191, 2, 9, v, (191, 192), (0, hd))], f"query rows = {v}")


@pytest.mark.parametrize("D", [384, 768, 1024, 1280])
def test_layernorm_bad_element_spoils_its_row(D):
    from gpu_util import layernorm
    g = torch.Generator(device="cuda").manual_seed(D)
    x = torch.randn(300, D, generator=g, device="cuda") * 3 + 0.5
    gam = torch.randn(D, generator=g, device="cuda") * 0.1 + 1
    bet = torch.randn(D, generator=g, device="cuda") * 0.1
    clean = layernorm(x, gam, bet)
    bad = x.clone()
    mask = np.zeros((300, D), bool)
    for r, d, v in ((0, 0, NAN), (1, D - 1, INF), (150, 77, -INF), (299, 5, NAN)):
        bad[r, d] = v
        mask[r] = True
    _check_mask(layernorm(bad, gam, bet), clean, mask, f"LayerNorm D={D}")


# ================================================================================================ engines
def _cfg(size, K, depth):
    from easy_vitpose_b200 import model_cfg
    cfg = model_cfg(size, K)
    cfg["backbone"] = dict(cfg["backbone"], depth=depth)
    return cfg


# name: (size, D, depth, heads, K, weight seed)
SPECS = {"s": ("s", 384, 12, 12, 17, 101), "b": ("b", 768, 12, 12, 17, 102), "h": ("h", 1280, 2, 16, 133, 104)}
MULTI_HEADS = (("coco", 17), ("aic", 14), ("wholebody", 133))
_sds, _engines = {}, {}


def _state_dict(name):
    if name not in _sds:
        if name == "multi":
            from oracle.multi_head import plus_state_dict
            _sds[name] = plus_state_dict("b", [k for _, k in MULTI_HEADS], 192, 31)
        else:
            _, D, depth, _, K, seed = SPECS[name]
            _sds[name] = O.make_state_dict(D, depth, K, seed, peaky=0.1, bumps=True)
    return _sds[name]


def _make(name, max_batch=MAX_BATCH):
    from easy_vitpose_b200 import ViTPose
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in _state_dict(name).items()}
    if name == "multi":
        m = ViTPose(_cfg("b", 17, 12), max_batch=max_batch, heads=MULTI_HEADS, expert_rows=192)
    else:
        size, _, depth, _, K, _ = SPECS[name]
        m = ViTPose(_cfg(size, K, depth), max_batch=max_batch)
    m.load_state_dict(sd)
    return m.to("cuda:0")


def _pair(name):
    """(clean engine, engine poisoned before every call) with the same weights"""
    if name not in _engines:
        _engines[name] = (_make(name), _make(name))
    return _engines[name]


DEFAULTS = {"chain": 0, "ln_fused": 0, "ln_in_gemm": 0, "resid_rmw": 0, "ln_ctl": 1}
# option set: (engine options over the defaults, vpb_debug_attention flags, forced GEMM tile width)
OPTIONS = {
    "defaults": ({}, -1, 0), "chain": ({"chain": 1}, -1, 0), "ln_fused": ({"ln_fused": 1}, -1, 0),
    "ln_in_gemm": ({"ln_in_gemm": 1}, -1, 0), "resid_rmw": ({"resid_rmw": 1}, -1, 0),
    "ln_ctl": ({"chain": 1, "ln_ctl": 0}, -1, 0), "fused_attention": ({}, FUSED, 0), "poly": ({}, 1, 0),
    "width128": ({}, -1, 128), "width192": ({}, -1, 192), "width256": ({}, -1, 256),
}


def _apply(engines, option):
    from easy_vitpose_b200 import _lib
    opts, att, width = OPTIONS[option]
    _lib.lib().vpb_debug_attention(att)
    _debug_gemm(width)
    for m in engines:
        for k, v in dict(DEFAULTS, **opts).items():
            m.set_option(k, v)            # every one of these drops the captured graphs, which embed the debug settings too


def _same(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert np.array_equal(_ints(u), _ints(v)), f"{what}: output {i} differs ({int((_ints(u) != _ints(v)).sum())} elements)"


def _flat(out):
    """an entry point's outputs as one list of arrays (per-frame lists concatenated)"""
    res = []
    for o in out:
        if isinstance(o, (list, tuple)):
            o = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in o]
            res.append(np.concatenate(o) if o else np.zeros(0))
        else:
            res.append(o.cpu().numpy() if isinstance(o, torch.Tensor) else o)
    return res


def _crops(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).cuda()
    org = torch.from_numpy(np.random.RandomState(seed).randint(64, 513, size=(n, 2)).astype(np.int32)).cuda()
    return x, org


_frames_cache = {}


def _frames(device):
    """two RGB frames, the second a column slice of a wider image (rows at a larger pitch, read in place)"""
    if device not in _frames_cache:
        rs = np.random.RandomState(77)
        a = rs.randint(0, 256, size=(360, 480, 3), dtype=np.uint8)
        wide = rs.randint(0, 256, size=(300, 640, 3), dtype=np.uint8)
        if device:
            _frames_cache[device] = [torch.from_numpy(a).cuda(), torch.from_numpy(wide).cuda()[:, 100:520]]
        else:
            _frames_cache[device] = [a, wide[:, 100:520]]
    return _frames_cache[device]


def _boxes(frames, n, seed, nv12=False):
    rs = np.random.RandomState(seed)
    counts = [n - n // 2, n // 2]
    out = []
    for f, c in zip(frames, counts):
        H, W = (f.shape[0] * 2 // 3 if nv12 else f.shape[0]), f.shape[1]
        x0, y0 = rs.randint(0, W - 60, c), rs.randint(0, H - 60, c)
        x1, y1 = np.minimum(x0 + rs.randint(40, 220, c), W), np.minimum(y0 + rs.randint(40, 220, c), H)
        out.append(np.stack([x0, y0, x1, y1], 1).astype(np.int32))
    return out


def _affine(boxes):
    mats, cs, ss = [], [], []
    for b in boxes:
        b = b.astype(np.float64)
        w, h = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
        s = np.minimum(192.0 / w, 256.0 / h)
        m = np.zeros((len(b), 2, 3))
        m[:, 0, 0] = m[:, 1, 1] = s
        m[:, 0, 2] = 96.0 - s * (b[:, 0] + w / 2)
        m[:, 1, 2] = 128.0 - s * (b[:, 1] + h / 2)
        mats.append(m)
        cs.append(np.stack([b[:, 0] + w / 2, b[:, 1] + h / 2], 1).astype(np.float32))
        ss.append(np.stack([192.0 / s, 256.0 / s], 1).astype(np.float32))
    return mats, cs, ss


def _nv12(frames_np):
    out = []
    for f in frames_np:
        H, W = f.shape[0] // 2 * 2, f.shape[1] // 2 * 2
        rs = np.random.RandomState(H + W)
        out.append(torch.from_numpy(rs.randint(16, 236, size=(3 * H // 2, W), dtype=np.uint8)).cuda())
    return out


def _infer_heads(m, x, org, segs, with_heatmaps=True):
    """vpb_infer_heads with an explicit segment list (infer_crops_heads would group the crops by head)"""
    from easy_vitpose_b200 import _lib
    n, Km = x.shape[0], m.num_keypoints_max
    kp = torch.zeros((n, Km, 3), dtype=torch.float32, device=x.device)
    idx = torch.zeros((n, Km), dtype=torch.int32, device=x.device)
    hm = torch.zeros((n, Km, 64, 48), dtype=torch.float32, device=x.device) if with_heatmaps else None
    arr = (_lib.VpbSegment * len(segs))(*[_lib.VpbSegment(h, c) for h, c in segs])
    m._call_on_stream((x, org, kp, idx, hm), lambda st: _lib.lib().vpb_infer_heads(
        m._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, len(segs), C.c_void_p(kp.data_ptr()),
        C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()) if hm is not None else None, st))
    return (kp, idx, hm) if with_heatmaps else (kp, idx)


def _alternating(n, H=len(MULTI_HEADS)):
    return [(i % H, 1) for i in range(n)]


def _entry(kind):
    """entry point kind -> call(engine, n, seed) returning its outputs"""
    def crops(m, n, s):
        x, org = _crops(n, s)
        return m.infer_crops(x, org, return_heatmaps=True)

    def features_head(m, n, s):
        f = m.forward_features(_crops(n, s)[0])
        return f, m.head_forward(f)

    def frames(m, n, s):
        fr = _frames(True)
        return m.infer_frames(fr, _boxes(fr, n, s))

    def affine(m, n, s):
        fr = _frames(True)
        return m.infer_affine(fr, *_affine(_boxes(fr, n, s)))

    def nv12(m, n, s):
        fr = _nv12(_frames(False))
        return m.infer_frames_nv12(fr, _boxes(fr, n, s, nv12=True))

    def host(m, n, s):
        x, org = _crops(n, s)
        return m.infer_host(x.cpu().numpy(), org.cpu().numpy())

    def pipelined(m, n, s):
        x, org = _crops(n, s)
        outs = []
        for slot in (0, 1):
            kp, idx = np.empty((n, m.num_keypoints, 3), np.float32), np.empty((n, m.num_keypoints), np.int32)
            m.submit_host(np.ascontiguousarray(x.cpu().numpy()[::-1] if slot else x.cpu().numpy()), org.cpu().numpy(), kp, idx, slot)
            outs.append((kp, idx))
        for slot in (0, 1):
            m.wait_host(slot)
        return [a for o in outs for a in o]

    def frames_host(m, n, s):
        fr = _frames(False)
        return m.infer_frames_host(fr, _boxes(fr, n, s))

    def affine_host(m, n, s):
        fr = _frames(False)
        return m.infer_affine_host(fr, *_affine(_boxes(fr, n, s)))

    def mixed(m, n, s):
        x, org = _crops(n, s)
        return _infer_heads(m, x, org, _alternating(n))

    def mixed_frames(m, n, s):
        fr = _frames(True)
        bx = _boxes(fr, n, s)
        return m.infer_frames_heads(fr, bx, [np.arange(len(b)) % len(MULTI_HEADS) for b in bx])

    return locals()[kind]


def _poisoned_sequence(name, kind, option, flip=None):
    """clean and poisoned engines through the same calls: ragged sizes, each size eager, captured and replayed, the largest
    call first so the smaller ones run on what it left behind"""
    engines = _pair(name)
    call = _entry(kind)
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    try:
        if flip is not None:
            for m in engines:
                if name == "multi":
                    m.set_flip_test_heads([COCO_FLIP_PAIRS, [], []], shift_heatmap=flip)
                else:
                    m.set_flip_test(COCO_FLIP_PAIRS if engines[0].num_keypoints == 17 else [], shift_heatmap=flip)
        _apply(engines, option)
        limit = engines[0].batch_limit
        for rep in range(3):
            for n in (limit, 1, 5, 7):
                seed = 1000 * rep + n
                want = _flat(call(engines[0], n, seed))
                engines[1].set_option("poison", 1)
                got = _flat(call(engines[1], n, seed))
                for w in want:
                    if w.dtype == np.float32:
                        assert np.isfinite(w).all(), f"{name} {kind} {option}: clean outputs must be finite"
                _same(got, want, f"{name} {kind} {option} flip={flip} n={n} call {rep}")
    finally:
        _apply(engines, "defaults")
        if flip is not None:
            for m in engines:
                (m.set_flip_test_heads if name == "multi" else m.set_flip_test)(None)


@pytest.mark.parametrize("option", list(OPTIONS))
def test_poisoned_workspace_vit_b_crops(debug_reset, option):
    _poisoned_sequence("b", "crops", option)


@pytest.mark.parametrize("kind", ["features_head", "frames", "affine", "nv12", "host", "pipelined", "frames_host", "affine_host"])
def test_poisoned_workspace_vit_b_entry_points(debug_reset, kind):
    _poisoned_sequence("b", kind, "defaults")


@pytest.mark.parametrize("kind,shift", [("crops", False), ("crops", True), ("frames", True), ("affine", False), ("host", True)])
def test_poisoned_workspace_vit_b_flip_test(debug_reset, kind, shift):
    _poisoned_sequence("b", kind, "defaults", flip=shift)


@pytest.mark.parametrize("option", ["defaults", "chain", "ln_in_gemm", "fused_attention", "poly", "width128", "width192"])
def test_poisoned_workspace_vit_s(debug_reset, option):
    """head_dim 32; D = 384 takes no 256-wide tiles"""
    _poisoned_sequence("s", "crops", option)


@pytest.mark.parametrize("kind,option,flip", [("crops", "defaults", None), ("crops", "chain", None), ("crops", "fused_attention", None),
                                              ("features_head", "defaults", None), ("crops", "defaults", True)])
def test_poisoned_workspace_vit_h(debug_reset, kind, option, flip):
    """head_dim 80, 133 keypoints (heatmap GEMM N padded to 144)"""
    _poisoned_sequence("h", kind, option, flip=flip)


@pytest.mark.parametrize("kind,option,flip", [("mixed", "defaults", None), ("mixed", "chain", None), ("mixed", "fused_attention", None),
                                              ("mixed", "width128", None), ("mixed", "defaults", False), ("mixed", "defaults", True),
                                              ("mixed_frames", "defaults", None)])
def test_poisoned_workspace_multi_head(debug_reset, kind, option, flip):
    """ViT-B with 192 expert rows and three heads (K = 17, 14, 133) in 1-crop segments of alternating heads: expert tiles
    straddle segments, and the smaller heads leave maps K..K_max of the workspace unwritten"""
    _poisoned_sequence("multi", kind, option, flip=flip)


# ================================================================================================ hostile neighbours
def _hostile(kind, seed):
    c = O.make_crops(1, seed)[0]
    if kind == "pixel":
        c[1, 5, 20] = np.nan                               # patch (0, 1): a key row the polynomial exponential serves
        return c
    return np.full_like(c, {"nan": np.nan, "+inf": np.inf, "-inf": -np.inf, "1e30": 1e30, "3.4e38": 3.4e38, "zeros": 0.0}[kind])


NON_FINITE_KINDS = ("nan", "+inf", "-inf", "pixel")         # every heatmap NaN
# crops c and c + 1 share the 128-row block floor(192 (c + 1) / 128) when c is even
LAYOUT_16 = {0: "nan", 3: "+inf", 6: "-inf", 9: "1e30", 10: "3.4e38", 13: "zeros", 15: "pixel"}
LAYOUT_FLIP_7 = {1: "nan", 4: "+inf", 6: "pixel"}          # crop 6 shares a block with the mirror image of crop 0 (model crop 7)


def _with_hostile(n, layout, seed):
    x, org = _crops(n, seed)
    xh = x.clone()
    for c, kind in layout.items():
        xh[c] = torch.from_numpy(_hostile(kind, seed + c))
    return x, xh, org


def _check_neighbours(clean_out, hostile_out, layout, what):
    n = clean_out[0].shape[0]
    keep = [c for c in range(n) if c not in layout]
    for i, (u, v) in enumerate(zip(clean_out, hostile_out)):
        u, v = _ints(u), _ints(v)
        for c in keep:
            assert np.array_equal(u[c], v[c]), f"{what}: clean crop {c} changed (output {i}) next to hostile crops {layout}"


def _check_own(kp, idx, hm, org, layout, what, K=None):
    """hostile crops: decode consistent with O.decode_maps of the engine's own maps; NaN maps and NaN scores where the crop
    is not finite"""
    kp, idx, hm, org = (t.cpu().numpy() for t in (kp, idx, hm, org))
    for c, kind in layout.items():
        k = K[c] if K is not None else hm.shape[1]
        h = hm[c:c + 1, :k]
        okp, oidx = O.decode_maps(np.ascontiguousarray(h), org[c:c + 1], wrap="crop")
        assert np.array_equal(idx[c, :k], oidx[0]), f"{what}: crop {c} ({kind}) argmax != decode of its maps"
        assert np.array_equal(kp[c, :k, 2], okp[0, :, 2], equal_nan=True), f"{what}: crop {c} ({kind}) scores"
        assert np.array_equal(np.isnan(kp[c, :k]), np.isnan(okp[0])), f"{what}: crop {c} ({kind}) NaN pattern of the keypoints"
        fin = np.isfinite(okp[0, :, :2])
        ref = okp[0, :, :2][fin]                                   # blur bit-exact; logf vs np.log differ by ulps
        tol = 2e-3 * float(org[c].max()) / 47 + 2e-3 * np.abs(ref)
        assert (np.abs(kp[c, :k, :2][fin] - ref) <= tol).all(), f"{what}: crop {c} ({kind}) keypoints"
        if kind in NON_FINITE_KINDS:
            assert np.isnan(h).all(), f"{what}: crop {c} ({kind}) must give NaN heatmaps everywhere, {int(np.isfinite(h).sum())} finite"
            assert np.isnan(kp[c, :k, 2]).all()


@pytest.mark.parametrize("name", ["s", "b", "h"])
def test_hostile_neighbours_crops(name):
    m = _pair(name)[0]
    n = MAX_BATCH
    x, xh, org = _with_hostile(n, LAYOUT_16, 5)
    for call in range(3):                                  # eager, captured, replayed
        clean = m.infer_crops(x, org, return_heatmaps=True)
        hostile = m.infer_crops(xh, org, return_heatmaps=True)
        _check_neighbours(clean, hostile, LAYOUT_16, f"ViT-{name} call {call}")
    _check_own(*hostile, org, LAYOUT_16, f"ViT-{name}")
    f_clean, f_host = m.forward_features(x), m.forward_features(xh)
    _check_neighbours([f_clean, m.head_forward(f_clean)], [f_host, m.head_forward(f_host)], LAYOUT_16, f"ViT-{name} features + head")
    kc, ic = m.infer_host(x.cpu().numpy(), org.cpu().numpy())
    kh, ih = m.infer_host(xh.cpu().numpy(), org.cpu().numpy())
    _check_neighbours([kc, ic], [kh, ih], LAYOUT_16, f"ViT-{name} host")


@pytest.mark.parametrize("shift", [False, True])
def test_hostile_neighbours_flip_test(shift):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    m = _pair("b")[0]
    x, xh, org = _with_hostile(7, LAYOUT_FLIP_7, 9)
    try:
        m.set_flip_test(COCO_FLIP_PAIRS, shift_heatmap=shift)
        for call in range(3):
            clean = m.infer_crops(x, org, return_heatmaps=True)
            hostile = m.infer_crops(xh, org, return_heatmaps=True)
            _check_neighbours(clean, hostile, LAYOUT_FLIP_7, f"flip test shift={shift} call {call}")
        _check_own(*hostile, org, LAYOUT_FLIP_7, f"flip test shift={shift}")
    finally:
        m.set_flip_test(None)


@pytest.mark.parametrize("flip", [None, False, True])
def test_hostile_neighbours_mixed_heads(flip):
    """1-crop segments of alternating heads: every hostile crop's neighbours are in another expert segment"""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    m = _pair("multi")[0]
    n = MAX_BATCH if flip is None else 7
    layout = LAYOUT_16 if flip is None else LAYOUT_FLIP_7
    x, xh, org = _with_hostile(n, layout, 13)
    segs = _alternating(n)
    K = [MULTI_HEADS[h][1] for h, _ in segs]
    try:
        if flip is not None:
            m.set_flip_test_heads([COCO_FLIP_PAIRS, [], []], shift_heatmap=flip)
        for call in range(3):
            clean = _infer_heads(m, x, org, segs)
            hostile = _infer_heads(m, xh, org, segs)
            _check_neighbours(clean, hostile, layout, f"mixed heads flip={flip} call {call}")
        _check_own(*hostile, org, layout, f"mixed heads flip={flip}", K=K)
    finally:
        if flip is not None:
            m.set_flip_test_heads(None)


# ================================================================================================ a non-finite crop's own result
@pytest.mark.parametrize("name", ["s", "b"])
def test_non_finite_crop_gives_nan_heatmaps_like_the_reference(name):
    """What the reference computes for a corrupt crop (oracle/torch_ref.py on the CPU: F.relu and softmax propagate NaN):
    NaN heatmaps everywhere.  The engine must agree, and so report NaN scores, not a finite pose near the crop's corner."""
    from oracle import torch_ref
    _, D, depth, heads, K, _ = SPECS[name]
    m = _pair(name)[0]
    kinds = ("nan", "+inf", "-inf", "pixel")
    x = torch.from_numpy(np.stack([_hostile(k, 3 + i) for i, k in enumerate(kinds)]))
    org = torch.tensor([[192, 256]] * len(kinds), dtype=torch.int32)
    sd = torch_ref.to_device(_state_dict(name), "cpu", torch.float32)
    with torch.no_grad(), np.errstate(all="ignore"):
        ref = torch_ref.forward(x, sd, depth, heads)
    assert torch.isnan(ref).all(), "the CPU reference propagates NaN through every layer"
    kp, idx, hm = (t.cpu() for t in m.infer_crops(x.cuda(), org.cuda(), return_heatmaps=True))
    assert torch.isnan(hm).all(), f"{int(torch.isfinite(hm).sum())} finite heatmap values from non-finite crops " \
                                  f"(per crop: {[int(torch.isfinite(hm[i]).sum()) for i in range(len(kinds))]})"
    with np.errstate(all="ignore"):
        okp, oidx = O.decode_maps(hm.numpy(), org.numpy(), wrap="crop")
    assert np.array_equal(idx.numpy(), oidx)
    assert np.array_equal(kp.numpy(), okp, equal_nan=True)
    assert torch.isnan(kp[..., 2]).all()


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("form", [FUSED, SEPARATE], ids=["fused", "separate"])
@pytest.mark.parametrize("name", ["s", "b"])
def test_bad_xn_row_spoils_its_crop_in_the_attention(debug_reset, name, form, poly):
    """The fused qkv + attention launch (and the two-launch form): a NaN pixel gives NaN patch row p, so NaN xn row p at block 0;
    that crop's q, k, v rows p are NaN in every head, so the whole crop's attention output must be NaN -- row p in a column the
    polynomial serves (p = 1) and in a MUFU column (p = 0) -- and every other crop keeps its clean bits.  The engine has one
    block, so the attention buffer read back is block 0's."""
    from easy_vitpose_b200 import ViTPose, _lib
    _, D, _, heads, K, seed = SPECS[name]
    size = SPECS[name][0]
    m = ViTPose(_cfg(size, K, 1), max_batch=8)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, 1, K, seed, peaky=0.1, bumps=True).items()})
    m.to("cuda:0")
    n = 6
    x, org = _crops(n, 21)
    _lib.lib().vpb_debug_attention(form | poly)
    m.set_option("graph", 0)

    def attn(inp):
        m.infer_crops(inp, org)
        torch.cuda.synchronize()
        return m.read_buffer("attn", (n * 192, D), "bf16")

    clean = attn(x)
    for c, (y, xx) in ((0, (5, 20)), (3, (5, 5)), (5, (200, 150))):      # patches 1 (polynomial column), 0 and 12 * 12 + 9
        xb = x.clone()
        xb[c, 0, y, xx] = NAN
        mask = np.zeros((n * 192, D), bool)
        mask[c * 192:(c + 1) * 192] = True
        _check_mask(attn(xb), clean, mask, f"ViT-{name} form {form} poly {poly}: NaN pixel in crop {c}")
