"""-m gpu: the engine at the limits its C ABI documents, which the other suites never reach: 1 and 144 keypoints (and the
heatmap GEMM's 32- and 144-wide tiles full and one past full), VPB_MAX_HEADS = 8 heads, VPB_MAX_SEGMENTS = 64 segments (128
expert segments with flip test, the whole ExpertParams table), the widest expert split P = D - 32, and batches past 64.

Engines run at depth 2: every kernel here is per layer, the depth only repeats it.  The references are the fp64 stage
references of test_gpu_stages (Checks, _check_block0_and_head, _check_tail), the decode oracles and the reference fixture
tests/golden/decode_k_edges.npz (oracle/make_golden_k_edges.py), and, for the multi-head and batch cases, single-head or
smaller calls that must give the same bits.

Tile widths pick_tile chooses on an H100 SXM (132 SMs), from its rule (least ceil(tiles / SMs) * width, ties to 192, then
256, then 128): at 64 crops (M = 12288) ViT-S patch / proj / fc2 192, qkv 128, fc1 192 and ViT-B 192 for all; at 256 crops
(M = 49152) ViT-S qkv 192, fc1 128 and ViT-B fc1 256, the others 192.  So the 256-crop calls below run other tile widths
than their 64-crop pieces, and the persistent tile loops run several waves of row blocks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import decode_modes_oracle as M, preproc_oracle as P, vitpose_oracle as O
from oracle import multi_head as MH
from oracle.make_golden_k_edges import COMBOS, KS, MODE_KS, N as DEC_N, centre_scale_of, org_of, seed_of
from test_gpu_stages import Checks, _check_block0_and_head, _check_tail

pytestmark = pytest.mark.gpu

DEPTH = 2
DIMS = {"s": (384, 12), "b": (768, 12)}              # embed_dim, attention heads
NAN_BITS, IDX_SENTINEL = 0x7FC00000, 0x7FFFFFFF
_cache = {}


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need an H100"
    return torch.device("cuda", 0)


def _lib():
    from easy_vitpose_b200 import _lib as L
    return L


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _sd(size, K, seed=71):
    key = ("sd", size, K, seed)
    if key not in _cache:
        _cache[key] = O.make_state_dict(DIMS[size][0], DEPTH, K, seed, peaky=0.1, bumps=True)
    return _cache[key]


def _single(size, K, max_batch=16):
    """a depth-2 single-head engine and its state dict"""
    from easy_vitpose_b200 import ViTPose, model_cfg
    key = ("single", size, K, max_batch)
    if key not in _cache:
        cfg = model_cfg(size, K)
        cfg["backbone"]["depth"] = DEPTH
        m = ViTPose(cfg, max_batch=max_batch)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in _sd(size, K).items()})
        _cache[key] = m.to("cuda:0")
    return _sd(size, K), _cache[key]


def _crops(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).to(_dev())
    org = torch.from_numpy(np.random.RandomState(seed).randint(64, 513, size=(n, 2)).astype(np.int32)).to(_dev())
    return x, org


def _pairs(K):
    """flip pairs: none for K = 1 (permutation [0]); for K = 144 a scrambled involution with 24 fixed points; else neighbours"""
    if K == 144:
        order = np.random.RandomState(9).permutation(K)
        return [(int(order[2 * i]), int(order[2 * i + 1])) for i in range(60)]
    return [(i, i + 1) for i in range(1, K - 1, 2)]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ 1. keypoint-count edges
SINGLE = [("s", K) for K in KS] + [("b", 1), ("b", 144)]


@pytest.mark.parametrize("size,K", SINGLE)
def test_head_stages_and_decode_at_keypoint_edges(size, K):
    """last norm, deconv 1, deconv 2 and the heatmaps against fp64 at 1, 5 and max_batch crops, and the decode of the
    engine's own maps against O.decode_maps(wrap="crop"): argmax and scores bit-exact, coordinates within 5e-3 px per
    heatmap pixel of crop size."""
    sd, m = _single(size, K)
    for n in (1, 5, m.max_batch):
        x, org = _crops(n, 100 * K + n)
        chk = Checks(f"vit-{size} K={K} {n} crops")
        with torch.no_grad():
            _check_tail(m, sd, x, chk)
        chk.done()
        kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
        org_np = org.cpu().numpy()
        okp, oidx = O.decode_maps(hm.cpu().numpy(), org_np, wrap="crop")
        assert np.array_equal(idx.cpu().numpy(), oidx)
        kp = kp.cpu().numpy()
        assert np.array_equal(kp[..., 2], okp[..., 2])
        vis = okp[..., 2] > 0.3
        if vis.any():
            assert np.abs(kp - okp)[vis].max() < 5e-3 * max(1.0, org_np.max() / 48.0)


def _ulp_sensitive(maps, org, wrap):
    """[N,K] mask of the keypoints whose refined coordinates move beyond the tolerance below when every log of the oracle's
    decode is off by 2 ulps: a max <= 0 map after a nearly flat one gives a nearly singular Hessian, where logf and np.log
    (which may differ by an ulp) can give answers pixels apart.  Those coordinates are not compared; argmax and score are."""
    base, _ = O.decode_maps(maps, org, wrap=wrap)
    out = np.zeros(base.shape[:2], bool)
    log = np.log
    try:
        for e in (2.0 ** -22, -2.0 ** -22):
            np.log = lambda v, e=e: log(v) * np.float32(1 + e)
            kp, _ = O.decode_maps(maps, org, wrap=wrap)
            out |= (np.abs(kp[..., :2] - base[..., :2]) > 2e-3 + 2e-3 * np.abs(base[..., :2])).any(-1)
    finally:
        np.log = log
    return out


def _assert_decode(kp, idx, maps, ref, K, what, sensitive):
    """test_gpu_kernels' criteria against a reference decode: argmax and scores bit-exact, real peaks within 2e-3 px, the
    other maps' coordinates relatively unless `sensitive` (_ulp_sensitive)"""
    N = maps.shape[0]
    assert np.array_equal(idx, np.argmax(maps.reshape(N, K, -1), -1)), what
    assert np.array_equal(kp[..., 2], ref[..., 2]), what
    err = np.abs(kp[..., :2] - ref[..., :2])
    well = np.isin((np.arange(N * K) % 10).reshape(N, K), [0, 1, 2, 3, 5, 7])
    assert not (well & sensitive).any() and sensitive.sum() <= max(2, N * K // 20), what
    print(f"{what}: {int(sensitive.sum())} of {N * K} coordinates ill-posed at the ulp level, not compared")
    assert err[well].max() < 2e-3, what
    rest = ~well & ~sensitive
    assert np.all(err[rest] <= 2e-3 + 2e-3 * np.abs(ref[..., :2][rest])), what


@pytest.mark.parametrize("K", KS)
def test_decode_kernel_at_keypoint_edges(golden_dir, K):
    """vpb_decode (wrap_batch 0 and 1) and vpb_decode_frame on 12 crops of synthetic maps with every sentinel kind, against
    the reference's per-crop postprocess and its batched call; at K = 1 the batched reference raises, so wrap_batch = 1 is
    checked against O.decode_maps(wrap="batch"), the formula with its intended shape (the sentinel reads the previous crop)."""
    L = _lib()
    g = np.load(os.path.join(golden_dir, "decode_k_edges.npz"))
    maps, org = O.make_decode_maps(DEC_N, K, seed_of(K)), org_of(K)
    offs = np.random.RandomState(K).randint(-300, 900, size=(DEC_N, 2)).astype(np.int32)
    hm, org_d, offs_d = (torch.from_numpy(a).to(_dev()) for a in (maps, org, offs))
    kp = torch.full((DEC_N, K, 3), float("nan"), device=_dev())
    idx = torch.full((DEC_N, K), IDX_SENTINEL, dtype=torch.int32, device=_dev())
    kf, idf = torch.empty_like(kp), torch.empty_like(idx)
    for wrap in (0, 1):
        L.check(L.lib().vpb_decode(C.c_void_p(hm.data_ptr()), DEC_N, K, C.c_void_p(org_d.data_ptr()), C.c_void_p(kp.data_ptr()),
                                   C.c_void_p(idx.data_ptr()), wrap, _stream()))
        L.check(L.lib().vpb_decode_frame(C.c_void_p(hm.data_ptr()), DEC_N, K, C.c_void_p(org_d.data_ptr()), C.c_void_p(offs_d.data_ptr()),
                                         C.c_void_p(kf.data_ptr()), C.c_void_p(idf.data_ptr()), wrap, _stream()))
        torch.cuda.synchronize()
        k_np, i_np = kp.cpu().numpy(), idx.cpu().numpy()
        if wrap == 0:
            ref = g[f"crop_{K}_kpts"]
        elif K == 1:
            assert int(g["batch_1_raises"]) == 1
            ref = O.decode_maps(maps, org, wrap="batch")[0]
            assert not np.array_equal(ref, O.decode_maps(maps, org, wrap="crop")[0])
        else:
            ref = g[f"batch_{K}_kpts"]
        _assert_decode(k_np, i_np, maps, ref, K, f"K={K} wrap_batch={wrap}", _ulp_sensitive(maps, org, "batch" if wrap else "crop"))
        assert np.array_equal(idf.cpu().numpy(), i_np)
        assert np.array_equal(kf.cpu().numpy().view(np.uint32), P.to_frame_coords(k_np, offs).view(np.uint32))


def _decode_modes(hm, n, k, mode, cs, kernel=11):
    L = _lib()
    kp = torch.full((n, k, 3), float("nan"), device=_dev())
    idx = torch.full((n, k), IDX_SENTINEL, dtype=torch.int32, device=_dev())
    L.check(L.lib().vpb_decode_modes_ex(C.c_void_p(hm.data_ptr()), n, k, mode, kernel, float(np.float32(0.0546875 * 64)),
                                        C.c_void_p(cs.data_ptr()), None, C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), _stream()))
    torch.cuda.synchronize()
    kp = kp.cpu().numpy()
    return np.ascontiguousarray(kp[..., 1::-1]), kp[..., 2:3].copy(), idx.cpu().numpy()


@pytest.mark.parametrize("K", MODE_KS)
def test_decode_modes_at_keypoint_edges(golden_dir, K):
    """vpb_decode_modes modes 0-4 on 12 crops against the reference's batched outputs; mode 4 at K = 1 (where the reference
    raises) against decode_modes_oracle, i.e. O.decode_maps(wrap="batch").  At K = 1 also mode 5 (CombinedTarget) per crop
    against the reference and batched against the oracle, and the Python wrapper at N = 1 (which the reference accepts)."""
    from easy_vitpose_b200 import keypoints_from_heatmaps
    g = np.load(os.path.join(golden_dir, "decode_k_edges.npz"))
    maps = O.make_decode_maps(DEC_N, K, seed_of(K))
    c, s = centre_scale_of(K)
    hm = torch.from_numpy(maps).to(_dev())
    cs = torch.from_numpy(np.concatenate([c, s], 1)).to(_dev())
    for pp, udp in COMBOS:
        key = f"k{K}_{pp}_{'udp' if udp else 'std'}"
        preds, maxvals, idx = _decode_modes(hm, DEC_N, K, 4 if udp else {None: 0, "default": 1, "unbiased": 2, "megvii": 3}[pp], cs)
        if int(g[key + "_raises"]):
            assert K == 1 and udp
            ref_p, ref_m, ref_i = M.keypoints_from_heatmaps(maps, c, s, post_process=pp, use_udp=True)
            assert np.array_equal(idx, ref_i), key
        else:
            ref_p, ref_m = g[key + "_preds"], g[key + "_maxvals"]
        assert np.array_equal(maxvals, ref_m, equal_nan=True), key
        assert np.array_equal(np.isnan(preds), np.isnan(ref_p)), key
        if pp in (None, "default", "megvii") and not udp:
            assert np.array_equal(preds, ref_p, equal_nan=True), key
        else:
            assert np.nanmax(np.abs(preds - ref_p)) < 2e-2, key
    if K != 1:
        return
    cmaps = M.make_combined_maps(DEC_N, 1, seed_of(1) + 3)
    chm = torch.from_numpy(cmaps).to(_dev())
    for n in range(DEC_N):
        p1, m1, _ = _decode_modes(chm[n:n + 1], 1, 1, 5, cs[n:n + 1])
        assert np.array_equal(m1[0], g["comb_maxvals"][n], equal_nan=True) and np.array_equal(p1[0], g["comb_preds"][n], equal_nan=True)
    pb, mb, ib = _decode_modes(chm, DEC_N, 1, 5, cs)
    op, om, oi = M.combined_target(cmaps, c, s, 11)
    assert np.array_equal(ib, oi) and np.array_equal(mb, om, equal_nan=True) and np.array_equal(pb, op, equal_nan=True)
    org = org_of(1)
    for n in range(3):
        p1, m1 = keypoints_from_heatmaps(maps[n:n + 1], org[n:n + 1] // 2, org[n:n + 1].astype(np.int64), unbiased=True, use_udp=True)
        ref = g["crop_1_kpts"][n:n + 1]
        assert np.array_equal(m1, ref[..., 2:3])
        assert np.abs(p1 - ref[..., 1::-1]).max() < 2e-3 + 2e-3 * np.abs(ref[..., :2]).max()


@pytest.mark.parametrize("K", [1, 144])
def test_flip_test_at_keypoint_edges(K):
    """K = 1 (permutation [0]) and K = 144 (an involution with fixed points), shift 0 and 1: keypoints, argmax and heatmaps
    bit-identical to forward -> vpb_flip_back -> average -> decode, eager, captured and replayed."""
    from easy_vitpose_b200 import decode_heatmaps
    _, m = _single("s", K)
    pairs = _pairs(K)
    try:
        for shift in (False, True):
            m.set_flip_test(pairs, shift)
            for n in (1, m.max_batch // 2):
                x, org = _crops(n, 60 + n + K)
                hm_r = m.forward_flip_test(x, pairs, shift)
                kp_r, idx_r = decode_heatmaps(hm_r, org)
                for call in range(3):
                    kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
                    assert _same(hm, hm_r) and _same(kp, kp_r) and _same(idx, idx_r), (K, shift, n, call)
    finally:
        m.set_flip_test(None)


@pytest.mark.parametrize("Kk,Npad", [(1, 32), (2, 32), (31, 32), (32, 32), (33, 144), (143, 144), (144, 144)])
def test_gemm_heatmap_nchw_channel_edges(Kk, Npad):
    """vpb_gemm epilogue 4 (the 1x1 conv) with the W rows and bias past Kk non-zero: channels 0..Kk-1 within the fp32
    accumulation bound of the fp64 product, and the sentinel after the last image's Kk channels kept bit for bit (a channel
    >= Kk written would land there or on the next image's channels)."""
    from gpu_util import EPI_F32_NCHW, gemm
    g = torch.Generator().manual_seed(Kk * 1000 + Npad)
    B, pix, K = 2, 3072, 256
    a = (torch.randn(B * pix, K, generator=g) * 0.5).bfloat16().to(_dev())
    w = (torch.randn(Npad, K, generator=g) * 0.05).bfloat16().to(_dev())
    bias = torch.randn(Npad, generator=g).to(_dev())
    valid = B * Kk * pix
    out = torch.full((valid + (Npad - Kk) * pix + 4096,), float("nan"), device=_dev())
    gemm(a, w, bias, out, EPI_F32_NCHW, aux=(Kk, pix, 0, 0))
    ref = (a.double() @ w.double().T + bias.double())[:, :Kk].reshape(B, pix, Kk).permute(0, 2, 1)
    mag = (a.double().abs() @ w.double().abs().T)[:, :Kk].reshape(B, pix, Kk).permute(0, 2, 1)
    bound = K * 2.0 ** -24 * mag + 2.0 ** -23 * ref.abs() + 1e-30
    r = float(((out[:valid].view(B, Kk, pix).double() - ref).abs() / bound).max())
    print(f"nchw Kk={Kk} Npad={Npad}: worst error / bound {r:.3f}")
    assert r <= 1.0
    assert bool((out[valid:].view(torch.int32) == NAN_BITS).all()), "a channel >= n_valid was written"


# ------------------------------------------------------------------------------------------------ 2. multi-head limits
HEADS8 = tuple((f"h{j}", K) for j, K in enumerate((1, 144, 17, 2, 33, 32, 14, 133)))
MULTI = [("s", 0), ("s", 32), ("s", 352), ("b", 736)]
MULTI_BATCH = 128


def _plus(size, P):
    """plus_state_dict at depth 2 (the expert GEMM and the heads are per layer)"""
    key = ("plus", size, P)
    if key not in _cache:
        saved = MH.SIZES[size]
        MH.SIZES[size] = (saved[0], DEPTH, saved[2])
        try:
            _cache[key] = {k: torch.from_numpy(np.asarray(v)) for k, v in MH.plus_state_dict(size, [k for _, k in HEADS8], P, 31).items()}
        finally:
            MH.SIZES[size] = saved
    return _cache[key]


def _engines8(size, P):
    """(8-head engine, [single-head engine per head]) built from split_vitpose_plus; one case kept on the device at a time"""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus
    key = ("multi", size, P)
    if key not in _cache:
        for k in [k for k in _cache if k[0] in ("multi", "single")]:
            del _cache[k]
        torch.cuda.empty_cache()
        plus = _plus(size, P)
        cfg = model_cfg(size, 17)
        cfg["backbone"]["depth"] = DEPTH
        multi = ViTPose(cfg, max_batch=MULTI_BATCH, heads=HEADS8, expert_rows=P)
        multi.load_state_dict(plus)
        multi.to("cuda:0")
        singles = []
        for (name, K), sd in zip(HEADS8, split_vitpose_plus(plus, [n for n, _ in HEADS8], [k for _, k in HEADS8]).values()):
            c = model_cfg(size, K)
            c["backbone"]["depth"] = DEPTH
            m = ViTPose(c, max_batch=MULTI_BATCH)
            m.load_state_dict(sd)
            singles.append(m.to("cuda:0"))
        _cache[key] = (multi, singles)
    return _cache[key]


def _sentinels(n, Km, maps=True):
    kp = torch.full((n, Km, 3), float("nan"), device=_dev())
    idx = torch.full((n, Km), IDX_SENTINEL, dtype=torch.int32, device=_dev())
    hm = torch.full((n, Km, 64, 48), float("nan"), device=_dev()) if maps else None
    return kp, idx, hm


def _expected_crops(singles, x, org, heads, Km):
    """each head's crops in one single-head infer_crops call, rows 0..K_j-1 of the sentinel-filled outputs"""
    kp, idx, hm = _sentinels(x.shape[0], Km)
    heads = torch.as_tensor(heads, device=_dev())
    for j, m in enumerate(singles):
        sel = torch.nonzero(heads == j).flatten()
        if sel.numel():
            k, i, h = m.infer_crops(x.index_select(0, sel), org.index_select(0, sel), return_heatmaps=True)
            K = m.num_keypoints
            kp[sel, :K], idx[sel, :K], hm[sel, :K] = k, i, h
    torch.cuda.synchronize()
    return kp, idx, hm


def _infer_heads(multi, x, org, segs, st):
    L = _lib()
    kp, idx, hm = _sentinels(x.shape[0], multi.num_keypoints_max)
    arr = (L.VpbSegment * len(segs))(*[L.VpbSegment(h, c) for h, c in segs])
    torch.cuda.synchronize()
    L.check(L.lib().vpb_infer_heads(multi._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, len(segs),
                                    C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()),
                                    C.c_void_p(st.cuda_stream)))
    st.synchronize()
    return kp, idx, hm


def _segment_layouts(limit):
    """64 one-crop segments cycling over the 8 heads; 64 segments of run lengths 1, 2, 3, 1, ... (at most `limit` crops)"""
    out = [[(j % 8, 1) for j in range(64)]]
    runs = [(j % 8 if j % 16 < 8 else 7 - j % 8, (1, 2, 3, 1)[j % 4]) for j in range(64)]
    if sum(c for _, c in runs) <= limit:
        out.append(runs)
    return out


def _check_heads_call(multi, singles, segs, seed, what):
    heads = [h for h, c in segs for _ in range(c)]
    x, org = _crops(len(heads), seed)
    want = _expected_crops(singles, x, org, heads, multi.num_keypoints_max)
    st = torch.cuda.Stream()
    for rep in range(3):                                   # eager (first use), graph capture, graph replay
        got = _infer_heads(multi, x, org, segs, st)
        for g_, w_, name in zip(got, want, ("keypoints", "argmax", "heatmaps")):
            assert _same(g_, w_), f"{what} rep {rep}: {name} differ (rows < K_j, or the sentinel at or beyond K_j)"


@pytest.mark.parametrize("size,P", MULTI)
def test_infer_heads_64_segments_bit_identical(size, P):
    """vpb_infer_heads with 64 segments over 8 heads (K = 1 .. 144) on max_batch 128: bit-identical to the single-head
    engines, and rows / maps at or beyond K_j still hold the caller's NaN / 0x7fffffff."""
    multi, singles = _engines8(size, P)
    for i, segs in enumerate(_segment_layouts(MULTI_BATCH)):
        assert len(segs) == 64
        _check_heads_call(multi, singles, segs, 700 + i, f"vit-{size} P={P} layout {i}")
    L = _lib()
    x, org = _crops(65, 5)
    arr = (L.VpbSegment * 65)(*[L.VpbSegment(j % 8, 1) for j in range(65)])
    kp = torch.empty((65, multi.num_keypoints_max, 3), device=_dev())
    assert L.lib().vpb_infer_heads(multi._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, 65,
                                   C.c_void_p(kp.data_ptr()), None, None, _stream()) == 1          # VPB_MAX_SEGMENTS + 1


@pytest.mark.parametrize("size,P", MULTI)
@pytest.mark.parametrize("shift", [False, True])
def test_flip_heads_128_expert_segments(size, P, shift):
    """vpb_set_flip_test_heads, 64 one-crop segments on max_batch 128: the crops and their mirror images make 128 expert
    segments, the whole expert table.  Bit-identical to each head's single-head engine with set_flip_test."""
    multi, singles = _engines8(size, P)
    try:
        multi.set_flip_test_heads([_pairs(K) for _, K in HEADS8], shift)
        for m, (_, K) in zip(singles, HEADS8):
            m.set_flip_test(_pairs(K), shift)
        segs = _segment_layouts(MULTI_BATCH // 2)[0]
        _check_heads_call(multi, singles, segs, 800 + int(shift), f"vit-{size} P={P} flip shift {int(shift)}")
    finally:
        multi.set_flip_test_heads(None)
        for m in singles:
            m.set_flip_test(None)


def _frame_entries(seed):
    """64 frame entries over 4 frames, heads cycling 0..7 (adjacent entries never share a head: 64 segments); head 0 (K = 1)
    entries hold 2 boxes, the others 1 or 2.  -> frames, [(frame, head, xywh boxes)]"""
    rs = np.random.RandomState(seed)
    frames = [P.make_frame(h, w, seed + j) for j, (h, w) in enumerate(((480, 640), (720, 1280), (300, 200), (256, 192)))]
    ents = []
    for e in range(64):
        f, h = frames[e % 4], e % 8
        n = 2 if h == 0 else 1 + e % 2
        x0, y0 = rs.randint(0, f.shape[1] - 40, n), rs.randint(0, f.shape[0] - 40, n)
        ents.append((e % 4, h, np.stack([x0, y0, rs.randint(20, 200, n), rs.randint(20, 200, n)], 1).astype(np.float64)))
    return frames, ents


def _frame_table(dfr, ents):
    L = _lib()
    return (L.VpbFrame * len(ents))(*[L.VpbFrame(dfr[f].data_ptr(), dfr[f].shape[0], dfr[f].shape[1], dfr[f].stride(0), len(b))
                                      for f, _, b in ents])


@pytest.mark.parametrize("size,P", MULTI)
def test_frames_and_affine_heads_full_tables(size, P):
    """vpb_infer_frames_heads and vpb_infer_affine_heads with 64 frame entries of alternating heads (a full frame table and
    a full segment table in one call), eager, captured and replayed.  Frames: bit-identical to per-head vpb_infer_frames.
    Affine: every segment bit-identical to the single-head vpb_infer_affine on that segment's boxes; the 2-box segments of
    the K = 1 head are the case the reference's keypoints_from_heatmaps cannot run, and there the single-head engine is
    held to decode_modes_oracle (O.decode_maps(wrap="batch")) on the maps of the same crops."""
    from easy_vitpose_b200 import topdown_args
    L = _lib()
    multi, singles = _engines8(size, P)
    frames, ents = _frame_entries(17)
    dfr = [torch.from_numpy(f).to(_dev()) for f in frames]
    farr = _frame_table(dfr, ents)
    ha = np.array([h for _, h, _ in ents], np.int32)
    n, Km = sum(len(b) for _, _, b in ents), multi.num_keypoints_max
    assert n <= MULTI_BATCH
    st = torch.cuda.Stream()
    # frames
    xyxy = [np.concatenate([b[:, :2], b[:, :2] + b[:, 2:]], 1).round().astype(np.int32) for _, _, b in ents]
    bb = torch.from_numpy(np.concatenate(xyxy)).to(_dev())
    want_k, want_i, _ = _sentinels(n, Km, maps=False)
    starts = np.cumsum([0] + [len(b) for b in xyxy])
    for j, m in enumerate(singles):
        sel = [e for e, (_, h, _) in enumerate(ents) if h == j]
        k, i = m.infer_frames([dfr[ents[e][0]] for e in sel], [xyxy[e] for e in sel])
        for e, ke, ie in zip(sel, k, i):
            want_k[starts[e]:starts[e + 1], :m.num_keypoints], want_i[starts[e]:starts[e + 1], :m.num_keypoints] = ke, ie
    for rep in range(3):
        kp, idx, _ = _sentinels(n, Km, maps=False)
        torch.cuda.synchronize()
        L.check(L.lib().vpb_infer_frames_heads(multi._handle, farr, len(ents), ha.ctypes.data_as(C.c_void_p), C.c_void_p(bb.data_ptr()),
                                               C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(st.cuda_stream)))
        st.synchronize()
        assert _same(kp, want_k) and _same(idx, want_i), f"frames rep {rep}"
    # affine
    args = [topdown_args(b, 1.25, True) for _, _, b in ents]
    Mt = torch.from_numpy(np.concatenate([a[0].reshape(-1, 6) for a in args])).to(_dev())
    CS = torch.from_numpy(np.concatenate([np.concatenate([a[1], a[2]], 1) for a in args]).astype(np.float32)).to(_dev())
    want_k, want_i, _ = _sentinels(n, Km, maps=False)
    for e, ((f, h, _), a) in enumerate(zip(ents, args)):                  # one single-head call per segment
        m = singles[h]
        k, i = m.infer_affine([dfr[f]], [a[0]], [a[1]], [a[2]])
        want_k[starts[e]:starts[e + 1], :m.num_keypoints], want_i[starts[e]:starts[e + 1], :m.num_keypoints] = k[0], i[0]
        if h == 0:                                                          # K = 1, 2 boxes: one decode over both crops
            hm = m.forward(m.preprocess_affine([dfr[f]], [a[0]])).cpu().numpy()
            op, om, oi = M.keypoints_from_heatmaps(hm, a[1], a[2], use_udp=True)
            k0 = k[0].cpu().numpy()
            assert np.array_equal(i[0].cpu().numpy(), oi) and np.array_equal(k0[..., 2:3], om)
            assert np.abs(k0[..., 1::-1] - op).max() < 2e-2
    for rep in range(3):
        kp, idx, _ = _sentinels(n, Km, maps=False)
        torch.cuda.synchronize()
        L.check(L.lib().vpb_infer_affine_heads(multi._handle, farr, len(ents), ha.ctypes.data_as(C.c_void_p), C.c_void_p(Mt.data_ptr()),
                                               C.c_void_p(CS.data_ptr()), C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()),
                                               C.c_void_p(st.cuda_stream)))
        st.synchronize()
        assert _same(kp, want_k) and _same(idx, want_i), f"affine rep {rep}"


# ------------------------------------------------------------------------------------------------ 3. batches past 64
@pytest.mark.parametrize("size", ["s", "b"])
def test_batch_256_invariant_and_against_fp64(size):
    """max_batch 256: a 256-crop infer_crops (with heatmaps) bit-identical to four 64-crop calls and to 256 one-crop calls;
    block 0 and the head against fp64 at 256 crops; a 128-crop flip-test call bit-identical to its composition."""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, decode_heatmaps
    for k in [k for k in _cache if k[0] in ("multi", "single")]:
        del _cache[k]
    torch.cuda.empty_cache()
    sd, m = _single(size, 17, max_batch=256)
    x, org = _crops(256, 256)
    full = m.infer_crops(x, org, return_heatmaps=True)
    for q in range(4):
        part = m.infer_crops(x[64 * q:64 * (q + 1)], org[64 * q:64 * (q + 1)], return_heatmaps=True)
        assert all(_same(a[64 * q:64 * (q + 1)], b) for a, b in zip(full, part)), f"64-crop call {q} differs"
    for i in range(256):
        one = m.infer_crops(x[i:i + 1], org[i:i + 1], return_heatmaps=True)
        assert all(_same(a[i:i + 1], b) for a, b in zip(full, one)), f"crop {i} alone differs"
    chk = Checks(f"vit-{size} 256 crops")
    with torch.no_grad():
        _check_block0_and_head(m, sd, DIMS[size][1], x, chk)
        _check_tail(m, sd, x, chk)
    chk.done()
    pairs = [tuple(int(v) for v in p) for p in COCO_FLIP_PAIRS]
    try:
        m.set_flip_test(pairs, True)
        xf, of = x[:128].contiguous(), org[:128].contiguous()
        hm_r = m.forward_flip_test(xf, pairs, True)
        kp_r, idx_r = decode_heatmaps(hm_r, of)
        for call in range(3):
            kp, idx, hm = m.infer_crops(xf, of, return_heatmaps=True)
            assert _same(hm, hm_r) and _same(kp, kp_r) and _same(idx, idx_r), f"flip call {call}"
    finally:
        m.set_flip_test(None)
