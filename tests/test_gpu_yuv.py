"""-m gpu: the YUV frame calls for every 8-bit layout (ViTPose.infer_frames_yuv / _host / submit_frames_yuv_host,
infer_affine_yuv / _host, infer_frames_heads_yuv / _host, infer_affine_heads_yuv / _host; vpb_*_yuv).  The reference for
every case is the engine's own RGB call on oracle.yuv_oracle.yuv_to_rgb(frame), which the RGB tests pin against the
reference project, or for the multi-head calls a single-head engine per head on those RGB frames: the YUV gathers convert
each tap and then run the RGB arithmetic, so the patch rows, keypoints and argmax indices must be BIT-IDENTICAL."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O
from oracle.multi_head import plus_state_dict
from oracle.yuv_oracle import LAYOUTS, rgb_to_yuv, yuv_to_rgb

pytestmark = pytest.mark.gpu

PACKED = ("yuyv", "uyvy")
FORMATS = [(m, f) for m in ("bt601", "bt709") for f in (False, True)]
_engines = {}


def _engine(size="s", max_batch=64):
    from easy_vitpose_b200 import ViTPose, model_cfg
    key = (size, max_batch)
    if key not in _engines:
        cfg = model_cfg(size, 17)
        D, depth = cfg["backbone"]["embed_dim"], cfg["backbone"]["depth"]
        m = ViTPose(cfg, max_batch=max_batch)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, 17, 101, peaky=0.1, bumps=True).items()})
        _engines[key] = m.to("cuda:0")
    return _engines[key]


def _random(layout, h, w, rs):
    return rs.randint(0, 256, size=(h, w, 2) if layout in PACKED else (3 * h // 2, w), dtype=np.uint8)


def _hd_boxes(n, seed=9):
    """1080p boxes: tiny ones, large ones, boxes clipped at every border (none empty after padding and clipping)."""
    rs = np.random.RandomState(seed)
    boxes = [[0, 0, 1920, 1080], [1915.5, 1070.5, 1990.0, 1100.0], [100.5, 200.5, 101.5, 201.5], [-30.5, 500.2, 60.7, 700.5],
             [1850.2, -40.5, 1930.7, 60.1]]
    for i in range(n - len(boxes)):
        w, h = (rs.randint(1, 60), rs.randint(1, 60)) if i % 4 == 0 else (rs.randint(20, 900), rs.randint(20, 1000))
        x0, y0 = rs.randint(-10, 1900), rs.randint(-10, 1060)
        boxes.append([x0 + rs.rand(), y0 + rs.rand(), x0 + w + rs.rand(), y0 + h + rs.rand()])
    return np.array(boxes[:n], np.float64)


def _gradient(h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([(xx * 255) // w, (yy * 255) // h, 255 - ((xx + yy) * 255) // (w + h)], -1).astype(np.uint8)


def _case(golden_dir, layout, matrix, full, n_hd=20, seed=17):
    """frame_a (random planes), a frame without boxes, frame_b (the golden frame converted) and a 1080p gradient converted, in
    the layout's stacked / packed form (odd sizes cropped to even)."""
    frames, boxes = [], []
    rs = np.random.RandomState(seed)
    for name in ("frame_a", "frame_b"):
        g = np.load(os.path.join(golden_dir, f"{name}.npz"))
        fh, fw, fseed = (int(v) for v in g["meta"][:3])
        rows = g["rows"].astype(np.float64)
        f = P.make_frame(fh, fw, fseed)[: fh & ~1, : fw & ~1]
        frames.append(_random(layout, f.shape[0], f.shape[1], rs) if name == "frame_a" else rgb_to_yuv(f, layout, matrix, full))
        boxes.append(rows[rows[:, 4] > 0.35, :4].round().astype(np.int32))
        if name == "frame_a":
            frames.append(_random(layout, 50, 70, rs))
            boxes.append(np.zeros((0, 4), np.int32))
    frames.append(rgb_to_yuv(_gradient(1080, 1920), layout, matrix, full))
    boxes.append(_hd_boxes(n_hd))
    return frames, boxes


def _cat(xs):
    return np.concatenate([x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in xs])


def _rows(m, n):
    return m.read_buffer("patch_rows", (n * 192, 768), "bf16").view(torch.int16).numpy().copy()


def _rgb(frames, layout, matrix, full):
    return [yuv_to_rgb(f, layout, matrix, full) for f in frames]


def _cuda(frames):
    return [torch.from_numpy(f).cuda() for f in frames]


def _affine_case(layout, matrix, full, n_per_frame=(5, 0, 4, 9), seed=3):
    """Frames (random planes and converted images) with boxes overhanging them; the matrices of topdown_args."""
    from easy_vitpose_b200 import topdown_args
    rs = np.random.RandomState(seed)
    sizes = [(240, 320), (64, 80), (480, 376), (1080, 1920)]
    frames, mats, cs, ss = [], [], [], []
    for j, ((h, w), k) in enumerate(zip(sizes, n_per_frame)):
        frames.append(_random(layout, h, w, rs) if j % 2 else rgb_to_yuv(P.make_frame(h, w, seed + j), layout, matrix, full))
        bw, bh = rs.uniform(8, w * 0.9, k), rs.uniform(8, h * 0.9, k)
        M, c, s = topdown_args(np.stack([rs.uniform(-0.3 * w, w) - bw / 2, rs.uniform(-0.3 * h, h) - bh / 2, bw, bh], 1))
        mats.append(np.asarray(M).reshape(-1, 2, 3)); cs.append(c); ss.append(s)
    return frames, mats, cs, ss


def _same(got, want):
    (gk, gi), (wk, wi) = got, want
    assert np.array_equal(_cat(gk), _cat(wk)) and np.array_equal(_cat(gi), _cat(wi))


@pytest.mark.parametrize("matrix,full", FORMATS)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_every_call_bit_identical_to_the_rgb_call(golden_dir, layout, matrix, full):
    """Device, host and pipelined frame calls and device and host affine calls, against the RGB calls on the converted
    frames; the patch rows too."""
    m = _engine("s")
    fmt = dict(layout=layout, matrix=matrix, full_range=full)
    frames, boxes = _case(golden_dir, layout, matrix, full)
    n = sum(len(b) for b in boxes)
    assert n <= m.batch_limit                                               # one call: the patch rows are all of it
    rgb = _rgb(frames, layout, matrix, full)
    want = m.infer_frames(_cuda(rgb), boxes)
    rows_r = _rows(m, n)
    got = m.infer_frames_yuv(_cuda(frames), boxes, **fmt)
    assert [len(k) for k in got[0]] == [len(b) for b in boxes]
    assert np.array_equal(_rows(m, n), rows_r)
    _same(got, want)
    _same(m.infer_frames_yuv_host(frames, boxes, **fmt), want)
    assert m.frame_status() == 0
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    ib = [np.ascontiguousarray(np.asarray(b).round().astype(np.int32)) for b in boxes]
    kp, idx = pin(np.empty((n, 17, 3), np.float32)), pin(np.empty((n, 17), np.int32))
    m.submit_frames_yuv_host([pin(f) for f in frames], ib, kp, idx, 1, **fmt)
    m.wait_host(1)
    assert np.array_equal(kp, _cat(want[0])) and np.array_equal(idx, _cat(want[1]))
    af, mats, cs, ss = _affine_case(layout, matrix, full)
    na = sum(len(x) for x in mats)
    want = m.infer_affine(_cuda(_rgb(af, layout, matrix, full)), mats, cs, ss, check=True)
    rows_r = _rows(m, na)
    _same(m.infer_affine_yuv(_cuda(af), mats, cs, ss, check=True, **fmt), want)
    assert np.array_equal(_rows(m, na), rows_r)
    _same(m.infer_affine_yuv_host(af, mats, cs, ss, **fmt), want)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_pipelined_slots_alternate(golden_dir, layout):
    m = _engine("s")
    fmt = dict(layout=layout, matrix="bt709", full_range=layout in ("i420", "yuyv"))
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    sets = []
    for i in range(4):
        frames, boxes = _case(golden_dir, layout, "bt709", fmt["full_range"], n_hd=6 + i, seed=30 + i)
        bs = [np.ascontiguousarray(np.asarray(b)[: len(b) - (i % 3)].round().astype(np.int32)) for b in boxes]
        sets.append(([pin(f) for f in frames], bs))
    want = [m.infer_frames_yuv_host(fs, bs, **fmt) for fs, bs in sets]
    outs = [(pin(np.empty((sum(len(b) for b in bs), 17, 3), np.float32)), pin(np.empty((sum(len(b) for b in bs), 17), np.int32)))
            for _, bs in sets]
    m.submit_frames_yuv_host(*sets[0], *outs[0], 0, **fmt)
    for i in range(1, 4):
        m.submit_frames_yuv_host(*sets[i], *outs[i], i % 2, **fmt)
        m.wait_host((i - 1) % 2)
    m.wait_host(1)
    for (wk, wi), (k, i) in zip(want, outs):
        assert np.array_equal(_cat(wk), k) and np.array_equal(_cat(wi), i)


@pytest.mark.parametrize("matrix,full", [("bt601", False), ("bt709", True)])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_flip_test(golden_dir, layout, matrix, full):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, B200PoseBackend, topdown_args
    m = _engine("s")
    fmt = dict(layout=layout, matrix=matrix, full_range=full)
    frames, boxes = _case(golden_dir, layout, matrix, full, n_hd=12)
    m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS], True)
    try:
        assert sum(len(b) for b in boxes) <= m.batch_limit
        want = m.infer_frames(_cuda(_rgb(frames, layout, matrix, full)), boxes)
        _same(m.infer_frames_yuv(_cuda(frames), boxes, **fmt), want)
        _same(m.infer_frames_yuv_host(frames, boxes, **fmt), want)
        be = B200PoseBackend(m)
        assert np.array_equal(_cat(be.inference_frames_yuv(frames, boxes, **fmt)), _cat(want[0]))
        af, mats, cs, ss = _affine_case(layout, matrix, full, (3, 2, 4, 6), seed=5)
        want = m.infer_affine(_cuda(_rgb(af, layout, matrix, full)), mats, cs, ss)
        _same(m.infer_affine_yuv(_cuda(af), mats, cs, ss, **fmt), want)
        xywh = [np.array([[10.5, 20.0, 120.0, 200.0], [-30.0, 40.0, 90.0, 150.0]]), np.array([[5.0, 5.0, 40.0, 50.0]])]
        tf = [af[0], af[2]]
        want = m.infer_affine_host(_rgb(tf, layout, matrix, full), *[[topdown_args(b)[i] for b in xywh] for i in range(3)])[0]
        assert np.array_equal(_cat(be.inference_topdown_yuv(tf, xywh, **fmt)), _cat(want))
    finally:
        m.set_flip_test(None)


def _wide(a, pad_left, pad_right, rs):
    """`a` (2-D) as a column slice of a wider random surface, at pitch a.shape[1] + pad_left + pad_right: (host view, device view)."""
    t = torch.from_numpy(rs.randint(0, 256, size=(a.shape[0], a.shape[1] + pad_left + pad_right), dtype=np.uint8))
    t[:, pad_left:pad_left + a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a))
    cols = slice(pad_left, pad_left + a.shape[1])
    return t.numpy()[:, cols], t.cuda()[:, cols]


@pytest.mark.parametrize("layout", LAYOUTS)
def test_separate_planes_at_odd_pitches(golden_dir, layout):
    """Planes in separate allocations and as column slices of wider surfaces at odd pitches (U and V of one pitch), on the
    device and on the host (the host forms stage them packed)."""
    from easy_vitpose_b200.model import yuv_planes
    m = _engine("s")
    frames, boxes = _case(golden_dir, layout, "bt601", True)
    f, b = frames[2], boxes[2]
    want = m.infer_frames(_cuda([yuv_to_rgb(f, layout, "bt601", True)]), [b])
    rs = np.random.RandomState(8)
    planes = [np.asarray(p) for p in yuv_planes(f, layout)[0]]
    if layout in PACKED:
        hw, dw = _wide(planes[0], 21, 17, rs)                               # [H, 2W] at pitch 2W + 38, and as [H, W, 2]
        forms = [(hw, dw), (hw.reshape(hw.shape[0], -1, 2), dw.reshape(dw.shape[0], -1, 2))]
    else:
        if layout in ("nv12", "nv21"):
            wide = [_wide(planes[0], 21, 17, rs), _wide(planes[1], 10, 55, rs)]
            packed = (planes[0].copy(), planes[1].copy())
        else:
            u, v = (planes[1], planes[2]) if layout == "i420" else (planes[2], planes[1])
            cw = _wide(np.concatenate([u, v], 1), 3, 6, rs)                  # U and V side by side in one surface: one pitch
            k = u.shape[1]
            wide = [_wide(planes[0], 21, 17, rs), (cw[0][:, :k], cw[1][:, :k]), (cw[0][:, k:], cw[1][:, k:])]
            packed = (planes[0].copy(), u.copy(), v.copy())
        forms = [(tuple(h for h, _ in wide), tuple(d for _, d in wide)), (packed, tuple(torch.from_numpy(p).cuda() for p in packed))]
    for host, dev in forms:
        _same(m.infer_frames_yuv([dev], [b], layout=layout, full_range=True), want)
        _same(m.infer_frames_yuv_host([host], [b], layout=layout, full_range=True), want)
    if layout in ("i420", "yv12"):                                         # U and V at different pitches: copied packed
        (hy, hu, _), (dy, du, _) = forms[0]
        hv, dv = _wide(v, 1, 1, rs)
        _same(m.infer_frames_yuv([(dy, du, dv)], [b], layout=layout, full_range=True), want)
        _same(m.infer_frames_yuv_host([(hy, hu, hv)], [b], layout=layout, full_range=True), want)


@pytest.mark.parametrize("layout", ["i420", "nv21", "uyvy"])
def test_chunking_over_the_batch_and_frame_limits(layout):
    """70 one-box frames (the first call is closed by the 64-frame limit), then a 1080p frame with 150 boxes (more than
    max_batch): three engine calls, equal to the RGB calls on the converted frames."""
    from easy_vitpose_b200 import B200PoseBackend
    m = _engine("s", max_batch=128)
    rs = np.random.RandomState(3)
    frames, boxes = [], []
    for j in range(70):
        h, w = 2 * int(rs.randint(20, 150)), 2 * int(rs.randint(20, 150))
        frames.append(_random(layout, h, w, rs))
        x0, y0 = int(rs.randint(-10, w - 5)), int(rs.randint(-10, h - 5))
        boxes.append(np.array([[x0, y0, x0 + int(rs.randint(5, 200)), y0 + int(rs.randint(5, 200))]], np.int32))
    frames.append(rgb_to_yuv(_gradient(1080, 1920), layout))
    boxes.append(_hd_boxes(150, seed=4))
    rgb = _rgb(frames, layout, "bt601", False)
    want = m.infer_frames(_cuda(rgb), boxes)
    _same(m.infer_frames_yuv(_cuda(frames), boxes, layout=layout), want)
    _same(m.infer_frames_yuv_host(frames, boxes, layout=layout), want)
    assert np.array_equal(_cat(B200PoseBackend(m).inference_frames_yuv(frames, boxes, layout=layout)), _cat(want[0]))
    mats = [np.tile(np.array([[[0.5, 0.0, 1.0], [0.0, 0.5, 2.0]]]), (len(b), 1, 1)) for b in boxes]
    cs = [np.tile([[96.0, 128.0]], (len(b), 1)) for b in boxes]
    ss = [np.tile([[192.0, 256.0]], (len(b), 1)) for b in boxes]
    _same(m.infer_affine_yuv_host(frames, mats, cs, ss, layout=layout), m.infer_affine_host(rgb, mats, cs, ss))


def test_nv12_through_the_yuv_calls_equals_the_nv12_calls(golden_dir):
    m = _engine("s")
    for matrix in ("bt601", "bt709"):
        frames, boxes = _case(golden_dir, "nv12", matrix, False)
        d = _cuda(frames)
        _same(m.infer_frames_yuv(d, boxes, layout="nv12", matrix=matrix), m.infer_frames_nv12(d, boxes, matrix))
        _same(m.infer_frames_yuv_host(frames, boxes, layout="nv12", matrix=matrix), m.infer_frames_nv12_host(frames, boxes, matrix))
        af, mats, cs, ss = _affine_case("nv12", matrix, False)
        _same(m.infer_affine_yuv(_cuda(af), mats, cs, ss, layout="nv12", matrix=matrix), m.infer_affine_nv12(_cuda(af), mats, cs, ss, matrix))
        _same(m.infer_affine_yuv_host(af, mats, cs, ss, layout="nv12", matrix=matrix), m.infer_affine_nv12_host(af, mats, cs, ss, matrix))


# ------------------------------------------------------------------------------------------------ multi-head engines
HEADS = (("coco", 17), ("aic", 14), ("ap10k", 17))
_heads_cache = {}


def _head_engines():
    """(ViT-S three-head engine, [single-head engine per head]) loaded from one ViTPose+ checkpoint"""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus
    if not _heads_cache:
        plus = {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("s", [k for _, k in HEADS], 96, 31).items()}
        multi = ViTPose(model_cfg("s", 17), max_batch=32, heads=HEADS, expert_rows=96)
        multi.load_state_dict(plus)
        singles = []
        for (_, K), sd in zip(HEADS, split_vitpose_plus(plus, [n for n, _ in HEADS], [k for _, k in HEADS]).values()):
            s = ViTPose(model_cfg("s", K), max_batch=32)
            s.load_state_dict(sd)
            singles.append(s.to("cuda:0"))
        _heads_cache["e"] = (multi.to("cuda:0"), singles)
    return _heads_cache["e"]


@pytest.mark.parametrize("layout,matrix,full", [("nv12", "bt601", False), ("i420", "bt709", True), ("yv12", "bt601", True),
                                                ("nv21", "bt709", False), ("yuyv", "bt601", False), ("uyvy", "bt709", True)])
def test_mixed_heads_equal_single_head_engines(golden_dir, layout, matrix, full):
    """A mixed-head batch (boxes of all three heads interleaved in every frame) against one single-head engine per head on
    the converted frames: frame calls device and host, affine calls device and host."""
    multi, singles = _head_engines()
    fmt = dict(layout=layout, matrix=matrix, full_range=full)
    frames, boxes = _case(golden_dir, layout, matrix, full, n_hd=8)
    rgb = _cuda(_rgb(frames, layout, matrix, full))
    heads = [np.arange(len(b)) % 3 for b in boxes]
    got_d = multi.infer_frames_heads_yuv(_cuda(frames), boxes, heads, **fmt)
    got_h = multi.infer_frames_heads_yuv_host(frames, boxes, heads, **fmt)
    for j, (s, (_, K)) in enumerate(zip(singles, HEADS)):
        want = s.infer_frames(rgb, [np.asarray(b)[h == j] for b, h in zip(boxes, heads)])
        for kp, idx in (got_d, got_h):
            assert np.array_equal(_cat([np.asarray(k.cpu() if isinstance(k, torch.Tensor) else k)[h == j, :K] for k, h in zip(kp, heads)]),
                                  _cat(want[0]))
            assert np.array_equal(_cat([np.asarray(i.cpu() if isinstance(i, torch.Tensor) else i)[h == j, :K] for i, h in zip(idx, heads)]),
                                  _cat(want[1]))
    af, mats, cs, ss = _affine_case(layout, matrix, full, (4, 0, 3, 5), seed=7)
    ah = [np.arange(len(x)) % 3 for x in mats]
    argb = _cuda(_rgb(af, layout, matrix, full))
    got_d = multi.infer_affine_heads_yuv(_cuda(af), mats, cs, ss, ah, **fmt)
    got_h = multi.infer_affine_heads_yuv_host(af, mats, cs, ss, ah, **fmt)
    for j, (s, (_, K)) in enumerate(zip(singles, HEADS)):
        sel = lambda xs: [np.asarray(x)[h == j] for x, h in zip(xs, ah)]
        want = s.infer_affine(argb, sel(mats), sel(cs), sel(ss))
        for kp, idx in (got_d, got_h):
            assert np.array_equal(_cat([np.asarray(k.cpu() if isinstance(k, torch.Tensor) else k)[h == j, :K] for k, h in zip(kp, ah)]),
                                  _cat(want[0]))
            assert np.array_equal(_cat([np.asarray(i.cpu() if isinstance(i, torch.Tensor) else i)[h == j, :K] for i, h in zip(idx, ah)]),
                                  _cat(want[1]))


def test_mixed_heads_backend_wrappers(golden_dir):
    from easy_vitpose_b200 import B200PoseBackend, topdown_args
    multi, _ = _head_engines()
    frames, boxes = _case(golden_dir, "i420", "bt601", False, n_hd=6)
    heads = [np.arange(len(b)) % 3 for b in boxes]
    be = B200PoseBackend(multi)
    rgb = _rgb(frames, "i420", "bt601", False)
    assert np.array_equal(_cat(be.inference_frames_heads_yuv(frames, boxes, heads)), _cat(multi.infer_frames_heads_host(rgb, boxes, heads)[0]))
    xywh = [np.array([[10.5, 20.0, 120.0, 200.0], [-30.0, 40.0, 90.0, 150.0]]), np.array([[5.0, 5.0, 40.0, 50.0]])]
    tf, hh = [frames[0], frames[2]], [np.array([0, 2]), np.array([1])]
    want = multi.infer_affine_heads_host([rgb[0], rgb[2]], *[[topdown_args(b)[i] for b in xywh] for i in range(3)], hh)[0]
    assert np.array_equal(_cat(be.inference_topdown_heads_yuv(tf, xywh, hh)), _cat(want))


# ------------------------------------------------------------------------------------------------ errors
def test_errors(golden_dir):
    from easy_vitpose_b200 import _lib
    m = _engine("s", max_batch=16)
    frames, boxes = _case(golden_dir, "i420", "bt601", False, n_hd=4)
    bad = [b.copy() for b in boxes]
    bad[2][1] = [500, 500, 520, 540]                                        # entirely outside frame_b
    with pytest.raises(ValueError, match="frame 2 box 1"):
        m.infer_frames_yuv_host(frames, bad)
    m.frame_status()
    d = _cuda(frames)
    m.infer_frames_yuv(d, bad)
    assert m.frame_status() & 1
    with pytest.raises(ValueError):
        m.infer_frames_yuv(d, bad, check=True)
    assert m.frame_status() == 0
    for kw in (dict(layout="nv16"), dict(matrix="bt2020"), dict(layout="p010")):
        with pytest.raises(ValueError):
            m.infer_frames_yuv(d, boxes, **kw)
    with pytest.raises(ValueError):
        m.infer_frames_yuv([torch.zeros((15, 21), dtype=torch.uint8, device="cuda")], [boxes[0]])          # odd width
    with pytest.raises(ValueError):
        m.infer_frames_yuv([torch.zeros((10, 7, 2), dtype=torch.uint8, device="cuda")], [boxes[0]], layout="yuyv")
    with pytest.raises(ValueError):
        m.infer_frames_yuv([(d[0][:10], d[0][10:15, :10], d[0][15:20, :12])], [boxes[0]])                  # mismatched chroma
    with pytest.raises(ValueError):                                         # the pipelined form cannot copy: U, V pitches differ
        u = np.zeros((5, 10), np.uint8)
        m.submit_frames_yuv_host([(np.zeros((10, 20), np.uint8), u, np.zeros((5, 30), np.uint8)[:, :10])], [np.zeros((1, 4), np.int32)],
                                 np.empty((1, 17, 3), np.float32), np.empty((1, 17), np.int32), 0)
    kp, idx = m.infer_frames_yuv(d[1:2], boxes[1:2])                         # no boxes at all: nothing launched
    assert len(kp) == 1 and kp[0].shape == (0, 17, 3)
    # raw ABI: VPB_ERR_ARG
    L = _lib.lib()
    fa = d[0]
    h, w = fa.shape[0] // 3 * 2, fa.shape[1]
    y, u, v = fa.data_ptr(), fa.data_ptr() + h * w, fa.data_ptr() + h * w + (h // 2) * (w // 2)
    bb = torch.zeros((32, 4), dtype=torch.int32, device="cuda")
    bb[:, 2:] = 50
    kp = torch.empty((32, 17, 3), dtype=torch.float32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    F = _lib.VpbFrameYuv

    def call(*fr, layout=2, matrix=0, rng=0):
        arr = (F * len(fr))(*fr)
        return L.vpb_infer_frames_yuv(m._handle, arr, len(arr), layout, matrix, rng, C.c_void_p(bb.data_ptr()), C.c_void_p(kp.data_ptr()),
                                      None, st)

    ok = F((y, u, v), 0, 0, h, w, 3)
    assert call(ok) == 0 and call(ok, matrix=1, rng=1) == 0 and call(ok, layout=3) == 0
    assert call(ok, layout=6) == 1 and call(ok, layout=-1) == 1            # unknown layout
    assert call(ok, matrix=2) == 1 and call(ok, rng=2) == 1 and call(ok, rng=-1) == 1
    assert b"range" in L.vpb_last_error()
    assert call(F((y, u, v), 0, 0, h, w, 17)) == 1                          # over max_batch
    assert call(F((y, u, v), 0, 0, h - 1, w, 3)) == 1                       # odd height in 4:2:0
    assert call(F((y, u, v), 0, 0, h, w - 1, 3)) == 1                       # odd width
    assert call(F((y, u, v), w - 1, 0, h, w, 3)) == 1                       # short y pitch
    assert call(F((y, u, v), 0, w // 2 - 1, h, w, 3)) == 1                  # short chroma pitch
    assert call(F((y, u, None), 0, 0, h, w, 3)) == 1                        # NULL plane the layout uses
    assert call(F((y, None, v), 0, 0, h, w, 3), layout=0) == 1
    assert call(F((y, u, None), 0, 0, h, w, 3), layout=0) == 0              # NV12 uses two planes
    assert call(F((y, u, None), 0, w - 1, h, w, 3), layout=0) == 1          # NV12 chroma rows are w bytes
    assert call(F((y, None, None), 0, 0, h - 1, w // 2, 3), layout=4) == 0  # 4:2:2: any height, one plane
    assert call(F((y, None, None), 2 * (w // 2) - 1, 0, h, w // 2, 3), layout=5) == 1      # short packed pitch
    assert call(F((y, None, None), 0, 0, h, w // 2 - 1 | 1, 3), layout=4) == 1             # odd width in 4:2:2
    assert call(F((None, None, None), 0, 0, h, w, 0), ok) == 0              # no boxes: skipped
    assert call(F((y, u, v), 0, 0, h, w, -1)) == 1
    hp = np.zeros((30, 20), np.uint8)
    assert L.vpb_infer_frames_yuv_host(m._handle, (F * 1)(F((hp.ctypes.data,) * 3, 0, 0, 20, 20, 1)), 1, 2, 5, 0,
                                       bb.cpu().numpy().ctypes.data_as(C.c_void_p), kp.cpu().numpy().ctypes.data_as(C.c_void_p),
                                       None, st) == 1
    assert b"matrix" in L.vpb_last_error()
    M = torch.tensor([[0.5, 0, 1, 0, 0.5, 2]] * 3, dtype=torch.float64, device="cuda")
    CS = torch.tensor([[96.0, 128, 192, 256]] * 3, device="cuda")
    assert L.vpb_infer_affine_yuv(m._handle, (F * 1)(F((y, u, v), 0, 0, h, w - 1, 3)), 1, 2, 0, 0, C.c_void_p(M.data_ptr()),
                                  C.c_void_p(CS.data_ptr()), C.c_void_p(kp.data_ptr()), None, st) == 1
    # affine: a non-finite matrix or a scale <= 0 sets status bit 1 on the device form and raises on the host form
    af, mats, cs, ss = _affine_case("yuyv", "bt601", True, (2, 0, 1, 1), seed=9)
    ss[0] = ss[0].copy(); ss[0][0, 0] = 0.0
    with pytest.raises(ValueError):
        m.infer_affine_yuv_host(af, mats, cs, ss, layout="yuyv", full_range=True)
    dm = [torch.from_numpy(np.asarray(x)).cuda() for x in mats]
    dc = [torch.from_numpy(np.asarray(x, np.float32)).cuda() for x in cs]
    m.infer_affine_yuv(_cuda(af), dm, dc, [torch.from_numpy(np.asarray(x, np.float32)).cuda() for x in ss], layout="yuyv", full_range=True)
    assert m.frame_status() & 2
    dm[3] = dm[3].clone(); dm[3][0, 1, 2] = float("nan")
    ss[0][0, 0] = 1.0
    m.infer_affine_yuv(_cuda(af), dm, dc, [torch.from_numpy(np.asarray(x, np.float32)).cuda() for x in ss], layout="yuyv", full_range=True)
    assert m.frame_status() & 2
    torch.cuda.synchronize()
    assert m.frame_status() == 0
