"""-m gpu: rotated frames (vpb_frame*.rotation; the `rotate` argument of the ViTPose frame methods and the B200PoseBackend
wrappers).  The reference for every case is the engine's own upright call on torch.rot90(stored, rotation // 90, dims=(0, 1))
-- for YUV frames on the rotated RGB conversion (oracle/yuv_oracle.py) -- which is cv2.rotate with the reference's
rotation_map (tests/test_rotation_cpu.py pins the direction).  The rotation only permutes the pixels the gathers read, so
keypoints, argmax indices, the status word and the patch rows must be BIT-IDENTICAL."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O
from oracle.multi_head import plus_state_dict
from oracle.yuv_oracle import LAYOUTS, rgb_to_yuv, yuv_to_rgb

pytestmark = pytest.mark.gpu

ROTATIONS = (0, 90, 180, 270)
_engines = {}


def _engine(max_batch=64):
    from easy_vitpose_b200 import ViTPose, model_cfg
    if max_batch not in _engines:
        cfg = model_cfg("s", 17)
        D, depth = cfg["backbone"]["embed_dim"], cfg["backbone"]["depth"]
        m = ViTPose(cfg, max_batch=max_batch)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, 17, 101, peaky=0.1, bumps=True).items()})
        _engines[max_batch] = m.to("cuda:0")
    return _engines[max_batch]


def _view(stored, rotation):
    """the view of a stored [H, W, ...] array or tensor: torch.rot90 / np.rot90 over the first two axes, made contiguous"""
    if isinstance(stored, torch.Tensor):
        return torch.rot90(stored, rotation // 90, dims=(0, 1)).contiguous()
    return np.ascontiguousarray(np.rot90(stored, rotation // 90, axes=(0, 1)))


def _view_hw(h, w, rotation):
    return (w, h) if rotation in (90, 270) else (h, w)


def _boxes(vh, vw, k, rs):
    """k float boxes in view pixels: some overhang every edge of the view, some are small; none is empty after clipping"""
    out = [[-25.5, -30.2, 0.4 * vw, 0.5 * vh], [0.6 * vw, 0.55 * vh, vw + 40.7, vh + 33.1]]
    while len(out) < k:
        bw, bh = rs.uniform(4, 0.8 * vw), rs.uniform(4, 0.8 * vh)
        x0, y0 = rs.uniform(-0.1 * vw, vw - 2), rs.uniform(-0.1 * vh, vh - 2)
        out.append([x0, y0, x0 + bw, y0 + bh])
    return np.array(out[:k], np.float64).reshape(-1, 4)


def _affine(vh, vw, k, rs):
    """topdown_args matrices / centres / scales of k person boxes in view pixels, some overhanging the view"""
    from easy_vitpose_b200 import topdown_args
    bw, bh = rs.uniform(8, vw * 0.9, k), rs.uniform(8, vh * 0.9, k)
    M, c, s = topdown_args(np.stack([rs.uniform(-0.3 * vw, vw) - bw / 2, rs.uniform(-0.3 * vh, vh) - bh / 2, bw, bh], 1))
    return np.asarray(M).reshape(-1, 2, 3), c, s


def _cat(xs):
    return np.concatenate([x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x) for x in xs])


def _same(got, want):
    (gk, gi), (wk, wi) = got, want
    assert np.array_equal(_cat(gk), _cat(wk)) and np.array_equal(_cat(gi), _cat(wi))


def _rows(m, n):
    return m.read_buffer("patch_rows", (n * 192, 768), "bf16").view(torch.int16).numpy().copy()


def _pin(a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()


# stored (h, w): odd and even, portrait and landscape; frame 1 has no boxes
SIZES = [(237, 311), (48, 70), (81, 64), (1080, 1920)]
COUNTS = [9, 0, 5, 14]


def _rgb_case(rotations, seed=5):
    """stored RGB frames (numpy), per-frame boxes in view pixels, and the views (numpy)"""
    rs = np.random.RandomState(seed)
    frames = [P.make_frame(h, w, seed + j) for j, (h, w) in enumerate(SIZES)]
    boxes = [_boxes(*_view_hw(h, w, r), k, rs) for (h, w), k, r in zip(SIZES, COUNTS, rotations)]
    return frames, boxes, [_view(f, r) for f, r in zip(frames, rotations)]


def _wide_cuda(f, rs, left=7, right=12):
    """an RGB frame as a column slice of a wider device surface: packed pixels at a larger row pitch"""
    t = torch.from_numpy(rs.randint(0, 256, size=(f.shape[0], f.shape[1] + left + right, 3), dtype=np.uint8)).cuda()
    t[:, left:left + f.shape[1]] = torch.from_numpy(f).cuda()
    return t[:, left:left + f.shape[1]]


def _wide_np(f, rs, left=5, right=9):
    """the same on the host: a numpy view at a larger row pitch"""
    a = rs.randint(0, 256, size=(f.shape[0], f.shape[1] + left + right, 3), dtype=np.uint8)
    a[:, left:left + f.shape[1]] = f
    return a[:, left:left + f.shape[1]]


@pytest.mark.parametrize("rotation", ROTATIONS)
def test_rgb_every_call_form(rotation):
    """One rotation for every frame: device, host and pipelined frame calls (padded pitches on the device and the host), device
    and host affine calls and vpb_preprocess_affine's f32 crops, against the upright calls on the rotated copies; patch rows
    and status word too."""
    m = _engine()
    rs = np.random.RandomState(rotation + 1)
    frames, boxes, views = _rgb_case([rotation] * 4, seed=rotation + 11)
    n = sum(COUNTS)
    dv = [torch.from_numpy(v).cuda() for v in views]
    m.frame_status()
    want = m.infer_frames(dv, boxes)
    rows = _rows(m, n)
    ds = [_wide_cuda(f, rs) if j % 2 == 0 else torch.from_numpy(f).cuda() for j, f in enumerate(frames)]
    assert ds[0].stride(0) > 3 * ds[0].shape[1]
    got = m.infer_frames(ds, boxes, rotate=rotation)
    assert np.array_equal(_rows(m, n), rows)
    _same(got, want)
    assert m.frame_status() == 0
    hs = [_wide_np(f, rs) if j == 2 else f for j, f in enumerate(frames)]
    assert hs[2].strides[0] > 3 * hs[2].shape[1]
    _same(m.infer_frames_host(hs, boxes, rotate=rotation), want)
    ib = [np.ascontiguousarray(b.round().astype(np.int32)) for b in boxes]
    kp, idx = _pin(np.empty((n, 17, 3), np.float32)), _pin(np.empty((n, 17), np.int32))
    m.submit_frames_host([_pin(f) for f in frames], ib, kp, idx, 1, rotate=rotation)
    m.wait_host(1)
    assert np.array_equal(kp, _cat(want[0])) and np.array_equal(idx, _cat(want[1]))
    aff = [_affine(*_view_hw(h, w, rotation), k, rs) for (h, w), k in zip(SIZES, COUNTS)]
    mats, cs, ss = ([a[i] for a in aff] for i in range(3))
    want = m.infer_affine(dv, mats, cs, ss, check=True)
    rows = _rows(m, n)
    _same(m.infer_affine(ds, mats, cs, ss, check=True, rotate=rotation), want)
    assert np.array_equal(_rows(m, n), rows)
    _same(m.infer_affine_host(hs, mats, cs, ss, rotate=rotation), want)
    crops = m.preprocess_affine(ds, mats, rotate=rotation)
    assert torch.equal(crops, m.preprocess_affine(dv, mats))


@pytest.mark.parametrize("flip", [False, True])
def test_mixed_rotations_in_one_call(flip):
    """Four frames of different sizes with all four rotations in one engine call (and the reversed assignment), with and
    without flip test; graphs: the rotated call replays the upright call's cached graph."""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, B200PoseBackend
    m = _engine()
    if flip:
        m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS], True)
    try:
        for rots in ([0, 90, 180, 270], [270, 180, 90, 0]):
            frames, boxes, views = _rgb_case(rots, seed=21 + rots[0])
            assert sum(COUNTS) <= m.batch_limit
            want = m.infer_frames([torch.from_numpy(v).cuda() for v in views], boxes)
            _same(m.infer_frames([torch.from_numpy(v).cuda() for v in views], boxes), want)
            graphs = m.cached_graphs()
            _same(m.infer_frames([torch.from_numpy(f).cuda() for f in frames], boxes, rotate=rots), want)
            assert m.cached_graphs() == graphs
            _same(m.infer_frames_host(frames, boxes, rotate=rots), want)
            be = B200PoseBackend(m)
            assert np.array_equal(_cat(be.inference_frames(frames, boxes, rotate=rots)), _cat(want[0]))
            rs = np.random.RandomState(3)
            xywh = [np.array([[10.5, 20.0, 40.0, 60.0], [-8.0, 12.0, 30.0, 50.0]])] * 4
            from easy_vitpose_b200 import topdown_args
            args = [topdown_args(b) for b in xywh]
            want_t = m.infer_affine_host(views, *[[a[i] for a in args] for i in range(3)])[0]
            assert np.array_equal(_cat(be.inference_topdown(frames, xywh, rotate=rots)), _cat(want_t))
            aff = [_affine(*_view_hw(h, w, r), k, rs) for (h, w), k, r in zip(SIZES, COUNTS, rots)]
            mats, cs, ss = ([a[i] for a in aff] for i in range(3))
            _same(m.infer_affine([torch.from_numpy(f).cuda() for f in frames], mats, cs, ss, rotate=rots),
                  m.infer_affine([torch.from_numpy(v).cuda() for v in views], mats, cs, ss))
    finally:
        if flip:
            m.set_flip_test(None)


def _yuv_case(layout, full, rotations, seed):
    """stored YUV frames (even sizes; 4:2:2 odd heights), boxes in view pixels and the RGB views"""
    rs = np.random.RandomState(seed)
    sizes = [(236, 310), (48, 70), (81 if layout in ("yuyv", "uyvy") else 80, 64), (1080, 1920)]
    frames, boxes, views = [], [], []
    for j, ((h, w), k, r) in enumerate(zip(sizes, COUNTS, rotations)):
        f = rgb_to_yuv(P.make_frame(h, w, seed + j), layout, "bt601", full)
        if j % 2:                                              # random chroma: a wrong chroma block shows
            f = rs.randint(0, 256, size=f.shape, dtype=np.uint8)
        frames.append(f)
        boxes.append(_boxes(*_view_hw(h, w, r), k, rs))
        views.append(_view(yuv_to_rgb(f, layout, "bt601", full), r))
    return frames, boxes, views


@pytest.mark.parametrize("full", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_yuv_layouts(layout, full):
    """Every layout and range: device and host frame calls (patch rows too), the pipelined form and the affine calls, with
    all four rotations in one call, against the upright RGB calls on the rotated conversions."""
    m = _engine()
    fmt = dict(layout=layout, full_range=full)
    for rots in ([0, 90, 180, 270], [180, 270, 0, 90]):
        frames, boxes, views = _yuv_case(layout, full, rots, seed=40 + rots[0])
        n = sum(len(b) for b in boxes)
        want = m.infer_frames([torch.from_numpy(v).cuda() for v in views], boxes)
        rows = _rows(m, n)
        dev = [torch.from_numpy(f).cuda() for f in frames]
        _same(m.infer_frames_yuv(dev, boxes, rotate=rots, **fmt), want)
        assert np.array_equal(_rows(m, n), rows)
        _same(m.infer_frames_yuv_host(frames, boxes, rotate=rots, **fmt), want)
        ib = [np.ascontiguousarray(b.round().astype(np.int32)) for b in boxes]
        kp, idx = _pin(np.empty((n, 17, 3), np.float32)), _pin(np.empty((n, 17), np.int32))
        m.submit_frames_yuv_host([_pin(f) for f in frames], ib, kp, idx, 0, rotate=rots, **fmt)
        m.wait_host(0)
        assert np.array_equal(kp, _cat(want[0])) and np.array_equal(idx, _cat(want[1]))
        rs = np.random.RandomState(rots[0])
        aff = [_affine(*v.shape[:2], k, rs) for v, k in zip(views, COUNTS)]
        mats, cs, ss = ([a[i] for a in aff] for i in range(3))
        want = m.infer_affine([torch.from_numpy(v).cuda() for v in views], mats, cs, ss, check=True)
        _same(m.infer_affine_yuv(dev, mats, cs, ss, check=True, rotate=rots, **fmt), want)
        _same(m.infer_affine_yuv_host(frames, mats, cs, ss, rotate=rots, **fmt), want)


def test_nv12_calls():
    """The _nv12 calls (device, host, pipelined, affine) with per-frame rotations."""
    m = _engine()
    rots = [90, 0, 270, 180]
    frames, boxes, views = _yuv_case("nv12", False, rots, seed=77)
    want = m.infer_frames([torch.from_numpy(v).cuda() for v in views], boxes)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    _same(m.infer_frames_nv12(dev, boxes, rotate=rots), want)
    _same(m.infer_frames_nv12_host(frames, boxes, rotate=rots), want)
    n = sum(len(b) for b in boxes)
    ib = [np.ascontiguousarray(b.round().astype(np.int32)) for b in boxes]
    kp, idx = _pin(np.empty((n, 17, 3), np.float32)), _pin(np.empty((n, 17), np.int32))
    m.submit_frames_nv12_host([_pin(f) for f in frames], ib, kp, idx, 1, rotate=rots)
    m.wait_host(1)
    assert np.array_equal(kp, _cat(want[0])) and np.array_equal(idx, _cat(want[1]))
    rs = np.random.RandomState(4)
    aff = [_affine(*v.shape[:2], k, rs) for v, k in zip(views, COUNTS)]
    mats, cs, ss = ([a[i] for a in aff] for i in range(3))
    want = m.infer_affine([torch.from_numpy(v).cuda() for v in views], mats, cs, ss)
    _same(m.infer_affine_nv12(dev, mats, cs, ss, rotate=rots), want)
    _same(m.infer_affine_nv12_host(frames, mats, cs, ss, rotate=rots), want)


def test_clipping_uses_the_view():
    """A box inside the stored frame's width but beyond the view's is empty after clipping: status bit 0 on the device form,
    VPB_ERR_ARG naming the frame and the box on the host forms; the same box is fine upright."""
    m = _engine()
    f = P.make_frame(100, 300, 3)                                   # stored 100 x 300: the 90-degree view is 300 x 100
    ok = np.array([[10.0, 20.0, 80.0, 250.0]])
    bad = np.array([[10.0, 20.0, 80.0, 250.0], [150.0, 20.0, 200.0, 60.0]])
    m.frame_status()
    m.infer_frames([torch.from_numpy(f).cuda()], [bad])
    assert m.frame_status() == 0                                    # upright: box 1 lies inside the 100 x 300 frame
    m.infer_frames([torch.from_numpy(f).cuda()], [bad], rotate=90)
    assert m.frame_status() & 1
    with pytest.raises(ValueError):
        m.infer_frames([torch.from_numpy(f).cuda()], [bad], rotate=[270], check=True)
    with pytest.raises(ValueError, match="frame 1 box 1"):
        m.infer_frames_host([f, f], [ok, bad], rotate=[0, 90])
    y = rgb_to_yuv(f, "i420")
    with pytest.raises(ValueError, match="frame 0 box 1"):
        m.infer_frames_yuv_host([y], [bad], layout="i420", rotate=270)
    m.infer_frames_yuv_host([y], [bad], layout="i420", rotate=180)
    _same(m.infer_frames_host([f], [ok], rotate=90), m.infer_frames([torch.from_numpy(_view(f, 90)).cuda()], [ok]))


# ------------------------------------------------------------------------------------------------ multi-head engines
HEADS = (("coco", 17), ("aic", 14), ("ap10k", 17))
_heads_cache = {}


def _multi():
    from easy_vitpose_b200 import ViTPose, model_cfg
    if not _heads_cache:
        plus = {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("s", [k for _, k in HEADS], 96, 31).items()}
        multi = ViTPose(model_cfg("s", 17), max_batch=32, heads=HEADS, expert_rows=96)
        multi.load_state_dict(plus)
        _heads_cache["m"] = multi.to("cuda:0")
    return _heads_cache["m"]


def test_multi_head_entries_keep_their_frames_rotation():
    """Boxes of all three heads interleaved in every frame, so a frame appears once per head: the frame, affine and YUV
    multi-head calls, device and host, against the same engine's upright calls on the rotated copies."""
    from easy_vitpose_b200 import B200PoseBackend
    multi = _multi()
    rots = [270, 0, 90, 180]
    frames, boxes, views = _rgb_case(rots, seed=61)
    boxes = [b[:6] for b in boxes]
    heads = [np.arange(len(b)) % 3 for b in boxes]
    dv = [torch.from_numpy(v).cuda() for v in views]
    want = multi.infer_frames_heads(dv, boxes, heads)
    _same(multi.infer_frames_heads([torch.from_numpy(f).cuda() for f in frames], boxes, heads, rotate=rots), want)
    _same(multi.infer_frames_heads_host(frames, boxes, heads, rotate=rots), want)
    assert np.array_equal(_cat(B200PoseBackend(multi).inference_frames_heads(frames, boxes, heads, rotate=rots)), _cat(want[0]))
    rs = np.random.RandomState(9)
    aff = [_affine(*v.shape[:2], len(b), rs) for v, b in zip(views, boxes)]
    mats, cs, ss = ([a[i] for a in aff] for i in range(3))
    want = multi.infer_affine_heads(dv, mats, cs, ss, heads)
    _same(multi.infer_affine_heads([torch.from_numpy(f).cuda() for f in frames], mats, cs, ss, heads, rotate=rots), want)
    _same(multi.infer_affine_heads_host(frames, mats, cs, ss, heads, rotate=rots), want)
    yf, yb, yv = _yuv_case("yuyv", True, rots, seed=62)
    yb = [b[:6] for b in yb]
    yh = [np.arange(len(b)) % 3 for b in yb]
    ydv = [torch.from_numpy(v).cuda() for v in yv]
    fmt = dict(layout="yuyv", full_range=True, rotate=rots)
    want = multi.infer_frames_heads(ydv, yb, yh)
    _same(multi.infer_frames_heads_yuv([torch.from_numpy(f).cuda() for f in yf], yb, yh, **fmt), want)
    _same(multi.infer_frames_heads_yuv_host(yf, yb, yh, **fmt), want)
    want = multi.infer_affine_heads(ydv, mats, cs, ss, heads)
    _same(multi.infer_affine_heads_yuv([torch.from_numpy(f).cuda() for f in yf], mats, cs, ss, heads, **fmt), want)
    _same(multi.infer_affine_heads_yuv_host(yf, mats, cs, ss, heads, **fmt), want)


def test_tracked_streams_with_their_own_rotations():
    """inference_frames_tracked with a rotation per stream equals the same step on the rotated copies (two trackers fed the
    same detections in view pixels)."""
    from easy_vitpose_b200 import B200PoseBackend
    from easy_vitpose_b200.track import DeviceSort
    m = _engine()
    be = B200PoseBackend(m)
    rots = [90, 180, 0, 270]
    frames, boxes, views = _rgb_case(rots, seed=83)
    a, b = DeviceSort(4, 1, 1, 0.3, 0), DeviceSort(4, 1, 1, 0.3, 0)
    for step in range(3):
        dets = [np.concatenate([bb + step, np.full((len(bb), 1), 0.9)], 1) for bb in boxes]
        got = be.inference_frames_tracked(frames, dets, a, rotate=rots)
        want = be.inference_frames_tracked(views, dets, b)
        assert [sorted(g) for g in got] == [sorted(w) for w in want]
        for g, w in zip(got, want):
            for i in g:
                assert np.array_equal(g[i], w[i])
    assert any(len(g) for g in got)


def test_invalid_rotation_is_an_argument_error():
    """Every C call that takes the frame structs returns VPB_ERR_ARG naming the frame for a rotation outside 0 / 90 / 180 /
    270, frames without boxes included; the Python methods raise ValueError before any launch."""
    from easy_vitpose_b200 import _lib
    m = _engine(16)
    L = _lib.lib()
    f = torch.from_numpy(P.make_frame(40, 60, 1)).cuda()
    bb = torch.tensor([[2, 2, 30, 30]] * 4, dtype=torch.int32, device="cuda")
    kp = torch.empty((4, 17, 3), dtype=torch.float32, device="cuda")
    M = torch.tensor([[0.5, 0, 1, 0, 0.5, 2]] * 4, dtype=torch.float64, device="cuda")
    CS = torch.tensor([[96.0, 128, 192, 256]] * 4, device="cuda")
    crops = torch.empty((4, 3, 256, 192), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    F, Y, N = _lib.VpbFrame, _lib.VpbFrameYuv, _lib.VpbFrameNv12
    hp, hu = f.data_ptr(), f.data_ptr() + 40 * 60
    heads = np.zeros(2, np.int32)
    for bad in (45, -90, 360, 1):
        arr = (F * 2)(F(f.data_ptr(), 40, 60, 0, 2, 0), F(f.data_ptr(), 40, 60, 0, 2, bad))
        assert L.vpb_infer_frames(m._handle, arr, 2, p(bb), p(kp), None, st) == 1
        assert b"frame 1" in L.vpb_last_error() and b"rotation" in L.vpb_last_error()
        assert L.vpb_infer_affine(m._handle, arr, 2, p(M), p(CS), p(kp), None, st) == 1
        assert L.vpb_preprocess_affine(arr, 2, p(M), p(crops), st) == 1
        assert L.vpb_infer_frames_heads(m._handle, arr, 2, heads.ctypes.data_as(C.c_void_p), p(bb), p(kp), None, st) == 1
        assert L.vpb_infer_affine_heads(m._handle, arr, 2, heads.ctypes.data_as(C.c_void_p), p(M), p(CS), p(kp), None, st) == 1
        empty = (F * 2)(F(f.data_ptr(), 40, 60, 0, 0, bad), F(f.data_ptr(), 40, 60, 0, 2, 0))   # no boxes: still checked
        assert L.vpb_infer_frames(m._handle, empty, 2, p(bb), p(kp), None, st) == 1
        assert b"frame 0" in L.vpb_last_error()
        yarr = (Y * 1)(Y((hp, hu, hu + 600), 0, 0, 40, 60, 2, bad))
        assert L.vpb_infer_frames_yuv(m._handle, yarr, 1, 2, 0, 0, p(bb), p(kp), None, st) == 1
        assert L.vpb_infer_affine_yuv(m._handle, yarr, 1, 2, 0, 0, p(M), p(CS), p(kp), None, st) == 1
        narr = (N * 1)(N(hp, 0, hu, 0, 40, 60, 2, bad))
        assert L.vpb_infer_frames_nv12(m._handle, narr, 1, 0, p(bb), p(kp), None, st) == 1
        assert L.vpb_infer_affine_nv12(m._handle, narr, 1, 0, p(M), p(CS), p(kp), None, st) == 1
    arr = (F * 1)(F(f.data_ptr(), 40, 60, 0, 2, 270))
    assert L.vpb_infer_frames(m._handle, arr, 1, p(bb), p(kp), None, st) == 0
    hf = P.make_frame(40, 60, 1)
    for rotate in (45, -90, 360, [0, 90]):
        with pytest.raises(ValueError):
            m.infer_frames([f], [bb[:2]], rotate=rotate)
        with pytest.raises(ValueError):
            m.infer_frames_host([hf], [bb[:2].cpu().numpy()], rotate=rotate)
        with pytest.raises(ValueError):
            m.infer_affine_yuv_host([rgb_to_yuv(hf, "i420")], [M[:2].cpu().numpy()], [CS[:2, :2].cpu().numpy()],
                                    [CS[:2, 2:].cpu().numpy()], layout="i420", rotate=rotate)
    torch.cuda.synchronize()
    assert m.frame_status() == 0
