"""-m gpu: the NV12 frame calls (ViTPose.infer_frames_nv12 / _host / submit_frames_nv12_host, infer_affine_nv12 / _host;
vpb_*_nv12).  The reference for every case is the engine's own RGB call on oracle.nv12_oracle.nv12_to_rgb(frame), which
the RGB tests pin against the reference project: the NV12 gathers convert each tap and then run the RGB arithmetic, so the
patch rows, keypoints and argmax indices must be BIT-IDENTICAL."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O
from oracle.nv12_oracle import nv12_to_rgb, rgb_to_nv12

pytestmark = pytest.mark.gpu

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


def _golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    fh, fw, fseed = (int(v) for v in g["meta"][:3])
    rows = g["rows"].astype(np.float64)
    return P.make_frame(fh, fw, fseed), rows[rows[:, 4] > 0.35, :4].round().astype(np.int32)


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


def _case(golden_dir, kind, matrix, n_hd=20):
    """frame_a, a frame without boxes, frame_b and a 1080p frame as stacked NV12 [3H/2, W] (odd sizes cropped to even):
    kind "random" = random planes, "image" = the frames (the 1080p one a smooth gradient) converted to NV12."""
    fa, ba = _golden(golden_dir, "frame_a")
    fb, bb = _golden(golden_dir, "frame_b")
    rgb = [fa, np.zeros((50, 70, 3), np.uint8), fb, _gradient(1080, 1920)]
    rs = np.random.RandomState(17)
    frames = []
    for f in rgb:
        h, w = f.shape[0] & ~1, f.shape[1] & ~1
        frames.append(rs.randint(0, 256, size=(3 * h // 2, w), dtype=np.uint8) if kind == "random" else rgb_to_nv12(f[:h, :w], matrix))
    return frames, [ba, np.zeros((0, 4), np.int32), bb, _hd_boxes(n_hd)]


def _cat(xs):
    return np.concatenate([x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in xs])


def _rows(m, n):
    return m.read_buffer("patch_rows", (n * 192, 768), "bf16").view(torch.int16).numpy().copy()


def _rgb_frames(frames, matrix):
    return [nv12_to_rgb(f, matrix) for f in frames]


@pytest.mark.parametrize("size,matrix,kind", [("s", "bt601", "random"), ("s", "bt709", "random"), ("s", "bt601", "image"),
                                              ("s", "bt709", "image"), ("b", "bt709", "image")])
def test_frames_bit_identical_to_the_rgb_call(golden_dir, size, matrix, kind):
    m = _engine(size)
    frames, boxes = _case(golden_dir, kind, matrix)
    n = sum(len(b) for b in boxes)
    assert n <= m.batch_limit                                               # one call: the patch rows are all of it
    kp_r, idx_r = m.infer_frames([torch.from_numpy(f).cuda() for f in _rgb_frames(frames, matrix)], boxes)
    rows_r = _rows(m, n)
    kp, idx = m.infer_frames_nv12([torch.from_numpy(f).cuda() for f in frames], boxes, matrix)
    assert [len(k) for k in kp] == [len(b) for b in boxes]
    assert np.array_equal(_rows(m, n), rows_r)
    assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
    assert m.frame_status() == 0


def test_eager_captured_and_replayed_calls_are_identical_and_share_the_graph_cache(golden_dir):
    """A fresh engine: the first NV12 call of a batch size runs eagerly, the second captures, the third replays; the RGB
    call of the same batch size then replays the same graph (the gather runs outside it), so no cache entry is added."""
    m = _engine("s", max_batch=48)
    frames, boxes = _case(golden_dir, "image", "bt601")
    dframes = [torch.from_numpy(f).cuda() for f in frames]
    assert m.cached_graphs() == (0, 0)
    outs = []
    for _ in range(3):
        kp, idx = m.infer_frames_nv12(dframes, boxes)
        outs.append((_cat(kp), _cat(idx)))
    assert m.cached_graphs() == (1, 1)
    kp_r, idx_r = m.infer_frames([torch.from_numpy(f).cuda() for f in _rgb_frames(frames, "bt601")], boxes)
    assert m.cached_graphs() == (1, 1)
    for kp, idx in outs:
        assert np.array_equal(kp, _cat(kp_r)) and np.array_equal(idx, _cat(idx_r))


def _rotated(M, deg):
    """M (image -> 192x256 crop) followed by a rotation of the crop about its centre."""
    t = np.deg2rad(deg)
    R = np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1]])
    c = np.array([[1, 0, 95.5], [0, 1, 127.5], [0, 0, 1]]) @ R @ np.array([[1, 0, -95.5], [0, 1, -127.5], [0, 0, 1]])
    return np.einsum("ij,njk->nik", c, np.concatenate([M, np.tile([[[0, 0, 1]]], (len(M), 1, 1))], 1))[:, :2]


def _affine_case(n_per_frame=(5, 0, 4, 9), seed=3):
    """NV12 frames (random planes and converted images) with boxes overhanging the frames; the matrices of topdown_args,
    every other frame's rotated by 25 / -40 degrees."""
    from easy_vitpose_b200 import topdown_args
    rs = np.random.RandomState(seed)
    sizes = [(240, 320), (64, 80), (480, 376), (1080, 1920)]
    frames, mats, cs, ss = [], [], [], []
    for j, ((h, w), k) in enumerate(zip(sizes, n_per_frame)):
        frames.append(rs.randint(0, 256, size=(3 * h // 2, w), dtype=np.uint8) if j % 2 else rgb_to_nv12(P.make_frame(h, w, seed + j)))
        bw, bh = rs.uniform(8, w * 0.9, k), rs.uniform(8, h * 0.9, k)
        boxes = np.stack([rs.uniform(-0.3 * w, w) - bw / 2, rs.uniform(-0.3 * h, h) - bh / 2, bw, bh], 1)
        M, c, s = topdown_args(boxes)
        if j % 2 == 0 and k:
            M = np.concatenate([M[: k // 2], _rotated(np.asarray(M[k // 2:]).reshape(-1, 2, 3), 25 if j == 0 else -40)])
        mats.append(np.asarray(M).reshape(-1, 2, 3)); cs.append(c); ss.append(s)
    return frames, mats, cs, ss


@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
def test_affine_bit_identical_to_the_rgb_call(matrix):
    m = _engine("s")
    frames, mats, cs, ss = _affine_case()
    n = sum(len(x) for x in mats)
    kp_r, idx_r = m.infer_affine([torch.from_numpy(f).cuda() for f in _rgb_frames(frames, matrix)], mats, cs, ss, check=True)
    rows_r = _rows(m, n)
    for _ in range(3):
        kp, idx = m.infer_affine_nv12([torch.from_numpy(f).cuda() for f in frames], mats, cs, ss, matrix, check=True)
        assert np.array_equal(_rows(m, n), rows_r)
        assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
    kp_h, idx_h = m.infer_affine_nv12_host(frames, mats, cs, ss, matrix)
    assert np.array_equal(_cat(kp_h), _cat(kp_r)) and np.array_equal(_cat(idx_h), _cat(idx_r))


@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
def test_flip_test_both_call_kinds(golden_dir, matrix):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, B200PoseBackend, topdown_args
    m = _engine("s")
    frames, boxes = _case(golden_dir, "image", matrix, n_hd=12)
    m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS], True)
    try:
        assert sum(len(b) for b in boxes) <= m.batch_limit
        rgb = _rgb_frames(frames, matrix)
        kp_r, idx_r = m.infer_frames([torch.from_numpy(f).cuda() for f in rgb], boxes)
        for _ in range(3):
            kp, idx = m.infer_frames_nv12([torch.from_numpy(f).cuda() for f in frames], boxes, matrix)
            assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
        kp_h, idx_h = m.infer_frames_nv12_host(frames, boxes, matrix)
        assert np.array_equal(_cat(kp_h), _cat(kp_r)) and np.array_equal(_cat(idx_h), _cat(idx_r))
        af, mats, cs, ss = _affine_case((3, 2, 4, 6), seed=5)
        kp_r, idx_r = m.infer_affine([torch.from_numpy(f).cuda() for f in _rgb_frames(af, matrix)], mats, cs, ss)
        kp, idx = m.infer_affine_nv12([torch.from_numpy(f).cuda() for f in af], mats, cs, ss, matrix)
        assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
        # B200PoseBackend.inference_topdown_nv12 takes xywh boxes and builds the same matrices
        xywh = [np.array([[10.5, 20.0, 120.0, 200.0], [-30.0, 40.0, 90.0, 150.0]]), np.array([[5.0, 5.0, 40.0, 50.0]])]
        tf = [af[0], af[2]]
        want = m.infer_affine_host(_rgb_frames(tf, matrix), *[[topdown_args(b)[i] for b in xywh] for i in range(3)])[0]
        got = B200PoseBackend(m).inference_topdown_nv12(tf, xywh, matrix=matrix)
        assert np.array_equal(_cat(got), _cat(want))
    finally:
        m.set_flip_test(None)


def test_chunking_over_the_batch_and_frame_limits(golden_dir):
    """70 one-box NV12 frames (the first call is closed by the 64-frame limit), then a 1080p frame with 150 boxes (more than
    max_batch): three engine calls, equal to the RGB calls on the converted frames."""
    m = _engine("s", max_batch=128)
    rs = np.random.RandomState(3)
    frames, boxes = [], []
    for j in range(70):
        h, w = 2 * int(rs.randint(20, 150)), 2 * int(rs.randint(20, 150))
        frames.append(rs.randint(0, 256, size=(3 * h // 2, w), dtype=np.uint8))
        x0, y0 = int(rs.randint(-10, w - 5)), int(rs.randint(-10, h - 5))
        boxes.append(np.array([[x0, y0, x0 + int(rs.randint(5, 200)), y0 + int(rs.randint(5, 200))]], np.int32))
    frames.append(rgb_to_nv12(_gradient(1080, 1920)))
    boxes.append(_hd_boxes(150, seed=4))
    rgb = _rgb_frames(frames, "bt601")
    kp_r, idx_r = m.infer_frames([torch.from_numpy(f).cuda() for f in rgb], boxes)
    kp, idx = m.infer_frames_nv12([torch.from_numpy(f).cuda() for f in frames], boxes)
    assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
    kp_h, idx_h = m.infer_frames_nv12_host(frames, boxes)
    assert np.array_equal(_cat(kp_h), _cat(kp_r)) and np.array_equal(_cat(idx_h), _cat(idx_r))
    from easy_vitpose_b200 import B200PoseBackend
    assert np.array_equal(_cat(B200PoseBackend(m).inference_frames_nv12(frames, boxes)), _cat(kp_r))
    mats = [np.tile(np.array([[[0.5, 0.0, 1.0], [0.0, 0.5, 2.0]]]), (len(b), 1, 1)) for b in boxes]
    cs = [np.tile([[96.0, 128.0]], (len(b), 1)) for b in boxes]
    ss = [np.tile([[192.0, 256.0]], (len(b), 1)) for b in boxes]
    kp_r, idx_r = m.infer_affine_host(rgb, mats, cs, ss)
    kp_h, idx_h = m.infer_affine_nv12_host(frames, mats, cs, ss)
    assert np.array_equal(_cat(kp_h), _cat(kp_r)) and np.array_equal(_cat(idx_h), _cat(idx_r))


def test_frame_layouts(golden_dir):
    """Stacked and split forms; planes as column slices of wider tensors (pitch > width); Y and UV in separate
    allocations; the host forms (which stage the pitched planes packed)."""
    m = _engine("s")
    frames, boxes = _case(golden_dir, "random", "bt601")
    fa, ba = frames[0], boxes[0]
    h, w = fa.shape[0] // 3 * 2, fa.shape[1]
    kp_r, idx_r = m.infer_frames([torch.from_numpy(nv12_to_rgb(fa)).cuda()], [ba])
    rs = np.random.RandomState(8)
    wy = torch.from_numpy(rs.randint(0, 256, size=(h, w + 38), dtype=np.uint8)).cuda()
    wuv = torch.from_numpy(rs.randint(0, 256, size=(h // 2, w + 66), dtype=np.uint8)).cuda()
    wy[:, 21:21 + w] = torch.from_numpy(fa[:h]).cuda()
    wuv[:, 10:10 + w] = torch.from_numpy(fa[h:]).cuda()
    y_view, uv_view = wy[:, 21:21 + w], wuv[:, 10:10 + w]
    assert y_view.stride() == (w + 38, 1) and uv_view.stride() == (w + 66, 1)
    stacked = torch.from_numpy(fa).cuda()
    separate = (torch.from_numpy(fa[:h].copy()).cuda(), torch.from_numpy(fa[h:].copy()).cuda())
    for f in (stacked, separate, (y_view, uv_view), fa, (fa[:h], fa[h:])):
        kp, idx = m.infer_frames_nv12([f], [ba])
        assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))
    hy, huv = wy.cpu().numpy()[:, 21:21 + w], wuv.cpu().numpy()[:, 10:10 + w]
    for f in (fa, (fa[:h].copy(), fa[h:].copy()), (hy, huv)):
        kp, idx = m.infer_frames_nv12_host([f], [ba])
        assert np.array_equal(_cat(kp), _cat(kp_r)) and np.array_equal(_cat(idx), _cat(idx_r))


def test_host_and_pipelined_forms_equal_the_device_form(golden_dir):
    m = _engine("s")
    frames, boxes = _case(golden_dir, "image", "bt709")
    kp_d, idx_d = m.infer_frames_nv12([torch.from_numpy(f).cuda() for f in frames], boxes, "bt709")
    kp_d, idx_d = _cat(kp_d), _cat(idx_d)
    for _ in range(2):
        kp_h, idx_h = m.infer_frames_nv12_host(frames, boxes, "bt709")
        assert np.array_equal(_cat(kp_h), kp_d) and np.array_equal(_cat(idx_h), idx_d)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    sets = []
    for i in range(4):
        hd = rgb_to_nv12(_gradient(1080, 1920)[:, ::-1] if i % 2 else _gradient(1080, 1920), "bt709")
        y, uv = hd[:1080], hd[1080:]
        fs = [pin(rgb_to_nv12(P.make_frame(360, 480, 11 + i), "bt709")), pin(frames[2]), (pin(y), pin(uv))]
        bs = [np.ascontiguousarray(boxes[0][: 7 - 2 * (i % 3)]), boxes[2], np.ascontiguousarray(_hd_boxes(6 + i, seed=20 + i).round().astype(np.int32))]
        sets.append((fs, bs))
    want = [m.infer_frames_nv12_host(fs, bs, "bt709") for fs, bs in sets]
    outs = []
    for fs, bs in sets:
        n = sum(len(b) for b in bs)
        outs.append((pin(np.empty((n, 17, 3), np.float32)), pin(np.empty((n, 17), np.int32))))
    m.submit_frames_nv12_host(*sets[0], *outs[0], 0, matrix="bt709")
    for i in range(1, 4):
        m.submit_frames_nv12_host(*sets[i], *outs[i], i % 2, matrix="bt709")
        m.wait_host((i - 1) % 2)
    m.wait_host(1)
    for (wk, wi), (k, i) in zip(want, outs):
        assert np.array_equal(_cat(wk), k) and np.array_equal(_cat(wi), i)


def test_errors(golden_dir):
    from easy_vitpose_b200 import _lib
    m = _engine("s", max_batch=16)
    frames, boxes = _case(golden_dir, "random", "bt601", n_hd=4)
    bad = [b.copy() for b in boxes]
    bad[2][1] = [500, 500, 520, 540]                                        # entirely outside frame_b
    with pytest.raises(ValueError, match="frame 2 box 1"):
        m.infer_frames_nv12_host(frames, bad)
    m.frame_status()
    dframes = [torch.from_numpy(f).cuda() for f in frames]
    m.infer_frames_nv12(dframes, bad)
    assert m.frame_status() & 1
    with pytest.raises(ValueError):
        m.infer_frames_nv12(dframes, bad, check=True)
    assert m.frame_status() == 0
    with pytest.raises(ValueError):
        m.infer_frames_nv12(dframes, boxes, "bt2020")
    with pytest.raises(ValueError):
        m.infer_frames_nv12([torch.zeros((15, 21), dtype=torch.uint8, device="cuda")], [boxes[0]])       # odd width
    with pytest.raises(ValueError):
        m.infer_frames_nv12([(dframes[0][:10], dframes[0][10:16])], [boxes[0]])                         # mismatched uv
    kp, idx = m.infer_frames_nv12(dframes[1:2], boxes[1:2])                  # no boxes at all: nothing launched
    assert len(kp) == 1 and kp[0].shape == (0, 17, 3)
    # raw ABI: VPB_ERR_ARG
    L = _lib.lib()
    fa = dframes[0]
    h, w = fa.shape[0] // 3 * 2, fa.shape[1]
    y, uv = fa.data_ptr(), fa.data_ptr() + h * w
    bb = torch.zeros((32, 4), dtype=torch.int32, device="cuda")
    bb[:, 2:] = 50
    kp = torch.empty((32, 17, 3), dtype=torch.float32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(*fr, matrix=0):
        arr = (_lib.VpbFrameNv12 * len(fr))(*fr)
        return L.vpb_infer_frames_nv12(m._handle, arr, len(arr), matrix, C.c_void_p(bb.data_ptr()), C.c_void_p(kp.data_ptr()), None, st)

    F = _lib.VpbFrameNv12
    assert call(F(y, 0, uv, 0, h, w, 3)) == 0
    assert call(F(y, 0, uv, 0, h, w, 3), matrix=1) == 0
    assert call(F(y, 0, uv, 0, h, w, 3), matrix=2) == 1                    # unknown matrix
    assert call(F(y, 0, uv, 0, h, w, 3), matrix=-1) == 1
    assert call(F(y, 0, uv, 0, h, w, 17)) == 1                              # over max_batch
    assert call(F(y, 0, uv, 0, h - 1, w, 3)) == 1                           # odd height
    assert call(F(y, 0, uv, 0, h, w - 1, 3)) == 1                           # odd width
    assert call(F(y, 0, uv, 0, 0, w, 3)) == 1
    assert call(F(y, w - 2, uv, 0, h, w, 3)) == 1                           # short y pitch
    assert call(F(y, 0, uv, w - 1, h, w, 3)) == 1                           # short uv pitch
    assert call(F(y, 0, None, 0, h, w, 3)) == 1                             # NULL uv
    assert call(F(None, 0, uv, 0, h, w, 3)) == 1                            # NULL y
    assert call(F(None, 0, None, 0, h, w, 0), F(y, 0, uv, 0, h, w, 3)) == 0   # no boxes: skipped
    assert call(F(y, 0, uv, 0, h, w, -1)) == 1
    hp = np.zeros((3, 20), np.uint8)
    assert L.vpb_infer_frames_nv12_host(m._handle, (F * 1)(F(hp.ctypes.data, 0, hp.ctypes.data, 0, 2, 20, 1)), 1, 5,
                                        bb.cpu().numpy().ctypes.data_as(C.c_void_p), kp.cpu().numpy().ctypes.data_as(C.c_void_p),
                                        None, st) == 1
    assert b"matrix" in L.vpb_last_error()
    M = torch.tensor([[0.5, 0, 1, 0, 0.5, 2]] * 3, dtype=torch.float64, device="cuda")
    CS = torch.tensor([[96.0, 128, 192, 256]] * 3, device="cuda")
    arr = (F * 1)(F(y, 0, uv, 0, h, w - 1, 3))
    assert L.vpb_infer_affine_nv12(m._handle, arr, 1, 0, C.c_void_p(M.data_ptr()), C.c_void_p(CS.data_ptr()),
                                   C.c_void_p(kp.data_ptr()), None, st) == 1
    # affine: a scale <= 0 sets status bit 1 on the device form and raises on the host form
    frames_a, mats, cs, ss = _affine_case((2, 0, 1, 1), seed=9)
    ss[0] = ss[0].copy(); ss[0][0, 0] = 0.0
    with pytest.raises(ValueError):
        m.infer_affine_nv12_host(frames_a, mats, cs, ss)
    m.infer_affine_nv12([torch.from_numpy(f).cuda() for f in frames_a], [torch.from_numpy(np.asarray(x)).cuda() for x in mats],
                        [torch.from_numpy(np.asarray(x, np.float32)).cuda() for x in cs],
                        [torch.from_numpy(np.asarray(x, np.float32)).cuda() for x in ss])
    assert m.frame_status() & 2
    torch.cuda.synchronize()
    assert m.frame_status() == 0
