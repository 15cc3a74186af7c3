"""-m gpu: the multi-frame calls (ViTPose.infer_frames / infer_frames_host / submit_frames_host; vpb_infer_frames and its host
forms).  The reference for every case is the engine's own per-frame infer_frame, which test_gpu_frame.py pins against the
reference's fixtures.  The forward is batch-invariant and the decode runs per crop, so a packed call must be BIT-IDENTICAL
to the per-frame calls it replaces."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O

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


def _hd_case(n, seed=9):
    """A seeded 1080p frame with float boxes: tiny ones, large ones, boxes clipped at every border.  None is empty after
    padding and clipping (x0, y0 >= -10), so the host forms accept them."""
    rs = np.random.RandomState(seed)
    frame = rs.randint(0, 256, size=(1080, 1920, 3), dtype=np.uint8)
    boxes = [[0, 0, 1920, 1080], [1915.5, 1070.5, 1990.0, 1100.0], [100.5, 200.5, 101.5, 201.5], [-30.5, 500.2, 60.7, 700.5]]
    for i in range(n - len(boxes)):
        w, h = (rs.randint(1, 60), rs.randint(1, 60)) if i % 4 == 0 else (rs.randint(20, 900), rs.randint(20, 1000))
        x0, y0 = rs.randint(-10, 1900), rs.randint(-10, 1060)
        boxes.append([x0 + rs.rand(), y0 + rs.rand(), x0 + w + rs.rand(), y0 + h + rs.rand()])
    return frame, np.array(boxes[:n], np.float64)


def _case(golden_dir, n_hd=20):
    """frame_a, a frame without boxes, frame_b and a 1080p frame."""
    fa, ba = _golden(golden_dir, "frame_a")
    fb, bb = _golden(golden_dir, "frame_b")
    fhd, bhd = _hd_case(n_hd)
    empty = np.zeros((50, 70, 3), np.uint8)
    return [fa, empty, fb, fhd], [ba, np.zeros((0, 4), np.int32), bb, bhd]


def _per_frame(m, frames, boxes, rows=False):
    """Concatenated per-frame infer_frame results (and the patch rows each call gathered)."""
    kps, ids, pr = [], [], []
    for f, b in zip(frames, boxes):
        f = f if isinstance(f, torch.Tensor) else torch.from_numpy(f).cuda()
        for s in range(0, len(b), m.batch_limit):
            kp, idx = m.infer_frame(f, b[s:s + m.batch_limit])
            kps.append(kp.cpu().numpy()); ids.append(idx.cpu().numpy())
            if rows:
                pr.append(m.read_buffer("patch_rows", (len(kp) * 192, 768), "bf16").view(torch.int16).numpy().copy())
    out = np.concatenate(kps), np.concatenate(ids)
    return out + (np.concatenate(pr),) if rows else out


def _cat(xs):
    return np.concatenate([x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in xs])


@pytest.mark.parametrize("size", ["s", "b"])
def test_packed_call_bit_identical_to_per_frame_calls(golden_dir, size):
    m = _engine(size)
    frames, boxes = _case(golden_dir)
    want_kp, want_idx, want_rows = _per_frame(m, frames, boxes, rows=True)
    n = len(want_kp)
    dframes = [torch.from_numpy(f).cuda() for f in frames]
    for _ in range(3):                                                      # eager, graph capture, graph replay
        kp, idx = m.infer_frames(dframes, boxes)
        assert [len(k) for k in kp] == [len(b) for b in boxes] and [len(i) for i in idx] == [len(b) for b in boxes]
        assert np.array_equal(_cat(kp), want_kp) and np.array_equal(_cat(idx), want_idx)
        rows = m.read_buffer("patch_rows", (n * 192, 768), "bf16").view(torch.int16).numpy()
        assert np.array_equal(rows, want_rows)
    assert m.frame_status() == 0


@pytest.mark.parametrize("shift", [False, True])
def test_packed_call_with_flip_test_bit_identical_to_per_frame_calls(golden_dir, shift):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    m = _engine("s")
    frames, boxes = _case(golden_dir, n_hd=12)
    assert sum(len(b) for b in boxes) <= m.max_batch // 2
    m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS], shift)
    try:
        want_kp, want_idx = _per_frame(m, frames, boxes)
        dframes = [torch.from_numpy(f).cuda() for f in frames]
        for _ in range(3):
            kp, idx = m.infer_frames(dframes, boxes)
            assert np.array_equal(_cat(kp), want_kp) and np.array_equal(_cat(idx), want_idx)
        kp_h, idx_h = m.infer_frames_host(frames, boxes)
        assert np.array_equal(_cat(kp_h), want_kp) and np.array_equal(_cat(idx_h), want_idx)
    finally:
        m.set_flip_test(None)


def test_chunking_over_the_batch_and_frame_limits(golden_dir):
    """70 one-box frames (the first call is closed by the 64-frame limit), then a 150-box frame (more than max_batch: it
    fills the rest of the second call and continues in a third)."""
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.model import plan_frame_chunks
    m = _engine("s", max_batch=128)
    rs = np.random.RandomState(3)
    frames, boxes = [], []
    for j in range(70):
        h, w = int(rs.randint(40, 300)), int(rs.randint(40, 300))
        frames.append(rs.randint(0, 256, size=(h, w, 3), dtype=np.uint8))
        x0, y0 = int(rs.randint(-10, w - 5)), int(rs.randint(-10, h - 5))
        boxes.append(np.array([[x0, y0, x0 + int(rs.randint(5, 200)), y0 + int(rs.randint(5, 200))]], np.int32))
    fhd, bhd = _hd_case(150, seed=4)
    frames.append(fhd); boxes.append(bhd)
    chunks = plan_frame_chunks([len(b) for b in boxes], m.batch_limit, _lib.MAX_FRAMES)
    assert [len(c) for c in chunks] == [_lib.MAX_FRAMES, 7, 1]
    assert [sum(e - s for _, s, e in c) for c in chunks] == [64, 128, 28]   # the 1080p frame spans the last two calls
    want_kp, want_idx = _per_frame(m, frames, boxes)
    kp, idx = m.infer_frames([torch.from_numpy(f).cuda() for f in frames], boxes)
    assert np.array_equal(_cat(kp), want_kp) and np.array_equal(_cat(idx), want_idx)
    kp_h, idx_h = m.infer_frames_host(frames, boxes)
    assert np.array_equal(_cat(kp_h), want_kp) and np.array_equal(_cat(idx_h), want_idx)


def test_pitched_frame_equals_its_contiguous_copy(golden_dir):
    m = _engine("s")
    fa, ba = _golden(golden_dir, "frame_a")
    rs = np.random.RandomState(8)
    wide = torch.from_numpy(rs.randint(0, 256, size=(fa.shape[0], fa.shape[1] + 77, 3), dtype=np.uint8)).cuda()
    wide[:, 21:21 + fa.shape[1]] = torch.from_numpy(fa).cuda()
    view = wide[:, 21:21 + fa.shape[1]]
    assert not view.is_contiguous() and view.stride() == (3 * wide.shape[1], 3, 1)
    want_kp, want_idx = _per_frame(m, [fa], [ba])
    kp, idx = m.infer_frames([view, view], [ba, ba[:3]])
    assert np.array_equal(_cat(kp), np.concatenate([want_kp, want_kp[:3]])) and np.array_equal(_cat(idx), np.concatenate([want_idx, want_idx[:3]]))
    hview = wide.cpu().numpy()[:, 21:21 + fa.shape[1]]                       # the host forms stage it packed with a 2D copy
    kp_h, idx_h = m.infer_frames_host([hview], [ba])
    assert np.array_equal(kp_h[0], want_kp) and np.array_equal(idx_h[0], want_idx)


def test_host_and_pipelined_forms_equal_the_device_form(golden_dir):
    from easy_vitpose_b200 import B200PoseBackend
    m = _engine("s")
    frames, boxes = _case(golden_dir)
    kp_d, idx_d = m.infer_frames([torch.from_numpy(f).cuda() for f in frames], boxes)
    kp_d, idx_d = _cat(kp_d), _cat(idx_d)
    for _ in range(3):
        kp_h, idx_h = m.infer_frames_host(frames, boxes)
        assert np.array_equal(_cat(kp_h), kp_d) and np.array_equal(_cat(idx_h), idx_d)
    assert np.array_equal(_cat(B200PoseBackend(m).inference_frames(frames, boxes)), kp_d)
    # two different frame sets in flight on slots 0 and 1, in pinned memory
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    sets = []
    for i in range(4):
        fs = [pin(P.make_frame(360, 480, 11 + i)), pin(frames[2]), pin(_hd_case(6, seed=20 + i)[0])]
        bs = [boxes[0][: 7 - 2 * (i % 3)], boxes[2], np.ascontiguousarray(_hd_case(6 + i, seed=20 + i)[1][:6 + i].round().astype(np.int32))]
        sets.append((fs, bs))
    want = [m.infer_frames_host(fs, bs) for fs, bs in sets]
    outs = []
    for fs, bs in sets:
        n = sum(len(b) for b in bs)
        outs.append((pin(np.empty((n, 17, 3), np.float32)), pin(np.empty((n, 17), np.int32))))
    m.submit_frames_host(*sets[0], *outs[0], 0)
    for i in range(1, 4):
        m.submit_frames_host(*sets[i], *outs[i], i % 2)
        m.wait_host((i - 1) % 2)
    m.wait_host(1)
    for (wk, wi), (k, i) in zip(want, outs):
        assert np.array_equal(_cat(wk), k) and np.array_equal(_cat(wi), i)


def test_errors(golden_dir):
    from easy_vitpose_b200 import _lib
    m = _engine("s", max_batch=16)
    frames, boxes = _case(golden_dir, n_hd=4)
    bad = [b.copy() for b in boxes]
    bad[2][1] = [500, 500, 520, 540]                                        # entirely outside the 131x97 frame_b
    with pytest.raises(ValueError, match="frame 2 box 1"):
        m.infer_frames_host(frames, bad)
    m.frame_status()
    dframes = [torch.from_numpy(f).cuda() for f in frames]
    m.infer_frames(dframes, bad)
    assert m.frame_status() & 1
    with pytest.raises(ValueError):
        m.infer_frames(dframes, bad, check=True)
    assert m.frame_status() == 0
    m.infer_frames(dframes, boxes, check=True)                              # good boxes: no raise
    kp, idx = m.infer_frames(dframes[1:2], boxes[1:2])                      # no boxes at all: nothing launched
    assert len(kp) == 1 and kp[0].shape == (0, 17, 3) and idx[0].shape == (0, 17)
    with pytest.raises(ValueError):
        m.infer_frames(dframes, boxes[:2])
    # raw ABI: VPB_ERR_ARG
    L = _lib.lib()
    fa = dframes[0]
    bb = torch.zeros((32, 4), dtype=torch.int32, device="cuda")
    bb[:, 2:] = 50
    kp = torch.empty((32, 17, 3), dtype=torch.float32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(*fr):
        arr = (_lib.VpbFrame * len(fr))(*fr)
        return L.vpb_infer_frames(m._handle, arr, len(arr), C.c_void_p(bb.data_ptr()), C.c_void_p(kp.data_ptr()), None, st)

    h, w = fa.shape[:2]
    assert call(_lib.VpbFrame(fa.data_ptr(), h, w, 0, 3)) == 0
    assert call(_lib.VpbFrame(fa.data_ptr(), h, w, 0, 17)) == 1                            # over max_batch
    assert call(_lib.VpbFrame(fa.data_ptr(), h, w, 0, 10), _lib.VpbFrame(fa.data_ptr(), h, w, 0, 7)) == 1
    assert call(_lib.VpbFrame(fa.data_ptr(), h, w, 0, -1), _lib.VpbFrame(fa.data_ptr(), h, w, 0, 3)) == 1   # negative count
    assert call(_lib.VpbFrame(None, h, w, 0, 3)) == 1                                      # null data with boxes
    assert call(_lib.VpbFrame(None, h, w, 0, 0), _lib.VpbFrame(fa.data_ptr(), h, w, 0, 3)) == 0   # null data, no boxes: skipped
    assert call(_lib.VpbFrame(fa.data_ptr(), h, w, 3 * w - 1, 3)) == 1                     # pitch below 3 * width
    assert call(_lib.VpbFrame(fa.data_ptr(), 0, w, 0, 3)) == 1
    assert call(*[_lib.VpbFrame(fa.data_ptr(), h, w, 0, 0)] * 100, _lib.VpbFrame(fa.data_ptr(), h, w, 0, 2)) == 0
    m2 = _engine("s", max_batch=128)
    arr = (_lib.VpbFrame * 65)(*[_lib.VpbFrame(fa.data_ptr(), h, w, 0, 1)] * 65)          # 65 frames with boxes
    kp2 = torch.empty((65, 17, 3), dtype=torch.float32, device="cuda")
    bb2 = bb[:1].repeat(65, 1)
    assert L.vpb_infer_frames(m2._handle, arr, 65, C.c_void_p(bb2.data_ptr()), C.c_void_p(kp2.data_ptr()), None, st) == 1
    assert b"VPB_MAX_FRAMES" in L.vpb_last_error()
    torch.cuda.synchronize()
    assert m.frame_status() == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_frame_on_another_device_raises(golden_dir):
    m = _engine("s")
    fa, ba = _golden(golden_dir, "frame_a")
    with pytest.raises(ValueError, match="lives on"):
        m.infer_frames([torch.from_numpy(fa).cuda(0), torch.from_numpy(fa).cuda(1)], [ba, ba])
