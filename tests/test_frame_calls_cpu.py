"""CPU: the call plumbing of ViTPose's multi-frame, affine and multi-head methods.  A recording fake stands in for the engine
library, and every host form is driven on seeded inputs: frames without boxes, more boxes than batch_limit (flip test off and
on), more than 64 frames, per-frame rotations, NV12 and the I420 / YUYV / NV21 layouts, mixed heads per frame.  Each engine
call is checked against expectations stated here box by box: the entry point and the number of calls, the decoded vpb_frame*
rows (pointers, sizes, pitches, box counts, rotations), the format ints, the heads array, the box / matrix / centre / scale
rows the call points at, the pointer offsets into the staged arrays and outputs, and where each output row lands in the
returned per-frame arrays (rows K_j..K_max-1 of a head-j box stay zero).  The pipelined submit forms, and which error wins
when an input has several faults, are pinned too.  The device forms run the same recorder under the gpu marker."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from easy_vitpose_b200 import _lib, model_cfg
from easy_vitpose_b200.model import ViTPose

STREAM = 0x5EED                                         # what the patched ViTPose._stream hands the host calls
HEADS = [17, 5, 3]                                      # keypoints of the multi-head engine's heads
LAYOUT = {"nv12": 0, "nv21": 1, "i420": 2, "yuyv": 4}   # VPB_YUV_* of include/vitpose_b200.h
MATRIX = {"bt601": 0, "bt709": 1}


def _row(f):
    """A decoded vpb_frame* struct: its fields in order, the YUV plane pointers as a tuple."""
    return tuple(tuple(getattr(f, n)) if n == "plane" else getattr(f, n) for n, _ in f._fields_)


def _view(ptr, dtype, shape):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(np.dtype(dtype)))), shape=shape)


class FakeLib:
    """Records every vpb_* call, decoding the multi-frame calls while their arguments are alive.  On the host it also reads
    the per-box rows through their pointers and writes (call, row, keypoint + 1) / 1000 * call + row + 1 into the keypoint
    columns of every output row that the engine would write (K_j of the row's head)."""

    def __init__(self, m, host):
        self.m, self.host, self.calls = m, host, []

    def __getattr__(self, name):
        if not name.startswith("vpb_"):
            raise AttributeError(name)
        return lambda *args: self._call(name, args)

    def _call(self, name, args):
        if name == "vpb_frame_status":
            return 0
        nfmt = 1 if "_nv12" in name else 3 if "_yuv" in name else 0
        widths = [(np.float64, 6), (np.float32, 4)] if "_affine" in name else [(np.int32, 4)]
        arr, n = args[1], args[2]
        rows = [_row(f) for f in arr]
        i = 3 + nfmt
        heads = None
        if "_heads" in name:
            heads = _view(args[i], np.int32, (n,)).copy()
            i += 1
        ptrs = args[i:i + len(widths)]
        kp, idx = args[i + len(widths)], args[i + len(widths) + 1]
        last = args[i + len(widths) + 2]
        nb = sum(r[-2] for r in rows)
        rec = dict(name=name, n=n, rows=rows, fmt=tuple(args[3:3 + nfmt]), heads=heads, ptrs=[p.value for p in ptrs],
                   kp=kp.value, idx=idx.value, last=last.value if isinstance(last, C.c_void_p) else last)
        if self.host:
            rec["per_box"] = [_view(p, dt, (nb, w)).copy() for p, (dt, w) in zip(ptrs, widths)]
            kw = self.m.num_keypoints_max if heads is not None else self.m.num_keypoints
            kpa, ida = _view(kp, np.float32, (nb, kw, 3)), _view(idx, np.int32, (nb, kw))
            r, call = 0, len(self.calls)
            for e, row in enumerate(rows):
                k = self.m.head_keypoints[heads[e]] if heads is not None else kw
                for _ in range(row[-2]):
                    kpa[r, :k] = [(call, r, q + 1) for q in range(k)]
                    ida[r, :k] = 1000 * call + r + 1
                    r += 1
        self.calls.append(rec)
        return 0


@pytest.fixture
def fake(monkeypatch):
    def make(m, host=True):
        lib = FakeLib(m, host)
        monkeypatch.setattr(_lib, "lib", lambda: lib)
        monkeypatch.setattr(ViTPose, "_ensure", lambda self: None)
        if host:
            monkeypatch.setattr(ViTPose, "_stream", lambda self: C.c_void_p(STREAM))
            monkeypatch.setattr(torch.cuda, "device", lambda *a: contextlib.nullcontext())
        return lib
    return make


def _engine(max_batch, flip, heads=False):
    m = ViTPose(model_cfg("s", 17), max_batch=max_batch, heads=HEADS if heads else None)
    m._flip = flip
    return m


# ------------------------------------------------------------------------------------------------ inputs
def _frames(rs, n, source, device=False):
    """n seeded frames of `source` ("rgb", "nv12" or a YUV layout) -> (frames, the vpb_frame* fields of each before
    num_boxes).  Every fifth host RGB frame is a column slice of a wider image (read in place at the wider pitch)."""
    frames, rows = [], []
    for j in range(n):
        H, W = 4 + 2 * (j % 2), 6 + 2 * (j % 3)
        if source == "rgb":
            f = rs.randint(0, 256, (H, W + 3, 3), dtype=np.uint8)[:, 1:1 + W] if j % 5 == 2 and not device else \
                rs.randint(0, 256, (H, W, 3), dtype=np.uint8)
        elif source == "yuyv":
            f = rs.randint(0, 256, (H, W, 2), dtype=np.uint8)
        else:
            f = rs.randint(0, 256, (H * 3 // 2, W), dtype=np.uint8)
        if device:
            f = torch.from_numpy(f).cuda()
        p = f.data_ptr() if device else f.ctypes.data
        if source == "rgb":
            rows.append((p, H, W, f.stride(0) if device else f.strides[0]))
        elif source == "nv12":
            rows.append((p, W, p + H * W, W, H, W))
        elif source == "nv21":
            rows.append(((p, p + H * W, None), W, W, H, W))
        elif source == "i420":
            rows.append(((p, p + H * W, p + H * W + H * W // 4), W, W // 2, H, W))
        else:
            rows.append(((p, None, None), 2 * W, 0, H, W))
        frames.append(f)
    return frames, rows


def _inputs(seed, counts, source, device=False):
    rs = np.random.RandomState(seed)
    frames, table = _frames(rs, len(counts), source, device)
    boxes = [np.round(rs.uniform(-5, 40, (c, 4)) * 2) / 2 for c in counts]       # halves: round-half-to-even shows
    mats = [rs.uniform(-2, 2, (c, 2, 3)) for c in counts]
    centers = [rs.uniform(0, 30, (c, 2)).astype(np.float32) for c in counts]
    scales = [rs.uniform(1, 9, (c, 2)).astype(np.float32) for c in counts]
    heads = [rs.randint(0, len(HEADS), c) for c in counts]
    return frames, table, boxes, mats, centers, scales, heads


def _counts(n_frames, seed):
    rs = np.random.RandomState(seed)
    return [0 if j % 7 == 3 else int(rs.randint(1, 5)) for j in range(n_frames)]


# (max_batch, flip test, box counts per frame, rotate)
CASES = [
    (8, False, [3, 0, 7, 5, 0, 2, 9], [0, 90, 180, 270, 90, 0, 180]),
    (8, True, [3, 0, 7, 5, 0, 2, 9], 270),
    (200, False, _counts(75, 1), [(90 * j) % 360 for j in range(75)]),
    (160, True, _counts(75, 2), 90),
    (64, False, [0, 0], 0),
]
CASE_IDS = ["over_limit", "over_limit_flip", "over_64_frames", "over_64_frames_flip", "no_boxes"]

# host form: (entry point, source, affine, heads, format keyword arguments, format ints)
HOST_FORMS = {
    "infer_frames_host": ("vpb_infer_frames_host", "rgb", False, False, {}, ()),
    "infer_affine_host": ("vpb_infer_affine_host", "rgb", True, False, {}, ()),
    "infer_frames_nv12_host": ("vpb_infer_frames_nv12_host", "nv12", False, False, {"matrix": "bt709"}, (1,)),
    "infer_affine_nv12_host": ("vpb_infer_affine_nv12_host", "nv12", True, False, {"matrix": "bt709"}, (1,)),
    "infer_frames_yuv_host": ("vpb_infer_frames_yuv_host", "yuv", False, False, None, None),
    "infer_affine_yuv_host": ("vpb_infer_affine_yuv_host", "yuv", True, False, None, None),
    "infer_frames_heads_host": ("vpb_infer_frames_heads_host", "rgb", False, True, {}, ()),
    "infer_affine_heads_host": ("vpb_infer_affine_heads_host", "rgb", True, True, {}, ()),
    "infer_frames_heads_yuv_host": ("vpb_infer_frames_heads_yuv_host", "yuv", False, True, None, None),
    "infer_affine_heads_yuv_host": ("vpb_infer_affine_heads_yuv_host", "yuv", True, True, None, None),
}
# the YUV forms run every layout here: (layout, matrix, full_range)
YUV = [("i420", "bt709", True), ("yuyv", "bt601", False), ("nv21", "bt709", False)]


def _forms(table):
    out = []
    for method, (name, source, affine, heads, kw, fmt) in table.items():
        if source != "yuv":
            out.append(pytest.param(method, name, source, affine, heads, kw, fmt, id=method))
            continue
        for lay, mat, full in YUV:
            out.append(pytest.param(method, name, lay, affine, heads, {"layout": lay, "matrix": mat, "full_range": full},
                                    (LAYOUT[lay], MATRIX[mat], int(full)), id=f"{method}-{lay}"))
    return out


# ------------------------------------------------------------------------------------------------ expectations
def _plan(counts, limit, heads=None):
    """The expected calls, stated box by box -> (entries, calls).  An entry is (frame, head, its boxes): every frame with
    boxes, or with heads one per (head, frame) pair that has boxes, head-major.  A call takes boxes in entry order until it
    holds `limit` boxes or would need a 65th entry; it is a list of (entry index, frame, head, boxes)."""
    entries = []
    for k in range(len(HEADS) if heads is not None else 1):
        for j, c in enumerate(counts):
            sel = [b for b in range(c) if heads is None or heads[j][b] == k]
            if sel:
                entries.append((j, k, sel))
    calls = []
    for e, (j, k, sel) in enumerate(entries):
        for b in sel:
            if not calls or sum(len(x[3]) for x in calls[-1]) == limit or (calls[-1][-1][0] != e and len(calls[-1]) == 64):
                calls.append([])
            if not calls[-1] or calls[-1][-1][0] != e:
                calls[-1].append((e, j, k, []))
            calls[-1][-1][3].append(b)
    return entries, calls


def _check_calls(fake, name, struct, table, rot, counts, per_box, fmt, limit, kw, heads=None, host=True, last=STREAM):
    """Asserts the recorded calls; per_box holds per frame the expected rows of every staged per-box array.  Returns
    {(frame, box): (call, row, K of its head)}."""
    entries, calls = _plan(counts, limit, heads)
    assert [c["name"] for c in fake.calls] == [name] * len(calls)
    where, done = {}, 0
    for ci, (rec, call) in enumerate(zip(fake.calls, calls)):
        slot = [e if heads is not None else j for e, j, _, _ in call]         # the table row of each entry of the call
        want = [_row(struct())] * (slot[-1] + 1)
        for s, (e, j, k, bs) in zip(slot, call):
            want[s] = tuple(table[j]) + (len(bs), rot[j])
        assert rec["n"] == len(want) and rec["rows"] == want, f"call {ci}"
        assert rec["fmt"] == fmt
        if heads is None:
            assert rec["heads"] is None
        else:
            assert rec["heads"].tolist() == [entries[e][1] for e in range(len(want))]
        items = [(j, b, k) for _, j, k, bs in call for b in bs]
        if host:
            for got, rows in zip(rec["per_box"], per_box):
                np.testing.assert_array_equal(got, np.stack([rows[j][b] for j, b, _ in items]))
            assert rec["last"] == last
        # every pointer points `done` rows past the first call's
        first = fake.calls[0]
        row_bytes = [a[0].dtype.itemsize * a[0].shape[1] for a in per_box]
        assert [p - p0 for p, p0 in zip(rec["ptrs"], first["ptrs"])] == [done * b for b in row_bytes]
        assert rec["kp"] - first["kp"] == done * kw * 3 * 4 and rec["idx"] - first["idx"] == done * kw * 4
        for r, (j, b, k) in enumerate(items):
            where[(j, b)] = (ci, r, HEADS[k] if heads is not None else kw)
        done += len(items)
    return where


def _check_outputs(kp, idx, counts, where, kw):
    assert len(kp) == len(idx) == len(counts)
    for j, c in enumerate(counts):
        assert isinstance(kp[j], np.ndarray) and isinstance(idx[j], np.ndarray)
        assert kp[j].shape == (c, kw, 3) and idx[j].shape == (c, kw)
        for b in range(c):
            call, r, k = where[(j, b)]
            want_k = np.zeros((kw, 3), np.float32)
            want_i = np.zeros((kw,), np.int32)
            for q in range(k):
                want_k[q] = (call, r, q + 1)
                want_i[q] = 1000 * call + r + 1
            np.testing.assert_array_equal(kp[j][b], want_k)
            np.testing.assert_array_equal(idx[j][b], want_i)


def _expected_per_box(boxes, mats, centers, scales, affine):
    if affine:
        return [[m.reshape(-1, 6) for m in mats], [np.concatenate([c, s], 1) for c, s in zip(centers, scales)]]
    return [[np.rint(b).astype(np.int32) for b in boxes]]


def _struct(source):
    return _lib.VpbFrame if source == "rgb" else _lib.VpbFrameNv12 if source == "nv12" else _lib.VpbFrameYuv


def _call(m, method, frames, boxes, mats, centers, scales, heads, affine, use_heads, kw, rotate, **extra):
    args = [frames] + ([mats, centers, scales] if affine else [boxes]) + ([heads] if use_heads else [])
    return getattr(m, method)(*args, **kw, rotate=rotate, **extra)


# ------------------------------------------------------------------------------------------------ the chunked host forms
@pytest.mark.parametrize("max_batch,flip,counts,rotate", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("method,name,source,affine,use_heads,kw,fmt", _forms(HOST_FORMS))
def test_host_form_calls_and_scatter(fake, method, name, source, affine, use_heads, kw, fmt, max_batch, flip, counts, rotate):
    m = _engine(max_batch, flip, use_heads)
    lib = fake(m)
    seed = 7 * len(counts) + max_batch + sum(map(ord, method + source))
    frames, table, boxes, mats, centers, scales, heads = _inputs(seed, counts, source)
    rot = rotate if isinstance(rotate, list) else [rotate] * len(counts)
    kp, idx = _call(m, method, frames, boxes, mats, centers, scales, heads, affine, use_heads, kw, rotate)
    kwid = max(HEADS) if use_heads else 17
    where = _check_calls(lib, name, _struct(source), table, rot, counts, _expected_per_box(boxes, mats, centers, scales, affine),
                         fmt, m.batch_limit, kwid, heads if use_heads else None)
    _check_outputs(kp, idx, counts, where, kwid)


@pytest.mark.parametrize("method,name,source,affine,use_heads,kw,fmt", _forms(HOST_FORMS))
def test_host_form_without_frames(fake, method, name, source, affine, use_heads, kw, fmt):
    m = _engine(8, False, use_heads)
    lib = fake(m)
    args = [[]] * (1 + (3 if affine else 1) + use_heads)
    assert getattr(m, method)(*args, **kw) == ([], [])
    assert lib.calls == []


# ------------------------------------------------------------------------------------------------ the submit forms
SUBMIT = [
    pytest.param("submit_frames_host", "vpb_submit_frames_host", "rgb", {}, (), id="rgb"),
    pytest.param("submit_frames_nv12_host", "vpb_submit_frames_nv12_host", "nv12", {"matrix": "bt709"}, (1,), id="nv12"),
] + [pytest.param("submit_frames_yuv_host", "vpb_submit_frames_yuv_host", lay,
                  {"layout": lay, "matrix": mat, "full_range": full}, (LAYOUT[lay], MATRIX[mat], int(full)), id=lay)
     for lay, mat, full in YUV]


@pytest.mark.parametrize("method,name,source,kw,fmt", SUBMIT)
def test_submit_form_makes_one_call_over_all_frames(fake, method, name, source, kw, fmt):
    m = _engine(64, False)
    lib = fake(m)
    counts, rot = [3, 0, 4, 1, 2], [90, 0, 270, 180, 0]
    frames, table, boxes, *_ = _inputs(11, counts, source)
    boxes = [np.rint(b).astype(np.int32) for b in boxes]
    n = sum(counts)
    kp, idx = np.zeros((n, 17, 3), np.float32), np.zeros((n, 17), np.int32)
    getattr(m, method)(frames, boxes, kp, idx, 5, **kw, rotate=rot)
    [rec] = lib.calls
    assert rec["name"] == name and rec["fmt"] == fmt and rec["heads"] is None and rec["last"] == 5
    assert rec["rows"] == [tuple(t) + (c, r) for t, c, r in zip(table, counts, rot)]
    np.testing.assert_array_equal(rec["per_box"][0], np.concatenate(boxes))
    assert rec["kp"] == kp.ctypes.data and rec["idx"] == idx.ctypes.data
    assert kp[4, 0].tolist() == [0, 4, 1] and idx[9, 16] == 10       # the outputs are the caller's arrays


@pytest.mark.parametrize("method,name,source,kw,fmt", SUBMIT)
def test_submit_form_errors(fake, method, name, source, kw, fmt):
    m = _engine(64, False)
    fake(m)
    frames, _, boxes, *_ = _inputs(12, [2, 1], source)
    boxes = [np.rint(b).astype(np.int32) for b in boxes]
    kp, idx = np.zeros((3, 17, 3), np.float32), np.zeros((3, 17), np.int32)
    call = getattr(m, method)
    with pytest.raises(ValueError, match="2 frames but 1 box arrays"):
        call(frames, boxes[:1], kp, idx, 0, **kw, rotate=45)
    with pytest.raises(ValueError, match="rotate"):
        call(frames, [boxes[0], boxes[1].astype(np.int64)], kp, idx, 0, **kw, rotate=45)
    with pytest.raises(TypeError, match="boxes of frame 1: int32"):
        call(frames, [boxes[0], boxes[1].astype(np.int64)], kp[:2], idx, 0, **kw)
    with pytest.raises(ValueError, match=f"{method}: outputs must be C-contiguous"):
        call(frames, boxes, kp[:2], idx, 0, **kw)
    with pytest.raises(ValueError, match=f"{method}: outputs must be C-contiguous"):
        call(frames, boxes, kp, idx.astype(np.int64), 0, **kw)


def test_submit_frame_and_box_checks_keep_their_order(fake):
    """submit_frames_host and submit_frames_nv12_host check each frame, then its boxes, frame by frame; submit_frames_yuv_host
    checks every frame's boxes before the frames."""
    m = _engine(64, False)
    fake(m)
    kp, idx = np.zeros((3, 17, 3), np.float32), np.zeros((3, 17), np.int32)
    good_b, bad_b = np.zeros((2, 4), np.int32), np.zeros((1, 4), np.float64)
    rgb = np.zeros((4, 6, 3), np.uint8)
    with pytest.raises(TypeError, match="boxes of frame 0"):
        m.submit_frames_host([rgb, rgb[::2]], [bad_b, good_b], kp, idx, 0)
    with pytest.raises(ValueError, match="frame 0: uint8"):
        m.submit_frames_host([rgb.astype(np.float32), rgb], [bad_b, good_b], kp, idx, 0)
    with pytest.raises(ValueError, match="frame 1: uint8"):
        m.submit_frames_host([rgb, rgb.astype(np.float32)], [good_b, bad_b], kp, idx, 0)
    nv = np.zeros((6, 6), np.uint8)
    with pytest.raises(TypeError, match="boxes of frame 0"):
        m.submit_frames_nv12_host([nv, nv[:, ::2]], [bad_b, good_b], kp, idx, 0)
    with pytest.raises(ValueError, match="frame 1: numpy NV12 planes with contiguous bytes"):
        m.submit_frames_nv12_host([nv, np.zeros((6, 12), np.uint8)[:, ::2]], [good_b, bad_b], kp, idx, 0)
    with pytest.raises(TypeError, match="boxes of frame 1"):
        m.submit_frames_yuv_host([nv, np.zeros((6, 12), np.uint8)[:, ::2]], [good_b, bad_b], kp, idx, 0)
    with pytest.raises(ValueError, match="frame 1: numpy i420 planes with contiguous bytes"):
        m.submit_frames_yuv_host([nv, np.zeros((6, 12), np.uint8)[:, ::2]], [good_b, good_b], kp, idx, 0)


# ------------------------------------------------------------------------------------------------ which error wins
def test_ensure_comes_first():
    m = ViTPose(model_cfg("s", 17), max_batch=8, heads=HEADS)          # no weights: _ensure raises
    for call in (lambda: m.infer_frames_yuv_host([1], [], layout="rgb", rotate=45),
                 lambda: m.infer_affine_heads_host([1], [], [], [], [], rotate=45),
                 lambda: m.submit_frames_nv12_host([1], [], None, None, 0, matrix="x"),
                 lambda: m.infer_frames([1], [], rotate=45)):
        with pytest.raises(RuntimeError, match="load_state_dict"):
            call()


@pytest.mark.parametrize("method,name,source,affine,use_heads,kw,fmt", _forms(HOST_FORMS))
def test_error_precedence(fake, method, name, source, affine, use_heads, kw, fmt):
    """format names, then the length check, then rotate, then the frames, then the boxes or matrices, then the heads."""
    m = _engine(8, False, use_heads)
    fake(m)
    frames, _, boxes, mats, centers, scales, heads = _inputs(5, [2, 3], source)
    bad_frame = [frames[0].astype(np.float32) if source == "rgb" else frames[0][..., :1] if source == "yuyv" else frames[0][:5],
                 frames[1]]
    bad_boxes = [np.zeros(3), boxes[1]]
    bad_mats = [np.zeros((2, 5)), mats[1]]
    bad_heads = [np.array([0, 9]), heads[1]]

    def run(frames=frames, boxes=boxes, mats=mats, heads=heads, short=False, rotate=0, kw=kw):
        fr = frames[:1] if short else frames
        return _call(m, method, fr, boxes, mats, centers, scales, heads, affine, use_heads, kw, rotate)

    if kw:
        bad_kw = dict(kw, **({"layout": "rgb24"} if "layout" in kw else {"matrix": "bt2020"}))
        with pytest.raises(ValueError, match="unknown YUV"):
            run(short=True, rotate=45, kw=bad_kw)
    with pytest.raises(ValueError, match=r"^1 frames(,| but)"):
        run(short=True, rotate=45, frames=bad_frame)
    with pytest.raises(ValueError, match="rotate"):
        run(rotate=45, frames=bad_frame, boxes=bad_boxes, mats=bad_mats)
    with pytest.raises(ValueError, match="^frame 0"):
        run(frames=bad_frame, boxes=bad_boxes, mats=bad_mats, heads=bad_heads)
    with pytest.raises(ValueError, match="matrices of frame 0" if affine else "reshape"):
        run(boxes=bad_boxes, mats=bad_mats, heads=bad_heads)
    if use_heads:
        with pytest.raises(ValueError, match="head indices"):
            run(heads=bad_heads)
        with pytest.raises(ValueError, match="2 boxes but 1 head indices in frame 0"):
            run(heads=[heads[0][:1], heads[1]])


# ------------------------------------------------------------------------------------------------ the device forms
DEVICE_FORMS = {
    "infer_frames": ("vpb_infer_frames", "rgb", False, False, {}, ()),
    "infer_affine": ("vpb_infer_affine", "rgb", True, False, {}, ()),
    "infer_frames_nv12": ("vpb_infer_frames_nv12", "nv12", False, False, {"matrix": "bt709"}, (1,)),
    "infer_affine_nv12": ("vpb_infer_affine_nv12", "nv12", True, False, {"matrix": "bt709"}, (1,)),
    "infer_frames_yuv": ("vpb_infer_frames_yuv", "yuv", False, False, None, None),
    "infer_affine_yuv": ("vpb_infer_affine_yuv", "yuv", True, False, None, None),
    "infer_frames_heads": ("vpb_infer_frames_heads", "rgb", False, True, {}, ()),
    "infer_affine_heads": ("vpb_infer_affine_heads", "rgb", True, True, {}, ()),
    "infer_frames_heads_yuv": ("vpb_infer_frames_heads_yuv", "yuv", False, True, None, None),
    "infer_affine_heads_yuv": ("vpb_infer_affine_heads_yuv", "yuv", True, True, None, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("max_batch,flip,counts,rotate", CASES[:4], ids=CASE_IDS[:4])
@pytest.mark.parametrize("method,name,source,affine,use_heads,kw,fmt", _forms(DEVICE_FORMS))
def test_device_form_calls(fake, method, name, source, affine, use_heads, kw, fmt, max_batch, flip, counts, rotate):
    m = _engine(max_batch, flip, use_heads)
    m._device = torch.cuda.current_device()
    lib = fake(m, host=False)
    seed = 7 * len(counts) + max_batch + sum(map(ord, method + source))
    frames, table, boxes, mats, centers, scales, heads = _inputs(seed, counts, source, device=True)
    rot = rotate if isinstance(rotate, list) else [rotate] * len(counts)
    kp, idx = _call(m, method, frames, boxes, mats, centers, scales, heads, affine, use_heads, kw, rotate)
    torch.cuda.synchronize()
    kwid = max(HEADS) if use_heads else 17
    _check_calls(lib, name, _struct(source), table, rot, counts, _expected_per_box(boxes, mats, centers, scales, affine),
                 fmt, m.batch_limit, kwid, heads if use_heads else None, host=False)
    assert [tuple(k.shape) for k in kp] == [(c, kwid, 3) for c in counts] and all(k.is_cuda for k in kp + idx)
