"""CPU: the rotated-frame contract (vpb_frame*.rotation, the `rotate` argument of the ViTPose frame methods).  Pins the
direction convention (rotation r is np.rot90(img, r // 90) and the reference's cv2.rotate code), the numpy restatement of
the gathers' view -> stored map (oracle/rotation_oracle.py) on RGB and on every YUV layout, the C structs' layout and the
Python-side validation of `rotate`."""
import ctypes as C

import numpy as np
import pytest

from oracle.rotation_oracle import ROTATION_MAP, ROTATIONS, rotate_view, stored_px, view_size, yuv_view_rgb
from oracle.yuv_oracle import LAYOUTS, rgb_to_yuv, yuv_to_rgb

SIZES = [(7, 5), (5, 9), (1, 4), (33, 18), (2, 2)]          # odd-sized and non-square (h, w)


def _rgb(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("rotation", ROTATIONS)
@pytest.mark.parametrize("h,w", SIZES)
def test_rot90_is_the_references_cv2_rotate(rotation, h, w):
    cv2 = pytest.importorskip("cv2")
    img = _rgb(h, w, 13 * h + w)
    ref = img if ROTATION_MAP[rotation] is None else cv2.rotate(img, getattr(cv2, ROTATION_MAP[rotation]))
    assert np.array_equal(np.rot90(img, k=rotation // 90), ref)


@pytest.mark.parametrize("rotation", ROTATIONS)
@pytest.mark.parametrize("h,w", SIZES)
def test_view_to_stored_map_reproduces_rot90(rotation, h, w):
    img = _rgb(h, w, 31 * h + w + rotation)
    view = rotate_view(img, rotation)
    assert view.shape[:2] == view_size(h, w, rotation)
    assert np.array_equal(view, np.rot90(img, k=rotation // 90))


@pytest.mark.parametrize("rotation", ROTATIONS)
def test_map_is_a_permutation_of_the_stored_pixels(rotation):
    h, w = 7, 12
    vh, vw = view_size(h, w, rotation)
    y, x = np.meshgrid(np.arange(vh), np.arange(vw), indexing="ij")
    sx, sy = stored_px(x, y, h, w, rotation)
    assert sx.min() >= 0 and sx.max() < w and sy.min() >= 0 and sy.max() < h
    assert len(set(zip(sx.ravel().tolist(), sy.ravel().tolist()))) == h * w


@pytest.mark.parametrize("full_range", [False, True])
@pytest.mark.parametrize("rotation", ROTATIONS)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_yuv_taps_read_the_stored_chroma_block(layout, rotation, full_range):
    packed = layout in ("yuyv", "uyvy")
    for h, w in ([(5, 6), (8, 4), (1, 10)] if packed else [(6, 10), (12, 4), (2, 2)]):
        rs = np.random.RandomState(h * 101 + w + LAYOUTS.index(layout))
        frame = rgb_to_yuv(rs.randint(0, 256, size=(h, w, 3), dtype=np.uint8), layout, "bt601", full_range)
        if not packed:                                     # random chroma too, so a wrong block shows
            frame[h:] = rs.randint(0, 256, size=frame[h:].shape, dtype=np.uint8)
        else:
            frame = rs.randint(0, 256, size=frame.shape, dtype=np.uint8)
        want = np.rot90(yuv_to_rgb(frame, layout, "bt601", full_range), k=rotation // 90)
        assert np.array_equal(yuv_view_rgb(frame, layout, rotation, "bt601", full_range), want), (h, w)


def test_bad_rotation_in_the_oracle():
    with pytest.raises(ValueError):
        view_size(4, 4, 45)


def test_struct_layout_keeps_sizes_and_offsets():
    from easy_vitpose_b200 import _lib
    expect = {
        _lib.VpbFrame: (32, {"data": 0, "height": 8, "width": 12, "pitch_bytes": 16, "num_boxes": 24, "rotation": 28}),
        _lib.VpbFrameNv12: (48, {"y": 0, "y_pitch": 8, "uv": 16, "uv_pitch": 24, "height": 32, "width": 36, "num_boxes": 40,
                                 "rotation": 44}),
        _lib.VpbFrameYuv: (56, {"plane": 0, "y_pitch": 24, "c_pitch": 32, "height": 40, "width": 44, "num_boxes": 48,
                                "rotation": 52}),
    }
    for struct, (size, offs) in expect.items():
        assert C.sizeof(struct) == size, struct.__name__
        assert {f: getattr(struct, f).offset for f, _ in struct._fields_} == offs, struct.__name__
        assert struct().rotation == 0                      # zero-initialised: upright
    assert _lib.ROTATIONS == ROTATIONS


def test_header_declares_rotation_last_in_every_frame_struct():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "vitpose_b200.h")).read()
    for name in ("vpb_frame", "vpb_frame_nv12", "vpb_frame_yuv"):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
        members = [ln.split("/*")[0].strip() for ln in body.strip().splitlines() if ln.split("/*")[0].strip()]
        assert members[-1] == "int32_t rotation;", name


@pytest.mark.parametrize("rotate", [45, -90, 360, 1, [0, 90], [0, 90, 180, 270], 90.0, True, "90", [[0, 90, 180]]])
def test_rotate_argument_is_validated(rotate):
    from easy_vitpose_b200.model import _rotations
    with pytest.raises(ValueError):
        _rotations(rotate, 3)


def test_rotate_argument_forms():
    import torch
    from easy_vitpose_b200.model import _rotations
    assert _rotations(0, 3) == [0, 0, 0]
    assert _rotations(270, 2) == [270, 270]
    assert _rotations(np.int64(90), 1) == [90]
    assert _rotations([0, 90, 180], 3) == [0, 90, 180]
    assert _rotations(np.array([270, 0], np.int32), 2) == [270, 0]
    assert _rotations(torch.tensor([180, 90]), 2) == [180, 90]
    assert _rotations([], 0) == [] and _rotations(90, 0) == []


def test_frame_array_carries_each_frames_rotation():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.model import _frame_array
    table = [(1000 + j, 10 + j, 20 + j, 60 + 3 * j) for j in range(4)]
    arr = _frame_array(table, [(1, 2, 5), (3, 0, 1)], rot=[0, 90, 180, 270])
    assert [(f.num_boxes, f.rotation) for f in arr] == [(0, 0), (3, 90), (0, 0), (1, 270)]
    ytab = [((1, 2, None), 8, 4, 6, 8)] * 2
    arr = _frame_array(ytab, [(0, 0, 2), (1, 0, 1)], _lib.VpbFrameYuv, [180, 90])
    assert [(f.num_boxes, f.rotation, f.height) for f in arr] == [(2, 180, 6), (1, 90, 6)]
    assert [f.rotation for f in _frame_array(table, [(0, 0, 1)])] == [0]


def test_head_planning_gives_each_entry_its_frames_rotation():
    """The multi-head methods map `rotate` through plan_head_calls' entries: a frame that appears once per head keeps its
    rotation in every entry."""
    from easy_vitpose_b200.model import _frame_array, _rotations, plan_head_calls
    rot = _rotations([90, 0, 270], 3)
    ents, _, chunks = plan_head_calls([2, 1, 3], [[0, 1], [1], [1, 0, 1]], 2, 64)
    erot = [rot[j] for j, _, _ in ents]
    assert [(j, k) for j, _, k in ents] == [(0, 0), (2, 0), (0, 1), (1, 1), (2, 1)]
    assert erot == [90, 270, 90, 0, 270]
    table = [(j, 8, 8, 24) for j, _, _ in ents]
    arr = _frame_array(table, chunks[0], rot=erot)
    assert [(f.data, f.rotation) for f in arr] == [(None, 90), (2, 270), (None, 90), (1, 0), (2, 270)]
