"""CPU: the YUV -> RGB oracle (oracle/yuv_oracle.py) that the GPU YUV gathers are held to, the splitting of YUV frames into
the planes of vpb_frame_yuv (easy_vitpose_b200.model.yuv_planes) and the host-side argument checks of the _yuv calls.
Limited-range BT.601 is pinned against cv2's COLOR_YUV2RGB_* for all six layouts, full-range BT.601 against
COLOR_YCrCb2RGB on every (Y, U, V) triple, and both BT.709 sets against the exact float formula."""
import numpy as np
import pytest

from oracle.nv12_oracle import nv12_to_rgb
from oracle.yuv_oracle import FULL_COEFS, LAYOUTS, convert, rgb_to_yuv, split_yuv, upsample, yuv_to_rgb

CV2_CODES = {"nv12": "COLOR_YUV2RGB_NV12", "nv21": "COLOR_YUV2RGB_NV21", "i420": "COLOR_YUV2RGB_I420",
             "yv12": "COLOR_YUV2RGB_YV12", "yuyv": "COLOR_YUV2RGB_YUY2", "uyvy": "COLOR_YUV2RGB_UYVY"}


def _random_frame(layout, h, w, seed):
    rs = np.random.RandomState(seed)
    shape = (h, w, 2) if layout in ("yuyv", "uyvy") else (3 * h // 2, w)
    return rs.randint(0, 256, size=shape, dtype=np.uint8)


def _all_triples():
    """A 512 x 32768 NV12 frame holding every (Y, U, V): chroma block b carries (U, V) = divmod(b // 64, 256) and the four Y
    values 4 (b % 64) + 0..3, so each (U, V) pair meets all 256 Y.  Returns the stacked frame and Y, U, V per pixel."""
    br, bc = np.meshgrid(np.arange(256), np.arange(16384), indexing="ij")
    b = br * 16384 + bc
    u, v = np.divmod(b // 64, 256)
    uv = np.stack([u, v], -1).reshape(256, 32768).astype(np.uint8)
    dy, dx = np.meshgrid(np.arange(2), np.arange(2), indexing="ij")
    y = ((4 * (b % 64))[:, None, :, None] + (2 * dy + dx)[None, :, None, :]).reshape(512, 32768).astype(np.uint8)
    U = np.repeat(np.repeat(u, 2, 0), 2, 1)
    V = np.repeat(np.repeat(v, 2, 0), 2, 1)
    return np.concatenate([y, uv], 0), y.astype(np.int64), U, V


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("h,w", [(2, 2), (10, 6), (34, 66), (6, 20), (1080, 1920)])
def test_limited_bt601_equals_cv2(layout, h, w):
    cv2 = pytest.importorskip("cv2")
    frame = _random_frame(layout, h, w, h * 7919 + w + LAYOUTS.index(layout))
    assert np.array_equal(yuv_to_rgb(frame, layout, "bt601"), cv2.cvtColor(frame, getattr(cv2, CV2_CODES[layout])))


def test_limited_nv12_is_the_nv12_oracle():
    frame = _random_frame("nv12", 34, 66, 1)
    for matrix in ("bt601", "bt709"):
        assert np.array_equal(yuv_to_rgb(frame, "nv12", matrix), nv12_to_rgb(frame, matrix))


def test_full_range_bt601_equals_cv2_ycrcb_on_every_triple():
    cv2 = pytest.importorskip("cv2")
    frame, Y, U, V = _all_triples()
    assert len(np.unique((Y << 16) | (U << 8) | V)) == 1 << 24
    ycrcb = np.stack([Y, V, U], -1).astype(np.uint8)
    assert np.array_equal(yuv_to_rgb(frame, "nv12", "bt601", True), cv2.cvtColor(ycrcb, cv2.COLOR_YCrCb2RGB))


@pytest.mark.parametrize("layout", LAYOUTS)
def test_full_range_bt601_is_nearest_chroma_then_cv2_ycrcb(layout):
    cv2 = pytest.importorskip("cv2")
    frame = _random_frame(layout, 18, 26, 40 + LAYOUTS.index(layout))
    Y, U, V = split_yuv(frame, layout)
    U, V = upsample(Y, U, V)
    ycrcb = np.stack([Y, V, U], -1).astype(np.uint8)
    assert np.array_equal(yuv_to_rgb(frame, layout, "bt601", True), cv2.cvtColor(ycrcb, cv2.COLOR_YCrCb2RGB))


def _exact(Y, U, V, matrix, full):
    kr, kb = (0.299, 0.114) if matrix == "bt601" else (0.2126, 0.0722)
    kg = 1 - kr - kb
    ys, cs = (1.0, 1.0) if full else (255 / 219, 255 / 224)
    yl = ys * (Y if full else np.maximum(Y - 16, 0)).astype(np.float64)
    u, v = cs * (U - 128).astype(np.float64), cs * (V - 128).astype(np.float64)
    out = np.stack([yl + 2 * (1 - kr) * v, yl - 2 * (1 - kb) * kb / kg * u - 2 * (1 - kr) * kr / kg * v, yl + 2 * (1 - kb) * u], -1)
    return np.clip(np.rint(out), 0, 255)


@pytest.mark.parametrize("matrix,full", [("bt709", True), ("bt601", True), ("bt709", False)])
def test_within_one_level_of_the_exact_formula_on_every_triple(matrix, full):
    _, Y, U, V = _all_triples()
    got = convert(Y, U, V, matrix, full).astype(np.float64)
    assert np.abs(got - _exact(Y, U, V, matrix, full)).max() <= 1


def test_full_range_coefficients_are_the_three_decimal_forms():
    assert FULL_COEFS["bt709"] == tuple(int(round(c * (1 << 14))) for c in (1.575, -0.468, -0.187, 1.856))
    assert FULL_COEFS["bt601"] == (22987, -11698, -5636, 29049)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("full", [False, True])
def test_round_trip_and_forms(layout, full):
    """rgb_to_yuv builds plausible inputs; the stacked / packed, split and [H, 2W] forms convert alike."""
    yy, xx = np.mgrid[0:34, 0:66]
    rgb = np.stack([xx * 3, yy * 7, 255 - xx * 2], -1).astype(np.uint8)              # smooth: the chroma blocks lose little
    f = rgb_to_yuv(rgb, layout, "bt709", full)
    assert f.dtype == np.uint8 and f.shape == ((34, 66, 2) if layout in ("yuyv", "uyvy") else (51, 66))
    assert np.abs(yuv_to_rgb(f, layout, "bt709", full).astype(int) - rgb).mean() < 3
    ref = yuv_to_rgb(f, layout, "bt601", full)
    if layout in ("yuyv", "uyvy"):
        assert np.array_equal(yuv_to_rgb(f.reshape(34, 132), layout, "bt601", full), ref)
    elif layout in ("nv12", "nv21"):
        assert np.array_equal(yuv_to_rgb((f[:34].copy(), f[34:].copy()), layout, "bt601", full), ref)
    else:
        c = f[34:].reshape(-1)
        a, b = c[:17 * 33].reshape(17, 33), c[17 * 33:].reshape(17, 33)
        u, v = (a, b) if layout == "i420" else (b, a)
        assert np.array_equal(yuv_to_rgb((f[:34], u, v), layout, "bt601", full), ref)


# ------------------------------------------------------------------------------------------------ the package's host side
@pytest.mark.parametrize("layout", LAYOUTS)
def test_yuv_planes_match_the_oracle(layout):
    """yuv_planes gives the planes in storage order as views; reading them with the layout's offsets (those the engine puts
    in its table) gives the oracle's Y, U and V, for numpy arrays and torch tensors."""
    import torch

    from easy_vitpose_b200.model import yuv_planes
    f = _random_frame(layout, 10, 14, 3)                                            # H/2 odd: I420 chroma is not row-aligned
    Y, U, V = split_yuv(f, layout)
    for frame in (f, torch.from_numpy(f)):
        planes, h, w = yuv_planes(frame, layout)
        assert (h, w) == (10, 14)
        p = [np.asarray(x) for x in planes]
        if layout in ("yuyv", "uyvy"):
            assert len(p) == 1 and p[0].shape == (10, 28)
            assert np.shares_memory(planes[0], f) or not isinstance(frame, np.ndarray)
            q = p[0].reshape(10, 7, 4).astype(np.int64)
            o = (0, 1, 3) if layout == "yuyv" else (1, 0, 2)
            assert np.array_equal(q[..., o[1]], U) and np.array_equal(q[..., o[2]], V)
            assert np.array_equal(np.stack([q[..., o[0]], q[..., o[0] + 2]], -1).reshape(10, 14), Y)
        elif layout in ("nv12", "nv21"):
            assert len(p) == 2 and p[1].shape == (5, 14)
            first, second = p[1][:, 0::2], p[1][:, 1::2]
            assert np.array_equal(*((first, U) if layout == "nv12" else (first, V)))
            assert np.array_equal(*((second, V) if layout == "nv12" else (second, U)))
        else:
            assert len(p) == 3 and p[1].shape == (5, 7) and p[2].shape == (5, 7)
            assert np.array_equal(p[1], U if layout == "i420" else V) and np.array_equal(p[2], V if layout == "i420" else U)
        assert layout in ("yuyv", "uyvy") or np.array_equal(p[0], Y)
    # the yuyv [H, W, 2] form and the [H, 2W] form give the same plane
    if layout in ("yuyv", "uyvy"):
        assert np.array_equal(yuv_planes(f.reshape(10, 28), layout)[0][0], yuv_planes(f, layout)[0][0])


def test_yuv_planes_rejects_bad_frames():
    import torch

    from easy_vitpose_b200.model import yuv_planes
    z = lambda *s: np.zeros(s, np.uint8)
    bad = [("i420", z(16, 20)), ("i420", z(15, 21)), ("yv12", z(3, 20)[:0]), ("i420", z(15, 20).astype(np.float32)),
           ("i420", (z(10, 20), z(5, 10))),                                        # two planes for a planar layout
           ("i420", (z(10, 20), z(5, 10), z(5, 11))),                              # mismatched chroma
           ("yv12", (z(10, 20), z(6, 10), z(6, 10))),
           ("i420", (z(9, 20), z(4, 10), z(4, 10))),                               # odd height
           ("i420", (z(10, 20), z(5, 10), torch.zeros((5, 10), dtype=torch.uint8))),   # mixed types
           ("nv21", (z(10, 20), z(5, 22))), ("nv12", z(15, 21)),
           ("yuyv", z(10, 7, 2)), ("uyvy", z(10, 14)), ("yuyv", z(10, 8, 3)), ("uyvy", (z(10, 16),)), ("yuyv", z(10, 16, 2, 1)),
           ("yuyv", z(10, 16).astype(np.int16))]
    for layout, f in bad:
        with pytest.raises(ValueError):
            yuv_planes(f, layout)
    for name in ("yuv444", "p010", "", None):
        with pytest.raises(ValueError):
            yuv_planes(z(15, 20), name)
    assert yuv_planes(z(3, 20), "yuyv")[1:] == (3, 10)                           # 4:2:2: any height


def test_format_names_and_host_table_checks():
    from easy_vitpose_b200.model import ViTPose, _yuv_format
    assert _yuv_format("I420", "BT709", True) == (2, 1, 1) and _yuv_format("uyvy", "bt601", False) == (5, 0, 0)
    for args in (("i444", "bt601", False), ("nv12", "bt2020", False), ("nv16", "bt709", True)):
        with pytest.raises(ValueError):
            _yuv_format(*args)
    f = _random_frame("i420", 10, 20, 4)
    keep, table = ViTPose._yuv_host_table([f], "i420")
    (ptrs, yp, cp, h, w), = table
    assert (yp, cp, h, w) == (20, 10, 10, 20) and ptrs[0] == f.ctypes.data and ptrs[1] == f.ctypes.data + 200
    assert ptrs[2] == f.ctypes.data + 250
    keep, table = ViTPose._yuv_host_table([_random_frame("yuyv", 6, 8, 5)], "yuyv")
    assert table[0][1:] == (16, 0, 6, 8) and table[0][0][1:] == (None, None)
    # short pitches (rows overlapping the next) and U / V planes of different pitches: copied packed, or refused where the
    # pipelined form cannot copy
    y = np.lib.stride_tricks.as_strided(np.zeros(400, np.uint8), (10, 20), (10, 1))
    u, v = np.zeros((5, 10), np.uint8), np.zeros((5, 30), np.uint8)[:, :10]
    for frame in ((y, u, u.copy()), (np.zeros((10, 20), np.uint8), u, v)):
        keep, table = ViTPose._yuv_host_table([frame], "i420")
        assert table[0][1] >= 20 and table[0][2] == 10
        with pytest.raises(ValueError):
            ViTPose._yuv_host_table([frame], "i420", copy=False)


def test_library_exports_every_declared_yuv_call():
    import ctypes
    import os
    import re

    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.build import LIB, build
    build()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vitpose_b200.h")).read()
    declared = set(re.findall(r"\b(vpb_\w*_yuv\w*)\s*\(", hdr))
    assert len(declared) == 9 and declared <= set(_lib.EXPORTS), declared - set(_lib.EXPORTS)
    lib = ctypes.CDLL(LIB)
    assert all(hasattr(lib, name) for name in declared)
    assert ctypes.sizeof(_lib.VpbFrameYuv) == 56
    for name, v in _lib.YUV_LAYOUTS.items():
        assert re.search(rf"#define VPB_YUV_{name.upper()} {v}\b", hdr)
    assert re.search(r"#define VPB_YUV_LIMITED 0\b", hdr) and re.search(r"#define VPB_YUV_FULL 1\b", hdr)
    assert _lib.YUV_RANGES == {"limited": 0, "full": 1}
