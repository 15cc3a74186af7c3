"""CPU: the NV12 -> RGB oracle (oracle/nv12_oracle.py) that the GPU NV12 gathers are held to, and the splitting of NV12
frames into planes (easy_vitpose_b200.model.nv12_planes).  BT.601 is pinned against cv2's COLOR_YUV2RGB_NV12 on every
(Y, U, V) triple and on frame sizes that run cv2's scalar tail; BT.709 against the exact float formula."""
import numpy as np
import pytest

from oracle.nv12_oracle import COEFS, nv12_to_rgb, rgb_to_nv12, split_nv12


def _all_triples():
    """One 512 x 32768 NV12 image holding every (Y, U, V): chroma block b carries (U, V) = divmod(b // 64, 256) and the
    four Y values 4 (b % 64) + 0..3, so each (U, V) pair meets all 256 Y.  Returns the stacked frame and Y, U, V per pixel."""
    br, bc = np.meshgrid(np.arange(256), np.arange(16384), indexing="ij")
    b = br * 16384 + bc
    u, v = np.divmod(b // 64, 256)
    uv = np.stack([u, v], -1).reshape(256, 32768).astype(np.uint8)
    dy, dx = np.meshgrid(np.arange(2), np.arange(2), indexing="ij")
    y4 = (4 * (b % 64))[:, None, :, None] + (2 * dy + dx)[None, :, None, :]       # [256, 2, 16384, 2]
    y = y4.reshape(512, 32768).astype(np.uint8)
    frame = np.concatenate([y, uv], 0)
    U = np.repeat(np.repeat(u, 2, 0), 2, 1)
    V = np.repeat(np.repeat(v, 2, 0), 2, 1)
    return frame, y.astype(np.int64), U, V


def test_the_exhaustive_image_holds_every_triple():
    _, Y, U, V = _all_triples()
    assert len(np.unique((Y << 16) | (U << 8) | V)) == 1 << 24


def test_bt601_equals_cv2_on_every_triple():
    cv2 = pytest.importorskip("cv2")
    frame = _all_triples()[0]
    assert np.array_equal(nv12_to_rgb(frame, "bt601"), cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12))


@pytest.mark.parametrize("h", [2, 10, 34, 1080])
@pytest.mark.parametrize("w", [2, 6, 18, 66, 1920])
def test_bt601_equals_cv2_on_random_frames(h, w):
    cv2 = pytest.importorskip("cv2")
    frame = np.random.RandomState(h * 7919 + w).randint(0, 256, size=(3 * h // 2, w), dtype=np.uint8)
    assert np.array_equal(nv12_to_rgb(frame, "bt601"), cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12))


def test_bt709_within_one_level_of_the_exact_formula():
    """The exact limited-range BT.709 inverse (Kr = 0.2126, Kb = 0.0722; luma 255/219, chroma 255/224), with cv2's clamp of
    Y below 16, rounded: the fixed-point constants stay within one level of it for every triple."""
    frame, Y, U, V = _all_triples()
    kr, kb = 0.2126, 0.0722
    kg = 1 - kr - kb
    ys, cs = 255 / 219, 255 / 224
    yl = ys * np.maximum(Y - 16, 0).astype(np.float64)
    u, v = (U - 128).astype(np.float64), (V - 128).astype(np.float64)
    exact = np.stack([yl + cs * 2 * (1 - kr) * v,
                      yl - cs * 2 * (1 - kb) * kb / kg * u - cs * 2 * (1 - kr) * kr / kg * v,
                      yl + cs * 2 * (1 - kb) * u], -1)
    exact = np.clip(np.rint(exact), 0, 255)
    got = nv12_to_rgb(frame, "bt709").astype(np.float64)
    assert np.abs(got - exact).max() <= 1
    assert not np.array_equal(nv12_to_rgb(frame, "bt709"), nv12_to_rgb(frame, "bt601"))


def test_coefficients_are_the_three_decimal_forms():
    for name, dec in (("bt601", (1.164, 1.596, -0.813, -0.391, 2.018)), ("bt709", (1.164, 1.793, -0.533, -0.213, 2.112))):
        assert COEFS[name] == tuple(int(round(c * (1 << 20))) for c in dec)


def test_stacked_and_split_forms_agree():
    rs = np.random.RandomState(5)
    frame = rs.randint(0, 256, size=(3 * 34 // 2, 66), dtype=np.uint8)
    y, uv = split_nv12(frame)
    assert y.shape == (34, 66) and uv.shape == (17, 66)
    assert np.array_equal(nv12_to_rgb(frame), nv12_to_rgb((y.copy(), uv.copy())))
    yy, xx = np.mgrid[0:34, 0:66]
    rgb = np.stack([xx * 3, yy * 7, 255 - xx * 2], -1).astype(np.uint8)              # smooth: the 2x2 chroma loses little
    for matrix in ("bt601", "bt709"):
        nv = rgb_to_nv12(rgb, matrix)
        assert nv.shape == (51, 66) and nv.dtype == np.uint8
        assert np.abs(nv12_to_rgb(nv, matrix).astype(int) - rgb).mean() < 3          # a plausible round trip, not an exact one


def test_nv12_planes_splits_and_rejects_odd_sizes():
    import torch

    from easy_vitpose_b200.model import nv12_planes
    rs = np.random.RandomState(6)
    frame = rs.randint(0, 256, size=(15, 20), dtype=np.uint8)                        # H = 10, W = 20
    y, uv = nv12_planes(frame)
    assert y.shape == (10, 20) and uv.shape == (5, 20) and np.shares_memory(y, frame) and np.shares_memory(uv, frame)
    assert np.array_equal(np.concatenate([y, uv]), frame)
    ty, tuv = nv12_planes(torch.from_numpy(frame))
    assert ty.shape == (10, 20) and tuv.shape == (5, 20) and tuv.data_ptr() == ty.data_ptr() + 200
    wide = rs.randint(0, 256, size=(10, 32), dtype=np.uint8)                         # planes as column slices: pitch > width
    wuv = rs.randint(0, 256, size=(5, 40), dtype=np.uint8)
    y2, uv2 = nv12_planes((wide[:, 4:24], wuv[:, 6:26]))
    assert y2.shape == (10, 20) and uv2.strides == (40, 1)
    for bad in (np.zeros((16, 20), np.uint8),                                       # rows not 3H/2
                np.zeros((15, 21), np.uint8),                                       # odd width
                np.zeros((3, 20), np.uint8)[:0],                                    # empty
                (np.zeros((9, 20), np.uint8), np.zeros((4, 20), np.uint8)),          # odd height
                (np.zeros((10, 20), np.uint8), np.zeros((5, 22), np.uint8)),         # mismatched uv
                (np.zeros((10, 20), np.uint8), np.zeros((6, 20), np.uint8)),
                (np.zeros((10, 20), np.uint8), torch.zeros((5, 20), dtype=torch.uint8)),   # mixed types
                np.zeros((15, 20), np.float32),
                np.zeros((15, 20, 1), np.uint8),
                (np.zeros((10, 20), np.uint8),)):
        with pytest.raises(ValueError):
            nv12_planes(bad)
    with pytest.raises(ValueError):
        split_nv12(np.zeros((15, 21), np.uint8))


def test_library_exports_every_declared_nv12_call():
    import ctypes
    import os
    import re

    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.build import LIB, build
    build()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vitpose_b200.h")).read()
    declared = set(re.findall(r"\b(vpb_[a-z0-9_]*nv12[a-z0-9_]*)\s*\(", hdr))
    assert declared == set(_lib.EXPORTS_NV12) and len(declared) == 5, declared ^ set(_lib.EXPORTS_NV12)
    lib = ctypes.CDLL(LIB)
    assert all(hasattr(lib, name) for name in declared)
    assert ctypes.sizeof(_lib.VpbFrameNv12) == 48
    assert re.search(r"#define VPB_YUV_BT601 0\b", hdr) and re.search(r"#define VPB_YUV_BT709 1\b", hdr)
    assert _lib.YUV_MATRICES == {"bt601": 0, "bt709": 1}


def test_unknown_matrix_is_rejected_in_python():
    from easy_vitpose_b200.model import _yuv_matrix
    assert _yuv_matrix("bt601") == 0 and _yuv_matrix("BT709") == 1
    with pytest.raises(ValueError):
        _yuv_matrix("bt2020")
