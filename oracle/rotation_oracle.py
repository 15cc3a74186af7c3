"""Rotated frames in numpy: the addressing contract of the frame gathers for vpb_frame*.rotation (preprocess.cuh: view_hw,
stored_px), restated as integer index arithmetic.

A frame stored as height x width with rotation r (0, 90, 180 or 270 degrees counter-clockwise, the reference's `--rotate`) is
seen as its VIEW, cv2.rotate(stored, ROTATION_MAP[r]) (easy_ViTPose/vit_utils/inference.py:6-11).  The view is width x height
for 90 and 270.  View pixel (x, y) shows stored pixel
  r = 0:   (x, y)            r = 90:  (W-1-y, x)
  r = 180: (W-1-x, H-1-y)    r = 270: (y, H-1-x)
with W, H the stored width and height.  A YUV tap reads that stored pixel's luma and the chroma pair of its STORED block, so a
rotated YUV view equals converting the stored frame and rotating the RGB result.
"""
from __future__ import annotations

import numpy as np

from oracle.yuv_oracle import convert, split_yuv

ROTATIONS = (0, 90, 180, 270)
# the cv2.rotate code of each rotation, by name (the reference's rotation_map, inference.py:173-175); None = no rotation
ROTATION_MAP = {0: None, 90: "ROTATE_90_COUNTERCLOCKWISE", 180: "ROTATE_180", 270: "ROTATE_90_CLOCKWISE"}


def view_size(height: int, width: int, rotation: int) -> "tuple[int, int]":
    """(view height, view width) of a stored height x width frame."""
    if rotation not in ROTATIONS:
        raise ValueError(f"rotation {rotation!r}: one of {ROTATIONS}")
    return (width, height) if rotation in (90, 270) else (height, width)


def stored_px(x, y, height: int, width: int, rotation: int) -> "tuple[np.ndarray, np.ndarray]":
    """View pixel coordinates (x, y) (int arrays of one shape) -> the stored pixel (sx, sy) each one shows: the device's
    axis swap for 90 / 270, then the reflection of stored x (90, 180) and of stored y (180, 270)."""
    code = ROTATIONS.index(rotation)
    x, y = np.asarray(x, np.int64), np.asarray(y, np.int64)
    a, b = (y, x) if code & 1 else (x, y)
    sx = width - 1 - a if code in (1, 2) else a
    sy = height - 1 - b if code & 2 else b
    return sx, sy


def _view_grid(height: int, width: int, rotation: int):
    vh, vw = view_size(height, width, rotation)
    y, x = np.meshgrid(np.arange(vh), np.arange(vw), indexing="ij")
    return stored_px(x, y, height, width, rotation)


def rotate_view(stored: np.ndarray, rotation: int) -> np.ndarray:
    """The view of a stored [H, W, ...] array, gathered pixel by pixel through stored_px."""
    sx, sy = _view_grid(stored.shape[0], stored.shape[1], rotation)
    return stored[sy, sx]


def yuv_view_rgb(frame_or_planes, layout: str, rotation: int, matrix: str = "bt601", full_range: bool = False) -> np.ndarray:
    """uint8 RGB view [H', W', 3] of a stored YUV frame (any yuv_oracle form), tap by tap as the gathers read it: each view
    pixel's stored luma and the chroma pair of its stored block (2x2 for 4:2:0, 2x1 for 4:2:2), then yuv_oracle.convert."""
    Y, U, V = split_yuv(frame_or_planes, layout)
    h, w = Y.shape
    vshift = 1 if U.shape[0] * 2 == h else 0
    sx, sy = _view_grid(h, w, rotation)
    return convert(Y[sy, sx], U[sy >> vshift, sx >> 1], V[sy >> vshift, sx >> 1], matrix, full_range)
