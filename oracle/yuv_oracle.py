"""YUV -> RGB in numpy int64 for every 8-bit layout: the contract of the engine's YUV gathers (vpb_infer_frames_yuv and the
other _yuv calls).  It extends oracle/nv12_oracle.py, whose limited-range formula it reuses unchanged.

Pixel (x, y) takes its own Y and the (U, V) pair of its chroma block (nearest chroma, as cv2 does): 2x2 pixels for the 4:2:0
layouts (NV12, NV21, I420, YV12), 2x1 for the packed 4:2:2 ones (YUYV, UYVY).  Then

  limited range   nv12_oracle's SHIFT-20 formula: cv2 4.13's COLOR_YUV2RGB_{NV12,NV21,I420,YV12,YUY2,UYVY} for bt601
                  (tests/test_yuv_oracle.py checks all six against cv2), its 3-decimal BT.709 form for bt709;
  full range      cv2's COLOR_YCrCb2RGB, SHIFT 14, D(s) = (s + 8192) >> 14, no offset or scale on Y:
                    R = clamp(Y + D(C0 (V - 128))), G = clamp(Y + D(C2 (U - 128) + C1 (V - 128))), B = clamp(Y + D(C3 (U - 128)))
                  bt601 C0..C3 = 22987, -11698, -5636, 29049 (cv2 bit for bit on all 2^24 triples); bt709 the same 3-decimal
                  form, round(2^14 x (1.575, -0.468, -0.187, 1.856)).

Frame forms (what cv2, ffmpeg and V4L2 deliver):
  nv12, nv21   [3H/2, W] with the planes stacked, or (y [H,W], uv [H/2,W]) (vu for nv21)
  i420, yv12   [3H/2, W] with each chroma plane H/2 x W/2 bytes packed after the luma (U first for i420, V first for yv12), or
               (y [H,W], u [H/2,W/2], v [H/2,W/2]) named by content
  yuyv, uyvy   [H, W, 2] or [H, 2W]: Y0 U Y1 V (yuyv) or U Y0 V Y1 (uyvy) per pixel pair
"""
from __future__ import annotations

import numpy as np

from oracle.nv12_oracle import COEFS

LAYOUTS = ("nv12", "nv21", "i420", "yv12", "yuyv", "uyvy")
#                    C0      C1      C2     C3
FULL_COEFS = {"bt601": (22987, -11698, -5636, 29049),
              "bt709": (25805, -7668, -3064, 30409)}
_KR_KB = {"bt601": (0.299, 0.114), "bt709": (0.2126, 0.0722)}


def split_yuv(frame_or_planes, layout: str) -> "tuple[np.ndarray, np.ndarray, np.ndarray]":
    """Any accepted form -> (Y [H,W], U, V) with U and V at chroma resolution ([H/2,W/2] or [H,W/2]), as int64."""
    if layout not in LAYOUTS:
        raise ValueError(f"unknown layout {layout!r}")
    if layout in ("yuyv", "uyvy"):
        f = np.asarray(frame_or_planes)
        h = f.shape[0]
        q = f.reshape(h, -1, 4).astype(np.int64)
        if layout == "yuyv":
            return np.stack([q[..., 0], q[..., 2]], -1).reshape(h, -1), q[..., 1], q[..., 3]
        return np.stack([q[..., 1], q[..., 3]], -1).reshape(h, -1), q[..., 0], q[..., 2]
    if layout in ("nv12", "nv21"):
        if isinstance(frame_or_planes, (tuple, list)):
            y, c = (np.asarray(p) for p in frame_or_planes)
        else:
            f = np.asarray(frame_or_planes)
            y, c = f[: f.shape[0] // 3 * 2], f[f.shape[0] // 3 * 2:]
        a, b = c[:, 0::2].astype(np.int64), c[:, 1::2].astype(np.int64)
        return (y.astype(np.int64),) + ((a, b) if layout == "nv12" else (b, a))
    if isinstance(frame_or_planes, (tuple, list)):
        y, u, v = (np.asarray(p) for p in frame_or_planes)
    else:
        f = np.asarray(frame_or_planes)
        h, w = f.shape[0] // 3 * 2, f.shape[1]
        y, flat = f[:h], np.ascontiguousarray(f[h:]).reshape(-1)
        q = (h // 2) * (w // 2)
        first, second = flat[:q].reshape(h // 2, w // 2), flat[q:].reshape(h // 2, w // 2)
        u, v = (first, second) if layout == "i420" else (second, first)
    return y.astype(np.int64), u.astype(np.int64), v.astype(np.int64)


def convert(Y, U, V, matrix: str = "bt601", full_range: bool = False) -> np.ndarray:
    """Per-pixel (Y, U, V) int arrays of one shape -> uint8 RGB [..., 3], exactly the formulas above."""
    Y, u, v = np.asarray(Y, np.int64), np.asarray(U, np.int64) - 128, np.asarray(V, np.int64) - 128
    if full_range:
        c0, c1, c2, c3 = FULL_COEFS[matrix]
        d = lambda s: (s + (1 << 13)) >> 14
        rgb = np.stack([Y + d(c0 * v), Y + d(c2 * u + c1 * v), Y + d(c3 * u)], -1)
    else:
        cy, cvr, cvg, cug, cub = COEFS[matrix]
        yy = np.maximum(Y - 16, 0) * cy + (1 << 19)
        rgb = np.stack([(yy + cvr * v) >> 20, (yy + cvg * v + cug * u) >> 20, (yy + cub * u) >> 20], -1)
    return np.clip(rgb, 0, 255).astype(np.uint8)


def upsample(Y, U, V) -> "tuple[np.ndarray, np.ndarray]":
    """Chroma at chroma resolution -> per pixel (nearest: each pair covers its 2x2 or 2x1 block)."""
    h, w = Y.shape
    ry = 2 if U.shape[0] * 2 == h else 1
    up = lambda c: np.repeat(np.repeat(c, ry, 0), 2, 1)[:h, :w]
    return up(U), up(V)


def yuv_to_rgb(frame_or_planes, layout: str, matrix: str = "bt601", full_range: bool = False) -> np.ndarray:
    """-> uint8 RGB [H, W, 3] of a frame in any accepted form."""
    Y, U, V = split_yuv(frame_or_planes, layout)
    return convert(Y, *upsample(Y, U, V), matrix, full_range)


def rgb_to_yuv(rgb: np.ndarray, layout: str, matrix: str = "bt601", full_range: bool = False) -> np.ndarray:
    """A test-input helper (not part of the contract): uint8 RGB [H, W, 3] (even width; even height for 4:2:0) -> the frame in
    its stacked form ([3H/2, W] for 4:2:0, [H, W, 2] for 4:2:2), chroma averaged over each block, limited or full range."""
    if layout not in LAYOUTS:
        raise ValueError(f"unknown layout {layout!r}")
    kr, kb = _KR_KB[matrix]
    f = np.asarray(rgb, np.float64)
    h, w = f.shape[:2]
    yl = kr * f[..., 0] + (1 - kr - kb) * f[..., 1] + kb * f[..., 2]
    cb = (f[..., 2] - yl) / (2 * (1 - kb))
    cr = (f[..., 0] - yl) / (2 * (1 - kr))
    ys, cs, y0 = (1.0, 1.0, 0.0) if full_range else (219 / 255, 224 / 255, 16.0)
    packed = layout in ("yuyv", "uyvy")
    ry = 1 if packed else 2
    pool = lambda c: c.reshape(h // ry, ry, w // 2, 2).mean((1, 3))
    Y = np.clip(np.rint(y0 + yl * ys), 0, 255).astype(np.uint8)
    U = np.clip(np.rint(128 + pool(cb) * cs), 0, 255).astype(np.uint8)
    V = np.clip(np.rint(128 + pool(cr) * cs), 0, 255).astype(np.uint8)
    if packed:
        y2 = Y.reshape(h, w // 2, 2)
        q = np.stack([y2[..., 0], U, y2[..., 1], V] if layout == "yuyv" else [U, y2[..., 0], V, y2[..., 1]], -1)
        return q.reshape(h, w, 2)
    if layout in ("nv12", "nv21"):
        c = np.stack([U, V] if layout == "nv12" else [V, U], -1).reshape(h // 2, w)
        return np.concatenate([Y, c], 0)
    first, second = (U, V) if layout == "i420" else (V, U)
    return np.concatenate([Y.reshape(-1), first.reshape(-1), second.reshape(-1)]).reshape(3 * h // 2, w)
