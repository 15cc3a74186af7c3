"""NV12 -> RGB in numpy int64: the contract of the engine's NV12 gathers (vpb_infer_frames_nv12 / vpb_infer_affine_nv12).

Pixel (x, y) of an even-sized NV12 frame takes Y = y_plane[y, x] and the (U, V) pair uv_plane[y // 2, 2 (x // 2) : +2]
(nearest chroma, one pair per 2x2 block, as cv2 does), then with SHIFT = 20, half = 1 << 19:

    yy = max(Y - 16, 0) * CY
    R  = clamp((yy + half + CVR (V - 128)) >> 20, 0, 255)
    G  = clamp((yy + half + CVG (V - 128) + CUG (U - 128)) >> 20, 0, 255)
    B  = clamp((yy + half + CUB (U - 128)) >> 20, 0, 255)

bt601 is cv2 4.13's COLOR_YUV2RGB_NV12 bit for bit (tests/test_nv12_oracle.py checks all 2^24 triples); bt709 uses
round(2^20 x (1.164, 1.793, -0.533, -0.213, 2.112)), the same 3-decimal form for limited-range BT.709.
"""
from __future__ import annotations

import numpy as np

#               CY       CVR      CVG      CUG      CUB
COEFS = {"bt601": (1220542, 1673527, -852492, -409993, 2116026),
         "bt709": (1220542, 1880097, -558891, -223347, 2214593)}


def split_nv12(frame_or_planes) -> "tuple[np.ndarray, np.ndarray]":
    """uint8 [3H/2, W] with the planes stacked, or a (y [H,W], uv [H/2,W]) pair -> (y, uv) numpy planes."""
    if isinstance(frame_or_planes, (tuple, list)):
        y, uv = (np.asarray(p) for p in frame_or_planes)
    else:
        f = np.asarray(frame_or_planes)
        if f.ndim != 2 or f.shape[0] % 3:
            raise ValueError(f"NV12 [3H/2, W] expected, got {f.shape}")
        y, uv = f[: f.shape[0] // 3 * 2], f[f.shape[0] // 3 * 2:]
    h, w = y.shape
    if h % 2 or w % 2 or uv.shape != (h // 2, w):
        raise ValueError(f"even-sized y plane and uv [H/2, W] expected, got {y.shape} / {uv.shape}")
    return y, uv


def nv12_to_rgb(frame_or_planes, matrix: str = "bt601") -> np.ndarray:
    """-> uint8 RGB [H, W, 3], exactly the formula above."""
    cy, cvr, cvg, cug, cub = COEFS[matrix]
    y, uv = split_nv12(frame_or_planes)
    h, w = y.shape
    Y = y.astype(np.int64)
    u = np.repeat(np.repeat(uv[:, 0::2].astype(np.int64) - 128, 2, 0), 2, 1)[:h, :w]
    v = np.repeat(np.repeat(uv[:, 1::2].astype(np.int64) - 128, 2, 0), 2, 1)[:h, :w]
    yy = np.maximum(Y - 16, 0) * cy + (1 << 19)
    rgb = np.stack([(yy + cvr * v) >> 20, (yy + cvg * v + cug * u) >> 20, (yy + cub * u) >> 20], -1)
    return np.clip(rgb, 0, 255).astype(np.uint8)


def rgb_to_nv12(rgb: np.ndarray, matrix: str = "bt601") -> np.ndarray:
    """A test-input helper (not part of the contract): uint8 RGB [H, W, 3], H and W even -> stacked NV12 [3H/2, W], limited
    range, chroma averaged over each 2x2 block."""
    kr, kb = (0.299, 0.114) if matrix == "bt601" else (0.2126, 0.0722)
    f = np.asarray(rgb, np.float64)
    h, w = f.shape[:2]
    yl = kr * f[..., 0] + (1 - kr - kb) * f[..., 1] + kb * f[..., 2]
    cb = (f[..., 2] - yl) / (2 * (1 - kb))
    cr = (f[..., 0] - yl) / (2 * (1 - kr))
    Y = np.clip(np.rint(16 + yl * 219 / 255), 0, 255)
    pool = lambda c: c.reshape(h // 2, 2, w // 2, 2).mean((1, 3))
    U = np.clip(np.rint(128 + pool(cb) * 224 / 255), 0, 255)
    V = np.clip(np.rint(128 + pool(cr) * 224 / 255), 0, 255)
    uv = np.stack([U, V], -1).reshape(h // 2, w)
    return np.concatenate([Y, uv], 0).astype(np.uint8)
