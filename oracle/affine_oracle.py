"""CPU restatement of the affine top-down crop (mmpose / HRNet style)  --  TEST INFRASTRUCTURE ONLY.

Only tests/ and the fixture generator (oracle/make_golden_affine.py) import this; the product path
(easy_vitpose_b200/csrc/preprocess.cuh: frame_to_patch_rows_affine, crop_warp_normalise) never does.

What the reference's top-down data path does per person box (x, y, w, h):
  easy_ViTPose/datasets/COCO.py:318-337   _xywh2cs: centre / scale (units of pixel_std = 200) at the 192:256 aspect, x1.25
  vit_utils/post_processing/post_transforms.py:312-340
                                          get_warp_matrix(rot, 2c, image_size - 1, s * 200): the UDP matrix (use_udp=True,
                                          every config's test_cfg)
  vit_utils/transform.py:46-75 (+ get_dir :89-96, get_3rd_point :84-86)
                                          get_affine_transform: the HRNet matrix COCO.py:288 uses
  COCO.py:289-294                         cv2.warpAffine(image, trans, (192, 256), flags=cv2.INTER_LINEAR)
  COCO.py:120-123, 300-302                torchvision ToTensor + Normalize: float32 (v / 255 - mean) / std

cv2's uint8 warpAffine with INTER_LINEAR and the constant (0) border is fixed-point; warp_affine_u8 restates it
(pinned bit for bit against cv2 4.13 by tests/test_affine_cpu.py and by the fixture generator):
  * the matrix is inverted in double: D = M0*M4 - M1*M3, D = 1/D (0 if D == 0), A11 = M4*D, A22 = M0*D, M1 *= -D, M3 *= -D,
    b1 = -A11*M2 - M1*M5, b2 = -M3*M2 - A22*M5
  * AB_BITS = 10, INTER_BITS = 5: adelta[x] = cvRound(M0*x*1024), bdelta[x] = cvRound(M3*x*1024),
    X0(y) = cvRound((M1*y + M2)*1024) + 16, Y0(y) = cvRound((M4*y + M5)*1024) + 16, X = (X0 + adelta) >> 5
  * integer tap X >> 5 (saturated to int16), fraction X & 31 (same for Y)
  * int16 weights of the 32 x 32 bilinear table: float32 (1 - fy/32 | fy/32) * (1 - fx/32 | fx/32) * 32768, rounded; every
    product is an exact integer here, so each set already sums to 32768 and cv2's sum correction never fires
  * pixel = (sum w * p + 2^14) >> 15; taps outside the image read 0 (so an output whose top-left tap is outside
    [-1, w) x [-1, h) is 0)
"""
from __future__ import annotations

import numpy as np

MEAN = (0.485, 0.456, 0.406)      # COCO.py:122 transforms.Normalize(mean=...)
STD = (0.229, 0.224, 0.225)       # COCO.py:122 transforms.Normalize(std=...)
IMAGE_SIZE = (192, 256)           # (width, height): data_cfg['image_size'] of configs/ViTPose_common.py
PIXEL_STD = 200                   # COCO.py:105
AB_BITS, INTER_BITS = 10, 5


def normalise_table() -> np.ndarray:
    """float32 [3, 256]: ToTensor (uint8 -> float32, / 255) then Normalize (float32 sub, div) of byte v in channel c."""
    v = np.arange(256, dtype=np.float32) / np.float32(255)
    return ((v[None, :] - np.asarray(MEAN, np.float32)[:, None]) / np.asarray(STD, np.float32)[:, None]).astype(np.float32)


def xywh2cs(box, padding: float = 1.25):
    """COCO.py:318-337 (_xywh2cs with aspect_ratio = 192 / 256, pixel_std = 200; the reference's x1.25 is `padding`)
    -> (centre float32 [2], scale float32 [2]) in units of 200 px."""
    x, y, w, h = (float(v) for v in box[:4])
    aspect = IMAGE_SIZE[0] * 1.0 / IMAGE_SIZE[1]
    center = np.zeros((2,), np.float32)
    center[0] = x + w * 0.5
    center[1] = y + h * 0.5
    if w > aspect * h:
        h = w * 1.0 / aspect
    elif w < aspect * h:
        w = h * aspect
    scale = np.array([w * 1.0 / PIXEL_STD, h * 1.0 / PIXEL_STD], np.float32)
    if center[0] != -1:
        scale = scale * padding
    return center, scale


def udp_matrix(center, scale, rot: float = 0.0) -> np.ndarray:
    """float32 [2, 3]: get_warp_matrix(rot, center * 2.0, image_size - 1.0, scale * 200.0)
    (post_transforms.py:312-340), with the scalar types numpy gives each term there."""
    import math
    size_in = np.asarray(center, np.float32) * 2.0                     # float32
    size_dst = np.array(IMAGE_SIZE) - 1.0                               # float64
    size_tg = np.asarray(scale, np.float32) * 200.0                     # float32
    theta = np.deg2rad(rot)
    cs, sn = math.cos(theta), math.sin(theta)
    sx = size_dst[0] / size_tg[0]                                       # float64
    sy = size_dst[1] / size_tg[1]
    m = np.zeros((2, 3), np.float32)
    m[0, 0] = cs * sx
    m[0, 1] = -sn * sx
    m[0, 2] = sx * (-0.5 * size_in[0] * cs + 0.5 * size_in[1] * sn + 0.5 * size_tg[0])   # bracket in float32
    m[1, 0] = sn * sy
    m[1, 1] = cs * sy
    m[1, 2] = sy * (-0.5 * size_in[0] * sn - 0.5 * size_in[1] * cs + 0.5 * size_tg[1])
    return m


def hrnet_points(center, scale, rot: float = 0.0):
    """The float32 point triples get_affine_transform (transform.py:46-75) hands to cv2.getAffineTransform."""
    center = np.asarray(center, np.float32)
    scale_tmp = np.asarray(scale, np.float32) * 1.0 * PIXEL_STD
    src_w = scale_tmp[0]
    dst_w, dst_h = IMAGE_SIZE
    rot_rad = np.pi * rot / 180
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)                           # get_dir, transform.py:89-96
    p = [0, src_w * -0.5]
    src_dir = [p[0] * cs - p[1] * sn, p[0] * sn + p[1] * cs]
    dst_dir = np.array([0, dst_w * -0.5], np.float32)
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0, :] = center
    src[1, :] = center + src_dir
    dst[0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[1, :] = np.array([dst_w * 0.5, dst_h * 0.5]) + dst_dir
    for a in (src, dst):                                                # get_3rd_point, transform.py:84-86
        d = a[0] - a[1]
        a[2] = a[1] + np.array([-d[1], d[0]], np.float32)
    return src, dst


def hrnet_matrix(center, scale, rot: float = 0.0) -> np.ndarray:
    """float64 [2, 3]: get_affine_transform(center, scale, 200, rot, (192, 256)) (transform.py:46-75).  The last step is
    cv2.getAffineTransform itself, so this one needs cv2."""
    import cv2
    src, dst = hrnet_points(center, scale, rot)
    return cv2.getAffineTransform(np.float32(src), np.float32(dst))


def inverse_matrix(M) -> "tuple[float, ...]":
    """cv::warpAffine's inversion of the 2x3 matrix, in double, one rounding per operation."""
    m0, m1, m2, m3, m4, m5 = (float(v) for v in np.asarray(M, np.float64).reshape(6))
    D = m0 * m4 - m1 * m3
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m4 * D, m0 * D
    m0, m1, m3, m4 = a11, m1 * -D, m3 * -D, a22
    b1 = -m0 * m2 - m1 * m5
    b2 = -m3 * m2 - m4 * m5
    return m0, m1, b1, m3, m4, b2


def _round(v: np.ndarray) -> np.ndarray:
    """cvRound: round half to even."""
    return np.rint(v).astype(np.int64)


def warp_coords(M, out_w: int = IMAGE_SIZE[0], out_h: int = IMAGE_SIZE[1]):
    """-> (X, Y) int64 [out_h, out_w]: the fixed-point source coordinates (INTER_BITS = 5 fractional bits)."""
    i0, i1, i2, i3, i4, i5 = inverse_matrix(M)
    x = np.arange(out_w, dtype=np.float64)
    y = np.arange(out_h, dtype=np.float64)
    scale = float(1 << AB_BITS)
    rd = (1 << AB_BITS) >> INTER_BITS >> 1
    adelta, bdelta = _round(i0 * x * scale), _round(i3 * x * scale)
    x0, y0 = _round((i1 * y + i2) * scale) + rd, _round((i4 * y + i5) * scale) + rd
    sh = AB_BITS - INTER_BITS
    return (x0[:, None] + adelta[None, :]) >> sh, (y0[:, None] + bdelta[None, :]) >> sh


def warp_affine_u8(img: np.ndarray, M, out_w: int = IMAGE_SIZE[0], out_h: int = IMAGE_SIZE[1]) -> np.ndarray:
    """cv2.warpAffine(img, M, (out_w, out_h), flags=cv2.INTER_LINEAR) (constant 0 border) for uint8 [h, w, c], bit-exact."""
    h, w = img.shape[:2]
    X, Y = warp_coords(M, out_w, out_h)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    fx, fy = X & 31, Y & 31
    p = img.astype(np.int64).reshape(h, w, -1)
    acc = np.zeros((out_h, out_w, p.shape[2]), np.int64)
    for ty, wy in ((0, 32 - fy), (1, fy)):
        for tx, wx in ((0, 32 - fx), (1, fx)):
            xx, yy = sx + tx, sy + ty
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            v = p[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)] * ok[..., None]
            acc += (wy * wx * 32)[..., None] * v
    out = (acc + (1 << 14)) >> 15
    return out.astype(np.uint8).reshape((out_h, out_w) + img.shape[2:])


def warp_normalise(img: np.ndarray, M) -> np.ndarray:
    """uint8 RGB [h, w, 3] -> float32 [3, 256, 192]: warpAffine then ToTensor + Normalize (COCO.py:289-302)."""
    r = warp_affine_u8(img, M)
    t = normalise_table()
    return np.stack([t[c][r[..., c]] for c in range(3)], 0)
