"""Arguments of the affine top-down crop (ViTPose.infer_affine): person boxes (x, y, w, h) -> warp matrices and the
centre / scale the keypoints are decoded with, as the reference's top-down data path computes them.

    easy_ViTPose/datasets/COCO.py:318-337            _xywh2cs: centre, scale (units of 200 px) at the 192:256 aspect, x1.25
    vit_utils/post_processing/post_transforms.py:312-340
                                                     get_warp_matrix(0, 2c, image_size - 1, s * 200): the UDP matrix of every
                                                     config's test_cfg (use_udp=True)
    vit_utils/transform.py:46-75                     get_affine_transform(c, s, 200, 0, image_size): the HRNet matrix
                                                     (COCO.py:288)

Centre, scale and the UDP matrix are bit-identical to the reference's (same float32 / float64 steps).  The HRNet matrix is
the exact solution of get_affine_transform's three float32 point pairs in float64; cv2.getAffineTransform solves the same
system with its own elimination order, so the two agree to a few units in the last place.
"""
from __future__ import annotations

import math

import numpy as np

__all__ = ["topdown_args", "xywh2cs", "udp_matrix", "hrnet_matrix"]

IMAGE_SIZE = (192, 256)           # (width, height) of the model input
PIXEL_STD = 200                   # COCO.py:105


def xywh2cs(box, padding: float = 1.25):
    """(x, y, w, h) -> (centre float32 [2], scale float32 [2] in units of 200 px), COCO.py:318-337 (`padding` is its x1.25)."""
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
    """float32 [2,3] = get_warp_matrix(rot, 2 * center, image_size - 1, 200 * scale) (post_transforms.py:312-340)."""
    size_in = np.asarray(center, np.float32) * 2.0
    size_dst = np.array(IMAGE_SIZE) - 1.0
    size_tg = np.asarray(scale, np.float32) * 200.0
    theta = np.deg2rad(rot)
    cs, sn = math.cos(theta), math.sin(theta)
    kx, ky = size_dst[0] / size_tg[0], size_dst[1] / size_tg[1]
    m = np.zeros((2, 3), np.float32)
    m[0, 0], m[0, 1] = cs * kx, -sn * kx
    m[0, 2] = kx * (-0.5 * size_in[0] * cs + 0.5 * size_in[1] * sn + 0.5 * size_tg[0])
    m[1, 0], m[1, 1] = sn * ky, cs * ky
    m[1, 2] = ky * (-0.5 * size_in[0] * sn - 0.5 * size_in[1] * cs + 0.5 * size_tg[1])
    return m


def hrnet_matrix(center, scale, rot: float = 0.0) -> np.ndarray:
    """float64 [2,3]: get_affine_transform(center, scale, 200, rot, (192, 256)) (transform.py:46-75) without cv2: the same
    float32 point triples, the 6x6 system solved in float64."""
    center = np.asarray(center, np.float32)
    st = np.asarray(scale, np.float32) * 1.0 * PIXEL_STD
    r = np.pi * rot / 180
    sn, cs = np.sin(r), np.cos(r)
    half = st[0] * -0.5
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0] = center
    src[1] = center + [0 * cs - half * sn, 0 * sn + half * cs]
    dst[0] = [IMAGE_SIZE[0] * 0.5, IMAGE_SIZE[1] * 0.5]
    dst[1] = np.array([IMAGE_SIZE[0] * 0.5, IMAGE_SIZE[1] * 0.5]) + np.array([0, IMAGE_SIZE[0] * -0.5], np.float32)
    for p in (src, dst):                                     # the third point: the second turned by 90 deg about the first
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], np.float32)
    a = np.zeros((6, 6))
    b = np.zeros(6)
    for k in range(3):
        a[k, 0:2] = a[k + 3, 3:5] = src[k]
        a[k, 2] = a[k + 3, 5] = 1.0
        b[k], b[k + 3] = dst[k]
    return np.linalg.solve(a, b).reshape(2, 3)


def topdown_args(bboxes_xywh, padding: float = 1.25, use_udp: bool = True):
    """Person boxes [n,4] (x, y, w, h) in image pixels -> (mats float64 [n,2,3], centers float32 [n,2], scales_px float32 [n,2]).
    mats are the UDP matrices (use_udp=True, what every reference config's test_cfg selects) or the HRNet ones, as float64;
    scales_px = scale * 200, the scale keypoints_from_heatmaps takes.  Feed them to ViTPose.infer_affine."""
    bb = np.asarray(bboxes_xywh, np.float64).reshape(-1, 4)
    n = bb.shape[0]
    mats = np.zeros((n, 2, 3), np.float64)
    centers = np.zeros((n, 2), np.float32)
    scales = np.zeros((n, 2), np.float32)
    for i, box in enumerate(bb):
        c, s = xywh2cs(box, padding)
        mats[i] = udp_matrix(c, s) if use_udp else hrnet_matrix(c, s)
        centers[i] = c
        scales[i] = s * 200.0
    return mats, centers, scales
