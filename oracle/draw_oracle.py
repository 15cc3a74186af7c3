"""Pose overlay of VitInference.draw() (easy_ViTPose/inference.py:283-312, vit_utils/visualization.py:360-481) restated in
exact integer / IEEE-double arithmetic, as the pixel sets cv2 4.13 paints.

cv2.circle(img, c, r, color, -1) is drawing.cpp's `Circle(fill=1)`: the integer midpoint loop, whose spans are tabulated by
`circle_half_widths`.  cv2.line(img, p0, p1, color, 2) first clips the integer segment with clipLine against the image grown
by the thickness on every side, Rect(-2, -2, w + 4, h + 4), and draws nothing when that rejects it (found by probing cv2
4.13 on small frames: without this step 15 % of the lines with an end point off the frame differ).  The clipped end points
then go to `ThickLine(flags=3)`: in 16.16 fixed point, a
perpendicular offset dp = cvRound((dy, dx) * 65536 / |p1 - p0|), the quad p0 +- dp, p1 -+ dp filled by
`FillConvexPoly(shift=16, LINE_8)` -- its four edges drawn by `Line2` (clipLine against the image scaled by 2^16, then a
fixed-point DDA plus the end pixel) and its scanlines stepped by the int64 `dx` of each edge -- and a radius-1 filled circle at
each end.  Every function returns coverage (pixels of an image of the given size); nothing is anti-aliased or blended, so
painting covered pixels in call order reproduces the reference's frame.

Also here: the palettes `draw()` passes (`reference_palettes`, through easy_vitpose_b200.draw) and `draw_poses`, the draw
loop over many frames.  This module is the checker of easy_vitpose_b200/csrc/draw.cuh; nothing on the product path imports
it.
"""
from __future__ import annotations

import math

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
DBL_EPSILON = 2.220446049250313e-16
THICKNESS = 2                  # cv2.line thickness of draw_skeleton
COORD_LIMIT = 1 << 31          # int(coordinate) outside int32 is not drawn (cv2 rejects such a point)


def _tdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


# ------------------------------------------------------------------------------------------------------------------ circle
def circle_half_widths(radius: int) -> np.ndarray:
    """hw[o] = half width of the filled circle's span on rows centre +- o (o = 0..radius), from Circle()'s midpoint loop:
    each step (dx, dy) paints rows +-dy over +-dx and rows +-dx over +-dy."""
    hw = np.full(radius + 1, -1, np.int64)
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    while dx >= dy:
        hw[dy] = max(hw[dy], dx)
        hw[dx] = max(hw[dx], dy)
        dy += 1
        err += plus
        plus += 2
        mask = (err <= 0) - 1
        err -= minus & mask
        dx += mask
        minus -= mask & 2
    return hw


def circle_spans(h: int, w: int, cx: int, cy: int, radius: int):
    """Filled circle as clipped row spans [(y, x0, x1)] (inclusive)."""
    hw = circle_half_widths(radius)
    out = []
    for o in range(-radius, radius + 1):
        y, half = cy + o, int(hw[abs(o)])
        if half < 0 or not 0 <= y < h:
            continue
        x0, x1 = max(cx - half, 0), min(cx + half, w - 1)
        if x0 <= x1:
            out.append((y, x0, x1))
    return out


# ------------------------------------------------------------------------------------------------------------------- lines
def clip_line(w: int, h: int, x1: int, y1: int, x2: int, y2: int):
    """drawing.cpp clipLine on an image of w x h (already scaled): the clipped segment, or None when it misses."""
    if w <= 0 or h <= 0:
        return None
    right, bottom = w - 1, h - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    if c1 | c2:
        return None
    return x1, y1, x2, y2


def line2_dda(h: int, w: int, p1, p2):
    """drawing.cpp Line2 (16.16 end points, 8-connected) as its DDA description, or None when clipLine rejects it:
    (x_major, a0, b0, step, count, end) -- pixel t = 0..count is (a0 + t, (b0 + t * step) >> 16) for an x-major line,
    ((b0 + t * step) >> 16, a0 + t) otherwise -- plus the separately painted end pixel `end` = (x, y)."""
    c = clip_line(w << XY_SHIFT, h << XY_SHIFT, p1[0], p1[1], p2[0], p2[1])
    if c is None:
        return None
    x1, y1, x2, y2 = c
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            dy = -dy
            x1, y1, x2, y2 = x2, y2, x1, y1
        step = _tdiv(dy << XY_SHIFT, ax | 1)
        count = (x2 - x1) >> XY_SHIFT
    else:
        if dy < 0:
            dx = -dx
            x1, y1, x2, y2 = x2, y2, x1, y1
        step = _tdiv(dx << XY_SHIFT, ay | 1)
        count = (y2 - y1) >> XY_SHIFT
    end = ((x2 + (XY_ONE >> 1)) >> XY_SHIFT, (y2 + (XY_ONE >> 1)) >> XY_SHIFT)
    x1 += XY_ONE >> 1
    y1 += XY_ONE >> 1
    if ax > ay:
        return True, x1 >> XY_SHIFT, y1, step, count, end
    return False, y1 >> XY_SHIFT, x1, step, count, end


def line2_pixels(h: int, w: int, p1, p2):
    """Pixels [(x, y)] Line2 paints inside the image."""
    d = line2_dda(h, w, p1, p2)
    if d is None:
        return []
    x_major, a0, b0, step, count, end = d
    t = np.arange(count + 1, dtype=object)
    b = [(b0 + int(k) * step) >> XY_SHIFT for k in t]
    pts = [(a0 + int(k), bb) if x_major else (bb, a0 + int(k)) for k, bb in zip(t, b)]
    pts.append(end)
    return [(x, y) for x, y in pts if 0 <= x < w and 0 <= y < h]


# -------------------------------------------------------------------------------------------------------- convex polygon
def fill_segments(h: int, w: int, v):
    """The scanline part of drawing.cpp FillConvexPoly(shift=16, LINE_8) for the 16.16 vertices v, as edge segments
    [(side, y0, y1, x, dx)]: on rows y0 <= y < y1 that side's edge sits at x + (y - y0) * dx; a row's span is
    [(left + 2^15) >> 16, (right + 2^15) >> 16].  Rows may be negative (the loop walks them without painting)."""
    delta = 1 << XY_SHIFT >> 1
    n = len(v)
    imin = 0
    for i in range(n):
        if v[i][1] < v[imin][1]:
            imin = i
    xmin = (min(p[0] for p in v) + delta) >> XY_SHIFT
    xmax = (max(p[0] for p in v) + delta) >> XY_SHIFT
    ymin = (v[imin][1] + delta) >> XY_SHIFT
    ymax = (max(p[1] for p in v) + delta) >> XY_SHIFT
    if n < 3 or xmax < 0 or ymax < 0 or xmin >= w or ymin >= h:
        return []
    ymax = min(ymax, h - 1)
    edges = n
    # per side: idx, di, ye, and the open segment (y0, x, dx)
    side = [dict(idx=imin, di=1, ye=ymin, seg=None), dict(idx=imin, di=n - 1, ye=ymin, seg=None)]
    segs = []
    y = ymin
    while True:
        for i in (0, 1):
            e = side[i]
            if y >= e["ye"]:
                idx0, di = e["idx"], e["di"]
                idx = (idx0 + di) % n
                while True:
                    old = edges
                    edges -= 1
                    if old <= 0:
                        break
                    ty = (v[idx][1] + delta) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        if e["seg"] is not None:
                            segs.append((i, e["seg"][0], y, e["seg"][1], e["seg"][2]))
                        e["seg"] = (y, xs, _tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y)))
                        e["ye"], e["idx"] = ty, idx
                        break
                    idx0 = idx
                    idx = (idx + di) % n
        if edges < 0:
            break
        nxt = min(side[0]["ye"], side[1]["ye"], ymax + 1)
        y = nxt
        if y > ymax:
            break
    for i in (0, 1):
        if side[i]["seg"] is not None:
            segs.append((i, side[i]["seg"][0], y, side[i]["seg"][1], side[i]["seg"][2]))
    return segs


def segment_spans(h: int, w: int, segs):
    """Clipped row spans [(y, x0, x1)] of fill_segments' output."""
    delta = XY_ONE >> 1
    out = []
    left = [s for s in segs if s[0] == 0]
    right = [s for s in segs if s[0] == 1]
    for s0 in left:
        for s1 in right:
            for y in range(max(s0[1], s1[1], 0), min(s0[2], s1[2], h)):
                xa = s0[3] + (y - s0[1]) * s0[4]
                xb = s1[3] + (y - s1[1]) * s1[4]
                lo, hi = (xb, xa) if xa > xb else (xa, xb)
                x0, x1 = (lo + delta) >> XY_SHIFT, (hi + delta) >> XY_SHIFT
                if x1 >= 0 and x0 < w:
                    out.append((y, max(x0, 0), min(x1, w - 1)))
    return out


def thick_line_parts(x0: int, y0: int, x1: int, y1: int):
    """ThickLine(thickness 2, LINE_8, shift 0): the 16.16 quad (or None for a zero-length line) and the end-circle
    centres (radius (2 << 15 + 2^15) >> 16 = 1)."""
    p0 = (x0 << XY_SHIFT, y0 << XY_SHIFT)
    p1 = (x1 << XY_SHIFT, y1 << XY_SHIFT)
    dx = (p0[0] - p1[0]) * (1.0 / XY_ONE)
    dy = (p1[1] - p0[1]) * (1.0 / XY_ONE)
    r = dx * dx + dy * dy
    quad = None
    if abs(r) > DBL_EPSILON:
        r = float(2 << (XY_SHIFT - 1)) / math.sqrt(r)
        dpx, dpy = round(dy * r), round(dx * r)           # cvRound: round half to even
        quad = [(p0[0] + dpx, p0[1] + dpy), (p0[0] - dpx, p0[1] - dpy),
                (p1[0] - dpx, p1[1] - dpy), (p1[0] + dpx, p1[1] + dpy)]
    return quad, [(x0, y0), (x1, y1)]


def preclip(h: int, w: int, x0: int, y0: int, x1: int, y1: int):
    """cv2.line's clip of the integer end points to Rect(-2, -2, w + 4, h + 4), or None when the segment misses it."""
    m = THICKNESS
    c = clip_line(w + 2 * m, h + 2 * m, x0 + m, y0 + m, x1 + m, y1 + m)
    return None if c is None else tuple(v - m for v in c)


def thick_line_spans(h: int, w: int, x0: int, y0: int, x1: int, y1: int):
    """Coverage of cv2.line(img, (x0, y0), (x1, y1), color, 2) as clipped row spans [(y, x0, x1)] (single pixels included)."""
    out = []
    c = preclip(h, w, x0, y0, x1, y1)
    if c is None:
        return out
    quad, ends = thick_line_parts(*c)
    if quad is not None:
        p0 = quad[-1]
        for p in quad:
            out += [(y, x, x) for x, y in line2_pixels(h, w, p0, p)]
            p0 = p
        out += segment_spans(h, w, fill_segments(h, w, quad))
    for cx, cy in ends:
        out += circle_spans(h, w, cx, cy, 1)
    return out


def thick_line_mask(h: int, w: int, x0: int, y0: int, x1: int, y1: int) -> np.ndarray:
    """Coverage of cv2.line(img, (x0, y0), (x1, y1), color, 2) as a bool [h, w] mask."""
    m = np.zeros((h, w), bool)
    for y, a, b in thick_line_spans(h, w, x0, y0, x1, y1):
        m[y, a:b + 1] = True
    return m


def circle_mask(h: int, w: int, cx: int, cy: int, radius: int) -> np.ndarray:
    """Coverage of cv2.circle(img, (cx, cy), radius, color, -1) as a bool [h, w] mask."""
    m = np.zeros((h, w), bool)
    for y, a, b in circle_spans(h, w, cx, cy, radius):
        m[y, a:b + 1] = True
    return m


# ---------------------------------------------------------------------------------------------------------------- draw loop
def _coord(v) -> int | None:
    """int() of a keypoint coordinate (truncation toward zero); None when it is not drawn (non-finite or outside int32)."""
    v = float(v)
    if not math.isfinite(v):
        return None
    t = int(v)
    return t if -COORD_LIMIT <= t < COORD_LIMIT else None


def draw_poses(frames, kpts, counts, skeleton, point_bgr, limb_bgr, person_index=None, threshold=0.5, radius=0,
               channel_order="rgb"):
    """The pose layer of draw() over many frames, painted in place: frames list of uint8 [H, W, 3]; kpts float32 [n, K, 3]
    (y, x, score) with the people of all frames concatenated (frame j owns the next counts[j] rows); person_index [n] colour
    index (None = position within its frame); colours BGR; radius <= 0 = max(1, min(H, W) // 150) per frame.  Scores are
    compared in float32, `score > threshold`."""
    kpts = np.asarray(kpts, np.float32)
    thr = np.float32(threshold)
    skeleton = np.asarray(skeleton, np.int64).reshape(-1, 2)
    point_bgr = np.asarray(point_bgr, np.uint8).reshape(-1, 3)
    limb_bgr = np.asarray(limb_bgr, np.uint8).reshape(-1, 3)
    rev = channel_order == "rgb"
    p = 0
    for j, img in enumerate(frames):
        h, w = img.shape[:2]
        r = radius if radius > 0 else max(1, min(h, w) // 150)
        for q in range(counts[j]):
            k = kpts[p]
            idx = q if person_index is None else int(person_index[p])
            col = limb_bgr[idx % len(limb_bgr)]
            col = col[::-1] if rev else col
            for a, b in skeleton:
                if k[a, 2] > thr and k[b, 2] > thr:
                    xa, ya, xb, yb = _coord(k[a, 1]), _coord(k[a, 0]), _coord(k[b, 1]), _coord(k[b, 0])
                    if None in (xa, ya, xb, yb):
                        continue
                    for yy, x0, x1 in thick_line_spans(h, w, xa, ya, xb, yb):
                        img[yy, x0:x1 + 1] = col
            for i in range(k.shape[0]):
                if k[i, 2] > thr:
                    x, y = _coord(k[i, 1]), _coord(k[i, 0])
                    if x is None or y is None:
                        continue
                    c = point_bgr[i % len(point_bgr)]
                    for yy, a, b in circle_spans(h, w, x, y, r):
                        img[yy, a:b + 1] = c[::-1] if rev else c
            p += 1
    return frames


def make_case(seed: int, h: int, w: int, n: int, k: int, far: bool = True):
    """Seeded frame u8 [h, w, 3] (a pattern, not zeros, so untouched pixels are checked too) and keypoints f32 [n, k, 3]
    (y, x, score): most inside the frame, some on its border, just outside, far outside (+-20000) and negative; some scores
    exactly at 0.5."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    frame = np.stack([(xx * 7 + yy * 3) % 256, (xx * 5 + yy * 11 + seed) % 256, (xx ^ yy) % 256], -1).astype(np.uint8)
    kp = np.zeros((n, k, 3), np.float32)
    cy, cx = rng.uniform(0, h, (n, 1)), rng.uniform(0, w, (n, 1))
    s = max(h, w) * 0.15 + 2
    kp[..., 0] = cy + rng.normal(0, s, (n, k))
    kp[..., 1] = cx + rng.normal(0, s, (n, k))
    pick = rng.uniform(size=(n, k))
    kp[..., 0] = np.where(pick < 0.05, rng.choice([-1.0, -0.7, 0.0, h - 1, h - 0.3, h, h + 1.5], (n, k)), kp[..., 0])
    kp[..., 1] = np.where((pick >= 0.05) & (pick < 0.1), rng.choice([-2.5, -0.7, 0.0, w - 1, w + 0.9, w + 2.5], (n, k)), kp[..., 1])
    if far:
        kp[..., 0] = np.where((pick >= 0.1) & (pick < 0.13), rng.uniform(-20000, 20000, (n, k)), kp[..., 0])
        kp[..., 1] = np.where((pick >= 0.13) & (pick < 0.16), rng.uniform(-20000, 20000, (n, k)), kp[..., 1])
    kp[..., 2] = rng.uniform(0, 1, (n, k))
    kp[..., 2] = np.where(rng.uniform(size=(n, k)) < 0.05, 0.5, kp[..., 2])
    return frame, kp
