"""The contract vpb_oks_nms / vpb_oks_iou are held to: the reference's oks_iou, oks_nms and soft_oks_nms
(easy_ViTPose/vit_utils/post_processing/nms.py:51-207), per frame, restated in numpy with every promotion and summation
order spelled out, plus HRNet's evaluation rescoring, which the reference's header and datasets/COCO.py:237-241 come from
but which the reference itself dropped (inference.py:272 leaves it as a TODO).

Per frame of n people, keypoints float32 [n, K, 3], area and score float64:

1. order: `scores.argsort()[::-1]`.  numpy's default argsort is not stable, so ties are defined by the same expression with
   a stable argsort (`tie="stable"`): equal scores put the later index first; NaN sorts above +inf.  soft_oks_nms applies
   it again every round to the remaining order, so its ties go to the later POSITION.  `tie="numpy"` uses the default sort.
2. OKS: dx, dy float32; dx**2 + dy**2 float32; / vars (float64, (2 sigma)^2) / ((a_g + a_d) / 2 + np.spacing(1)) / 2 left to
   right; np.exp; np.sum, whose pairwise order `pairwise_sum` states; / len; stored as float32; 0 for an empty mask.
3. mask: `list(vg > vis_thr) and list(vd > vis_thr)` is the candidate's mask alone; vis_thr None = no mask.
4. hard: `oks <= thr` compares in float32 with thr rounded to float32 (NEP 50), so a NaN OKS suppresses.
5. soft: scores * np.exp(-o**2 / thr), the OKS term in float32, the product float64; re-sort; stop at max_dets.
6. rescoring (`rescore`): float32 sum of the keypoint scores > in_vis_thr in keypoint order, float32 divide by the count (0
   when none), times the box score rounded to float32; widened to float64.

`flag_ambiguous` names the frames where the device's exp may decide differently from numpy's: a consulted OKS whose float64
mean, moved by 4 ulps, rounds to float32 values on both sides of float32(thr), or in soft NMS two neighbouring rescored
scores that are not equal but lie within r * 2^-20 of each other (relative) after round r.  A round multiplies every
remaining score by one float32 exp factor, and the device's factor may differ from numpy's by a few float32 ulps (its expf,
and an OKS one ulp off), about 2^-21 relative per score; so after r rounds two scores may have drifted apart by up to
r * 2^-20.  Round 1 uses the 2^-20 bound alone.
"""
from __future__ import annotations

import importlib.util
import os

import numpy as np

COCO_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0
MAX_PEOPLE = 256
MAX_K = 144
MAX_DETS = 256
STATUS_TOO_MANY_PEOPLE = 1
STATUS_BAD_ROWS = 2
SOFT_TIE_REL = 2.0 ** -20                 # per round of soft NMS (flag_ambiguous)


def load_reference_nms():
    """The unmodified post_processing/nms.py, loaded by file path (it imports only numpy)."""
    from oracle import ref_import
    path = os.path.join(ref_import.REF_PKG, "vit_utils", "post_processing", "nms.py")
    if not os.path.exists(path):
        raise RuntimeError(f"reference nms.py not found at {path}")
    spec = importlib.util.spec_from_file_location("_reference_post_processing_nms", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def kpts_db(kpts, areas, scores):
    """Arrays of one frame -> the reference's list of {'keypoints', 'area', 'score'} (Python floats, as HRNet builds them)."""
    return [dict(keypoints=np.asarray(k, np.float32), area=float(a), score=float(s)) for k, a, s in zip(kpts, areas, scores)]


# ------------------------------------------------------------------------------------------------------------- arithmetic
def _block(a):
    """numpy's pairwise_sum for 8 <= n <= 128: eight strided partial sums, ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), the tail."""
    n = len(a)
    r = [a[j] for j in range(8)]
    m8 = n - n % 8
    for i in range(8, m8, 8):
        for j in range(8):
            r[j] = r[j] + a[i + j]
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for i in range(m8, n):
        res = res + a[i]
    return res


def pairwise_sum(a) -> np.float64:
    """np.sum of a float64 vector, in numpy's pairwise order."""
    a = np.asarray(a, np.float64)
    n = len(a)
    if n < 8:
        res = np.float64(0.0)
        for v in a:
            res = res + v
        return np.float64(res)
    if n <= 128:
        return np.float64(0.0) + _block(a)
    h = n // 2
    h -= h % 8
    return np.float64(pairwise_sum(a[:h]) + pairwise_sum(a[h:]))


def _vars(sigmas, k):
    s = COCO_SIGMAS if sigmas is None else np.asarray(sigmas, np.float64)
    if len(s) != k:
        raise ValueError(f"{len(s)} sigmas for {k} keypoints")
    return (s * 2) ** 2


def oks_means(g, d, a_g, a_d, sigmas=None, vis_thr=None):
    """The float64 means oks_iou rounds to float32: g [K, 3], d [m, K, 3] float32, a_g float, a_d float64 [m]."""
    g = np.asarray(g, np.float32).reshape(-1, 3)
    d = np.asarray(d, np.float32).reshape(-1, g.shape[0], 3)
    var = _vars(sigmas, g.shape[0])
    out = np.zeros(len(d), np.float64)
    for j in range(len(d)):
        dx = d[j, :, 0] - g[:, 0]
        dy = d[j, :, 1] - g[:, 1]
        e = (dx * dx + dy * dy) / var / ((a_g + a_d[j]) / 2 + np.spacing(1)) / 2
        if vis_thr is not None:
            e = e[d[j, :, 2] > np.float32(vis_thr)]
        out[j] = np.sum(np.exp(-e)) / len(e) if len(e) else 0.0       # np.sum's order is pairwise_sum's (tested)
    return out


def oks_iou(g, d, a_g, a_d, sigmas=None, vis_thr=None):
    """float32 [m]: the reference oks_iou with (y, x, score) or (x, y, score) rows."""
    with np.errstate(invalid="ignore", over="ignore"):
        return oks_means(g, d, a_g, np.asarray(a_d, np.float64), sigmas, vis_thr).astype(np.float32)


def oks_matrix(kpts, areas, sigmas=None, vis_thr=None):
    """float32 [n, n]: row i, column j = oks_iou(g = person i, d = person j) (what vpb_oks_iou writes)."""
    kpts = np.asarray(kpts, np.float32)
    areas = np.asarray(areas, np.float64)
    return np.stack([oks_iou(kpts[i], kpts, areas[i], areas, sigmas, vis_thr) for i in range(len(kpts))]) if len(kpts) else \
        np.zeros((0, 0), np.float32)


def order_desc(scores, tie: str = "stable"):
    """`scores.argsort()[::-1]`: tie="stable" the device's rule, "numpy" the reference's default sort."""
    s = np.asarray(scores, np.float64)
    return (np.argsort(s, kind="stable") if tie == "stable" else s.argsort())[::-1]


def rescore(kpts, box_scores, in_vis_thr):
    """HRNet's evaluate rescoring -> float64 [n]: float32(mean of keypoint scores > in_vis_thr, 0 when none) * float32(box)."""
    kpts = np.asarray(kpts, np.float32)
    thr = np.float32(in_vis_thr)
    out = np.zeros(len(kpts), np.float64)
    for i, (k, b) in enumerate(zip(kpts, np.asarray(box_scores, np.float64))):
        s, c = np.float32(0.0), 0
        for t in k[:, 2]:
            if t > thr:
                s = np.float32(s + t)
                c += 1
        m = np.float32(s / np.float32(c)) if c else np.float32(0.0)
        with np.errstate(invalid="ignore", over="ignore"):
            out[i] = np.float64(np.float32(m * np.float32(b)))
    return out


# ---------------------------------------------------------------------------------------------------------------- NMS
def oks_nms(kpts, areas, scores, thr, sigmas=None, vis_thr=None, tie="stable", trace=None):
    """The reference oks_nms on arrays of one frame -> kept indices (int64).  `trace` (a list) collects the float64 means of
    every OKS the sweep consults."""
    kpts = np.asarray(kpts, np.float32)
    areas = np.asarray(areas, np.float64)
    order = order_desc(scores, tie)
    thr32 = np.float32(thr)
    keep = []
    while len(order) > 0:
        i = order[0]
        keep.append(i)
        with np.errstate(invalid="ignore", over="ignore"):
            m = oks_means(kpts[i], kpts[order[1:]], areas[i], areas[order[1:]], sigmas, vis_thr)
        if trace is not None:
            trace.extend(m.tolist())
        order = order[np.where(m.astype(np.float32) <= thr32)[0] + 1]
    return np.array(keep, np.int64)


def soft_oks_nms(kpts, areas, scores, thr, max_dets=20, sigmas=None, vis_thr=None, tie="stable", trace=None):
    """The reference soft_oks_nms on arrays of one frame -> kept indices.  `trace` collects every re-sorted score vector."""
    kpts = np.asarray(kpts, np.float32)
    areas = np.asarray(areas, np.float64)
    scores = np.asarray(scores, np.float64)
    order = order_desc(scores, tie)
    scores = scores[order]
    thr32 = np.float32(thr)
    keep = []
    while len(order) > 0 and len(keep) < max_dets:
        i = order[0]
        o = oks_iou(kpts[i], kpts[order[1:]], areas[i], areas[order[1:]], sigmas, vis_thr)
        order = order[1:]
        with np.errstate(invalid="ignore", over="ignore"):
            scores = scores[1:] * np.exp(-(o * o) / thr32)
        tmp = order_desc(scores, tie)
        order, scores = order[tmp], scores[tmp]
        if trace is not None:
            trace.append(scores.copy())
        keep.append(i)
    return np.array(keep, np.int64)


def run_frame(kpts, areas, scores, thr, sigmas=None, vis_thr=None, soft=False, max_dets=20, rescore_vis_thr=None, tie="stable"):
    """One frame as vpb_oks_nms computes it -> (kept indices, the scores the sort used)."""
    s = rescore(kpts, scores, rescore_vis_thr) if rescore_vis_thr is not None else np.asarray(scores, np.float64)
    if soft:
        return soft_oks_nms(kpts, areas, s, thr, max_dets, sigmas, vis_thr, tie), s
    return oks_nms(kpts, areas, s, thr, sigmas, vis_thr, tie), s


def flag_ambiguous(kpts, areas, scores, thr, sigmas=None, vis_thr=None, soft=False, max_dets=20, rescore_vis_thr=None) -> bool:
    """True when a 1-ulp difference in exp could change the frame's kept list (see the module docstring)."""
    s = rescore(kpts, scores, rescore_vis_thr) if rescore_vis_thr is not None else np.asarray(scores, np.float64)
    thr32 = np.float32(thr)
    if not soft:
        trace = []
        oks_nms(kpts, areas, s, thr, sigmas, vis_thr, trace=trace)
        m = np.asarray(trace, np.float64)
        m = m[np.isfinite(m)]
        step = 4 * np.spacing(m)
        with np.errstate(over="ignore"):
            lo, hi = (m - step).astype(np.float32), (m + step).astype(np.float32)
        return bool(np.any((lo <= thr32) != (hi <= thr32)))
    trace = []
    soft_oks_nms(kpts, areas, s, thr, max_dets, sigmas, vis_thr, trace=trace)
    for r, v in enumerate(trace):
        a, b = v[:-1], v[1:]
        with np.errstate(invalid="ignore"):
            close = (a != b) & (np.abs(a - b) <= (r + 1) * SOFT_TIE_REL * np.maximum(np.abs(a), np.abs(b)))
        if np.any(close):
            return True
    return False
