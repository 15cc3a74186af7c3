"""CPU: oracle/draw_oracle.py, the restatement vpb_draw_poses is held to, is bit-equal to live cv2.line(..., 2) /
cv2.circle(..., -1) on a seeded sweep, and its draw loop reproduces frames the unmodified reference drew
(tests/golden/draw_poses.npz, oracle/make_golden_draw.py); easy_vitpose_b200.draw's palettes and argument checks."""
import zlib

import numpy as np
import pytest

from oracle import draw_oracle as D

cv2 = pytest.importorskip("cv2")

SIZES = [(1, 1), (7, 5), (33, 17), (1080, 1920)]        # (h, w)


def _cv_line(h, w, a, b):
    img = np.zeros((h, w, 3), np.uint8)
    cv2.line(img, a, b, (255, 255, 255), 2)
    return img[..., 0] > 0


def _cv_circle(h, w, c, r):
    img = np.zeros((h, w, 3), np.uint8)
    cv2.circle(img, c, r, (255, 255, 255), -1)
    return img[..., 0] > 0


def _point(rng, h, w, mode):
    if mode == 0:                                                              # inside
        return int(rng.integers(0, w)), int(rng.integers(0, h))
    if mode == 1:                                                              # on the border
        return int(rng.choice([0, w - 1])), int(rng.integers(0, h))
    if mode == 2:                                                              # just outside (up to 3 px)
        return int(rng.integers(-3, w + 3)), int(rng.choice([-3, -2, -1, h, h + 1, h + 2]))
    if mode == 3:                                                              # far outside
        return int(rng.integers(-20000, 20001)), int(rng.integers(-20000, 20001))
    return int(rng.integers(-40, 0)), int(rng.integers(-40, h + 40))           # negative


def _limbs(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(count):
        h, w = SIZES[t % len(SIZES)]
        a = _point(rng, h, w, int(rng.integers(0, 5)))
        kind = t % 6
        if kind == 0:
            b = _point(rng, h, w, int(rng.integers(0, 5)))
        elif kind == 1:                                                        # horizontal
            b = (int(rng.integers(-50, w + 50)), a[1])
        elif kind == 2:                                                        # vertical
            b = (a[0], int(rng.integers(-50, h + 50)))
        elif kind == 3:                                                        # 45 degrees
            d = int(rng.integers(-60, 61))
            b = (a[0] + d, a[1] + d * int(rng.choice([-1, 1])))
        elif kind == 4:                                                        # near-degenerate
            b = (a[0] + int(rng.integers(-1, 2)), a[1] + int(rng.integers(-1, 2)))
        else:                                                                  # zero length
            b = a
        out.append((h, w, a, b))
    return out


@pytest.mark.parametrize("part", range(4))
def test_thick_line_bit_equal_to_cv2(part):
    bad = [(h, w, a, b) for h, w, a, b in _limbs(100 + part, 400) if not np.array_equal(_cv_line(h, w, a, b), D.thick_line_mask(h, w, *a, *b))]
    assert not bad, bad[:5]


def test_thick_line_off_frame_cases():
    """The case that shows cv2.line's clip to Rect(-2, -2, w + 4, h + 4): a 1 x 1 frame, (0, 2) -> (-3, 0) paints the pixel."""
    assert D.thick_line_mask(1, 1, 0, 2, -3, 0).tolist() == [[True]] == _cv_line(1, 1, (0, 2), (-3, 0)).tolist()
    for a, b in [((-20000, 5), (20000, 6)), ((3, -20000), (4, 20000)), ((-20000, -20000), (20000, 20000)), ((-5, -5), (-4, -100))]:
        assert np.array_equal(D.thick_line_mask(33, 17, *a, *b), _cv_line(33, 17, a, b)), (a, b)


def test_filled_circle_bit_equal_to_cv2():
    rng = np.random.default_rng(7)
    bad = []
    for t in range(1000):
        h, w = SIZES[t % len(SIZES)]
        r = int(rng.integers(1, 13))
        c = _point(rng, h, w, int(rng.integers(0, 5))) if t % 3 else (int(rng.integers(-15, w + 15)), int(rng.integers(-15, h + 15)))
        if not np.array_equal(_cv_circle(h, w, c, r), D.circle_mask(h, w, *c, r)):
            bad.append((h, w, c, r))
    assert not bad, bad[:5]


def _reference_like(frame, kp, ids, skeleton, thr, pts, lms):
    """draw()'s loop with live cv2 on a BGR copy (the reference's calls, with the palettes passed in)."""
    img = np.ascontiguousarray(frame[..., ::-1])
    h, w = img.shape[:2]
    r = max(1, min(h, w) // 150)
    for idx, k in zip(ids, kp):
        for a, b in skeleton:
            if k[a, 2] > thr and k[b, 2] > thr:
                cv2.line(img, (int(k[a, 1]), int(k[a, 0])), (int(k[b, 1]), int(k[b, 0])), tuple(int(v) for v in lms[idx % len(lms)]), 2)
        for i, p in enumerate(k):
            if p[2] > thr:
                cv2.circle(img, (int(p[1]), int(p[0])), r, tuple(int(v) for v in pts[i % len(pts)]), -1)
    return np.ascontiguousarray(img[..., ::-1])


def test_draw_loop_matches_reference_fixture(golden_dir):
    """The oracle's draw loop and the same loop on live cv2 both reproduce the reference-drawn frames (CRC-32 of the frame
    and a patch), for every case of oracle/make_golden_draw.py."""
    import os

    from easy_vitpose_b200.draw import reference_palettes
    from oracle.make_golden_draw import CASES, patch
    g = np.load(os.path.join(golden_dir, "draw_poses.npz"))
    pts, lms = reference_palettes()
    for c, (seed, h, w, ds, n, ids, thr) in enumerate(CASES):
        frame, kp = D.make_case(seed, h, w, n, int(g[f"num_keypoints_{ds}"]))
        sk = g[f"skeleton_{ds}"]
        mine = D.draw_poses([frame.copy()], kp, [n], sk, pts, lms, person_index=ids, threshold=thr)[0]
        assert zlib.crc32(mine.tobytes()) == int(g["case_crc32"][c]), (c, ds)
        assert np.array_equal(patch(mine, kp), g["case_patch"][c])
        live = _reference_like(frame, kp, ids if ids is not None else range(n), sk, np.float32(thr), pts, lms)
        assert np.array_equal(live, mine), c


def test_fixture_skeletons_fit_the_table_limits(golden_dir):
    import os

    from easy_vitpose_b200.draw import MAX_LIMBS
    g = np.load(os.path.join(golden_dir, "draw_poses.npz"))
    assert "wholebody" in g["datasets"] and len(g["skeleton_wholebody"]) == 65 and int(g["num_keypoints_wholebody"]) == 133
    for ds in g["datasets"]:
        sk = g[f"skeleton_{ds}"]
        assert len(sk) <= MAX_LIMBS and sk.min() >= 0 and sk.max() < int(g[f"num_keypoints_{ds}"]), ds


def test_restated_palettes_match_matplotlib():
    mpl = pytest.importorskip("matplotlib")
    from easy_vitpose_b200.draw import RestatedColormap, palette
    x = np.linspace(0, 1, 1001)
    for name in ("gist_rainbow", "jet"):
        assert np.array_equal(RestatedColormap(name)(x), mpl.colormaps[name](x)), name
    for name, s in (("gist_rainbow", 10), ("jet", 8)):
        want = np.round(np.array(mpl.colormaps[name](np.linspace(0, 1, s))) * 255).astype(np.uint8)[:, -2::-1]
        assert np.array_equal(palette(name, s), want)


def test_restated_palettes_shape_and_ends():
    """Without matplotlib: the tables draw() passes, and the colormap end points from the published segment data."""
    from easy_vitpose_b200.draw import RestatedColormap, reference_palettes
    pts, lms = reference_palettes()
    assert pts.shape == (10, 3) and lms.shape == (8, 3) and pts.dtype == lms.dtype == np.uint8
    assert RestatedColormap("jet")(np.array([0.0, 1.0]))[:, :3].tolist() == [[0, 0, 0.5], [0.5, 0, 0]]
    assert RestatedColormap("gist_rainbow")(np.array([0.0, 1.0]))[:, :3].tolist() == [[1, 0, 0.16], [1, 0, 0.75]]
    assert lms[0].tolist() == [128, 0, 0] and lms[-1].tolist() == [0, 0, 128]           # BGR of jet's dark blue and dark red


def test_plan_checks_arguments():
    from easy_vitpose_b200 import draw as Dr
    sk = [[0, 1], [1, 2]]
    p = Dr.plan([(10, 20), (5, 5)], [60, 15], 3, 4, [2, 1], sk, channel_order="bgr", radius=3, confidence_threshold=0.25)
    assert p.n == 3 and p.k == 4 and p.channel_order == 1 and p.radius == 3 and p.threshold == 0.25
    assert p.limbs.tolist() == sk and p.point_bgr.shape == (10, 3) and p.limb_bgr.shape == (8, 3)
    assert (p.canvases[0].height, p.canvases[0].width, p.canvases[0].pitch_bytes, p.canvases[0].num_people) == (10, 20, 60, 2)
    bad = [dict(channel_order="yuv"), dict(counts=[2, 2]), dict(counts=[3]), dict(counts=[-1, 4]), dict(skeleton=[[0, 4]]),
           dict(skeleton=[[0, 1]] * 129), dict(skeleton=[[-1, 0]]), dict(point_colors=np.zeros((0, 3))), dict(limb_colors=np.zeros((65, 3))),
           dict(limb_colors=np.zeros((4, 4))), dict(point_colors=[[256, 0, 0]]), dict(radius=1024), dict(pitches=[59, 15]),
           dict(shapes=[(0, 20), (5, 5)]), dict(k=0)]
    for kw in bad:
        args = dict(shapes=[(10, 20), (5, 5)], pitches=[60, 15], n=3, k=4, counts=[2, 1], skeleton=sk)
        args.update(kw)
        with pytest.raises(ValueError):
            Dr.plan(**args)
    # frames without people are not checked and do not count towards the frame limit
    Dr.plan([(0, 0)] + [(4, 4)] * 64, [0] + [12] * 64, 64, 2, [0] + [1] * 64, [[0, 1]])
    with pytest.raises(ValueError):
        Dr.plan([(4, 4)] * 65, [12] * 65, 65, 2, [1] * 65, [[0, 1]])


def test_header_declares_the_draw_calls():
    import os
    import re

    from easy_vitpose_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vitpose_b200.h")).read()
    assert {"vpb_draw_poses", "vpb_draw_workspace_bytes"} <= set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr)) <= set(_lib.EXPORTS)
    assert re.search(r"#define VPB_DRAW_RGB 0", hdr) and re.search(r"#define VPB_DRAW_BGR 1", hdr)
