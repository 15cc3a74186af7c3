"""CPU: oracle/preproc_oracle.py (SURVEY.md section 8 row f1) against the fixtures the UNMODIFIED reference produced
(oracle/make_golden_frames.py, oracle/make_golden_reference_checks.py) and against cv2 where it is installed."""
import os

import numpy as np
import pytest

from oracle import preproc_oracle as P


def _case(golden_dir, name):
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    fh, fw, fseed = (int(v) for v in g["meta"][:3])
    rows = g["rows"].astype(np.float64)
    boxes = rows[rows[:, 4] > 0.35, :4].round().astype(int)            # easy_ViTPose/inference.py:240,253
    return g, P.make_frame(fh, fw, fseed), boxes


@pytest.mark.parametrize("name", ["frame_a", "frame_b"])
def test_preprocess_matches_reference_fixture(golden_dir, name):
    g, frame, boxes = _case(golden_dir, name)
    crops, org_wh, offs = P.preprocess_frame(frame, boxes)
    assert np.array_equal(P.normalise_lut(), g["lut"])
    assert np.array_equal(org_wh, g["org_wh"]) and np.array_equal(offs, g["offs_yx"])
    for i in range(len(boxes)):
        canvas, _ = P.crop_canvas(frame, boxes[i])
        assert np.array_equal(P.resize_linear_u8(canvas), g["resized"][i])
        want = np.stack([g["lut"][c][g["resized"][i][..., c]] for c in range(3)], 0)
        assert np.array_equal(crops[i], want)


def test_pad_geometry_is_the_reference_rule():
    """pad_image decides with floats (w / h < 3 / 4, int(0.75 * h), int(w / 0.75)); the oracle with integers."""
    for w in range(1, 140):
        for h in range(1, 140):
            ar = w / h
            if ar < 3 / 4:
                tw = int(3 / 4 * h); want = (tw, h, (tw - w) // 2, 0)
            else:
                th = int(w / (3 / 4)); want = (w, th, 0, (th - h) // 2)
            assert P.pad_geometry(w, h) == want, (w, h)
    with pytest.raises(ValueError):
        P.pad_geometry(0, 5)


def test_padded_box_clips_to_frame():
    assert P.padded_box((5, 3, 50, 40), 100, 200) == (0, 0, 60, 50)
    assert P.padded_box((150, 80, 260, 130), 100, 200) == (140, 70, 200, 100)
    assert P.padded_box((300, 300, 310, 310), 100, 200) == (200, 100, 200, 100)      # empty: the reference raises later


def test_resize_matches_cv2_on_random_sizes():
    cv2 = pytest.importorskip("cv2")
    rs = np.random.RandomState(0)
    sizes = [(rs.randint(1, 700), rs.randint(1, 600)) for _ in range(25)] + [(256, 192), (512, 384), (1, 1), (2, 3), (1080, 810)]
    for h, w in sizes:
        img = rs.randint(0, 256, size=(h, w, 3), dtype=np.uint8)
        assert np.array_equal(P.resize_linear_u8(img), cv2.resize(img, (192, 256), interpolation=cv2.INTER_LINEAR)), (h, w)


def test_to_frame_coords_is_one_rounding():
    rs = np.random.RandomState(1)
    kp = (rs.rand(4, 17, 3) * 400).astype(np.float32)
    offs = rs.randint(-50, 2000, size=(4, 2)).astype(np.int32)
    out = P.to_frame_coords(kp, offs)
    assert np.array_equal(out[..., :2], kp[..., :2] + offs[:, None, :].astype(np.float32))     # float32 add == f64 add then cast
    assert np.array_equal(out[..., 2], kp[..., 2])


def test_against_reference_pad_image_and_pre_img(golden_dir):
    """The oracle's canvas and pre_img against the unmodified reference's pad_image / pre_img on seeded boxes (stored by
    oracle/make_golden_reference_checks.py: whole canvases; pre_img's whole output for the first boxes, a seeded sample of it
    for the others)."""
    from oracle.make_golden_reference_checks import PRE_FULL, pre_boxes, pre_sample_index, unpack_exact
    g = np.load(os.path.join(golden_dir, "reference_checks.npz"))
    frame = P.make_frame(200, 260, 5)
    cases = pre_boxes()
    assert np.array_equal(np.array([b for b, _ in cases]), g["pre_boxes"])
    for i, (box, (bx0, by0, _, _)) in enumerate(cases):
        left, top = (int(v) for v in g["pre_left_top"][i])
        canvas, off = P.crop_canvas(frame, box)
        assert np.array_equal(canvas, g[f"canvas_{i}"]) and off == (by0 - top, bx0 - left)
        x = P.pre_img(canvas)
        assert np.array_equal(np.asarray(x, np.float32).reshape(-1)[pre_sample_index(i)], g["pre_x_sample"][i])
        if i < PRE_FULL:
            assert np.array_equal(np.asarray(x, np.float32), unpack_exact(g[f"pre_x_table_{i}"], g[f"pre_x_index_{i}"]))
        assert tuple(canvas.shape[:2]) == tuple(int(v) for v in g["pre_org_hw"][i])
