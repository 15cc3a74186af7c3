"""Writes tests/golden/draw_poses.npz: every dataset's skeleton from the reference's joints_dict() and CRC-32s of frames the
UNMODIFIED reference draw_points_and_skeleton drew, in VitInference.draw()'s loop (easy_ViTPose/inference.py:302-312).

matplotlib is not installed here: its stub gets a `get_cmap` that returns easy_vitpose_b200.draw's restated colormaps, so the
palette values themselves are not pinned against matplotlib; the loop semantics are (painter's order, int() truncation, the
strict threshold, person_index % 8, i % 10, the per-frame circle radius).  Run: python -m oracle.make_golden_draw
"""
from __future__ import annotations

import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easy_vitpose_b200.draw import RestatedColormap  # noqa: E402
from oracle import draw_oracle as D, ref_import  # noqa: E402

# (seed, height, width, dataset, people, person ids or None, threshold)
CASES = [(1, 1, 1, "coco", 3, None, 0.5), (2, 7, 5, "coco", 4, None, 0.5), (3, 33, 17, "coco_25", 5, [7, 3, 12, 0, 9], 0.5),
         (4, 120, 160, "wholebody", 3, None, 0.3), (5, 240, 320, "ap10k", 9, [0, 1, 2, 3, 4, 5, 6, 7, 8], 0.5),
         (6, 1080, 1920, "coco", 12, [5, 17, 2, 9, 30, 1, 8, 4, 11, 6, 3, 10], 0.5), (7, 480, 640, "mpii", 6, None, 0.5),
         (8, 360, 480, "aic", 6, None, 0.7)]


def reference_draw(vis, frame_rgb, kpts, ids, skeleton, thr):
    img = np.array(frame_rgb)[..., ::-1]
    for idx, k in zip(ids, kpts):
        img = vis.draw_points_and_skeleton(img.copy(), k, skeleton, person_index=idx, points_color_palette="gist_rainbow",
                                           skeleton_color_palette="jet", points_palette_samples=10, confidence_threshold=thr)
    return np.ascontiguousarray(img[..., ::-1])


def patch(img, kp):
    """The 16 x 16 patch (zero-padded) around the first keypoint of the first person (the frame centre if it is outside)."""
    h, w = img.shape[:2]
    y = int(kp[0, 0, 0]) if 0 <= kp[0, 0, 0] < h else h // 2
    x = int(kp[0, 0, 1]) if 0 <= kp[0, 0, 1] < w else w // 2
    return np.pad(img, ((8, 8), (8, 8), (0, 0)))[y:y + 16, x:x + 16]


def main():
    import importlib
    ref_import.load()
    sys.modules["matplotlib.pyplot"].get_cmap = RestatedColormap
    vis = importlib.import_module("vit_utils.visualization")
    joints = vis.joints_dict()
    out = {"datasets": np.array(sorted(joints))}
    for name in sorted(joints):
        out[f"skeleton_{name}"] = np.asarray(joints[name]["skeleton"], np.int32).reshape(-1, 2)
        out[f"num_keypoints_{name}"] = np.int32(len(joints[name]["keypoints"]))
    crcs, patches = [], []
    for seed, h, w, ds, n, ids, thr in CASES:
        frame, kp = D.make_case(seed, h, w, n, int(out[f"num_keypoints_{ds}"]))
        got = reference_draw(vis, frame, kp, ids if ids is not None else range(n), joints[ds]["skeleton"], thr)
        crcs.append(zlib.crc32(got.tobytes()))
        patches.append(patch(got, kp))
    out["case_crc32"] = np.array(crcs, np.uint32)
    out["case_patch"] = np.stack(patches)
    path = os.path.join(ROOT, "tests", "golden", "draw_poses.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
