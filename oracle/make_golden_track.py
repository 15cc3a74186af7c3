"""Generates tests/golden/track_sort.npz: what the UNMODIFIED easy_ViTPose/sort.py returns on seeded multi-stream sequences.

Each case runs one reference `Sort` per stream, updated round-robin in one process (`KalmanBoxTracker.count` starts at 0),
loaded by sort_oracle.load_reference_sort(): matplotlib / skimage stubbed, filterpy's KalmanFilter restated, and `import lap`
raising ImportError so that scipy's linear_sum_assignment is used, as in the reference environment.  The detections are
regenerated from seeds by sort_oracle.make_sequence.  Stored per case: every output's row count and CRC-32 (of the float64
bytes, -0.0 written as +0.0), the raw rows of the first stream over its first RAW_FRAMES frames, and the id counter at the end.

    python -m oracle.make_golden_track
"""
from __future__ import annotations

import os
import zlib

import numpy as np

from oracle import sort_oracle as SO

# (name, max_age, min_hits, yolo_step, frames, streams: (kind, people, width, height, seed))
CASES = [
    ("mixed", 1, 3, 1, 80, [("walk", 9, 1920, 1080, 1), ("crowd", 100, 900, 600, 2), ("jump", 12, 1920, 1080, 3), ("dup", 6, 1920, 1080, 4),
                            ("shrink", 8, 1920, 1080, 5), ("empty", 5, 1920, 1080, 6)]),
    ("cadence3", 3, 1, 3, 90, [("walk", 9, 1920, 1080, 11), ("crowd", 40, 700, 500, 12), ("jump", 10, 1920, 1080, 13),
                               ("shrink", 8, 1920, 1080, 14), ("occlude", 9, 1920, 1080, 15)]),
    ("gaps", 5, 1, 1, 80, [("occlude", 9, 1920, 1080, 21), ("walk", 9, 1920, 1080, 22), ("crowd", 60, 800, 600, 23)]),
]


RAW_FRAMES = 30                      # raw rows of stream 0 are kept for the first frames of a case


def case_inputs(case):
    """Per frame, the list of per-stream detection arrays the case feeds (empty where the detector is skipped: frames with
    frame_counter >= 3 and frame_counter % yolo_step != 0, inference.py:234-236)."""
    name, max_age, min_hits, step, frames, streams = case
    seqs = [SO.make_sequence(seed, frames, people, kind, float(w), float(h)) for kind, people, w, h, seed in streams]
    empty = np.empty((0, 5))
    return [[seq[f] if (f < 3 or f % step == 0) else empty for seq in seqs] for f in range(frames)]


def crc(rows: np.ndarray) -> int:
    return zlib.crc32(np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 6) + 0.0).tobytes())


def run_reference(ref, case):
    """(counts [F, S], crcs [F, S], first-stream rows of the first RAW_FRAMES frames, final count) from S reference Sorts."""
    name, max_age, min_hits, step, frames, streams = case
    ref.KalmanBoxTracker.count = 0
    sorts = [ref.Sort(max_age=max_age, min_hits=min_hits, iou_threshold=0.3) for _ in streams]
    counts, crcs, first = [], [], []
    for f, dl in enumerate(case_inputs(case)):
        outs = [s.update(d) for s, d in zip(sorts, dl)]
        counts.append([len(o) for o in outs])
        crcs.append([crc(o) for o in outs])
        if f < RAW_FRAMES:
            first.append(outs[0].reshape(-1, 6))
    return np.array(counts, np.int32), np.array(crcs, np.uint32), np.concatenate(first), int(ref.KalmanBoxTracker.count)


def main():
    ref = SO.load_reference_sort()
    out = {"names": np.array([c[0] for c in CASES])}
    for case in CASES:
        counts, crcs, first, final = run_reference(ref, case)
        out[f"{case[0]}_counts"] = counts
        out[f"{case[0]}_crc32"] = crcs
        out[f"{case[0]}_stream0_rows"] = first
        out[f"{case[0]}_next_id"] = np.array(final)
        print(case[0], "rows", int(counts.sum()), "ids", final)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "track_sort.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
