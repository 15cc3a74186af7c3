"""Generates tests/golden/smooth_one_euro.npz: what the UNMODIFIED reference `OneEuroFilter`, composed per track id as
oracle/one_euro_oracle.py states, returns on seeded multi-stream sequences.

The ids are SORT's: oracle/sort_oracle.SortOracle run on a case of oracle/make_golden_track.py, so they carry the reference
tracker's churn, gaps and min_hits silences.  Each output row gets keypoints drawn inside its box around a per-id pose, with
jitter, some coordinates at or below 0 (missing keypoints), as float32 [K, 3].  Cases cover K = 17 and 133, fps mode and
realtime mode (uneven timestamps with one dropped frame), non-default (min_cutoff, beta, d_cutoff, dx0), max_gap 0 and 30.
Stored per case: every update's per-stream row count and CRC-32 of the float64 output (NaN canonical, -0.0 written as
+0.0), and the raw output rows of the first stream over the first RAW_FRAMES updates.

    python -m oracle.make_golden_smooth
"""
from __future__ import annotations

import os
import zlib

import numpy as np

from oracle import make_golden_track as MT
from oracle import one_euro_oracle as OE
from oracle import sort_oracle as SO

# (name, tracking case, K, filter parameters, max_gap)
CASES = [
    ("fps17", "mixed", 17, dict(fps=30.0), 30),
    ("fps133_gap0", "cadence3", 133, dict(fps=25.0), 0),
    ("realtime17", "gaps", 17, dict(fps=None), 30),
    ("realtime133_custom", "cadence3", 133, dict(fps=None, min_cutoff=0.8, beta=0.05, d_cutoff=15.0, dx0=0.25), 0),
    ("fps17_custom", "gaps", 17, dict(fps=30.0, min_cutoff=0.5, beta=0.7, dx0=-1.5), 30),
]
RAW_FRAMES = 4


def tracked_rows(track_case: str):
    """Per frame, the per-stream SORT output rows [m, 6] (x1, y1, x2, y2, score, id + 1) of a make_golden_track case."""
    case = next(c for c in MT.CASES if c[0] == track_case)
    o = SO.SortOracle(len(case[5]), case[1], case[2], 0.3)
    return [o.update(dl) for dl in MT.case_inputs(case)]


def keypoints(rows: np.ndarray, K: int, frame: int, seed: int) -> np.ndarray:
    """float32 [m, K, 3] (y, x, score): each id's pose (seeded by the id) placed in its box, jittered per frame; about 4% of
    the coordinates are 0 or negative."""
    out = np.zeros((len(rows), K, 3), np.float32)
    rng = np.random.default_rng([seed, frame])
    for r, row in enumerate(rows):
        pose = np.random.default_rng([seed, int(row[5])]).uniform(0.05, 0.95, (K, 2))
        h, w = row[3] - row[1], row[2] - row[0]
        y = row[1] + pose[:, 0] * h + rng.normal(0, 1.5, K)
        x = row[0] + pose[:, 1] * w + rng.normal(0, 1.5, K)
        yx = np.stack([y, x], 1)
        missing = rng.uniform(size=(K, 2)) < 0.04
        yx[missing] = rng.choice([0.0, -3.25, -40.0], size=int(missing.sum()))
        out[r, :, :2] = yx
        out[r, :, 2] = rng.uniform(0, 1, K)
    return out


def timestamps(frames: int, seed: int) -> np.ndarray:
    """Uneven capture times in seconds around 30 fps, with frame 7's slot dropped (a double interval)."""
    rng = np.random.default_rng(seed)
    dt = rng.uniform(0.9, 1.1, frames) / 30.0
    dt[7] *= 2.0
    return 1.7e9 + np.cumsum(dt)


def case_inputs(case):
    """Per update: (per-stream keypoints [m, K, 3], per-stream ids, per-stream clock or None)."""
    name, track_case, K, params, max_gap = case
    seed = zlib.crc32(name.encode())
    outs = []
    ts = timestamps(200, seed) if params.get("fps") is None else None
    for f, rows_s in enumerate(tracked_rows(track_case)):
        kl = [keypoints(r, K, f, seed + s) for s, r in enumerate(rows_s)]
        il = [r[:, 5].astype(np.int64).tolist() for r in rows_s]
        clock = None if ts is None else [float(ts[f])] * len(rows_s)
        outs.append((kl, il, clock))
    return outs


def make_oracle(case, num_streams: int, filter_cls=None, limit: bool = False) -> OE.SmoothOracle:
    name, track_case, K, params, max_gap = case
    return OE.SmoothOracle(num_streams, max_gap=max_gap, filter_cls=filter_cls, limit=limit, **params)


def crc(out: np.ndarray) -> int:
    a = np.asarray(out, np.float64) + 0.0
    a = np.where(np.isnan(a), np.nan, a)
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def run(case, filter_cls=None):
    """(counts [F, S], crcs [F, S], first-stream rows of the first RAW_FRAMES updates)."""
    inputs = case_inputs(case)
    o = make_oracle(case, len(inputs[0][0]), filter_cls)
    counts, crcs, first = [], [], []
    for f, (kl, il, clock) in enumerate(inputs):
        outs = o.update(kl, il, clock)
        counts.append([len(x) for x in outs])
        crcs.append([crc(x) for x in outs])
        if f < RAW_FRAMES:
            first.append(outs[0].reshape(-1, case[2], 2))
    return np.array(counts, np.int32), np.array(crcs, np.uint32), np.concatenate(first)


def main():
    ref = OE.load_reference_one_euro()
    out = {"names": np.array([c[0] for c in CASES])}
    for case in CASES:
        counts, crcs, first = run(case, ref)
        out[f"{case[0]}_counts"] = counts
        out[f"{case[0]}_crc32"] = crcs
        out[f"{case[0]}_stream0_rows"] = first
        print(case[0], "updates", len(counts), "rows", int(counts.sum()))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "smooth_one_euro.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
