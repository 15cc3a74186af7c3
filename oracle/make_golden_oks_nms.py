"""Writes tests/golden/oks_nms.npz from the UNMODIFIED reference oks_iou / oks_nms / soft_oks_nms (post_processing/nms.py).

Each case is a set of frames (K = 17 or 133, separated crowds and duplicate-heavy ones with many jittered copies of a few
people, and frames of 0 and 1 person) run through the reference per frame with its thr / vis_thr / soft settings.  Cases with
`rescore` first apply HRNet's rescoring (oracle/oks_nms_oracle.rescore, which the reference dropped) to the box scores and
hand the reference the rescored values.  Scores are continuous draws, redrawn until no frame is ambiguous
(oks_nms_oracle.flag_ambiguous) and no score ties, so the reference's unstable sort and the device's stable one agree; the
script asserts that.  Stored per K (k17_*, k133_*): keypoints, areas, counts and sigmas (empty = the COCO-17 table); per
case: the box scores, the scores the sort used, the kept indices (concatenated, per-frame counts in keep_counts), and the
reference's float32 OKS matrix of every frame (concatenated row-major n_f x n_f blocks).

    python -m oracle.make_golden_oks_nms
"""
from __future__ import annotations

import os

import numpy as np

from oracle import oks_nms_oracle as O

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "oks_nms.npz")

# (name, K, soft, vis_thr, thr, rescore_vis_thr)
CASES = [(f"k{K}_{'soft' if soft else 'hard'}_{'vis' if vis is not None else 'all'}_t{int(thr * 10)}", K, soft, vis, thr,
          vis if (vis is not None and thr == 0.9) else None)
         for K in (17, 133) for soft in (False, True) for vis in (None, 0.2) for thr in (0.5, 0.9)]
FRAMES = 10


def sigmas_for(K):
    return None if K == 17 else np.random.default_rng(K).uniform(0.02, 0.11, K)


def _frame(rng, K, n, dup):
    """n people: separated (dup False) or jittered copies of a few (dup True), float32 (y, x, score), areas, box scores."""
    people = max(1, n // 4) if dup else n
    base = rng.uniform(0, 640, (people, 1, 2)) + rng.normal(0, 40, (people, K, 2))
    src = rng.integers(0, people, n) if dup else np.arange(n)
    kp = np.zeros((n, K, 3), np.float32)
    kp[:, :, :2] = base[src] + rng.normal(0, 1, (n, 1, 1)) * rng.choice([0.3, 2.0, 8.0], (n, 1, 1)) * rng.normal(0, 1, (n, K, 2))
    kp[:, :, 2] = rng.uniform(0, 1, (n, K))
    areas = rng.uniform(2e3, 6e4, people)[src] * (rng.uniform(0.9, 1.1, n) if dup else 1.0)
    return kp, areas


def frames_for(K):
    """The frames every case of K runs on: keypoints, areas, counts (seeded by K)."""
    rng = np.random.default_rng(K)
    out = []
    for f in range(FRAMES):
        n = [0, 1, 2, 40, 25][f] if f < 5 else int(rng.integers(3, 40 if K == 17 else 24))
        out.append(_frame(rng, K, n, dup=f % 2 == 1))
    return out


def make_case(case):
    """-> per-case arrays: box_scores and the scores the sort used [n], keep / keep_counts, the OKS matrices."""
    name, K, soft, vis, thr, rsc = case
    rng = np.random.default_rng([ord(c) for c in name])
    sig = sigmas_for(K)
    R = O.load_reference_nms()
    box, used, keep, kc, oks = [], [], [], [], []
    for f, (kp, ar) in enumerate(frames_for(K)):
        n = len(kp)
        for _ in range(100):
            b = rng.uniform(0.05, 1.0, n)
            s = O.rescore(kp, b, rsc) if rsc is not None else b
            if len(np.unique(s)) == n and not O.flag_ambiguous(kp, ar, b, thr, sig, vis, soft, 20, rsc):
                break
        else:
            raise AssertionError(f"{name} frame {f}: no unambiguous scores in 100 draws")
        db = O.kpts_db(kp, ar, s)
        k = R.soft_oks_nms(db, thr, 20, sig, vis) if soft else R.oks_nms(db, thr, sig, vis)
        k = np.asarray(k, np.int64).reshape(-1)
        mine, _ = O.run_frame(kp, ar, b, thr, sig, vis, soft, 20, rsc)
        assert np.array_equal(k, mine), (name, f)
        flat = kp.reshape(n, K * 3)
        m = np.stack([R.oks_iou(flat[i], flat, ar[i], ar, sig, vis) for i in range(n)]) if n else np.zeros((0, 0), np.float32)
        box.append(b); used.append(s); keep.append(k); kc.append(len(k)); oks.append(m.reshape(-1))
    return dict(box_scores=np.concatenate(box), scores=np.concatenate(used), keep=np.concatenate(keep),
                keep_counts=np.array(kc, np.int32), oks=np.concatenate(oks).astype(np.float32))


def inputs_for(K):
    fr = frames_for(K)
    sig = sigmas_for(K)
    return dict(kpts=np.concatenate([f[0] for f in fr]), areas=np.concatenate([f[1] for f in fr]),
                counts=np.array([len(f[0]) for f in fr], np.int32), sigmas=np.zeros(0) if sig is None else sig)


def main():
    out = {f"k{K}_{k}": v for K in (17, 133) for k, v in inputs_for(K).items()}
    for case in CASES:
        for k, v in make_case(case).items():
            out[f"{case[0]}_{k}"] = v
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(CASES)} cases")


if __name__ == "__main__":
    main()
