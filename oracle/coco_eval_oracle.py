"""COCO keypoint evaluation with its intermediate arrays  --  TEST INFRASTRUCTURE ONLY.

oracle/coco_oks_eval.py's `evaluate` returns the ten summary numbers.  `evaluate_full` runs the same evaluateImg (its
`_evaluate_img`, `load_results`, thresholds and area ranges) and the same accumulate / summarize, and also returns what
vpb_coco_eval is compared on: the precision [3, 10, 101] and recall [3, 10] arrays (area all / medium / large) and each image's
matches.  `flag_ambiguous` names the sets where CUDA's exp (not numpy's) could change a result: an OKS within a few ulps of a
threshold, or of a different OKS of the same detection that the greedy matching compares it with.
"""
from __future__ import annotations

import numpy as np

from oracle import coco_oks_eval as E

AREAS = tuple(E.AREA_RNG)               # ("all", "medium", "large"), the order of the device arrays
STAT_NAMES = ("AP", "AP50", "AP75", "AP_medium", "AP_large", "AR", "AR50", "AR75", "AR_medium", "AR_large")


def _per_image(gt_annotations, results, image_ids):
    dts_all = E.load_results(results)
    for img in image_ids:
        gts = [g for g in gt_annotations if g["image_id"] == img and g.get("category_id", 1) == 1]
        dts = [d for d in dts_all if d["image_id"] == img and d.get("category_id", 1) == 1]
        yield img, gts, dts


def evaluate_full(gt_annotations, results, image_ids, sigmas=E.KPT_OKS_SIGMAS) -> dict:
    """E.evaluate's computation, returning {"stats": {name: value}, "precision": [3, 10, 101], "recall": [3, 10],
    "evals": {area: [per image None or evaluateImg's dict]}}."""
    per = list(_per_image(gt_annotations, results, image_ids))
    T, R = len(E.IOU_THRS), len(E.REC_THRS)
    precision, recall = -np.ones((3, T, R)), -np.ones((3, T))
    evals_by_area = {}
    for a, (a_name, a_rng) in enumerate(E.AREA_RNG.items()):
        evs = [E._evaluate_img([dict(g) for g in gts], dts, a_rng, sigmas) for _, gts, dts in per]
        evals_by_area[a_name] = evs
        evals = [e for e in evs if e is not None]
        if not evals:
            continue
        dt_scores = np.concatenate([e["dtScores"][0:E.MAX_DETS] for e in evals])
        inds = np.argsort(-dt_scores, kind="mergesort")
        dtm = np.concatenate([e["dtMatches"][:, 0:E.MAX_DETS] for e in evals], axis=1)[:, inds]
        dt_ig = np.concatenate([e["dtIgnore"][:, 0:E.MAX_DETS] for e in evals], axis=1)[:, inds]
        gt_ig = np.concatenate([e["gtIgnore"] for e in evals])
        npig = np.count_nonzero(gt_ig == 0)
        if npig == 0:
            continue
        tp_sum = np.cumsum(np.logical_and(dtm, np.logical_not(dt_ig)), axis=1).astype(dtype=float)
        fp_sum = np.cumsum(np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig)), axis=1).astype(dtype=float)
        for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
            nd = len(tp)
            rc = tp / npig
            pr = (tp / (fp + tp + np.spacing(1))).tolist()
            q = np.zeros((R,))
            recall[a, t] = rc[-1] if nd else 0
            for i in range(nd - 1, 0, -1):
                if pr[i] > pr[i - 1]:
                    pr[i - 1] = pr[i]
            for ri, pi in enumerate(np.searchsorted(rc, E.REC_THRS, side="left")):
                if pi < nd:
                    q[ri] = pr[pi]
            precision[a, t] = q

    def _mean(arr):
        arr = arr[arr > -1]
        return float(np.mean(arr)) if arr.size else -1.0
    vals = [_mean(precision[0]), _mean(precision[0, 0]), _mean(precision[0, 5]), _mean(precision[1]), _mean(precision[2]),
            _mean(recall[0]), _mean(recall[0, 0:1]), _mean(recall[0, 5:6]), _mean(recall[1]), _mean(recall[2])]
    return {"stats": dict(zip(STAT_NAMES, vals)), "precision": precision, "recall": recall, "evals": evals_by_area}


def flag_ambiguous(gt_annotations, results, image_ids, sigmas=E.KPT_OKS_SIGMAS, ulps: int = 4) -> list:
    """(image id, detection, reason) for every OKS of a scored detection (the first 20 by score) that can reach the matching
    (>= the lowest threshold) and lies within `ulps` ulps of an OKS threshold or of a different OKS of the same detection.  Equal OKS values (duplicate ground truths) are not flagged: the
    device computes them from the same inputs the same way."""
    thrs = np.minimum(E.IOU_THRS, 1 - 1e-10)
    out = []
    for img, gts, dts in _per_image(gt_annotations, results, image_ids):
        if not gts or not dts:
            continue
        order = np.argsort([-d["score"] for d in dts], kind="mergesort")[:E.MAX_DETS]
        oks = E.compute_oks(gts, [dts[i] for i in order], sigmas)
        for d, row in enumerate(oks):
            for o in row:
                tol = ulps * np.spacing(max(abs(o), 1e-300))
                if np.isnan(o) or o < thrs[0] - tol:                      # never compared with anything that decides
                    continue
                if np.any(np.abs(thrs - o) <= tol):
                    out.append((img, d, f"OKS {o!r} near a threshold"))
                near = np.abs(row - o) <= tol
                if np.any(near & (row != o)):
                    out.append((img, d, f"OKS {o!r} near another OKS of the detection"))
    return out


def random_set(seed, K, n_img=40):
    """A seeded evaluation set -> (gts, records, image_ids sorted, sigmas or None for K = 17): every fifth image has ground
    truths only and the next detections only; up to 40 detections per image, a share of them tied or NaN; crowd, duplicate and
    no-visible-keypoint ground truths; areas from small through large."""
    rng = np.random.default_rng(seed)
    sig = None if K == 17 else rng.uniform(0.02, 0.12, K)
    image_ids = sorted(int(v) for v in rng.choice(np.arange(1, 10 ** 6), n_img, replace=False))
    gts, recs, gid = [], [], 1
    tied = [0.25, 0.5, 0.75]
    for j, img in enumerate(image_ids):
        kind = j % 5                                       # 0: gts only, 1: dets only, others both
        G = 0 if kind == 1 else int(rng.choice([1, 2, 3, 6, 12]))
        people = []
        for _ in range(G):
            w, h = rng.uniform(8, 260, 2)                  # areas from small through medium to large
            x, y = rng.uniform(0, 600, 2)
            kp = np.zeros((K, 3))
            kp[:, 0], kp[:, 1] = x + rng.uniform(0, w, K), y + rng.uniform(0, h, K)
            kp[:, 2] = rng.choice([0, 1, 2], K, p=[0.3, 0.2, 0.5])
            crowd = int(rng.uniform() < 0.1)
            if rng.uniform() < 0.12:                       # no visible keypoint: the bbox-distance OKS, num_keypoints 0
                kp[:, 2] = 0
            num = int(np.count_nonzero(kp[:, 2] > 0))
            g = {"id": gid, "image_id": img, "category_id": 1, "iscrowd": crowd, "num_keypoints": num,
                 "keypoints": kp.reshape(-1).tolist(), "bbox": [float(x), float(y), float(w), float(h)],
                 "area": float(w * h * rng.uniform(0.5, 1.0))}
            gid += 1
            gts.append(g)
            people.append(g)
            if rng.uniform() < 0.15:                       # a duplicate: equal OKS, the later ground truth wins
                gts.append(dict(g, id=gid))
                gid += 1
        if kind == 0:
            continue
        D = int(rng.choice([1, 3, 8, 25, 40]))
        for _ in range(D):
            if people and rng.uniform() < 0.85:
                g = people[int(rng.integers(len(people)))]
                base = np.array(g["keypoints"]).reshape(K, 3)[:, :2]
                spread = rng.choice([0.0, 0.02, 0.1, 0.3]) * np.sqrt(g["area"])
                xy = base + rng.normal(0, 1, (K, 2)) * spread
            else:
                xy = rng.uniform(0, 800, (K, 2))
            u = rng.uniform()
            score = float(rng.choice(tied)) if u < 0.4 else (float("nan") if u < 0.45 else float(rng.uniform()))
            kp = np.concatenate([xy, np.zeros((K, 1))], 1)
            recs.append({"image_id": img, "category_id": 1, "score": score, "keypoints": kp.reshape(-1).tolist()})
    order = rng.permutation(len(recs))                     # interleave the images' records
    recs = [recs[i] for i in sorted(order[:len(order) // 2])] + [recs[i] for i in sorted(order[len(order) // 2:])]
    return gts, recs, image_ids, sig
