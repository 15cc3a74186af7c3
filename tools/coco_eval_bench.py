"""Times COCO keypoint evaluation (coco_eval / vpb_coco_eval) on a seeded set shaped like COCO val2017 person keypoints:
5000 images, about 6.4 k ground-truth people (about half the images have none; crowds and num_keypoints == 0 people among
them), up to 20 kept detections per image (jittered copies of the image's people plus false positives):
  device_replay   coco_eval_device captured once in a CUDA graph and replayed (CUDA events around all replays)
  device_eager    coco_eval_device on inputs already on the device (CUDA events)
  host_dropin     coco_eval.evaluate(gts, records, image_ids): packing, upload, the device call and the read-back (host clock)
  oracle_cpu_subset  oracle/coco_oks_eval.evaluate on the host CPU (host clock, one run), on the first --oracle-images images
                  only: its per-image filtering scans every annotation, so its time grows with the square of the set size
Before timing, the device's ten stats, precision and recall on that subset are checked bit for bit against the oracle.
Three runs of every other arm after a warm-up; prints one JSON line with the card's name and power limit.

    python tools/coco_eval_bench.py [--iters 50] [--oracle-images 1000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import coco_eval_oracle as CO  # noqa: E402
from oracle import coco_oks_eval as E  # noqa: E402

RUNS = 3


def val2017_like(seed=2017, n_img=5000, K=17):
    """(gts, records, image_ids): about 6.4 k people over 5000 images, at most 20 detections per image."""
    rng = np.random.default_rng(seed)
    image_ids = sorted(int(v) for v in rng.choice(np.arange(1, 600000), n_img, replace=False))
    gts, recs, gid = [], [], 1
    for img in image_ids:
        G = int(rng.choice([0, 1, 2, 3, 4, 6, 10], p=[0.46, 0.25, 0.12, 0.07, 0.05, 0.03, 0.02]))
        people = []
        for _ in range(G):
            w, h = rng.uniform(10, 400), rng.uniform(20, 480)
            x, y = rng.uniform(0, 640 - w / 2), rng.uniform(0, 480 - h / 2)
            kp = np.stack([x + rng.uniform(0, w, K), y + rng.uniform(0, h, K), rng.choice([0.0, 1.0, 2.0], K, p=[0.4, 0.1, 0.5])], 1)
            if rng.uniform() < 0.1:
                kp[:, 2] = 0
            g = {"id": gid, "image_id": img, "category_id": 1, "iscrowd": int(rng.uniform() < 0.01),
                 "num_keypoints": int(np.count_nonzero(kp[:, 2])), "keypoints": kp.reshape(-1).tolist(),
                 "bbox": [float(x), float(y), float(w), float(h)], "area": float(w * h * rng.uniform(0.4, 0.9))}
            gid += 1
            gts.append(g)
            people.append(kp)
        D = min(20, G + int(rng.integers(0, 4)) + (2 * G if rng.uniform() < 0.3 else 0))
        for _ in range(D):
            if people and rng.uniform() < 0.8:
                base = people[int(rng.integers(len(people)))][:, :2]
                xy = np.round(base + rng.normal(0, rng.choice([1.0, 4.0, 15.0]), base.shape))
            else:
                xy = np.round(rng.uniform(0, 640, (K, 2)))
            recs.append({"image_id": img, "category_id": 1, "score": float(rng.uniform()),
                         "keypoints": np.concatenate([xy, np.zeros((K, 1))], 1).reshape(-1).tolist()})
    return gts, recs, image_ids


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = out[0].split(", ")
        return name, power
    except Exception as exc:                                            # reported, never guessed
        return f"unknown ({exc})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--oracle-images", type=int, default=1000)
    a = ap.parse_args()
    import torch

    from easy_vitpose_b200 import coco_eval
    warnings.simplefilter("ignore", RuntimeWarning)
    name, power = card()
    gts, recs, ids = val2017_like()

    # exactness on the oracle's subset first
    sub = ids[:a.oracle_images]
    sub_set = set(sub)
    sgts = [g for g in gts if g["image_id"] in sub_set]
    srecs = [r for r in recs if r["image_id"] in sub_set]
    flagged = len(CO.flag_ambiguous(sgts, srecs, sub))
    want = CO.evaluate_full(sgts, srecs, sub)
    ev = coco_eval.DeviceCocoEval(sgts, sub)
    ev.add(srecs)
    got = ev.evaluate()
    exact = (all(np.float64(got[k]).tobytes() == np.float64(want["stats"][k]).tobytes() for k in CO.STAT_NAMES)
             and np.array_equal(got["precision"].cpu().numpy(), want["precision"])
             and np.array_equal(got["recall"].cpu().numpy(), want["recall"]))

    # the full set on the device
    ev = coco_eval.DeviceCocoEval(gts, ids)
    ev.add(recs)
    stats = ev.evaluate()
    dev = ev.device
    args = [torch.cat([c[j] for c in ev._chunks]) for j in range(6)]
    ws = torch.empty(coco_eval.workspace_bytes(len(ids), args[2].shape[0]), dtype=torch.uint8, device=dev)
    out = coco_eval.CocoEvalResult(torch.empty(10, dtype=torch.float64, device=dev), torch.empty((3, 10, 101), dtype=torch.float64, device=dev),
                                   torch.empty((3, 10), dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))

    def call():
        coco_eval.coco_eval_device(*ev._gt, *args, workspace=ws, out=out)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    g.replay()
    torch.cuda.synchronize()
    assert int(out.status.item()) == 0 and np.array_equal(out.stats.cpu().numpy(), [stats[k] for k in CO.STAT_NAMES])

    def events(fn):
        ms = []
        for _ in range(RUNS):
            fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            ms.append(t0.elapsed_time(t1) / a.iters)
        return ms

    def host(fn, n):
        ms = []
        fn()
        for _ in range(RUNS):
            t0 = time.perf_counter()
            for _ in range(n):
                fn()
            ms.append((time.perf_counter() - t0) * 1e3 / n)
        return ms

    arms = {"device_replay": events(g.replay), "device_eager": events(call),
            "host_dropin": host(lambda: coco_eval.evaluate(gts, recs, ids), 1)}
    t0 = time.perf_counter()
    E.evaluate(sgts, srecs, sub)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    arms["oracle_cpu_subset"] = [oracle_ms]
    res = {"card": name, "power_limit": power, "images": len(ids), "gt_people": len(gts), "detections": len(recs), "iters": a.iters,
           "ms": {k: [round(v, 4) for v in vs] for k, vs in arms.items()},
           "median_ms": {k: round(float(np.median(vs)), 4) for k, vs in arms.items()},
           "oracle_images": len(sub), "oracle_gt_people": len(sgts), "oracle_detections": len(srecs),
           "subset_bit_exact": bool(exact), "subset_flagged": flagged, "stats": {k: stats[k] for k in CO.STAT_NAMES}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
