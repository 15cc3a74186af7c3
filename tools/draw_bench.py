"""Times the device pose overlay (vpb_draw_poses) against draw()'s CPU loop on the ap10k-streams shape: 16 1920x1080 RGB
frames, 143 people, the COCO skeleton.

The CPU arm is VitInference.draw()'s pose loop (easy_ViTPose/inference.py:302-312) without its matplotlib calls: a BGR flip,
per person a copy of the whole frame, cv2.line per limb and cv2.circle per keypoint, and the flip back.  Both arms draw the same
seeded keypoints and are checked bit-identical before anything is timed.  Device time: one draw_poses call (setup + raster
launches) captured in a CUDA graph, CUDA events around `steps` back-to-back replays, divided by the steps.  Call time: the same
with eager draw_poses calls, host work (argument checks, workspace allocation, ctypes) included.  Each run is repeated and the
median of the runs reported.  Prints one JSON line, with the card's name and power limit.

    python tools/draw_bench.py [--steps 200] [--runs 3] [--cpu-steps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COCO_SKELETON = [[15, 13], [13, 11], [16, 14], [14, 12], [11, 12], [5, 11], [6, 12], [5, 6], [5, 7], [6, 8], [7, 9], [8, 10], [1, 2],
                 [0, 1], [0, 2], [1, 3], [2, 4], [3, 5], [4, 6]]          # COCO's 19 limbs (joints_dict()['coco']['skeleton'])


def workload(frames=16, people=143, h=1080, w=1920, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 7 + yy * 3) % 256, (xx * 5 + yy * 11) % 256, (xx ^ yy) % 256], -1).astype(np.uint8)
    imgs = [np.roll(base, 13 * j, axis=1) for j in range(frames)]
    counts = [people // frames + (j < people % frames) for j in range(frames)]
    kp = np.zeros((people, 17, 3), np.float32)
    hgt = rng.uniform(120, 420, people)                                   # person height in pixels
    cy, cx = rng.uniform(0, h, people), rng.uniform(0, w, people)
    kp[..., 0] = cy[:, None] + rng.uniform(-0.5, 0.5, (people, 17)) * hgt[:, None]
    kp[..., 1] = cx[:, None] + rng.uniform(-0.2, 0.2, (people, 17)) * hgt[:, None]
    kp[..., 2] = rng.uniform(0.2, 1.0, (people, 17))
    return imgs, kp, counts


def cpu_draw(imgs, kp, counts, pts, lms, thr=0.5):
    import cv2
    out, p = [], 0
    for img, c in zip(imgs, counts):
        img = np.array(img)[..., ::-1]
        r = max(1, min(img.shape[:2]) // 150)
        for idx in range(c):
            img = img.copy()
            k = kp[p]
            for a, b in COCO_SKELETON:
                if k[a, 2] > thr and k[b, 2] > thr:
                    img = cv2.line(img, (int(k[a, 1]), int(k[a, 0])), (int(k[b, 1]), int(k[b, 0])), tuple(lms[idx % 8].tolist()), 2)
            for i, q in enumerate(k):
                if q[2] > thr:
                    img = cv2.circle(img, (int(q[1]), int(q[0])), r, tuple(pts[i % 10].tolist()), -1)
            p += 1
        out.append(np.ascontiguousarray(img[..., ::-1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=5)
    args = ap.parse_args()
    import torch

    from easy_vitpose_b200.draw import draw_poses, reference_palettes
    assert torch.cuda.is_available(), "draw_bench needs a GPU"
    pts, lms = reference_palettes()
    imgs, kp, counts = workload()
    dev = [torch.from_numpy(im).cuda() for im in imgs]
    kd = torch.from_numpy(kp).cuda()
    draw_poses(dev, kd, counts, COCO_SKELETON)
    want = cpu_draw(imgs, kp, counts, pts, lms)
    same = all(np.array_equal(d.cpu().numpy(), w) for d, w in zip(dev, want))
    assert same, "device and CPU frames differ"
    covered = int(sum((w != im).any(-1).sum() for w, im in zip(want, imgs)))
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        draw_poses(dev, kd, counts, COCO_SKELETON)
    torch.cuda.synchronize()

    def timed(fn):
        for _ in range(10):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    dev_runs, call_runs, cpu_runs = [], [], []
    for _ in range(args.runs):
        dev_runs.append(timed(graph.replay))
        call_runs.append(timed(lambda: draw_poses(dev, kd, counts, COCO_SKELETON)))
        ts = []
        for _ in range(args.cpu_steps):
            t0 = time.perf_counter()
            cpu_draw(imgs, kp, counts, pts, lms)
            ts.append((time.perf_counter() - t0) * 1e3)
        cpu_runs.append(float(np.median(ts)))
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                                                  # the timing stands without the label
        card = f"unknown ({exc})"
    print(json.dumps({"workload": "ap10k-streams draw: 16 x 1920x1080, 143 people, coco skeleton", "bit_identical": same,
                      "changed_pixels": covered, "device_ms_per_step": float(np.median(dev_runs)), "device_ms_runs": dev_runs,
                      "call_ms_per_step": float(np.median(call_runs)), "call_ms_runs": call_runs,
                      "cpu_ms_per_step": float(np.median(cpu_runs)), "cpu_ms_runs": cpu_runs, "cpu_threads": os.cpu_count(), "card": card}))


if __name__ == "__main__":
    main()
