#!/usr/bin/env python
"""Per-frame calls against packed multi-frame calls on the video workload of bench.py --config ap10k-streams: ViT-B/17, a step
= 16 consecutive 1080p frames with Poisson(10) detector boxes each (bench.py's stream_workload, rank 0, clipped to 1..32), the
frames and boxes resident in HBM.
  per_frame   16 infer_frame calls per step (what bench.py times)
  packed      one infer_frames call per step, split into engine calls of at most max_batch boxes
at max_batch 32 and 64.  Before timing, the packed outputs of every step are checked to equal the per-frame outputs bit for
bit.  Reported: ms per step and crops/s (CUDA events around `steps` back-to-back steps; the arms alternate, three runs each,
medians), and the per-frame latency: the time from the start of a step until the call that holds a frame's boxes has
finished, averaged over the frames of a step (a packed frame waits for its whole call).  Prints the card, its power limit and
maximum SM clock first: the numbers belong to them.

    python tools/multi_frame_bench.py [--steps 50] [--warmup 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import stream_workload  # noqa: E402
from easy_vitpose_b200 import ViTPose, model_cfg  # noqa: E402
from easy_vitpose_b200.model import plan_frame_chunks  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402

FRAMES_PER_STEP, MAX_BOXES = 16, 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    imgs, boxes, counts = stream_workload(0, FRAMES_PER_STEP, MAX_BOXES)
    d_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    d_boxes = [torch.from_numpy(b).cuda() for b in boxes]
    crops = int(counts.sum())
    print(f"{FRAMES_PER_STEP} frames per step, {crops} crops ({int(counts.min())}..{int(counts.max())} per frame)", flush=True)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    results = {"card": card, "frames_per_step": FRAMES_PER_STEP, "crops_per_step": crops, "box_counts": counts.tolist(), "runs": {}}

    for mb in (32, 64):
        m = ViTPose(model_cfg("b", 17), max_batch=mb)
        m.load_state_dict(sd).to("cuda:0")
        frames_of = lambda i: [d_imgs[(i * FRAMES_PER_STEP + f) % 4] for f in range(FRAMES_PER_STEP)]

        def per_frame(i):
            return [m.infer_frame(fr, b) for fr, b in zip(frames_of(i), d_boxes)]

        def packed(i):
            return m.infer_frames(frames_of(i), d_boxes)

        arms = {"per_frame": per_frame, "packed": packed}
        for i in range(4):                                             # the 4 frame rotations: identical outputs
            want = per_frame(i)
            kp, idx = packed(i)
            for (wk, wi), k, x in zip(want, kp, idx):
                assert torch.equal(wk, k) and torch.equal(wi, x), f"max_batch {mb}, step {i}: packed != per-frame"
        for name, fn in arms.items():
            for i in range(args.warmup):
                fn(i)
        torch.cuda.synchronize()

        def time_steps(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.steps):
                fn(i)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / args.steps

        ms = {a: [] for a in arms}
        for _ in range(3):
            for name, fn in arms.items():
                ms[name].append(time_steps(fn))

        # per-frame latency: an event after every engine call of a step; a frame is ready when its call has finished
        chunks = plan_frame_chunks(counts, m.batch_limit)

        def latency(arm):
            per_step = []
            for i in range(args.steps):
                fr = frames_of(i)
                start = torch.cuda.Event(enable_timing=True)
                start.record()
                ready = [None] * FRAMES_PER_STEP
                if arm == "per_frame":
                    for f in range(FRAMES_PER_STEP):
                        m.infer_frame(fr[f], d_boxes[f])
                        ready[f] = torch.cuda.Event(enable_timing=True)
                        ready[f].record()
                else:
                    for chunk in chunks:                                  # the calls infer_frames makes, one at a time
                        m.infer_frames([fr[f] for f, _, _ in chunk], [d_boxes[f][s:e] for f, s, e in chunk])
                        ev = torch.cuda.Event(enable_timing=True)
                        ev.record()
                        for f, _, _ in chunk:
                            ready[f] = ev                                 # a split frame: its last call wins
                torch.cuda.synchronize()
                per_step.append(float(np.mean([start.elapsed_time(ev) for ev in ready])))
            return float(np.median(per_step))

        lat = {a: latency(a) for a in arms}
        run = {}
        for a in arms:
            med = float(np.median(ms[a]))
            run[a] = {"ms_per_step": med, "runs_ms": ms[a], "crops_per_s": crops / med * 1e3, "mean_frame_latency_ms": lat[a]}
        run["engine_calls_per_step"] = {"per_frame": FRAMES_PER_STEP, "packed": len(chunks)}
        results["runs"][f"max_batch_{mb}"] = run
        print(f"max_batch {mb}: " + "; ".join(
            f"{a} {run[a]['ms_per_step']:.3f} ms/step (runs {', '.join(f'{t:.3f}' for t in ms[a])}), {run[a]['crops_per_s']:.0f} crops/s, "
            f"mean frame latency {lat[a]:.3f} ms" for a in arms) + f"; packed = {len(chunks)} engine calls per step", flush=True)
        del m
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
