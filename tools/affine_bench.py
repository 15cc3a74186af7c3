#!/usr/bin/env python
"""Affine top-down crops on the device against the CPU warp, and against the frame path at the same number of people.
Workload: ViT-B/17, max_batch 64, a step = 16 1080p frames with Poisson(10) detector boxes each (bench.py's stream_workload,
rank 0, clipped to 1..32), the boxes turned into centre / scale and UDP matrices by topdown_args (the reference's COCO
top-down recipe), frames resident in HBM.
  affine      one infer_affine call per step (warp fused into the patch gather, chunked by max_batch), matrices and
              centre / scale already on the device
  cpu_warp    cv2.warpAffine + torchvision ToTensor / Normalize per box on the CPU, H2D of the f32 crops, infer_crops
              (what a user of the reference's data path does without this feature)
  frames      infer_frames on the same frames and boxes (the easy_ViTPose crop), same number of crops
Before timing, the device crops of step 0 are checked to equal the CPU arm's crops bit for bit.  Reported: ms per step and
crops/s (host clock around `steps` steps that end in a device synchronise; arms alternate, three runs each, medians).
Prints the card, its power limit and maximum SM clock first: the numbers belong to them.

    python tools/affine_bench.py [--steps 50] [--warmup 10] [--cpu-steps 5] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import stream_workload  # noqa: E402
from easy_vitpose_b200 import ViTPose, model_cfg, topdown_args  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402

FRAMES_PER_STEP, MAX_BOXES, MAX_BATCH = 16, 32, 64


def main():
    import cv2
    from torchvision import transforms
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cpu-steps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    imgs, boxes, counts = stream_workload(0, FRAMES_PER_STEP, MAX_BOXES)
    d_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    d_boxes = [torch.from_numpy(b).cuda() for b in boxes]
    targs = [topdown_args(np.concatenate([b[:, :2], b[:, 2:] - b[:, :2]], 1).astype(np.float64)) for b in boxes]
    mats = [torch.from_numpy(a[0]).cuda() for a in targs]
    centers = [torch.from_numpy(a[1]).cuda() for a in targs]
    scales = [torch.from_numpy(a[2]).cuda() for a in targs]
    crops = int(counts.sum())
    print(f"{FRAMES_PER_STEP} frames per step, {crops} crops ({int(counts.min())}..{int(counts.max())} per frame)", flush=True)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=MAX_BATCH)
    m.load_state_dict(sd).to("cuda:0")
    tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    frames_of = lambda i: [(i * FRAMES_PER_STEP + f) % 4 for f in range(FRAMES_PER_STEP)]

    def cpu_crops(i):
        return torch.stack([tf(cv2.warpAffine(imgs[fi], mm, (192, 256), flags=cv2.INTER_LINEAR))
                            for fi, a in zip(frames_of(i), targs) for mm in a[0]])

    def affine(i):
        return m.infer_affine([d_imgs[f] for f in frames_of(i)], mats, centers, scales)

    def cpu_warp(i):
        x = cpu_crops(i).cuda()
        org = torch.tensor([[192, 256]] * x.shape[0], dtype=torch.int32)
        return [m.infer_crops(x[s:s + MAX_BATCH], org[s:s + MAX_BATCH]) for s in range(0, x.shape[0], MAX_BATCH)]

    def frames(i):
        return m.infer_frames([d_imgs[f] for f in frames_of(i)], d_boxes)

    dev = m.preprocess_affine([d_imgs[f] for f in frames_of(0)], mats).cpu()
    assert torch.equal(dev, cpu_crops(0)), "device affine crops differ from cv2.warpAffine + torchvision"
    print("device crops of step 0 equal cv2.warpAffine + torchvision bit for bit", flush=True)
    arms = {"affine": (affine, args.steps), "cpu_warp": (cpu_warp, args.cpu_steps), "frames": (frames, args.steps)}
    for name, (fn, _) in arms.items():
        for i in range(args.warmup if name != "cpu_warp" else 2):
            fn(i)
    torch.cuda.synchronize()

    def time_steps(fn, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(steps):
            fn(i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / steps

    ms = {a: [] for a in arms}
    for _ in range(3):
        for name, (fn, steps) in arms.items():
            ms[name].append(time_steps(fn, steps))
    results = {"card": card, "frames_per_step": FRAMES_PER_STEP, "crops_per_step": crops, "max_batch": MAX_BATCH, "arms": {}}
    for a in arms:
        med = float(np.median(ms[a]))
        results["arms"][a] = {"ms_per_step": med, "runs_ms": ms[a], "crops_per_s": crops / med * 1e3, "steps": arms[a][1]}
        print(f"{a}: {med:.3f} ms/step (runs {', '.join(f'{t:.3f}' for t in ms[a])}), {crops / med * 1e3:.0f} crops/s", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
