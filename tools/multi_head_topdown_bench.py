"""Several datasets in one evaluation-quality step: the multi_head_bench.py workload run as affine top-down crops with flip
test.  ViT-B, P = 192, 32 people per step -- 20 coco, 8 ap10k, 4 wholebody -- in four 1080p frames, served three ways:

    mixed   one multi-head engine (max_batch 64), set_flip_test_heads, one infer_affine_heads call per step
    split   three single-head engines (model_split.py's checkpoints) with set_flip_test, one infer_affine call each per step
    floor   one single-head engine running all 32 people as coco with affine crops and flip test (one 64-crop forward)

The coco head flips with COCO_FLIP_PAIRS; the reference defines no pairs for the other datasets, so they take a fixed
choice of neighbouring keypoints.  Outputs of the mixed and split arms are checked bit-identical before timing.  Reports ms
per step, people/s and the device memory each arm's engines hold, plus the card and its power limit, read in the same run.
Median of three alternating runs.

    python tools/multi_head_topdown_bench.py --steps 50 --warmup 10 [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easy_vitpose_b200 import COCO_FLIP_PAIRS, ViTPose, model_cfg, split_vitpose_plus, topdown_args  # noqa: E402
from oracle import preproc_oracle as PP  # noqa: E402
from oracle.multi_head import plus_state_dict  # noqa: E402

HEADS = (("coco", 17), ("ap10k", 17), ("wholebody", 133))
COUNTS = (20, 8, 4)
P = 192
FRAMES = 4


def _pairs(name, K):
    return [tuple(int(v) for v in p) for p in COCO_FLIP_PAIRS] if name == "coco" else [(i, i + 1) for i in range(1, K - 1, 2)]


def _engine(sd, K, max_batch, **kw):
    m = ViTPose(model_cfg("b", K), max_batch=max_batch, **kw)
    m.load_state_dict(sd)
    return m.to("cuda:0")


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

    plus = {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("b", [k for _, k in HEADS], P, 5).items()}
    parts = list(split_vitpose_plus(plus, [n for n, _ in HEADS], [k for _, k in HEADS]).values())
    pairs = [_pairs(n, k) for n, k in HEADS]
    n = sum(COUNTS)

    # four 1080p frames; every person gets a box (x, y, w, h) and a head, spread over the frames
    rs = np.random.RandomState(9)
    frames = [torch.from_numpy(PP.make_frame(1080, 1920, 20 + f)).cuda() for f in range(FRAMES)]
    head_of = np.repeat(np.arange(len(HEADS)), COUNTS)
    frame_of = rs.permutation(np.arange(n) % FRAMES)
    boxes = np.stack([rs.uniform(0, 1700, n), rs.uniform(0, 800, n), rs.uniform(60, 220, n), rs.uniform(120, 420, n)], 1)
    per_frame = [np.nonzero(frame_of == f)[0] for f in range(FRAMES)]
    fargs = [topdown_args(boxes[s], 1.25, True) for s in per_frame]
    fheads = [head_of[s] for s in per_frame]

    mixed = _engine(plus, 17, 64, heads=HEADS, expert_rows=P)
    mixed.set_flip_test_heads(pairs, False)
    split = [_engine(sd, K, 2 * c) for sd, (_, K), c in zip(parts, HEADS, COUNTS)]
    for m, p in zip(split, pairs):
        m.set_flip_test(p, False)
    floor = _engine(parts[0], 17, 64)
    floor.set_flip_test(pairs[0], False)
    mem_mixed, mem_split, mem_floor = mixed.device_bytes(), sum(m.device_bytes() for m in split), floor.device_bytes()

    def split_args(j):
        sel = [np.nonzero(h == j)[0] for h in fheads]
        return [a[0][s] for a, s in zip(fargs, sel)], [a[1][s] for a, s in zip(fargs, sel)], [a[2][s] for a, s in zip(fargs, sel)]
    sargs = [split_args(j) for j in range(len(HEADS))]
    margs = ([a[0] for a in fargs], [a[1] for a in fargs], [a[2] for a in fargs])

    kp_m, idx_m = mixed.infer_affine_heads(frames, *margs, fheads)
    for j, m in enumerate(split):
        kp, idx = m.infer_affine(frames, *sargs[j])
        K = HEADS[j][1]
        for f in range(FRAMES):
            sel = np.nonzero(fheads[f] == j)[0]
            t = torch.as_tensor(sel, device="cuda")
            assert torch.equal(kp_m[f].index_select(0, t)[:, :K], kp[f]) and torch.equal(idx_m[f].index_select(0, t)[:, :K], idx[f]), HEADS[j][0]

    arms = {
        "mixed": lambda: mixed.infer_affine_heads(frames, *margs, fheads),
        "split": lambda: [m.infer_affine(frames, *sargs[j]) for j, m in enumerate(split)],
        "floor": lambda: floor.infer_affine(frames, *margs),
    }
    runs = {k: [] for k in arms}
    for _ in range(3):
        for k, fn in arms.items():
            runs[k].append(_time(fn, args.steps, args.warmup))
    res = {"gpu": gpu, "model": "vit-b", "people_per_step": dict(zip([h for h, _ in HEADS], COUNTS)), "frames": "4 x 1920x1080",
           "expert_rows": P, "affine": True, "flip_test": True, "steps": args.steps, "bit_identical": True}
    for k, mem in (("mixed", mem_mixed), ("split", mem_split), ("floor", mem_floor)):
        ms = float(np.median(runs[k]))
        res[k] = {"ms_per_step": round(ms, 3), "runs_ms": [round(v, 3) for v in runs[k]], "people_per_s": round(n / ms * 1e3, 1),
                  "device_mb": round(mem / 2**20, 1)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
