"""Several datasets in one step: ViT-B, 64 crops per step -- 40 coco, 16 ap10k, 8 wholebody -- served three ways:

    mixed   one multi-head engine (ViTPose+ experts, P = 192), one infer_crops_heads call per step
    split   three single-head engines (model_split.py's checkpoints), one infer_crops call each per step
    floor   one single-head engine running all 64 crops as coco (the cost of one 64-crop forward)

Outputs of the mixed and split arms are checked bit-identical before timing.  Reports ms per step, crops/s and the device
memory each arm's engines hold (vpb_device_bytes: packed weights, workspace, staging), plus the card and its power limit, read
in the same run.  Median of three alternating runs.

    python tools/multi_head_bench.py --steps 50 --warmup 10 [--out FILE.json]
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

from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus  # noqa: E402
from oracle import vitpose_oracle as O  # noqa: E402
from oracle.multi_head import plus_state_dict  # noqa: E402

HEADS = (("coco", 17), ("ap10k", 17), ("wholebody", 133))
COUNTS = (40, 16, 8)
P = 192


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
    n = sum(COUNTS)
    heads = np.repeat(np.arange(len(HEADS)), COUNTS)
    x = torch.from_numpy(O.make_crops(n, 9)).cuda()
    org = torch.from_numpy(np.random.RandomState(9).randint(40, 400, size=(n, 2)).astype(np.int32)).cuda()
    bounds = np.cumsum((0,) + COUNTS)

    mixed = _engine(plus, 17, n, heads=HEADS, expert_rows=P)
    split = [_engine(sd, K, c) for sd, (_, K), c in zip(parts, HEADS, COUNTS)]
    floor = _engine(parts[0], 17, n)
    mem_mixed, mem_split, mem_floor = mixed.device_bytes(), sum(m.device_bytes() for m in split), floor.device_bytes()

    kp_m, idx_m = mixed.infer_crops_heads(x, org, heads)
    for j, m in enumerate(split):
        kp, idx = m.infer_crops(x[bounds[j]:bounds[j + 1]], org[bounds[j]:bounds[j + 1]])
        K = HEADS[j][1]
        assert torch.equal(kp_m[bounds[j]:bounds[j + 1], :K], kp) and torch.equal(idx_m[bounds[j]:bounds[j + 1], :K], idx), HEADS[j][0]

    arms = {
        "mixed": lambda: mixed.infer_crops_heads(x, org, heads),
        "split": lambda: [m.infer_crops(x[bounds[j]:bounds[j + 1]], org[bounds[j]:bounds[j + 1]]) for j, m in enumerate(split)],
        "floor": lambda: floor.infer_crops(x, org),
    }
    runs = {k: [] for k in arms}
    for _ in range(3):
        for k, fn in arms.items():
            runs[k].append(_time(fn, args.steps, args.warmup))
    res = {"gpu": gpu, "model": "vit-b", "crops_per_step": dict(zip([h for h, _ in HEADS], COUNTS)), "expert_rows": P,
           "steps": args.steps, "bit_identical": True}
    for k, mem in (("mixed", mem_mixed), ("split", mem_split), ("floor", mem_floor)):
        ms = float(np.median(runs[k]))
        res[k] = {"ms_per_step": round(ms, 3), "runs_ms": [round(v, 3) for v in runs[k]], "crops_per_s": round(n / ms * 1e3, 1),
                  "device_mb": round(mem / 2**20, 1)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
