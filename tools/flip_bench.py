#!/usr/bin/env python
"""Cost of the flip test on the keypoint path (seeded random weights and crops, CUDA-event timing of back-to-back calls, every
arm warmed up first, the arms alternated in one process and each measured three times):
  flip          infer_crops at n people with flip test on: one forward over the n crops + n mirror images, the flip-back
                average, the decode
  composition   forward_flip_test + decode_heatmaps at n: two forwards of n crops, torch.flip, flip_back, the average in torch
  plain_2n      infer_crops at 2n crops with flip test off: the same model work as `flip`, without the average
Configs: ViT-B/17 with n = 32, ViT-H/133 with n = 16 (synthetic flip pairs).  Prints the card, its power limit and maximum SM
clock first: the numbers belong to them.

    python tools/flip_bench.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from easy_vitpose_b200 import COCO_FLIP_PAIRS, ViTPose, decode_heatmaps, model_cfg  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip(), flush=True)


def ms_per_call(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters


def run(size, K, n, pairs, iters=20, rounds=3):
    m = ViTPose(model_cfg(size, K), max_batch=2 * n)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict(size, K, seed=1).items()}).to("cuda:0")
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, 3, 256, 192, generator=g, device="cuda")
    x2 = torch.randn(2 * n, 3, 256, 192, generator=g, device="cuda")
    org, org2 = torch.full((n, 2), 256, dtype=torch.int32), torch.full((2 * n, 2), 256, dtype=torch.int32)
    org_d = org.cuda()
    arms = {
        "flip": (True, lambda: m.infer_crops(x, org)),
        "composition": (False, lambda: decode_heatmaps(m.forward_flip_test(x, pairs), org_d)),
        "plain_2n": (False, lambda: m.infer_crops(x2, org2)),
    }
    res = {a: [] for a in arms}
    for r in range(rounds + 1):                                       # round 0: warm-up (graph capture, allocator) only
        for name, (flip, fn) in arms.items():
            m.set_flip_test(pairs if flip else None)
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            if r:
                res[name].append(ms_per_call(fn, iters))
    m.set_flip_test(None)
    print(f"ViT-{size.upper()}/{K}, n = {n} people: " + "; ".join(
        f"{a} {np.median(v):.3f} ms per call (runs {', '.join(f'{t:.3f}' for t in v)})" for a, v in res.items()), flush=True)


run("b", 17, 32, list(COCO_FLIP_PAIRS))
rs = np.random.RandomState(0)
order = rs.permutation(133)
run("h", 133, 16, [(int(order[2 * i]), int(order[2 * i + 1])) for i in range(60)])
