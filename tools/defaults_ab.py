#!/usr/bin/env python
"""A/B of the engine defaults that depend on the GPU (ViT-B COCO-17, seeded random weights and crops, CUDA-event timing of
back-to-back calls, each arm measured twice in alternation):
  l2       the L2 persisting window over the fp32 token stream (default) against none (VPB_L2_PERSIST=0), at 64 crops
  tiles    standalone GEMMs (unchained path) with the tile-width rule of engine.cu pick_tile (default) against 128-wide tiles
           everywhere (vpb_debug_gemm flag 8 around the narrow arm's calls)
  chain    chained launches against one kernel per GEMM, per batch size: where chain_min_batch belongs
Prints the card and its power limit first: the numbers belong to them.

    python tools/defaults_ab.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from easy_vitpose_b200 import ViTPose, _lib, model_cfg  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip(), flush=True)
SD = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1).items()}


def engine(l2=True):
    os.environ["VPB_L2_PERSIST"] = "1" if l2 else "0"
    m = ViTPose(model_cfg("b", 17), max_batch=64)
    m.load_state_dict(SD).to("cuda:0")
    os.environ.pop("VPB_L2_PERSIST")
    return m


def ms_per_call(m, n, iters=30):
    g = torch.Generator(device="cuda").manual_seed(n)
    xs = [torch.randn(n, 3, 256, 192, generator=g, device="cuda") for _ in range(4)]
    org = torch.tensor([[192, 256]] * n, dtype=torch.int32, device="cuda")
    for i in range(5):
        m.infer_crops(xs[i % 4], org)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        m.infer_crops(xs[i % 4], org)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


base, no_l2, narrow = engine(), engine(l2=False), engine()
for m in (base, no_l2, narrow):
    m.set_option("chain_min_batch", 1)

r = []
for _ in range(2):
    r.append((ms_per_call(base, 64), ms_per_call(no_l2, 64)))
print("l2 (64 crops, chained) ms/call  window on / off: " + "  ".join(f"{a:.3f} / {b:.3f}" for a, b in r), flush=True)

for n in (1, 4, 9, 16, 32, 48, 64):
    cells = []
    for _ in range(2):
        for m in (base, narrow):
            m.set_option("chain", 0)
        wide_t = ms_per_call(base, n)
        _lib.lib().vpb_debug_gemm(8 << 8, None)
        narrow_t = ms_per_call(narrow, n)
        _lib.lib().vpb_debug_gemm(0, None)
        base.set_option("chain", 1)
        chain_t = ms_per_call(base, n)
        cells.append(f"{wide_t:.3f} / {narrow_t:.3f} / {chain_t:.3f}")
    print(f"{n:2d} crops ms/call  unchained rule / unchained 128-wide / chained:  " + "  |  ".join(cells), flush=True)
