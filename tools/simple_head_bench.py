"""Classic vs simple decoder on the same backbone, in one run, alternating the two engines:

    b17x64    ViT-B, COCO (K = 17), 64 crops per step
    h133x32   ViT-H, K = 133, 32 crops per step

For each: infer_crops step time and crops/s, the head alone (vpb_head on [B, D, 16, 12] features: the features -> tokens
conversion and the head's launches), and the engine's device memory at max_batch 64 (cudaMemGetInfo before and after
construction, and vpb_device_bytes).  For the simple engine also the simple_head kernel's own time (the engine's per-kernel
CUDA events) and its achieved FLOP/s and bytes/s from shapes, against the H100 SXM data-sheet bounds (989 TFLOP/s dense
BF16, 3.35 TB/s).  Median of three alternating runs; the card's name and power limit are read in the same run.

    python tools/simple_head_bench.py --steps 30 --warmup 5 [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from easy_vitpose_b200 import ViTPose, _lib, model_cfg  # noqa: E402
from easy_vitpose_b200.synthetic import random_crops, random_state_dict  # noqa: E402

CASES = (("b17x64", "b", 17, 64), ("h133x32", "h", 133, 32))
DIMS = {"b": 768, "h": 1280}
PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12


def _engine(size, K, decoder):
    free0 = torch.cuda.mem_get_info()[0]
    m = ViTPose(model_cfg(size, K, decoder), max_batch=64)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in random_state_dict(size, K, seed=3, decoder=decoder).items()})
    m.to("cuda:0")
    torch.cuda.synchronize()
    return m, free0 - torch.cuda.mem_get_info()[0]


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def _head_fn(m, feats, out):
    L, st = _lib.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: _lib.check(L.vpb_head(m._handle, C.c_void_p(feats.data_ptr()), feats.shape[0], C.c_void_p(out.data_ptr()), st))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "steps": args.steps, "cases": {}}
    for name, size, K, B in CASES:
        D = DIMS[size]
        engines = {d: _engine(size, K, d) for d in ("classic", "simple")}
        x = torch.from_numpy(random_crops(B, seed=4)).cuda()
        org = torch.tensor([[192, 256]] * B, dtype=torch.int32, device="cuda")
        feats = engines["simple"][0].forward_features(x)
        out = torch.empty((B, K, 64, 48), dtype=torch.float32, device="cuda")
        step, head = {d: [] for d in engines}, {d: [] for d in engines}
        for _ in range(3):
            for d, (m, _) in engines.items():
                step[d].append(_time(lambda: m.infer_crops(x, org), args.steps, args.warmup))
                head[d].append(_time(_head_fn(m, feats, out), args.steps * 4, args.warmup))
        r = {}
        for d, (m, mem) in engines.items():
            ms = float(np.median(step[d]))
            r[d] = {"step_ms": ms, "crops_per_s": B / ms * 1e3, "head_ms": float(np.median(head[d])),
                    "step_ms_runs": step[d], "head_ms_runs": head[d], "mem_get_info_bytes": int(mem), "device_bytes": m.device_bytes()}
        m = engines["simple"][0]
        m.set_option("profile", 1)
        m.profile_collect()
        fn = _head_fn(m, feats, out)
        for _ in range(args.steps * 4):
            fn()
        prof = m.profile_collect()
        m.set_option("profile", 0)
        k_ms, k_n = prof["simple_head"]
        k_s = k_ms / k_n * 1e-3
        G = -(-K // 16)
        flops = 2.0 * B * 192 * D * 9 * K                                       # the tap GEMM (the stencil's FMAs are ~1 %)
        bytes_ = B * G * 192 * D * 2 + G * 144 * D * 2 + B * K * 3072 * 4 + K * 4   # xn once per group, W, heatmaps
        r["simple_kernel"] = {"ms": k_s * 1e3, "tflops": flops / k_s / 1e12, "tb_s": bytes_ / k_s / 1e12,
                              "share_of_peak": max(flops / PEAK_FLOPS, bytes_ / PEAK_BW) / k_s,
                              "bound_by": "flops" if flops / PEAK_FLOPS > bytes_ / PEAK_BW else "bytes"}
        res["cases"][name] = r
        print(name, json.dumps(r), flush=True)
        del engines, m, feats, out
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
