"""A/B of the fused qkv + attention launch (csrc/qkv_attention.cuh) against the qkv GEMM + attention pair, per ViT size and
batch: the measurements behind fuse_qkv_attention's rule in engine.cu.

    python tools/qkv_attention_ab.py [--sizes s,b,l,h] [--batches 1,2,...] [--calls 20] [--rounds 3] [--out FILE]

For every (size, batch) it first checks that both forms give the same bits (heatmaps, keypoints, argmax, the attention
buffer), then times whole keypoint calls (vpb_infer with its CUDA graph) in each form, alternating the forms `rounds` times;
the graph cache is dropped between forms so each form is captured anew.  Prints one JSON line per (size, batch): median ms per
call of each form and fused / separate.  Random weights at full depth, K = 17."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import vitpose_oracle as O  # noqa: E402

FUSED, SEPARATE = 2, 4
DIMS = {"s": (384, 12), "b": (768, 12), "l": (1024, 24), "h": (1280, 32)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="s,b,l,h")
    ap.add_argument("--batches", default="1,2,4,8,11,12,16,20,24,32,44,48,64")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from easy_vitpose_b200 import ViTPose, _lib, model_cfg
    L = _lib.lib()
    batches = [int(b) for b in a.batches.split(",")]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
    rows = []
    for size in a.sizes.split(","):
        D, depth = DIMS[size]
        m = ViTPose(model_cfg(size, 17), max_batch=max(batches))
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, 17, 7, peaky=0.1, bumps=True).items()})
        m.to("cuda:0")
        for n in batches:
            x = torch.from_numpy(O.make_crops(n, n)).cuda()
            org = torch.from_numpy(np.random.RandomState(n).randint(64, 513, size=(n, 2)).astype(np.int32))
            outs = {}
            for form in (SEPARATE, FUSED):
                L.vpb_debug_attention(form)
                m.set_option("graph", 0)
                kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
                torch.cuda.synchronize()
                attn = m.read_buffer("attn", (n * 192, D), "bf16").view(torch.int16)
                outs[form] = [t.cpu() for t in (kp, idx, hm)] + [attn]
                m.set_option("graph", 1)
            same = all(torch.equal(u, v) for u, v in zip(outs[FUSED], outs[SEPARATE]))
            times = {FUSED: [], SEPARATE: []}
            for _ in range(a.rounds):
                for form in (SEPARATE, FUSED):
                    L.vpb_debug_attention(form)
                    m.set_flip_test(None)                      # drops the cached graphs: capture this form
                    for _ in range(3):                         # eager, capture, replay
                        m.infer_crops(x, org)
                    torch.cuda.synchronize()
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0.record()
                    for _ in range(a.calls):
                        m.infer_crops(x, org)
                    t1.record()
                    t1.synchronize()
                    times[form].append(t0.elapsed_time(t1) / a.calls)
            L.vpb_debug_attention(-1)
            m.set_flip_test(None)
            sep, fus = float(np.median(times[SEPARATE])), float(np.median(times[FUSED]))
            r = {"size": size, "batch": n, "items": n * {384: 6, 768: 12, 1024: 16, 1280: 16}[D],
                 "bit_identical": same, "separate_ms": round(sep, 4), "fused_ms": round(fus, 4), "fused_over_separate": round(fus / sep, 4),
                 "separate_all": [round(t, 4) for t in times[SEPARATE]], "fused_all": [round(t, 4) for t in times[FUSED]]}
            rows.append(r)
            print(json.dumps(r), flush=True)
        del m
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    if not all(r["bit_identical"] for r in rows):
        sys.exit("fused and separate forms differ")


if __name__ == "__main__":
    main()
