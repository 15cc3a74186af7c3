#!/usr/bin/env python
"""Where the attention launches spend their cycles: the per-CTA phase counters of the fused qkv + attention launch
(QkvAttnParams::dbg) at ViT-B and ViT-L with 64 crops, and of attention_wgmma (AttnParams::dbg) at head_dim 32, 64 and 80.
Prints cycles per item, averaged over the CTAs (thread 0 of each), and the launch time by CUDA events without the counters.

    python tools/attn_phases.py [--poly]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from easy_vitpose_b200 import _lib  # noqa: E402
from gpu_util import EPI_BF16, gemm, ptr  # noqa: E402

FUSED = ("gemm", "of which full waits", "hand-off", "S", "softmax", "PV", "store")
STANDALONE = ("lifetime", "operand wait", "loop rest", "S", "softmax", "PV", "store")


def run(name, launch, items, labels, calls=20):
    dev = torch.device("cuda", 0)
    for _ in range(3):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        launch()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / calls
    n = min(items, torch.cuda.get_device_properties(0).multi_processor_count)
    dbg = torch.zeros(n * 8, dtype=torch.int64, device=dev)
    L = _lib.lib()
    L.vpb_debug_gemm(0, C.c_void_p(dbg.data_ptr()))
    try:
        launch()
        torch.cuda.synchronize()
    finally:
        L.vpb_debug_gemm(0, None)
    d = dbg.cpu().view(n, 8).double()
    per_item = d[:, :7].sum(0) / d[:, 7].sum()
    cols = ", ".join(f"{lab} {v:.0f}" for lab, v in zip(labels, per_item.tolist()) if lab != "lifetime")
    print(f"{name}: {us:.1f} us/launch, {items} items on {n} CTAs; cycles per item: {cols}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poly", action="store_true", help="every 4th exponential by ex2_poly (VPB_ATT_POLY)")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip() or torch.cuda.get_device_name(0))
    L = _lib.lib()
    L.vpb_debug_attention(1 if args.poly else 0)
    g = torch.Generator(device="cuda").manual_seed(0)
    try:
        for vit, heads, hd, B in (("ViT-B", 12, 64, 64), ("ViT-L", 16, 64, 64)):
            D = heads * hd
            xn = (torch.randn(B * 192, D, device="cuda", generator=g) * 0.5).bfloat16()
            w = (torch.randn(3 * D, D, device="cuda", generator=g) * D ** -0.5).bfloat16()
            bias = torch.randn(3 * D, device="cuda", generator=g) * 0.1
            out = torch.empty(B * 192, D, dtype=torch.bfloat16, device="cuda")
            launch = lambda: _lib.check(L.vpb_qkv_attention(ptr(xn), ptr(w), ptr(bias), B, heads, hd, ptr(out), None))  # noqa: E731
            run(f"qkv_attention_wgmma {vit} hd {hd}, {B} crops", launch, B * heads, FUSED)
        for heads, hd, B in ((6, 32, 64), (12, 64, 64), (16, 80, 32)):
            D = heads * hd
            xn = (torch.randn(B * 192, D, device="cuda", generator=g) * 0.5).bfloat16()
            w = (torch.randn(3 * D, D, device="cuda", generator=g) * D ** -0.5).bfloat16()
            bias = torch.randn(3 * D, device="cuda", generator=g) * 0.1
            qkv = torch.empty(B * 192, 3 * D, dtype=torch.bfloat16, device="cuda")
            gemm(xn, w, bias, qkv, EPI_BF16)
            out = torch.empty(B * 192, D, dtype=torch.bfloat16, device="cuda")
            launch = lambda: _lib.check(L.vpb_attention(ptr(qkv), B, heads, hd, ptr(out), None))  # noqa: E731
            run(f"attention_wgmma hd {hd}, {B} crops x {heads} heads", launch, B * heads, STANDALONE)
    finally:
        L.vpb_debug_attention(-1)


if __name__ == "__main__":
    main()
