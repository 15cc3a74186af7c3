#!/usr/bin/env python
"""Times the standalone GEMM of each transformer linear (qkv, proj, fc1 + GELU, fc2) with every tile width that divides its N,
forced through the vpb_debug_gemm width override, and prints the width the engine's rule (engine.cu: pick_tile) takes.  This
table is the evidence behind the rule and its tie-break.  Seeded random operands, CUDA-event timing of back-to-back launches,
the widths of one cell measured in alternation, best of three rounds.  Prints the card and its power limit first: the numbers
belong to them.

    python tools/gemm_width_ab.py [--dims 768,1024,1280] [--crops 1,8,32,64]"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from easy_vitpose_b200 import _lib  # noqa: E402

EPI_BF16, EPI_BF16_GELU, EPI_F32_ADD = 0, 1, 5
WIDTHS = (128, 192, 256)
TIE_ORDER = (128, 256, 192)      # engine.cu kTileWidths: on equal cost the later width wins


def ptr(t):
    return C.c_void_p(t.data_ptr())


def rule(M, N, sms):
    """engine.cu pick_tile without overrides: least ceil(tiles / SMs) * BN, ties by TIE_ORDER"""
    best = None
    for w in TIE_ORDER:
        if N % w:
            continue
        cost = -(-((M + 127) // 128) * (N // w) // sms) * w
        if best is None or cost <= best[1]:
            best = (w, cost)
    return best[0]


def time_gemm(M, N, K, epi, width, iters):
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, generator=g, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, generator=g, device="cuda") * 0.1
    out = torch.zeros(M, N, device="cuda", dtype=torch.float32 if epi == EPI_F32_ADD else torch.bfloat16)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.vpb_debug_gemm((width << 8) << 8, None)
    try:
        def launch():
            _lib.check(L.vpb_gemm(ptr(a), ptr(w), ptr(bias), ptr(out), M, N, K, epi, None, 0, 0, 0, 0, 0, st))
        for _ in range(3):
            launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters
    finally:
        L.vpb_debug_gemm(0, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="768,1024,1280")
    ap.add_argument("--crops", default="1,8,32,64")
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"{sms} SMs; us per launch (best of 3 alternating rounds), TFLOP/s in brackets; * = the rule's width", flush=True)
    for D in (int(d) for d in args.dims.split(",")):
        classes = [("qkv", 3 * D, D, EPI_BF16), ("proj", D, D, EPI_F32_ADD), ("fc1_gelu", 4 * D, D, EPI_BF16_GELU),
                   ("fc2", D, 4 * D, EPI_F32_ADD)]
        for crops in (int(c) for c in args.crops.split(",")):
            M = crops * 192
            for name, N, K, epi in classes:
                widths = [w for w in WIDTHS if N % w == 0]
                best = {w: float("inf") for w in widths}
                for _ in range(3):
                    for w in widths:
                        best[w] = min(best[w], time_gemm(M, N, K, epi, w, args.iters))
                pick = rule(M, N, sms)
                cells = "  ".join(f"{w}{'*' if w == pick else ' '} {best[w]:8.1f} ({2 * M * N * K / best[w] / 1e6:5.0f})" for w in widths)
                print(f"D={D:4d} crops={crops:3d} {name:9s} M={M:6d} N={N:5d} K={K:5d}  {cells}", flush=True)


if __name__ == "__main__":
    main()
