#!/usr/bin/env python
"""GEMM diagnostics on the GPU: time vs ring depth, and where the MMA / producer / epilogue threads wait."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import ctypes as C
import torch
from easy_vitpose_b200 import _lib
from gpu_util import EPI_BF16, EPI_BF16_GELU, EPI_F32_ADD, gemm

dev = torch.device("cuda", 0)
L = _lib.lib()
M, D = 12288, 768
shapes = {"qkv": (D, 3 * D, EPI_BF16), "proj": (D, D, EPI_F32_ADD), "fc1": (D, 4 * D, EPI_BF16_GELU), "fc2": (4 * D, D, EPI_F32_ADD)}
torch.manual_seed(0)
for name, (K, N, epi) in shapes.items():
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.03).bfloat16()
    bias = torch.randn(N, device=dev)
    out = torch.zeros(M, N, dtype=torch.float32 if epi == EPI_F32_ADD else torch.bfloat16, device=dev)
    for stages in (0, 8 << 8):   # bits 8..: 1 same A, 2 same W, 4 m-fastest order, 8 force BN=128
        L.vpb_debug_gemm(stages, None)
        for _ in range(3):
            gemm(a, w, bias, out, epi)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            _lib.check(L.vpb_gemm(C.c_void_p(a.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(bias.data_ptr()), C.c_void_p(out.data_ptr()),
                                  M, N, K, epi, None, 0, 0, 0, 0, 0, None))
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 100
        print(f"{name:5s} flags={stages >> 8} {us:8.1f} us  {2*M*N*K/us/1e6:8.1f} TFLOP/s")
    SMS = torch.cuda.get_device_properties(0).multi_processor_count    # the GEMM grid is at most one CTA per SM
    dbg = torch.zeros(SMS * 8, dtype=torch.int64, device=dev)
    L.vpb_debug_gemm(0, C.c_void_p(dbg.data_ptr()))
    gemm(a, w, bias, out, epi)
    d = dbg.cpu().reshape(SMS, 8).double()
    m = d.mean(0)
    print(f"      cycles/CTA: consumer total {m[0]:.0f} wait for operands {m[1]:.0f} ({m[1]/max(m[0],1):.0%}) | "
          f"producer total {m[3]:.0f} wait_empty {m[4]:.0f} ({m[4]/max(m[3],1):.0%}) | CTA lifetime {m[7]:.0f}")
    life_cyc = d[:, 7].mean(); life_ns = d[1::2, 0].mean()
    print(f"      CTA lifetime {life_cyc:.0f} cycles = {life_ns/1e3:.1f} us -> SM clock {life_cyc/life_ns:.2f} GHz")
    L.vpb_debug_gemm(0, None)
