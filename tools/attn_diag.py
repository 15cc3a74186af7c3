#!/usr/bin/env python
"""Where the attention kernel's threads spend their cycles (AttnParams::dbg counters)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import ctypes as C
import torch
from easy_vitpose_b200 import _lib
from gpu_util import attention

dev = torch.device("cuda", 0)
L = _lib.lib()
import itertools
for (heads, hd, B), flags in itertools.product(((12, 64, 64), (16, 64, 64), (16, 80, 32), (12, 32, 64)), (0, 1, 2, 3)):
    if hd == 80 and flags >= 2:
        continue
    L.vpb_debug_attention(flags)
    print("--- exponentials:", "every 4th on the FMA pipe (ex2_poly)" if flags & 1 else "all on the MUFU", "| half tiles:",
          "PACKED (attention_pack.cuh)" if flags & 2 else "one step each")
    D = heads * hd
    qkv = (torch.randn(B * 192, 3 * D, device=dev) * 0.5).bfloat16()
    for _ in range(3):
        attention(qkv, B, heads, hd)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = torch.empty((B * 192, D), dtype=torch.bfloat16, device=dev)
    e0.record()
    for _ in range(10):
        _lib.check(L.vpb_attention(C.c_void_p(qkv.data_ptr()), B, heads, hd, C.c_void_p(out.data_ptr()), None))
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 100
    n = min(B * heads, torch.cuda.get_device_properties(0).multi_processor_count)
    dbg = torch.zeros(n * 8, dtype=torch.int64, device=dev)
    L.vpb_debug_gemm(0, C.c_void_p(dbg.data_ptr()))
    attention(qkv, B, heads, hd)
    L.vpb_debug_gemm(0, None)
    d = dbg.cpu().reshape(n, 8).double()
    m = d.mean(0)
    steps = m[7]
    flops = 4 * B * heads * 192 * 192 * hd
    print(f"hd={hd} B={B} heads={heads}: {us:.1f} us/launch = {flops / us / 1e6:.0f} TFLOP/s; per CTA: lifetime {m[0]:.0f} cyc (max {d[:,0].max():.0f}), "
          f"{steps:.2f} items (max {d[:,7].max():.0f}) -> {m[0]/max(steps, 1):.0f} cyc/item, of which waiting for operands {m[1]/max(steps, 1):.0f}")
L.vpb_debug_attention(-1)
