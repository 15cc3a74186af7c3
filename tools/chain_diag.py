#!/usr/bin/env python
"""Where the chained launches (chain.cuh) spend their cycles: per phase, the MMA thread's total / operand-wait / accumulator-wait
cycles, the producer's dependency and ring waits, the epilogue's busy and wait cycles (ChainParams::dbg counters, leader CTAs)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ctypes as C
import numpy as np, torch
from easy_vitpose_b200 import ViTPose, model_cfg, _lib
from easy_vitpose_b200.synthetic import random_state_dict

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
m = ViTPose(model_cfg("b", 17), max_batch=B)
m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1).items()}).to("cuda:0")
m.set_option("graph", 0)
x = torch.randn(B, 3, 256, 192, device="cuda"); org = torch.tensor([[192, 256]] * B, dtype=torch.int32, device="cuda")
side = torch.cuda.Stream()
with torch.cuda.stream(side):
    for _ in range(3):
        m.forward_features(x)
    torch.cuda.synchronize()
    SMS = torch.cuda.get_device_properties(0).multi_processor_count   # the chained grid is at most one CTA per SM
    dbg = torch.zeros(SMS * 4 * 12, dtype=torch.int64, device="cuda")
    _lib.lib().vpb_debug_gemm(0, C.c_void_p(dbg.data_ptr()))
    m.forward_features(x)                  # backbone only: the head's GEMMs share the debug pointer
    torch.cuda.synchronize()
    _lib.lib().vpb_debug_gemm(0, None)
d = dbg.cpu().numpy().reshape(SMS, 4, 12).astype(np.float64)
# launch 0 (patch -> qkv) lands in phases 0,1 too: 13 launches accumulate; block launches dominate (12 of 13)
names = ["proj(+patch)", "fc1(+qkv0)", "fc2", "qkv"]
print(f"B={B}: cycles per CTA over one forward (13 chained launches)")
for ph in range(4):
    _, wf, _, dep, ring, eb, _, n = d[:, ph, :8].mean(0)
    print(f"  {names[ph]:13s} tiles/CTA {n:5.1f} | consumer wait for operands {wf / max(n, 1):6.0f}/tile, epilogue {eb / max(n, 1):6.0f}/tile "
          f"| producer: dependency wait {dep / max(n, 1):6.0f}/tile ({d[:, ph, 11].mean() / max(dep, 1):.0%} of it on the CTA's first tile of the phase), ring wait {ring / max(n, 1):6.0f}/tile")
for st, ph in ((0, 0), (1, 2)):
    w, b, n = d[:, ph, 8:11].mean(0)
    rows, other, pub = d[:, ph + 1, 8:11].mean(0)
    print(f"  LayerNorm stage {st} (first LayerNorm warp): jobs/CTA {n:5.1f}, busy {b / max(n, 1):7.0f} cyc/job (own rows {rows / max(n, 1):.0f}, waiting for the other "
          f"three warps {other / max(n, 1):.0f}, fence + release {pub / max(n, 1):.0f}), wait for the residual rows {w / max(n, 1):7.0f} cyc/job")
