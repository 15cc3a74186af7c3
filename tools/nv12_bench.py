#!/usr/bin/env python
"""NV12 video frames read directly by the engine against the RGB workarounds, on the video workload of bench.py --config
ap10k-streams (tools/multi_frame_bench.py): ViT-B/17, max_batch 64, a step = 16 1080p frames with Poisson(10) detector boxes
each.  The frames are the workload's four seeded images converted to limited-range BT.601 NV12 (oracle/nv12_oracle.py).
  dev_nv12        device NV12 frames -> infer_frames_nv12 (the gather converts only the taps it reads)
  dev_torch_rgb   device NV12 frames -> whole-frame RGB by the formula in torch ops -> infer_frames
  host_nv12       pinned host NV12 frames -> infer_frames_nv12_host (H2D of 1.5 B per pixel)
  host_rgb        pinned host RGB frames (already converted: the CPU conversion is not timed) -> infer_frames_host (3 B per pixel)
Before timing, the keypoints and argmax indices of all four arms are checked bit-identical on every frame rotation.  Reported:
ms per step and crops/s (host clock around `steps` steps ending in a device synchronise; the arms alternate, three runs each,
medians), and for the device arms the engine's `crop_preprocess` class time per step from profile_collect() in a separate profiled
run (plus, for dev_torch_rgb, the torch conversion's time by CUDA events).  Prints the card and its power limit first.

    python tools/nv12_bench.py [--steps 50] [--warmup 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import stream_workload  # noqa: E402
from easy_vitpose_b200 import ViTPose, model_cfg  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402
from oracle.nv12_oracle import COEFS, nv12_to_rgb, rgb_to_nv12  # noqa: E402

FRAMES_PER_STEP, MAX_BOXES, MAX_BATCH = 16, 32, 64


def torch_nv12_to_rgb(f: torch.Tensor, matrix: str = "bt601") -> torch.Tensor:
    """The obvious workaround: the whole frame converted by the fixed-point formula in torch int32 ops."""
    cy, cvr, cvg, cug, cub = COEFS[matrix]
    h, w = f.shape[0] // 3 * 2, f.shape[1]
    y = f[:h].int()
    uv = (f[h:].view(h // 2, w // 2, 2).int() - 128).repeat_interleave(2, 0).repeat_interleave(2, 1)
    u, v = uv[..., 0], uv[..., 1]
    yy = (y - 16).clamp_min(0) * cy + (1 << 19)
    return torch.stack([(yy + cvr * v) >> 20, (yy + cvg * v + cug * u) >> 20, (yy + cub * u) >> 20], -1).clamp(0, 255).to(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    imgs, boxes, counts = stream_workload(0, FRAMES_PER_STEP, MAX_BOXES)
    nv = [rgb_to_nv12(im) for im in imgs]
    rgb = [nv12_to_rgb(f) for f in nv]                                  # what cv2.cvtColor(COLOR_YUV2RGB_NV12) gives
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    h_nv, h_rgb = [pin(f) for f in nv], [pin(f) for f in rgb]
    d_nv = [torch.from_numpy(f).cuda() for f in nv]
    d_boxes = [torch.from_numpy(b).cuda() for b in boxes]
    h_boxes = [np.ascontiguousarray(b) for b in boxes]
    crops = int(counts.sum())
    print(f"{FRAMES_PER_STEP} frames per step, {crops} crops ({int(counts.min())}..{int(counts.max())} per frame); "
          f"H2D per step: NV12 {sum(f.nbytes for f in nv) * 4 / 1e6:.1f} MB, RGB {sum(f.nbytes for f in rgb) * 4 / 1e6:.1f} MB", flush=True)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=MAX_BATCH)
    m.load_state_dict(sd).to("cuda:0")
    rot = lambda i, fr: [fr[(i * FRAMES_PER_STEP + f) % len(fr)] for f in range(FRAMES_PER_STEP)]

    def dev_nv12(i):
        return m.infer_frames_nv12(rot(i, d_nv), d_boxes)

    def dev_torch_rgb(i):
        return m.infer_frames([torch_nv12_to_rgb(f) for f in rot(i, d_nv)], d_boxes)

    def host_nv12(i):
        return m.infer_frames_nv12_host(rot(i, h_nv), h_boxes)

    def host_rgb(i):
        return m.infer_frames_host(rot(i, h_rgb), h_boxes)

    arms = {"dev_nv12": dev_nv12, "dev_torch_rgb": dev_torch_rgb, "host_nv12": host_nv12, "host_rgb": host_rgb}
    for i in range(4):                                                  # the 4 frame rotations: identical outputs
        outs = {a: fn(i) for a, fn in arms.items()}
        want_k = np.concatenate([k.cpu().numpy() if torch.is_tensor(k) else k for k in outs["host_rgb"][0]])
        want_i = np.concatenate([x.cpu().numpy() if torch.is_tensor(x) else x for x in outs["host_rgb"][1]])
        for a, (kp, idx) in outs.items():
            k = np.concatenate([x.cpu().numpy() if torch.is_tensor(x) else x for x in kp])
            x = np.concatenate([x.cpu().numpy() if torch.is_tensor(x) else x for x in idx])
            assert np.array_equal(k, want_k) and np.array_equal(x, want_i), f"step {i}: {a} != host_rgb"
    print("outputs of all arms bit-identical", flush=True)
    for fn in arms.values():
        for i in range(args.warmup):
            fn(i)
    torch.cuda.synchronize()

    def time_steps(fn):
        t0 = time.perf_counter()
        for i in range(args.steps):
            fn(i)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    ms = {a: [] for a in arms}
    for _ in range(3):
        for name, fn in arms.items():
            ms[name].append(time_steps(fn))

    # profiled run (eager launches, per-class events): the gather's time per step on the device arms
    prof = {}
    m.set_option("profile", 1)
    for a in ("dev_nv12", "dev_torch_rgb"):
        m.profile_collect()
        for i in range(args.steps):
            arms[a](i)
        torch.cuda.synchronize()
        cls = m.profile_collect()
        pre = cls["crop_preprocess"]                                  # the frame gather's kernel class
        prof[a] = {"preprocess_ms_per_step": pre[0] / args.steps, "preprocess_launches_per_step": pre[1] / args.steps}
    m.set_option("profile", 0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        [torch_nv12_to_rgb(f) for f in rot(i, d_nv)]
    e1.record()
    e1.synchronize()
    prof["dev_torch_rgb"]["torch_conversion_ms_per_step"] = e0.elapsed_time(e1) / args.steps

    results = {"card": card, "frames_per_step": FRAMES_PER_STEP, "crops_per_step": crops, "max_batch": MAX_BATCH, "arms": {}}
    for a in arms:
        med = float(np.median(ms[a]))
        results["arms"][a] = {"ms_per_step": med, "runs_ms": ms[a], "crops_per_s": crops / med * 1e3, **prof.get(a, {})}
        extra = "".join(f", {k} {v:.3f}" for k, v in prof.get(a, {}).items())
        print(f"{a}: {med:.3f} ms/step (runs {', '.join(f'{t:.3f}' for t in ms[a])}), {crops / med * 1e3:.0f} crops/s{extra}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
