#!/usr/bin/env python
"""YUV video frames read directly by the engine against the RGB workarounds, on the video workload of bench.py --config
ap10k-streams (tools/multi_frame_bench.py): ViT-B/17, max_batch 64, a step = 16 1080p frames with Poisson(10) detector boxes
each.  The frames are the workload's four seeded images converted to limited-range BT.601 I420, YUYV and NV12
(oracle/yuv_oracle.py).
  dev_i420 / dev_yuyv / dev_nv12     device frames -> infer_frames_yuv (the gather converts only the taps it reads)
  dev_torch_i420 / dev_torch_yuyv    device frames -> whole-frame RGB by the formula in torch ops -> infer_frames
  host_i420                          pinned host I420 frames -> infer_frames_yuv_host (H2D of 1.5 B per pixel)
  host_rgb                           pinned host RGB frames (already converted: the CPU conversion is not timed) -> infer_frames_host
Before timing, the keypoints and argmax indices of all arms are checked bit-identical on every frame rotation.  Reported:
ms per step and crops/s (host clock around `steps` steps ending in a device synchronise; the arms alternate, three runs each,
medians), and for the device arms the engine's `crop_preprocess` class time per step from profile_collect() in a separate profiled
run (plus, for the torch arms, the torch conversion's time by CUDA events).  Prints the card and its power limit first.

    python tools/yuv_bench.py [--steps 50] [--warmup 10] [--json out.json]"""
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
from oracle.nv12_oracle import COEFS  # noqa: E402
from oracle.yuv_oracle import rgb_to_yuv, yuv_to_rgb  # noqa: E402

FRAMES_PER_STEP, MAX_BOXES, MAX_BATCH = 16, 32, 64


def _torch_convert(y, u, v, matrix="bt601"):
    """limited-range fixed-point formula on full-resolution int32 planes"""
    cy, cvr, cvg, cug, cub = COEFS[matrix]
    u, v = u - 128, v - 128
    yy = (y - 16).clamp_min(0) * cy + (1 << 19)
    return torch.stack([(yy + cvr * v) >> 20, (yy + cvg * v + cug * u) >> 20, (yy + cub * u) >> 20], -1).clamp(0, 255).to(torch.uint8)


def torch_i420_to_rgb(f: torch.Tensor) -> torch.Tensor:
    """The obvious workaround for I420: the whole frame converted in torch int32 ops."""
    h, w = f.shape[0] // 3 * 2, f.shape[1]
    flat, q = f[h:].reshape(-1), (h // 2) * (w // 2)
    up = lambda c: c.view(h // 2, w // 2).int().repeat_interleave(2, 0).repeat_interleave(2, 1)
    return _torch_convert(f[:h].int(), up(flat[:q]), up(flat[q:]))


def torch_yuyv_to_rgb(f: torch.Tensor) -> torch.Tensor:
    """The same for YUYV [H, W, 2]."""
    h, w = f.shape[0], f.shape[1]
    q = f.view(h, w // 2, 4).int()
    y = torch.stack([q[..., 0], q[..., 2]], -1).view(h, w)
    return _torch_convert(y, q[..., 1].repeat_interleave(2, 1), q[..., 3].repeat_interleave(2, 1))


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
    i420 = [rgb_to_yuv(im, "i420") for im in imgs]
    yuyv = [rgb_to_yuv(im, "yuyv") for im in imgs]
    nv12 = [rgb_to_yuv(im, "nv12") for im in imgs]
    rgb_i420 = [yuv_to_rgb(f, "i420") for f in i420]                   # what cv2.cvtColor(COLOR_YUV2RGB_I420) gives
    rgb_yuyv = [yuv_to_rgb(f, "yuyv") for f in yuyv]
    assert all(np.array_equal(a, yuv_to_rgb(f, "nv12")) for a, f in zip(rgb_i420, nv12))   # I420 and NV12 carry the same samples
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
    h_i420, h_rgb = [pin(f) for f in i420], [pin(f) for f in rgb_i420]
    d_i420, d_yuyv, d_nv12 = ([torch.from_numpy(f).cuda() for f in fs] for fs in (i420, yuyv, nv12))
    d_boxes = [torch.from_numpy(b).cuda() for b in boxes]
    h_boxes = [np.ascontiguousarray(b) for b in boxes]
    crops = int(counts.sum())
    mb = lambda fs: sum(f.nbytes for f in fs) * 4 / 1e6
    print(f"{FRAMES_PER_STEP} frames per step, {crops} crops ({int(counts.min())}..{int(counts.max())} per frame); "
          f"H2D per step: I420 {mb(i420):.1f} MB, YUYV {mb(yuyv):.1f} MB, RGB {mb(rgb_i420):.1f} MB", flush=True)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=MAX_BATCH)
    m.load_state_dict(sd).to("cuda:0")
    rot = lambda i, fr: [fr[(i * FRAMES_PER_STEP + f) % len(fr)] for f in range(FRAMES_PER_STEP)]
    arms = {
        "dev_i420": lambda i: m.infer_frames_yuv(rot(i, d_i420), d_boxes, layout="i420"),
        "dev_yuyv": lambda i: m.infer_frames_yuv(rot(i, d_yuyv), d_boxes, layout="yuyv"),
        "dev_nv12": lambda i: m.infer_frames_yuv(rot(i, d_nv12), d_boxes, layout="nv12"),
        "dev_torch_i420": lambda i: m.infer_frames([torch_i420_to_rgb(f) for f in rot(i, d_i420)], d_boxes),
        "dev_torch_yuyv": lambda i: m.infer_frames([torch_yuyv_to_rgb(f) for f in rot(i, d_yuyv)], d_boxes),
        "host_i420": lambda i: m.infer_frames_yuv_host(rot(i, h_i420), h_boxes, layout="i420"),
        "host_rgb": lambda i: m.infer_frames_host(rot(i, h_rgb), h_boxes),
    }
    cat = lambda xs: np.concatenate([x.cpu().numpy() if torch.is_tensor(x) else x for x in xs])
    for i in range(4):                                                  # the 4 frame rotations: identical outputs
        want = m.infer_frames_host(rot(i, rgb_yuyv), h_boxes)
        ref = {a: (cat(want[0]), cat(want[1])) for a in ("dev_yuyv", "dev_torch_yuyv")}
        want = arms["host_rgb"](i)
        for a, fn in arms.items():
            kp, idx = fn(i)
            wk, wi = ref.get(a, (cat(want[0]), cat(want[1])))
            assert np.array_equal(cat(kp), wk) and np.array_equal(cat(idx), wi), f"step {i}: {a} != its RGB call"
    print("outputs of all arms bit-identical to the RGB calls on the converted frames", flush=True)
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
    for a in ("dev_i420", "dev_yuyv", "dev_nv12", "dev_torch_i420", "dev_torch_yuyv"):
        m.profile_collect()
        for i in range(args.steps):
            arms[a](i)
        torch.cuda.synchronize()
        pre = m.profile_collect()["crop_preprocess"]                  # the frame gather's kernel class
        prof[a] = {"preprocess_ms_per_step": pre[0] / args.steps, "preprocess_launches_per_step": pre[1] / args.steps}
    m.set_option("profile", 0)
    for a, conv, frames in (("dev_torch_i420", torch_i420_to_rgb, d_i420), ("dev_torch_yuyv", torch_yuyv_to_rgb, d_yuyv)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            [conv(f) for f in rot(i, frames)]
        e1.record()
        e1.synchronize()
        prof[a]["torch_conversion_ms_per_step"] = e0.elapsed_time(e1) / args.steps

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
