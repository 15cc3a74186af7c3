#!/usr/bin/env python
"""Rotated video frames (the `rotate` argument) read in place by the engine, against the upright floor and today's workaround,
on the video workload of bench.py --config ap10k-streams (ViT-B/17, max_batch 64, a step = 16 frames with Poisson(10) detector
boxes each).  The stored frames are the workload's four seeded 1920x1080 (w x h) images; rotated by 90 or 270 degrees they are
seen as 1080x1920 portrait views, with person-like boxes drawn in the portrait view; at 0 and 180 degrees the view is
landscape and the boxes are the workload's own.  Per layout (RGB, I420, NV12; limited-range BT.601 for YUV):
  rot<r>       stored frames -> the frame call with rotate=r (the gather reads the stored frame through the rotation)
  floor        frames rotated by 90 degrees beforehand (I420 / NV12: each plane rotated, still 4:2:0) -> the upright call
  workaround   what a user does without `rotate`: RGB torch.rot90(frame).contiguous(); YUV a whole-frame torch conversion to
               RGB, then torch.rot90(...).contiguous(); then the upright RGB call
Before timing, the outputs of rot90, floor and workaround are checked bit-identical.  Reported: ms per step (host clock around
`steps` steps ending in a device synchronise; the arms alternate, three runs each, medians), and the frame gather's time per
step (the engine's `crop_preprocess` kernel class, CUDA events around each launch with option "profile", in a separate run:
the figure tools/yuv_bench.py reports).  Prints the card and its power limit first.

    python tools/rotation_bench.py [--steps 50] [--warmup 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import stream_workload  # noqa: E402
from easy_vitpose_b200 import ViTPose, model_cfg  # noqa: E402
from easy_vitpose_b200.synthetic import random_state_dict  # noqa: E402
from oracle.yuv_oracle import rgb_to_yuv  # noqa: E402
from yuv_bench import _torch_convert, torch_i420_to_rgb  # noqa: E402

FRAMES_PER_STEP, MAX_BOXES, MAX_BATCH = 16, 32, 64
ROTATIONS = (0, 90, 180, 270)


def portrait_boxes(counts, seed=4100):
    """person-like boxes in a 1080x1920 (w x h) portrait view, drawn as bench.stream_workload draws them in landscape"""
    rs = np.random.RandomState(seed)
    VH, VW = 1920, 1080
    out = []
    for n in counts:
        w = rs.randint(90, 420, size=n); h = (w * rs.uniform(1.6, 2.6, size=n)).astype(np.int64)
        x0 = rs.randint(0, VW - 100, size=n); y0 = rs.randint(0, VH - 200, size=n)
        out.append(np.ascontiguousarray(np.stack([x0, y0, x0 + w, y0 + h], 1).astype(np.int32)))
    return out


def torch_nv12_to_rgb(f: torch.Tensor) -> torch.Tensor:
    """The whole-frame workaround for NV12, as yuv_bench.torch_i420_to_rgb does it for I420."""
    h, w = f.shape[0] // 3 * 2, f.shape[1]
    uv = f[h:].view(h // 2, w // 2, 2).int()
    up = lambda c: c.repeat_interleave(2, 0).repeat_interleave(2, 1)
    return _torch_convert(f[:h].int(), up(uv[..., 0]), up(uv[..., 1]))


def rot90_yuv(f: np.ndarray, layout: str) -> np.ndarray:
    """a stacked 4:2:0 frame turned by 90 degrees counter-clockwise plane by plane: the 4:2:0 frame of the rotated picture"""
    h, w = f.shape[0] // 3 * 2, f.shape[1]
    y = np.rot90(f[:h])
    if layout == "nv12":
        uv = np.rot90(f[h:].reshape(h // 2, w // 2, 2)).reshape(w // 2, h)
        return np.ascontiguousarray(np.concatenate([y, uv], 0))
    flat, q = f[h:].reshape(-1), (h // 2) * (w // 2)
    u, v = (np.rot90(c.reshape(h // 2, w // 2)).reshape(-1) for c in (flat[:q], flat[q:]))
    return np.ascontiguousarray(np.concatenate([y.reshape(-1), u, v]).reshape(3 * w // 2, h))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    imgs, land, counts = stream_workload(0, FRAMES_PER_STEP, MAX_BOXES)
    port = portrait_boxes(counts)
    boxes = {r: [torch.from_numpy(b).cuda() for b in (port if r in (90, 270) else land)] for r in ROTATIONS}
    stored = {"rgb": imgs, "i420": [rgb_to_yuv(im, "i420") for im in imgs], "nv12": [rgb_to_yuv(im, "nv12") for im in imgs]}
    pre = {"rgb": [np.ascontiguousarray(np.rot90(im)) for im in imgs]}
    pre.update({lay: [rot90_yuv(f, lay) for f in stored[lay]] for lay in ("i420", "nv12")})
    dev = {lay: [torch.from_numpy(f).cuda() for f in fs] for lay, fs in stored.items()}
    dpre = {lay: [torch.from_numpy(f).cuda() for f in fs] for lay, fs in pre.items()}
    crops = int(counts.sum())
    print(f"{FRAMES_PER_STEP} frames per step, {crops} crops ({int(counts.min())}..{int(counts.max())} per frame)", flush=True)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=MAX_BATCH)
    m.load_state_dict(sd).to("cuda:0")
    pick = lambda i, fr: [fr[(i * FRAMES_PER_STEP + f) % len(fr)] for f in range(FRAMES_PER_STEP)]
    conv = {"i420": torch_i420_to_rgb, "nv12": torch_nv12_to_rgb}

    def call(lay, frames, bb, rotate=0):
        if lay == "rgb":
            return m.infer_frames(frames, bb, rotate=rotate)
        return m.infer_frames_yuv(frames, bb, layout=lay, rotate=rotate)

    arms = {}
    for lay in stored:
        for r in ROTATIONS:
            arms[f"{lay}_rot{r}"] = (lambda lay, r: lambda i: call(lay, pick(i, dev[lay]), boxes[r], r))(lay, r)
        arms[f"{lay}_floor"] = (lambda lay: lambda i: call(lay, pick(i, dpre[lay]), boxes[90]))(lay)
        if lay == "rgb":
            arms["rgb_workaround"] = lambda i: m.infer_frames([torch.rot90(f, 1, dims=(0, 1)).contiguous() for f in pick(i, dev["rgb"])],
                                                              boxes[90])
        else:
            arms[f"{lay}_workaround"] = (lambda lay: lambda i: m.infer_frames(
                [torch.rot90(conv[lay](f), 1, dims=(0, 1)).contiguous() for f in pick(i, dev[lay])], boxes[90]))(lay)
    cat = lambda xs: np.concatenate([x.cpu().numpy() for x in xs])
    for i in range(4):                                                  # the 4 frame rotations of the step
        for lay in stored:
            outs = [arms[f"{lay}_{a}"](i) for a in ("rot90", "floor", "workaround")]
            for kp, idx in outs[1:]:
                assert np.array_equal(cat(kp), cat(outs[0][0])) and np.array_equal(cat(idx), cat(outs[0][1])), f"{lay} step {i}"
    print("rot90, floor and workaround outputs bit-identical on every layout", flush=True)
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

    prof = {}
    m.set_option("profile", 1)
    for a, fn in arms.items():
        m.profile_collect()
        for i in range(args.steps):
            fn(i)
        torch.cuda.synchronize()
        pre_ms = m.profile_collect()["crop_preprocess"]
        prof[a] = pre_ms[0] / args.steps
    m.set_option("profile", 0)

    results = {"card": card, "frames_per_step": FRAMES_PER_STEP, "crops_per_step": crops, "max_batch": MAX_BATCH, "arms": {}}
    for a in arms:
        med = float(np.median(ms[a]))
        results["arms"][a] = {"ms_per_step": med, "runs_ms": ms[a], "gather_ms_per_step": prof[a]}
        print(f"{a}: {med:.3f} ms/step (runs {', '.join(f'{t:.3f}' for t in ms[a])}), gather {prof[a]:.4f} ms/step", flush=True)
    for lay in stored:
        f = prof[f"{lay}_floor"]
        print(f"{lay}: gather rotated / upright (floor): " + ", ".join(f"{r}: {prof[f'{lay}_rot{r}'] / f:.2f}" for r in ROTATIONS), flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
