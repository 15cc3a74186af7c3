"""Times SORT on the device (track.DeviceSort / vpb_tracker_update) on the ap10k-streams shape: 16 streams of about 9 people,
300 frames, at yolo_step 1 (max_age 1, min_hits 3, detections every frame) and yolo_step 3 (max_age 3, min_hits 1, empty
detections on 2 frames of 3).  Per step (one update of all 16 streams):
  device_eager    update_device on detections already on the device (CUDA events around the 300 steps)
  device_replay   the same update captured once in a CUDA graph: copy the step's detections into the static input, replay
  host_update     DeviceSort.update on numpy arrays: one upload, the update, one read-back (host clock)
  oracle_cpu      oracle/sort_oracle.py on this host's CPU (the numpy restatement; host clock)
  reference_cpu   the unmodified easy_ViTPose/sort.py, 16 Sort objects round-robin, when the reference tree is present
Every arm's rows are checked equal to the oracle's before timing.  Then the tracker's added cost in a pose step: ViT-B/17,
max_batch 32, 16 1080p device frames, `inference_frames_tracked` (tracker update + count read-back + infer_frames on the
tracker's device boxes) against `infer_frames` alone on the same boxes (host clock, synchronised per step).  Prints one JSON
line with the card's name and power limit.

    python tools/track_bench.py [--frames 300] [--pose-steps 40] [--reference]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import sort_oracle as SO  # noqa: E402

STREAMS, PEOPLE = 16, 9


def workload(frames: int, step: int):
    seqs = [SO.make_sequence(500 + s, frames, PEOPLE, "walk") for s in range(STREAMS)]
    empty = np.empty((0, 5))
    return [[sq[f] if (f < 3 or f % step == 0) else empty for sq in seqs] for f in range(frames)]


def oracle_rows(dl_all, max_age, min_hits):
    o = SO.SortOracle(STREAMS, max_age, min_hits, 0.3)
    return [o.update(dl) for dl in dl_all]


def cpu_ms(fn, frames):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3 / frames


def bench_tracker(torch, dl_all, max_age, min_hits, want, reference):
    from easy_vitpose_b200.track import DeviceSort
    F = len(dl_all)
    packer = DeviceSort(STREAMS, max_age, min_hits)
    packed = [packer.pack(dl) for dl in dl_all]
    res = {}

    def check(rows_per_frame, what):
        for f, (g, w) in enumerate(zip(rows_per_frame, want)):
            assert all(np.array_equal(a, b) and a.shape == b.shape for a, b in zip(g, w)), f"{what}: frame {f} differs from the oracle"

    # host form (also the correctness check of the device path)
    t = DeviceSort(STREAMS, max_age, min_hits)
    check([t.update(dl) for dl in dl_all], "host_update")
    t = DeviceSort(STREAMS, max_age, min_hits)
    torch.cuda.synchronize()
    res["host_update_ms"] = cpu_ms(lambda: [t.update(dl) for dl in dl_all], F)

    # eager device calls
    t = DeviceSort(STREAMS, max_age, min_hits)
    outs = [t.update_device(d, c) for d, c in packed]
    rows = [[r[s, :int(n[s])].cpu().numpy() for s in range(STREAMS)] for r, _, n in outs]
    check(rows, "device_eager")
    t = DeviceSort(STREAMS, max_age, min_hits)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for d, c in packed:
        t.update_device(d, c)
    e1.record()
    e1.synchronize()
    res["device_eager_ms"] = e0.elapsed_time(e1) / F

    # graph replays
    g_t = DeviceSort(STREAMS, max_age, min_hits)
    dets = torch.zeros_like(packed[0][0])
    counts = torch.zeros_like(packed[0][1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        g_rows, _, g_n = g_t.update_device(dets, counts)
    torch.cuda.synchronize()
    got = []
    for d, c in packed:
        dets.copy_(d)
        counts.copy_(c)
        graph.replay()
        n = g_n.cpu()
        got.append([g_rows[s, :int(n[s])].cpu().numpy() for s in range(STREAMS)])
    check(got, "device_replay")
    g_t.reset()
    e0.record()
    for d, c in packed:
        dets.copy_(d)
        counts.copy_(c)
        graph.replay()
    e1.record()
    e1.synchronize()
    res["device_replay_ms"] = e0.elapsed_time(e1) / F

    res["oracle_cpu_ms"] = cpu_ms(lambda: oracle_rows(dl_all, max_age, min_hits), F)
    if reference:
        ref = SO.load_reference_sort()
        ref.KalmanBoxTracker.count = 0
        sorts = [ref.Sort(max_age, min_hits, 0.3) for _ in range(STREAMS)]
        res["reference_cpu_ms"] = cpu_ms(lambda: [[s.update(d) for s, d in zip(sorts, dl)] for dl in dl_all], F)
    return res


def bench_pose(torch, dl_all, steps):
    from bench import stream_workload
    from easy_vitpose_b200 import B200PoseBackend, ViTPose, model_cfg
    from easy_vitpose_b200.synthetic import random_state_dict
    from easy_vitpose_b200.track import DeviceSort
    imgs, _, _ = stream_workload(0, STREAMS, 32)
    d_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    frames = [d_imgs[s % len(d_imgs)] for s in range(STREAMS)]
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=32)
    m.load_state_dict(sd).to("cuda:0")
    backend = B200PoseBackend(m)
    want = oracle_rows(dl_all[:steps], 1, 3)
    boxes = [[torch.from_numpy(np.round(r[:, :4]).astype(np.int32)).cuda() for r in rows] for rows in want]
    t = DeviceSort(STREAMS, 1, 3, device=0)
    for f in range(steps):                                            # same keypoints and ids, and warm-up
        got = backend.inference_frames_tracked(frames, dl_all[f], t)
        kps, _ = m.infer_frames(frames, boxes[f])
        for s in range(STREAMS):
            assert list(got[s]) == want[f][s][:, 5].astype(int).tolist()
            assert all(np.array_equal(a, b) for a, b in zip(got[s].values(), kps[s].cpu().numpy())), f"pose step {f} stream {s}"
    t = DeviceSort(STREAMS, 1, 3, device=0)
    torch.cuda.synchronize()
    tracked = cpu_ms(lambda: [backend.inference_frames_tracked(frames, dl_all[f], t) for f in range(steps)], steps)

    def untracked():
        for f in range(steps):
            kps, _ = m.infer_frames(frames, boxes[f])
            [k.cpu() for k in kps]
    untracked_ms = cpu_ms(untracked, steps)
    return {"tracked_pose_ms": tracked, "infer_frames_ms": untracked_ms, "crops_per_step": float(np.mean([sum(len(r) for r in w) for w in want]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--pose-steps", type=int, default=40)
    ap.add_argument("--reference", action="store_true", help="also time the unmodified sort.py (needs the reference tree)")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "track_bench needs a GPU"
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                                                  # the timing stands without the label
        card = f"unknown ({exc})"
    out = {"workload": f"{STREAMS} streams x {PEOPLE} people, {args.frames} frames", "card": card, "cpu_threads": os.cpu_count()}
    for step in (1, 3):
        max_age, min_hits = step, 3 if step == 1 else 1
        dl_all = workload(args.frames, step)
        out[f"yolo_step_{step}"] = bench_tracker(torch, dl_all, max_age, min_hits, oracle_rows(dl_all, max_age, min_hits), args.reference)
    out["pose"] = bench_pose(torch, workload(args.pose_steps, 1), args.pose_steps)
    out["pose"]["tracker_added_ms"] = out["pose"]["tracked_pose_ms"] - out["pose"]["infer_frames_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
