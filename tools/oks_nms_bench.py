"""Times OKS NMS on the device (nms.oks_nms_device / vpb_oks_nms) against the reference functions on the host CPU, per call
(every frame of the shape once):
  device_replay   the call captured once in a CUDA graph and replayed (CUDA events around all replays)
  device_eager    oks_nms_device on inputs already on the device (CUDA events)
  reference_cpu   the unmodified reference oks_nms / soft_oks_nms, looped over the frames (host clock); needs the reference
                  tree (`oracle.ref_import`); where it is absent, oracle/oks_nms_oracle.py's numpy restatement, which follows
                  the same steps, is timed instead and the arm is named restatement_cpu
on four shapes: 64 frames x 100 people at K = 17, hard and soft; the ap10k-streams shape, 16 frames and 143 people (about
9 per frame) at K = 17, hard; and 16 frames x 256 people at K = 133, hard.  People are jittered copies of a few poses
(duplicate-heavy, as a detector's overlapping boxes make them).  Every device arm's kept lists are checked against the
oracle first.  Three runs of every arm after a warm-up; prints one JSON line with the card's name and power limit.

    python tools/oks_nms_bench.py [--iters 200] [--cpu-iters 2]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import oks_nms_oracle as O  # noqa: E402

# name: (frames, people per frame (list or int), K, soft)
SHAPES = {"f64_p100_k17_hard": (64, 100, 17, False), "f64_p100_k17_soft": (64, 100, 17, True),
          "ap10k_streams_hard": (16, [9] * 15 + [8], 17, False), "f16_p256_k133_hard": (16, 256, 133, False)}
RUNS = 3


def workload(frames, people, K, seed):
    rng = np.random.default_rng(seed)
    per = people if isinstance(people, list) else [people] * frames
    sig = None if K == 17 else rng.uniform(0.02, 0.1, K)
    kps, ars, scs = [], [], []
    for n in per:
        poses = max(1, n // 3)
        base = rng.uniform(0, 1500, (poses, 1, 2)) + rng.normal(0, 40, (poses, K, 2))
        src = rng.integers(0, poses, n)
        kp = np.zeros((n, K, 3), np.float32)
        kp[:, :, :2] = base[src] + rng.choice([1.0, 4.0, 12.0], (n, 1, 1)) * rng.normal(0, 1, (n, K, 2))
        kp[:, :, 2] = rng.uniform(0, 1, (n, K))
        kps.append(kp)
        ars.append(rng.uniform(5e3, 8e4, poses)[src])
        scs.append(rng.uniform(0, 1, n))
    return kps, ars, scs, sig


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = out[0].split(", ")
        return name, power
    except Exception as exc:                                            # reported, never guessed
        return f"unknown ({exc})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--cpu-iters", type=int, default=2)
    a = ap.parse_args()
    import torch

    from easy_vitpose_b200.nms import OksNmsResult, check, oks_nms_device
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    warnings.simplefilter("ignore", RuntimeWarning)
    try:
        R = O.load_reference_nms()
        ref_name = "reference_cpu"
    except RuntimeError:
        R, ref_name = None, "restatement_cpu"
    dev = torch.device("cuda", 0)
    name, power = card()
    result = {"card": name, "power_limit": power, "iters": a.iters, "shapes": {}}
    for tag, (frames, people, K, soft) in SHAPES.items():
        kps, ars, scs, sig = workload(frames, people, K, len(tag))
        kp = torch.from_numpy(np.concatenate(kps)).to(dev)
        cnt = torch.tensor([len(k) for k in kps], dtype=torch.int32, device=dev)
        ar = torch.from_numpy(np.concatenate(ars)).to(dev)
        sc = torch.from_numpy(np.concatenate(scs)).to(dev)
        n = kp.shape[0]
        out = OksNmsResult(torch.empty(n, dtype=torch.int32, device=dev), torch.empty(frames, dtype=torch.int32, device=dev),
                           torch.empty(n, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        call = lambda: oks_nms_device(kp, cnt, ar, sc, 0.9, sig, None, soft, 20, None, out=out)   # noqa: E731
        call()
        check(out)
        keep, kc = out.keep.cpu().numpy(), out.keep_counts.cpu().numpy()
        r, mism = 0, 0
        for f, k in enumerate(kps):
            want = (O.soft_oks_nms(k, ars[f], scs[f], 0.9, 20, sig) if soft else O.oks_nms(k, ars[f], scs[f], 0.9, sig))
            if not np.array_equal(keep[r:r + kc[f]], want):
                assert O.flag_ambiguous(k, ars[f], scs[f], 0.9, sig, None, soft, 20), (tag, f)
                mism += 1
            r += len(k)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            call()
        arms = {"device_replay": graph.replay, "device_eager": call}
        times = {k: [] for k in arms}
        for k, fn in arms.items():
            for _ in range(10):
                fn()
        for _ in range(RUNS):
            for k, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.iters)
        cpu = []
        dbs = [O.kpts_db(k, ars[f], scs[f]) for f, k in enumerate(kps)]
        for _ in range(RUNS):
            t0 = time.perf_counter()
            for _ in range(a.cpu_iters):
                for f, db in enumerate(dbs):
                    if R is not None:
                        (R.soft_oks_nms(db, 0.9, 20, sig) if soft else R.oks_nms(db, 0.9, sig))
                    else:
                        (O.soft_oks_nms(kps[f], ars[f], scs[f], 0.9, 20, sig) if soft else O.oks_nms(kps[f], ars[f], scs[f], 0.9, sig))
            cpu.append((time.perf_counter() - t0) * 1e3 / a.cpu_iters)
        times[ref_name] = cpu
        result["shapes"][tag] = {"frames": frames, "people": n, "K": K, "soft": soft, "ambiguous_frames_differing": mism,
                                 "ms_median": {k: float(np.median(v)) for k, v in times.items()},
                                 "ms_runs": {k: [round(x, 5) for x in v] for k, v in times.items()}}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
