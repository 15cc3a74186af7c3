"""Times keypoint smoothing on the device (smooth.DeviceOneEuro / vpb_smoother_update), per step (one update of every stream):
  device_replay   the update captured once in a CUDA graph: copy the step's keypoints, ids and counts into the static
                  inputs, replay (CUDA events around all steps; the copies are included)
  device_eager    update_device on inputs already on the device (CUDA events)
  host_update     DeviceOneEuro.update on numpy arrays: one upload, the update, one read-back (host clock)
  numpy_cpu       the per-id dict of oracle/one_euro_oracle.py's numpy restatement of the reference filter on this host's CPU
                  (what a user composing the reference class by hand runs; host clock)
on two shapes: ap10k-streams (16 streams, 143 people, K = 17, --steps steps, ids with churn) and a stress shape (64 full
streams of 128 people, K = 133, 15% of --steps: its inputs are 12 MB a step), fps mode.  Every device arm's output is
checked equal to the oracle's first.  Then the smoother's added cost in a pose step: ViT-B/17, max_batch 32, 16 1080p device
frames of 9 tracked people, `inference_frames_tracked` with and without a smoother (host clock, synchronised per step, the
two arms alternated).  Three runs of every arm after a warm-up; prints one JSON line with the card's name and power limit.

    python tools/smooth_bench.py [--steps 200] [--cpu-steps 20] [--pose-steps 40]
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

from oracle import one_euro_oracle as OE  # noqa: E402
from oracle import sort_oracle as SO  # noqa: E402

SHAPES = {"ap10k_streams": (16, 143, 17, 1.0), "stress": (64, 128 * 64, 133, 0.15)}   # (S, people, K, share of --steps)
RUNS = 3


def workload(S, people, K, steps, seed):
    """Per step (per-stream float32 [n, K, 3], per-stream ids): `people` spread over the streams (at most 128 each), every
    step about 5% of them missing and, unless a stream is full, 2% replaced by new ids."""
    rng = np.random.default_rng(seed)
    per = np.full(S, people // S)
    per[:people % S] += 1
    churn = 0.02 if per.max() < 128 else 0.0
    ids = [np.arange(100000 * s, 100000 * s + n) for s, n in enumerate(per)]
    nxt = [100000 * s + n for s, n in enumerate(per)]
    base = rng.uniform(1, 1000, (S, 128, K, 2))
    out = []
    for _ in range(steps):
        kl, il = [], []
        for s in range(S):
            new = np.nonzero(rng.uniform(size=len(ids[s])) < churn)[0]
            ids[s][new] = nxt[s] + np.arange(len(new))
            nxt[s] += len(new)
            keep = np.nonzero(rng.uniform(size=len(ids[s])) > 0.05)[0]
            k = np.zeros((len(keep), K, 3), np.float32)
            k[:, :, :2] = base[s, keep] + rng.normal(0, 1.5, (len(keep), K, 2))
            k[:, :, 2] = rng.uniform(0, 1, (len(keep), K))
            kl.append(k)
            il.append(ids[s][keep].tolist())
        out.append((kl, il))
    return out


def stats(xs):
    return {"median": float(np.median(xs)), "runs": [float(x) for x in xs]}


def bench_update(torch, S, people, K, steps, cpu_steps):
    from easy_vitpose_b200.smooth import DeviceOneEuro
    wl = workload(S, people, K, steps, S + K)
    o = OE.SmoothOracle(S, fps=30.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        want = [o.update(kl, il) for kl, il in wl[:10]]
    packed = []
    for kl, il in wl:
        packed.append((torch.from_numpy(np.concatenate(kl)).cuda(), torch.tensor([len(x) for x in il], dtype=torch.int32).cuda(),
                       torch.tensor([i for x in il for i in x], dtype=torch.int32).cuda()))
    F = len(wl)
    res = {"streams": S, "people": int(sum(len(x) for x in wl[0][1])), "K": K}

    def check(outs, what):
        for f, (g, w) in enumerate(zip(outs, want)):
            assert all(np.array_equal(a, b) for a, b in zip(g, w)), f"{what}: step {f} differs from the oracle"

    s = DeviceOneEuro(S, K, fps=30.0)
    check([s.update(kl, il) for kl, il in wl[:10]], "host_update")
    host = []
    for _ in range(RUNS):
        s = DeviceOneEuro(S, K, fps=30.0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for kl, il in wl:
            s.update(kl, il)
        host.append((time.perf_counter() - t0) * 1e3 / F)
    res["host_update_ms"] = stats(host)

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s = DeviceOneEuro(S, K, fps=30.0)
    outs = []
    for kp, c, i in packed[:10]:
        out = torch.empty((kp.shape[0], K, 2), dtype=torch.float64, device="cuda")
        s.update_device(kp.clone(), c, i, out=out)
        offs = np.cumsum([0] + c.tolist())
        r = out.cpu().numpy()
        outs.append([r[offs[j]:offs[j + 1]] for j in range(S)])
    check(outs, "device_eager")
    eager = []
    for _ in range(RUNS):
        s = DeviceOneEuro(S, K, fps=30.0)
        work = [kp.clone() for kp, _, _ in packed]                    # the update smooths its input in place
        torch.cuda.synchronize()
        e0.record()
        for kp, (_, c, i) in zip(work, packed):
            s.update_device(kp, c, i)
        e1.record()
        e1.synchronize()
        eager.append(e0.elapsed_time(e1) / F)
    res["device_eager_ms"] = stats(eager)

    cap = max(p[0].shape[0] for p in packed)
    skp = torch.zeros((cap, K, 3), dtype=torch.float32, device="cuda")
    sids = torch.zeros(cap, dtype=torch.int32, device="cuda")
    scounts = torch.zeros(S, dtype=torch.int32, device="cuda")
    sout = torch.zeros((cap, K, 2), dtype=torch.float64, device="cuda")
    graphs = []
    for _ in range(RUNS + 1):
        g_s = DeviceOneEuro(S, K, fps=30.0)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
            g_s.update_device(skp, scounts, sids, None, sout)
        torch.cuda.synchronize()
        graphs.append((g_s, graph))
    got = []
    for (kl, il), (kp, c, i) in zip(wl[:10], packed[:10]):
        n = kp.shape[0]
        skp[:n].copy_(kp)
        sids[:n].copy_(i)
        scounts.copy_(c)
        graphs[0][1].replay()
        offs = np.cumsum([0] + c.tolist())
        r = sout[:n].cpu().numpy()
        got.append([r[offs[j]:offs[j + 1]] for j in range(S)])
    check(got, "device_replay")
    replay = []
    for _, graph in graphs[1:]:
        torch.cuda.synchronize()
        e0.record()
        for kp, c, i in packed:
            n = kp.shape[0]
            skp[:n].copy_(kp)
            sids[:n].copy_(i)
            scounts.copy_(c)
            graph.replay()
        e1.record()
        e1.synchronize()
        replay.append(e0.elapsed_time(e1) / F)
    res["device_replay_ms"] = stats(replay)

    cpu = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for _ in range(RUNS):
            o = OE.SmoothOracle(S, fps=30.0)
            t0 = time.perf_counter()
            for kl, il in wl[:cpu_steps]:
                o.update(kl, il)
            cpu.append((time.perf_counter() - t0) * 1e3 / min(cpu_steps, F))
    res["numpy_cpu_ms"] = stats(cpu)
    return res


def bench_pose(torch, steps):
    from bench import stream_workload
    from easy_vitpose_b200 import B200PoseBackend, ViTPose, model_cfg
    from easy_vitpose_b200.smooth import DeviceOneEuro
    from easy_vitpose_b200.synthetic import random_state_dict
    from easy_vitpose_b200.track import DeviceSort
    S = 16
    imgs, _, _ = stream_workload(0, S, 32)
    d_imgs = [torch.from_numpy(im).cuda() for im in imgs]
    frames = [d_imgs[s % len(d_imgs)] for s in range(S)]
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in random_state_dict("b", 17, seed=1, peaks=True).items()}
    m = ViTPose(model_cfg("b", 17), max_batch=32)
    m.load_state_dict(sd).to("cuda:0")
    backend = B200PoseBackend(m)
    seqs = [SO.make_sequence(500 + s, steps, 9, "walk") for s in range(S)]
    dl_all = [[sq[f] for sq in seqs] for f in range(steps)]

    def run(smooth):
        t = DeviceSort(S, 1, 3, device=0)
        sm = DeviceOneEuro(S, 17, fps=30.0, device=0) if smooth else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in range(steps):
            backend.inference_frames_tracked(frames, dl_all[f], t, smoother=sm)
        return (time.perf_counter() - t0) * 1e3 / steps

    run(False)
    run(True)                                                           # warm-up of both arms
    plain, smoothed = [], []
    for _ in range(RUNS):
        plain.append(run(False))
        smoothed.append(run(True))
    return {"tracked_pose_ms": stats(plain), "tracked_smoothed_pose_ms": stats(smoothed),
            "smoother_added_ms": float(np.median(smoothed) - np.median(plain))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--cpu-steps", type=int, default=20)
    ap.add_argument("--pose-steps", type=int, default=40)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "smooth_bench needs a GPU"
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:                                                  # the timing stands without the label
        card = f"unknown ({exc})"
    out = {"card": card, "cpu_threads": os.cpu_count(), "steps": args.steps, "cpu_steps": args.cpu_steps}
    for name, (S, people, K, share) in SHAPES.items():
        out[name] = bench_update(torch, S, people, K, max(10, int(args.steps * share)), args.cpu_steps)
    out["pose"] = bench_pose(torch, args.pose_steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
