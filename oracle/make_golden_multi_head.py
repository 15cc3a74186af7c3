"""Generate the multi-head (ViTPose+) fixtures from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Run here (the container that has /root/reference or baseline/_ref):   python oracle/make_golden_multi_head.py

For each case a seeded synthetic ViTPose+ state_dict with all six heads of model_split.py (oracle/multi_head.py: every head
has its own bump pathway, every expert its own random rows) is saved as a checkpoint and split by the UNMODIFIED
model_split.py (`main()` with sys.argv pointing at a temporary directory).  Each split checkpoint the case serves is loaded
into the UNMODIFIED reference ViTPose (`dyn_model_import(dataset, size)`, strict) and run on seeded crops; the keypoints come
from VitInference.postprocess (restated around the reference's keypoints_from_heatmaps by oracle/ref_import.py).  Stored per
case in tests/golden/multi_head_{s,b}.npz:
    crc [6, n_keys] CRC-32 of every tensor of every split checkpoint (keys: the sorted key set, identical for all six)
    per served head j: kpts [n,K_max,3], idx [n,K_max] (np.argmax of the reference heatmaps), org_wh [n,2], range (min, max),
    map_sum [n,K_max] float64, sample_hm [4,64,48] = maps kp_ids[j] of crop 0 (rows / maps past K_j are zero)
The crops are regenerated from seeds (make_crops(n, xseed + j)).  Before writing, the generator asserts that the experts and the
heads matter: the reference run with a swapped expert, and separately with a swapped head, moves the heatmaps of a head far
beyond the 1 % of range the engine is held to.
    s: ViT-S, all six heads served, P = 96 (D - P = 288)      b: ViT-B, coco + ap10k + wholebody served, P = 192"""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import, vitpose_oracle as O  # noqa: E402
from oracle.multi_head import SIZES, plus_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
ALL_HEADS = (("coco", 17), ("aic", 14), ("mpii", 16), ("ap10k", 17), ("apt36k", 17), ("wholebody", 133))  # model_split.py:71-74
# name -> (size, P, served heads, weight seed, crop seed, crops per head)
CASES = {
    "multi_head_s": ("s", 96, ("coco", "aic", "mpii", "ap10k", "apt36k", "wholebody"), 131, 231, 4),
    "multi_head_b": ("b", 192, ("coco", "ap10k", "wholebody"), 132, 232, 4),
}
PREFIX = "vitpose-x-"


def crc(t) -> int:
    return zlib.crc32(np.ascontiguousarray(t.numpy()).tobytes())


def org_sizes(n: int, seed: int) -> np.ndarray:
    rs = np.random.RandomState(seed + 7)
    return np.stack([rs.randint(64, 513, size=n), rs.randint(64, 513, size=n)], 1).astype(np.int32)


def run_model_split(sd: dict, workdir: str) -> "dict[str, dict]":
    """The unmodified model_split.py on `sd` -> {dataset: split state_dict}."""
    import torch
    src = os.path.join(workdir, "plus.pth")
    torch.save({"state_dict": {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}}, src)
    spec = importlib.util.spec_from_file_location("model_split", os.path.join(ref_import.REF_ROOT, "model_split.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    argv = sys.argv
    sys.argv = ["model_split.py", "--source", src, "--prefix", PREFIX, "--target", workdir]
    try:
        mod.main()
    finally:
        sys.argv = argv
    return {n: torch.load(os.path.join(workdir, f"{PREFIX}{n}.pth"), map_location="cpu", weights_only=True)["state_dict"]
            for n, _ in ALL_HEADS}


def reference_heatmaps(ns, size, dataset, sd, x):
    import torch
    # the reference's per-dataset config modules patch the dicts of ViTPose_common in place (ViTPose_wholebody sets 133
    # channels on the shared model dicts), so within one process the last dataset imported wins: re-import them fresh, as a
    # new process running that dataset would
    for m in [m for m in sys.modules if m == "configs" or m.startswith("configs.")]:
        del sys.modules[m]
    model = ns.ViTPose(ns.dyn_model_import(dataset, size)).eval()
    model.load_state_dict(sd, strict=True)
    return np.concatenate([model(torch.from_numpy(x[s:s + 8])).numpy() for s in range(0, len(x), 8)], 0).astype(np.float32)


def main() -> None:
    import torch
    torch.set_grad_enabled(False)
    ns = ref_import.load()
    only = set(sys.argv[1:])
    for name, (size, P, served, wseed, xseed, n) in CASES.items():
        if only and name not in only:
            continue
        D, depth, heads = SIZES[size]
        with tempfile.TemporaryDirectory() as wd:
            split = run_model_split(plus_state_dict(size, [k for _, k in ALL_HEADS], P, wseed), wd)
        keys = sorted(split["coco"])
        assert all(sorted(d) == keys for d in split.values())
        crcs = np.array([[crc(split[h][k]) for k in keys] for h, _ in ALL_HEADS], np.uint32)
        Ks = [dict(ALL_HEADS)[h] for h in served]
        Km = max(Ks)
        H = len(served)
        kpts, idx = np.zeros((H, n, Km, 3), np.float32), np.zeros((H, n, Km), np.int32)
        map_sum, rng = np.zeros((H, n, Km), np.float64), np.zeros((H, 2), np.float32)
        orgs, sample, kp_ids = np.zeros((H, n, 2), np.int32), np.zeros((H, 4, 64, 48), np.float32), np.zeros((H, 4), np.int32)
        for j, (h, K) in enumerate(zip(served, Ks)):
            x = O.make_crops(n, xseed + j)
            hm = reference_heatmaps(ns, size, h, split[h], x)
            org = org_sizes(n, xseed + j)
            kp = np.concatenate([ref_import.postprocess(ns, hm[i:i + 1], int(org[i, 0]), int(org[i, 1])) for i in range(n)], 0)
            kpts[j, :, :K], idx[j, :, :K] = kp, hm.reshape(n, K, -1).argmax(-1)
            map_sum[j, :, :K] = hm.reshape(n, K, -1).sum(-1, dtype=np.float64)
            rng[j] = hm.min(), hm.max()
            orgs[j] = org
            kp_ids[j] = np.sort(np.random.RandomState(xseed + 50 + j).choice(K, size=4, replace=False))
            sample[j] = hm[0, kp_ids[j]]
            vis = kp[..., 2] > 0.3
            print(name, h, "range", float(hm.min()), float(hm.max()), "visible (score > 0.3)", int(vis.sum()), "/", vis.size, flush=True)
            if h == "ap10k":                  # the experts and the heads matter (coco has the same K)
                r = float(hm.max() - hm.min())
                for swap in ("expert", "head"):
                    sd = dict(split[h])
                    for k in sd:
                        if (".mlp.fc2." in k) if swap == "expert" else k.startswith("keypoint_head."):
                            sd[k] = split["coco"][k]
                    moved = float(np.abs(reference_heatmaps(ns, size, h, sd, x) - hm).max())
                    print(name, f"swapped {swap}: heatmaps move by {moved / r:.1%} of range", flush=True)
                    assert moved > 0.05 * r, f"a swapped {swap} moves the heatmaps by only {moved / r:.2%} of range"
        np.savez_compressed(os.path.join(OUT, f"{name}.npz"), keys=np.array(keys), crc=crcs, heads=np.array(served),
                            keypoints=np.array(Ks, np.int32), kpts=kpts, idx=idx, org_wh=orgs, range=rng, map_sum=map_sum,
                            kp_ids=kp_ids, sample_hm=sample, meta=np.array([D, depth, heads, P, n, wseed, xseed], np.int64))


if __name__ == "__main__":
    main()
