"""Generate tests/golden/decode_k_edges.npz from the UNMODIFIED reference keypoints_from_heatmaps  --  TEST INFRASTRUCTURE ONLY.

Run here:  python oracle/make_golden_k_edges.py
The decode at the keypoint counts the C ABI promises but the other fixtures never use: K = 1, 2, 32, 33 and 144 (1..144 per
head; the heatmap GEMM's 32- and 144-wide tiles full and one past full).  Maps regenerate from the seeds
(vitpose_oracle.make_decode_maps, N = 12 crops so that every sentinel kind occurs and, at K = 1, sentinel maps follow other
crops' maps); stored per K:
  crop_K_kpts     VitInference.postprocess per crop (one reference call per crop, N = 1), (y, x, score)
  batch_K_kpts    one keypoints_from_heatmaps(unbiased=True, use_udp=True) call on the whole [N,K,64,48] array, where it runs
  batch_K_raises  1 where that call raises: post_dark_udp's `.squeeze()` (top_down_eval.py:414) drops the K = 1 axis for N > 1
and for K = 1 and 144 the other decode modes on float32 centre / scale (the keys of decode_modes.npz: `{pp}_{std|udp}_preds`,
`_maxvals`, `_raises`), plus CombinedTarget (mode 5) at K = 1, one reference call per crop (`comb_preds`, `comb_maxvals`).
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import decode_modes_oracle as M, ref_import, vitpose_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "decode_k_edges.npz")
N = 12
KS = (1, 2, 32, 33, 144)
MODE_KS = (1, 144)
COMBOS = [(None, False), ("default", False), ("unbiased", False), ("megvii", False), ("default", True)]


def seed_of(K: int) -> int:
    return 800 + K


def org_of(K: int) -> np.ndarray:
    rs = np.random.RandomState(seed_of(K) + 1)
    return np.stack([rs.randint(64, 513, size=N), rs.randint(64, 513, size=N)], 1).astype(np.int32)


def centre_scale_of(K: int) -> "tuple[np.ndarray, np.ndarray]":
    rs = np.random.RandomState(seed_of(K) + 2)
    c = np.stack([rs.uniform(50, 600, N), rs.uniform(50, 400, N)], 1).astype(np.float32)
    s = np.stack([rs.uniform(60, 400, N), rs.uniform(80, 520, N)], 1).astype(np.float32)
    return c, s


def _call(ns, *args, **kw):
    """the reference call -> (preds, maxvals) or None where it raises ValueError"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return ns.keypoints_from_heatmaps(*args, **kw)
        except ValueError as e:
            print("  reference raises:", str(e)[:90])
            return None


def main() -> None:
    ns = ref_import.load()
    out = {"meta": np.array([N, *KS], np.int64)}
    for K in KS:
        maps, org = O.make_decode_maps(N, K, seed_of(K)), org_of(K)
        out[f"crop_{K}_kpts"] = np.concatenate([ref_import.postprocess(ns, maps[i:i + 1], int(org[i, 0]), int(org[i, 1]))
                                                for i in range(N)], 0).astype(np.float32)
        r = _call(ns, heatmaps=maps.copy(), center=np.stack([org[:, 0] // 2, org[:, 1] // 2], 1), scale=org.astype(np.int64),
                  unbiased=True, use_udp=True)
        out[f"batch_{K}_raises"] = np.int64(r is None)
        out[f"batch_{K}_kpts"] = (np.zeros((0,), np.float32) if r is None
                                  else np.concatenate([r[0][:, :, ::-1], r[1]], 2).astype(np.float32))
        print(f"K={K}: per-crop postprocess stored; batched call {'raises' if r is None else 'stored'}")
    for K in MODE_KS:
        maps = O.make_decode_maps(N, K, seed_of(K))
        c, s = centre_scale_of(K)
        for pp, udp in COMBOS:
            key = f"k{K}_{pp}_{'udp' if udp else 'std'}"
            r = _call(ns, maps.copy(), c, s, unbiased=False, post_process=pp, kernel=11, use_udp=udp)
            out[key + "_raises"] = np.int64(r is None)
            out[key + "_preds"] = np.zeros((0,), np.float32) if r is None else r[0].astype(np.float32)
            out[key + "_maxvals"] = np.zeros((0,), np.float32) if r is None else r[1].astype(np.float32)
            print(key, "raises" if r is None else "stored")
    # CombinedTarget with one keypoint: [N, 3, 64, 48], one call per crop (the only batch size its index arithmetic accepts)
    cmaps = M.make_combined_maps(N, 1, seed_of(1) + 3)
    c, s = centre_scale_of(1)
    pr, mv = [], []
    for n in range(N):
        p1, m1 = _call(ns, cmaps[n:n + 1].copy(), c[n:n + 1], s[n:n + 1], post_process="default", kernel=11, use_udp=True,
                       target_type="CombinedTarget")
        pr.append(p1[0]); mv.append(m1[0])
    out["comb_preds"] = np.stack(pr).astype(np.float32)
    out["comb_maxvals"] = np.stack(mv).astype(np.float32)
    np.savez_compressed(OUT, **out)
    print("written", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
