"""Generate tests/golden/multi_head_topdown_s.npz (flip test + affine top-down crops on several heads) from the UNMODIFIED
reference  --  TEST INFRASTRUCTURE ONLY.

Run where the reference tree is available:   python oracle/make_golden_multi_head_topdown.py

Recipe (ViT-S with all six ViTPose+ heads, P = 96):
  * weights: multi_head_flip.flip_plus_state_dict -- a ViTPose+ state_dict whose heads each own their bump channels (17 + 14 + 16 +
    17 + 17 + 133 = 214 of the 256), placed flip-symmetrically under that head's pairs (multi_head_flip.topdown_pairs: COCO's for coco,
    neighbouring keypoints for the others, for which the reference defines none); split by the UNMODIFIED model_split.py;
  * two synthetic frames (preproc_oracle.make_frame) and three boxes (x, y, w, h) per head spread over them;
  * per box: COCODataset._xywh2cs and the UDP get_warp_matrix of the reference (asserted equal to topdown_args' steps in
    affine_oracle), cv2.warpAffine + the dataset's torchvision ToTensor / Normalize, asserted bit-equal to affine_oracle;
  * per head, on that head's split checkpoint in the UNMODIFIED reference ViTPose: output = model(x), output_flipped =
    keypoint_head.inference_model(backbone(flip(x)), pairs) with test_cfg shift_heatmap False and True, their average, and
    ONE keypoints_from_heatmaps(hm, c, s * 200, unbiased=True, use_udp=True) call on the head's boxes (what one segment of
    vpb_infer_affine_heads decodes);
  * every averaged map's peak must beat its best competitor more than 4 cells away by more than 2 % of the range
    (make_golden_flip.check_margins).
Stored: pairs (flat, with per-head counts), frames, boxes, matrices, centre / scale in pixels, head and frame of every box (boxes
in call order: head-major, frame order inside a head), a CRC-32 of every warped uint8 crop, CRC-32s of the unsplit weights and of
every split checkpoint, and per shift keypoints (y, x, score) [N, K_max, 3], argmax, per-head range, per-map sums and 2 sampled
heatmaps per head (crop 0 of the head).
"""
from __future__ import annotations

import os
import sys
import tempfile
import types
import warnings
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import affine_oracle as A, preproc_oracle as P  # noqa: E402
from oracle.make_golden_affine import load_reference  # noqa: E402
from oracle.make_golden_flip import MIN_MARGIN, far_margin  # noqa: E402
from oracle.make_golden_multi_head import ALL_HEADS, run_model_split  # noqa: E402
from oracle.multi_head import SIZES  # noqa: E402
from oracle.multi_head_flip import flip_plus_state_dict, topdown_pairs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "multi_head_topdown_s.npz")
SIZE, P_ROWS, WSEED, BSEED = "s", 96, 141, 241
FRAMES = [(360, 480, 81), (480, 640, 82)]            # (height, width, seed)
PER_HEAD = 3


def crc(a) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def boxes_for(j: int):
    """three (frame, x, y, w, h) boxes of head j, in frame order; some reach past the frame's border"""
    rs = np.random.RandomState(BSEED + j)
    out = []
    for _ in range(PER_HEAD):
        f = int(rs.randint(0, len(FRAMES)))
        h, w = FRAMES[f][:2]
        bw, bh = rs.uniform(40, 0.6 * w), rs.uniform(60, 0.8 * h)
        out.append((f, float(rs.uniform(-0.2 * bw, w - 0.8 * bw)), float(rs.uniform(-0.2 * bh, h - 0.8 * bh)), bw, bh))
    return sorted(out, key=lambda b: b[0])


def reference_model(ns, dataset, sd):
    """the unmodified reference ViTPose for `dataset`, strict-loaded with sd; the per-dataset config modules patch shared dicts
    in place, so they are re-imported for every dataset (as make_golden_multi_head.reference_heatmaps does)"""
    for m in [m for m in sys.modules if m == "configs" or m.startswith("configs.")]:
        del sys.modules[m]
    model = ns.ViTPose(ns.dyn_model_import(dataset, SIZE)).eval()
    model.load_state_dict(sd, strict=True)
    return model


def main() -> None:
    import cv2
    import torch
    from torchvision import transforms
    torch.set_grad_enabled(False)
    ns = load_reference()
    tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    ds = types.SimpleNamespace(aspect_ratio=192 * 1.0 / 256, pixel_std=200)
    D, depth, nheads = SIZES[SIZE]
    names = [n for n, _ in ALL_HEADS]
    Ks = [k for _, k in ALL_HEADS]
    Km = max(Ks)
    pairs = [topdown_pairs(n, k) for n, k in ALL_HEADS]
    sd = flip_plus_state_dict(SIZE, Ks, P_ROWS, WSEED, pairs)
    wkeys = sorted(sd)
    with tempfile.TemporaryDirectory() as wd:
        split = run_model_split(sd, wd)
    skeys = sorted(split["coco"])
    frames = [P.make_frame(h, w, s) for h, w, s in FRAMES]
    image_size = np.array([192, 256])

    rows = [(j,) + b for j in range(len(ALL_HEADS)) for b in boxes_for(j)]
    N = len(rows)
    mats, cs_px, crcs = np.zeros((N, 2, 3), np.float64), np.zeros((N, 4), np.float32), np.zeros(N, np.uint32)
    xs = []
    for i, (j, f, x, y, w, h) in enumerate(rows):
        c, s = ns.COCODataset._xywh2cs(ds, x, y, w, h)
        c2, s2 = A.xywh2cs((x, y, w, h))
        assert np.array_equal(c, c2) and np.array_equal(s, s2), i
        m = ns.get_warp_matrix(0, c * 2.0, image_size - 1.0, s * 200.0)
        assert np.array_equal(m, A.udp_matrix(c, s)), i
        img = cv2.warpAffine(frames[f], m, (192, 256), flags=cv2.INTER_LINEAR)
        assert np.array_equal(img, A.warp_affine_u8(frames[f], m)), i
        xt = tf(img).numpy()
        assert np.array_equal(xt, A.warp_normalise(frames[f], m)), i
        mats[i], cs_px[i], crcs[i] = m, np.concatenate([c, s * 200.0]), crc(img)
        xs.append(xt)
    head_of = np.array([r[0] for r in rows], np.int32)
    out = dict(meta=np.array([D, depth, nheads, P_ROWS, WSEED, PER_HEAD], np.int64), heads=np.array(names),
               keypoints=np.array(Ks, np.int32), pairs=np.array([p for pp in pairs for p in pp], np.int32).reshape(-1, 2),
               pair_counts=np.array([len(pp) for pp in pairs], np.int32), frames=np.array(FRAMES, np.int64),
               boxes=np.array([r[2:] for r in rows], np.float64), frame_id=np.array([r[1] for r in rows], np.int32), head_id=head_of,
               mats=mats, cs_px=cs_px, crc=crcs, weight_keys=np.array(wkeys), weight_crc=np.array([crc(sd[k]) for k in wkeys], np.uint32),
               split_keys=np.array(skeys), split_crc=np.array([[crc(split[n][k].numpy()) for k in skeys] for n in names], np.uint32))
    rs = np.random.RandomState(5)
    sample_kps = np.stack([np.sort(rs.choice(K, size=2, replace=False)) for K in Ks]).astype(np.int32)
    out["sample_kps"] = sample_kps
    for shift in (0, 1):
        kpts, idx = np.zeros((N, Km, 3), np.float32), np.zeros((N, Km), np.int32)
        map_sum, rng = np.zeros((N, Km), np.float64), np.zeros((len(Ks), 2), np.float32)
        sample = np.zeros((len(Ks), 2, 64, 48), np.float32)
        near = np.zeros((N, Km), bool)
        for j, (name, K) in enumerate(ALL_HEADS):
            sel = np.nonzero(head_of == j)[0]
            x = torch.from_numpy(np.stack([xs[i] for i in sel]))
            model = reference_model(ns, name, split[name])
            model.keypoint_head.test_cfg["shift_heatmap"] = bool(shift)
            hm = ((model(x).numpy() + model.keypoint_head.inference_model(model.backbone(torch.flip(x, [3])), pairs[j])) * 0.5).astype(np.float32)
            m = far_margin(hm) / float(hm.max() - hm.min())
            low = m <= MIN_MARGIN
            print(f"{name} shift={shift}: margin to the best far competitor, fraction of range: min {m.min():.4f} median "
                  f"{np.median(m):.4f}; {int(low.sum())} of {m.size} maps at or below {MIN_MARGIN}", flush=True)
            near[sel, :K] |= low
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", DeprecationWarning)
                pts, prob = ns.keypoints_from_heatmaps(heatmaps=hm, center=cs_px[sel, :2], scale=cs_px[sel, 2:], unbiased=True, use_udp=True)
            kpts[sel, :K] = np.concatenate([pts[:, :, ::-1], prob], axis=2)
            idx[sel, :K] = hm.reshape(len(sel), K, -1).argmax(-1)
            map_sum[sel, :K] = hm.reshape(len(sel), K, -1).sum(-1, dtype=np.float64)
            rng[j] = hm.min(), hm.max()
            sample[j] = hm[0, sample_kps[j]]
            vis = prob[..., 0] > 0.3
            print(name, f"shift={shift}", "range", float(hm.min()), float(hm.max()), "visible", int(vis.sum()), "/", vis.size, flush=True)
        out.update({f"kpts_{shift}": kpts, f"idx_{shift}": idx, f"map_sum_{shift}": map_sum, f"range_{shift}": rng,
                    f"sample_hm_{shift}": sample, f"near_tie_{shift}": near})
        # 214 bump channels leak into every map through the random weights; a few maps keep a second peak close to the first
        assert near.sum() <= 0.01 * (N // len(Ks)) * sum(Ks), (shift, int(near.sum()))
    np.savez_compressed(OUT, **out)
    print("written", OUT, os.path.getsize(OUT), "bytes", flush=True)


if __name__ == "__main__":
    main()
