"""Generate tests/golden/flip_{s,b}_coco.npz (flip test) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Run here (the container that has /root/reference):   python oracle/make_golden_flip.py

Recipe, per model size (ViT-S and ViT-B, COCO, K = 17), with the reference's own modules (oracle/ref_import.py):
  * weights: flip_weights.flip_symmetric_state_dict(..., COCO_FLIP_PAIRS) -- make_state_dict(..., peaky=0.1, bumps=True) with
    the bumps placed flip-symmetrically (without it every averaged map has two peaks of similar height and the bf16-vs-fp32
    argmax would jump between them);
  * crops: vitpose_oracle.make_crops(B, xseed), org sizes as make_golden_batch.org_sizes;
  * for shift_heatmap in (False, True): the fp32 reference ViTPose, output = model(x),
    output_flipped = keypoint_head.inference_model(backbone(torch.flip(x, [3])), flip_pairs) with
    keypoint_head.test_cfg['shift_heatmap'] set (head/topdown_heatmap_simple_head.py:195-218), the average
    (output + output_flipped) * 0.5, then VitInference.postprocess one crop at a time (ref_import.postprocess);
  * one frame + boxes case (shift_heatmap False): preproc_oracle.make_frame and the boxes of make_golden_frames' frame_a
    except its 1x1 box,
    through the reference's per-person loop -- box pad / clip, crop, pad_image, VitInference.pre_img -- then the same flip
    composition, postprocess and the frame offset (easy_ViTPose/inference.py:258-272).
Stored like the batch_* fixtures: keypoints, argmax (np.argmax of the averaged maps), heatmap range, per-map checksums and a
sample of heatmaps.  For every averaged map the script prints the margin between its maximum and its best far competitor
(Chebyshev distance > FAR_CELLS from the arg-max) and asserts that one peak dominates.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import decode_modes_oracle as DM, preproc_oracle as P, ref_import, vitpose_oracle as O  # noqa: E402
from oracle.flip_weights import flip_symmetric_state_dict  # noqa: E402
from oracle.make_golden_batch import org_sizes  # noqa: E402
from oracle.make_golden_frames import FRAME_CASES  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
PAIRS = [tuple(p) for p in DM.COCO_FLIP_PAIRS]
FAR_CELLS = 4                 # a bump spans about 10 heatmap cells; a competitor farther than this is another peak
MIN_MARGIN = 0.02             # of the heatmap range: twice the engine's heatmap tolerance, so bf16 cannot swap the peaks

# name -> (size, B, weight seed, crop seed)
CASES = {"flip_s_coco": ("s", 8, 121, 221), "flip_b_coco": ("b", 8, 122, 222)}


def far_margin(hm: np.ndarray) -> np.ndarray:
    """[N,K,64,48] -> [N,K]: max - best value farther than FAR_CELLS (Chebyshev) from the arg-max."""
    N, K = hm.shape[:2]
    flat = hm.reshape(N, K, -1)
    am = flat.argmax(-1)
    yy, xx = np.divmod(np.arange(64 * 48), 48)
    dist = np.maximum(np.abs(yy[None, None] - (am // 48)[..., None]), np.abs(xx[None, None] - (am % 48)[..., None]))
    return flat.max(-1) - np.where(dist > FAR_CELLS, flat, -np.inf).max(-1)


def check_margins(tag: str, hm: np.ndarray) -> None:
    rng = float(hm.max() - hm.min())
    m = far_margin(hm) / rng
    print(f"{tag}: averaged-map margin to the best far competitor, fraction of range: min {m.min():.4f} median "
          f"{np.median(m):.4f} (bar {MIN_MARGIN})", flush=True)
    assert m.min() > MIN_MARGIN, (tag, np.unravel_index(m.argmin(), m.shape), m.min())


def main() -> None:
    import torch
    torch.set_grad_enabled(False)
    ns = ref_import.load()
    inf = ref_import.load_vitinference()
    vi = object.__new__(inf.VitInference)              # only pre_img is used: it needs target_size
    vi.target_size = (192, 256)
    fh, fw, fseed, _, _, _, _, rows = FRAME_CASES["frame_a"]
    # without frame_a's 1x1 box (a 21x21 pure upscale): its nearly flat crop leaves one averaged map with two peaks 0.8 % of
    # the range apart, a near-tie where bf16 may pick either
    rows = np.asarray([r for r in rows if r[2] - r[0] > 1], np.float64)
    boxes = rows[rows[:, 4] > 0.35, :4].round().astype(int)
    frame = P.make_frame(fh, fw, fseed)
    os.makedirs(OUT, exist_ok=True)
    for name, (size, B, wseed, xseed) in CASES.items():
        D, depth, heads = O.MODEL_DIMS[size]
        K = 17
        model = ns.ViTPose(ns.dyn_model_import("coco", size)).eval()
        sd = flip_symmetric_state_dict(D, depth, K, wseed, PAIRS)
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)

        def flip_test(x: np.ndarray, shift: bool) -> np.ndarray:
            xt = torch.from_numpy(x)
            out = model(xt).numpy()
            model.keypoint_head.test_cfg["shift_heatmap"] = shift
            out_f = model.keypoint_head.inference_model(model.backbone(torch.flip(xt, [3])), PAIRS)
            return ((out + out_f) * 0.5).astype(np.float32)

        x = O.make_crops(B, xseed)
        org_wh = org_sizes(B, xseed)
        rs = np.random.RandomState(xseed + 9)
        crop_ids = np.sort(rs.choice(B, size=4, replace=False)).astype(np.int32)
        kp_ids = np.sort(rs.choice(K, size=8, replace=False)).astype(np.int32)
        out = dict(org_wh=org_wh, crop_ids=crop_ids, kp_ids=kp_ids, frame_rows=rows.astype(np.float32),
                   meta=np.array([D, depth, heads, K, B, wseed, xseed, fh, fw, fseed], np.int64))
        for shift in (0, 1):
            hm = flip_test(x, bool(shift))
            check_margins(f"{name} shift={shift}", hm)
            kp = np.concatenate([ref_import.postprocess(ns, hm[i:i + 1], int(org_wh[i, 0]), int(org_wh[i, 1])) for i in range(B)], 0)
            out[f"kpts_{shift}"] = kp.astype(np.float32)
            out[f"idx_{shift}"] = hm.reshape(B, K, -1).argmax(-1).astype(np.int32)
            out[f"range_{shift}"] = np.array([hm.min(), hm.max()], np.float32)
            out[f"map_sum_{shift}"] = hm.reshape(B, K, -1).sum(-1, dtype=np.float64)
            out[f"sample_hm_{shift}"] = hm[crop_ids][:, kp_ids]
            vis = kp[..., 2] > 0.3
            print(name, f"shift={shift}", "range", float(hm.min()), float(hm.max()), "visible", int(vis.sum()), "/", vis.size, flush=True)

        # frame + boxes, the reference's per-person loop (easy_ViTPose/inference.py:258-272)
        kps, orgs, hms = [], [], []
        for bb in boxes.copy():
            bb[[0, 2]] = np.clip(bb[[0, 2]] + [-10, 10], 0, frame.shape[1])
            bb[[1, 3]] = np.clip(bb[[1, 3]] + [-10, 10], 0, frame.shape[0])
            img, (left_pad, top_pad) = inf.pad_image(frame[bb[1]:bb[3], bb[0]:bb[2]], 3 / 4)
            xi, org_h, org_w = vi.pre_img(img)
            hm = flip_test(xi, False)
            kp = ref_import.postprocess(ns, hm, org_w, org_h)[0]
            kp[:, :2] += bb[:2][::-1] - [top_pad, left_pad]
            kps.append(kp); orgs.append((org_w, org_h)); hms.append(hm[0])
        hm = np.stack(hms, 0)
        check_margins(f"{name} frame", hm)
        out["frame_kpts"] = np.stack(kps, 0).astype(np.float32)
        out["frame_org_wh"] = np.array(orgs, np.int32)
        out["frame_idx"] = hm.reshape(len(hms), K, -1).argmax(-1).astype(np.int32)
        out["frame_range"] = np.array([hm.min(), hm.max()], np.float32)
        np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **out)
        print(name, "written", os.path.getsize(os.path.join(OUT, f"{name}.npz")), "bytes", flush=True)


if __name__ == "__main__":
    main()
