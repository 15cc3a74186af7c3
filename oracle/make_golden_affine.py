"""Generate tests/golden/affine_b_coco.npz (affine top-down crops) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Run where the reference tree is available:   python oracle/make_golden_affine.py

Recipe, with the reference's own modules (oracle/ref_import.py; pycocotools, json_tricks and munkres are stubbed the way
ref_import stubs matplotlib / ffmpeg: datasets/COCO.py and vit_utils/transform.py import them but the functions used here
never touch them):
  * three synthetic frames (preproc_oracle.make_frame) and CASES below: boxes (x, y, w, h) inside, partly and wholly outside
    their frame, tiny (up-sampling) and huge (down-sampling) ones; the rotated (+-30 deg) and HRNet-matrix cases are used
    for the matrix / crop checks only;
  * centre / scale from COCODataset._xywh2cs (datasets/COCO.py:318-337), called unbound on a light object that has the
    dataset's aspect_ratio and pixel_std;
  * the matrix from get_warp_matrix(rot, 2c, image_size - 1, s * 200) (post_transforms.py:312-340, use_udp=True) or
    get_affine_transform(c, s, 200, rot, image_size) (transform.py:46-75);
  * cv2.warpAffine(frame, M, (192, 256), flags=cv2.INTER_LINEAR), then the dataset's torchvision ToTensor + Normalize
    (COCO.py:120-123, 289-302).  affine_oracle is asserted bit-equal to cv2, torchvision and the reference on every case;
  * ViT-B/17 with make_state_dict(bumps=True), the fp32 reference ViTPose on the forward cases, then
    keypoints_from_heatmaps(heatmaps, c, s * 200, use_udp=True) (top_down_eval.py:576-579) in one call on the whole array;
  * the flip test with flip_weights.flip_symmetric_state_dict: (model(x) + keypoint_head.inference_model(
    backbone(flip(x)), flip_pairs)) * 0.5 with shift_heatmap off, decoded the same way.
Stored: matrices, centre / scale, the warped uint8 crops of CROP_CASES whole and a CRC-32 of every warped crop, keypoints
(y, x, score), argmax, heatmap range, per-map sums and a sample of heatmaps.
"""
from __future__ import annotations

import importlib
import os
import sys
import types
import warnings
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import affine_oracle as A, decode_modes_oracle as DM, preproc_oracle as P, ref_import, vitpose_oracle as O  # noqa: E402
from oracle.flip_weights import flip_symmetric_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "affine_b_coco.npz")
PAIRS = [tuple(p) for p in DM.COCO_FLIP_PAIRS]
FRAMES = [(360, 480, 71), (480, 640, 72), (300, 420, 73)]        # (height, width, seed)
WSEED, FLIP_WSEED = 131, 132
# (frame, x, y, w, h, rot, builder 0 = UDP / 1 = HRNet, forward): the forward cases are unrotated UDP crops
CASES = [
    (0, 120.0, 60.0, 90.0, 210.0, 0, 0, 1),          # inside
    (0, 300.5, 20.25, 150.0, 120.0, 0, 0, 1),        # wide box
    (0, -40.0, 200.0, 110.0, 190.0, 0, 0, 1),        # partly outside, left / bottom
    (0, 400.0, -60.0, 120.0, 160.0, 0, 0, 1),        # partly outside, top / right
    (1, 250.0, 100.0, 7.0, 9.0, 0, 0, 1),            # tiny: strong up-sampling
    (1, -300.0, -200.0, 1200.0, 900.0, 0, 0, 1),     # huge: down-sampling, frame inside the crop
    (1, 700.0, 100.0, 80.0, 160.0, 0, 0, 1),         # wholly outside: a black crop
    (1, 33.3, 211.7, 140.2, 250.9, 0, 0, 1),
    (2, 10.0, 10.0, 400.0, 280.0, 0, 0, 1),
    (2, 150.0, 50.0, 60.0, 200.0, 0, 0, 1),
    (2, 380.0, 250.0, 100.0, 100.0, 0, 0, 1),        # partly outside, bottom right
    (2, 200.0, -1000.0, 50.0, 60.0, 0, 0, 1),        # wholly outside, far
    (0, 120.0, 60.0, 90.0, 210.0, 30, 0, 0),         # matrix / crop only
    (1, 250.0, 120.0, 160.0, 300.0, -30, 0, 0),
    (2, 100.0, 40.0, 200.0, 180.0, 17.5, 0, 0),
    (0, 120.0, 60.0, 90.0, 210.0, 0, 1, 0),          # HRNet matrices
    (1, -40.0, 300.0, 200.0, 260.0, -30, 1, 0),
    (2, 150.0, 50.0, 60.0, 200.0, 24, 1, 0),
]
CROP_CASES = [2, 12]                  # stored whole (uint8 [256,192,3]); every other crop as its CRC-32


def load_reference():
    ns = ref_import.load()
    for name in ("pycocotools", "pycocotools.coco", "json_tricks", "munkres"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                mod = types.ModuleType(name)
                mod.COCO = object
                sys.modules[name] = mod
    ns.COCODataset = importlib.import_module("datasets.COCO").COCODataset
    ns.get_warp_matrix = importlib.import_module("vit_utils.post_processing.post_transforms").get_warp_matrix
    ns.get_affine_transform = importlib.import_module("vit_utils.transform").get_affine_transform
    return ns


def crc(a: np.ndarray) -> int:
    return zlib.crc32(np.ascontiguousarray(a).tobytes())


def main() -> None:
    import cv2
    import torch
    from torchvision import transforms
    torch.set_grad_enabled(False)
    ns = load_reference()
    tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    ds = types.SimpleNamespace(aspect_ratio=192 * 1.0 / 256, pixel_std=200)
    frames = [P.make_frame(h, w, s) for h, w, s in FRAMES]
    image_size = np.array([192, 256])
    N = len(CASES)
    centers, scales, mats = np.zeros((N, 2), np.float32), np.zeros((N, 2), np.float32), np.zeros((N, 2, 3), np.float64)
    crcs, xs = np.zeros(N, np.uint32), []
    for i, (f, x, y, w, h, rot, builder, _) in enumerate(CASES):
        c, s = ns.COCODataset._xywh2cs(ds, x, y, w, h)
        c2, s2 = A.xywh2cs((x, y, w, h))
        assert c.dtype == c2.dtype == np.float32 and s.dtype == s2.dtype == np.float32
        assert np.array_equal(c, c2) and np.array_equal(s, s2), i
        if builder == 0:
            m = ns.get_warp_matrix(rot, c * 2.0, image_size - 1.0, s * 200.0)
            m2 = A.udp_matrix(c, s, rot)
        else:
            m = ns.get_affine_transform(c, s, 200, rot, (192, 256))
            m2 = A.hrnet_matrix(c, s, rot)
        assert m.dtype == m2.dtype and np.array_equal(m, m2), i
        img = cv2.warpAffine(frames[f], m, (192, 256), flags=cv2.INTER_LINEAR)
        assert np.array_equal(img, A.warp_affine_u8(frames[f], m)), i
        x_t = tf(img).numpy()
        assert x_t.dtype == np.float32 and np.array_equal(x_t, A.warp_normalise(frames[f], m)), i
        centers[i], scales[i], mats[i], crcs[i] = c, s, m, crc(img)
        xs.append(x_t)
    fwd = np.array([i for i, case in enumerate(CASES) if case[7]], np.int32)
    x = np.stack([xs[i] for i in fwd], 0)
    B, K = len(fwd), 17
    cs_px = np.concatenate([centers[fwd], scales[fwd] * 200.0], 1).astype(np.float32)
    D, depth, heads = O.MODEL_DIMS["b"]
    out = dict(meta=np.array([D, depth, heads, K, WSEED, FLIP_WSEED], np.int64), frames=np.array(FRAMES, np.int64),
               boxes=np.array([c[1:5] for c in CASES], np.float64), rot=np.array([c[5] for c in CASES], np.float64),
               builder=np.array([c[6] for c in CASES], np.int32), frame_id=np.array([c[0] for c in CASES], np.int32),
               centers=centers, scales=scales, mats=mats, crc=crcs, crop_ids=np.array(CROP_CASES, np.int32),
               crops=np.stack([cv2.warpAffine(frames[CASES[i][0]], mats[i], (192, 256), flags=cv2.INTER_LINEAR) for i in CROP_CASES]),
               fwd=fwd, cs_px=cs_px)
    rs = np.random.RandomState(5)
    sample_crops = np.sort(rs.choice(B, size=2, replace=False)).astype(np.int32)      # the fixture stays small: 2 x 4 maps
    sample_kps = np.sort(rs.choice(K, size=4, replace=False)).astype(np.int32)
    out.update(sample_crops=sample_crops, sample_kps=sample_kps)
    for tag, sd in (("plain", O.make_state_dict(D, depth, K, WSEED, peaky=0.1, bumps=True)),
                    ("flip", flip_symmetric_state_dict(D, depth, K, FLIP_WSEED, PAIRS))):
        model = ns.ViTPose(ns.dyn_model_import("coco", "b")).eval()
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        xt = torch.from_numpy(x)
        hm = model(xt).numpy()
        if tag == "flip":
            model.keypoint_head.test_cfg["shift_heatmap"] = False
            hm = ((hm + model.keypoint_head.inference_model(model.backbone(torch.flip(xt, [3])), PAIRS)) * 0.5).astype(np.float32)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            pts, prob = ns.keypoints_from_heatmaps(heatmaps=hm, center=cs_px[:, :2], scale=cs_px[:, 2:], unbiased=True, use_udp=True)
        kp = np.concatenate([pts[:, :, ::-1], prob], axis=2).astype(np.float32)
        out[f"kpts_{tag}"] = kp
        out[f"idx_{tag}"] = hm.reshape(B, K, -1).argmax(-1).astype(np.int32)
        out[f"range_{tag}"] = np.array([hm.min(), hm.max()], np.float32)
        out[f"map_sum_{tag}"] = hm.reshape(B, K, -1).sum(-1, dtype=np.float64)
        out[f"sample_hm_{tag}"] = hm[sample_crops][:, sample_kps]
        print(tag, "range", float(hm.min()), float(hm.max()), "visible", int((kp[..., 2] > 0.3).sum()), "/", kp[..., 2].size, flush=True)
    np.savez_compressed(OUT, **out)
    print("written", OUT, os.path.getsize(OUT), "bytes", flush=True)


if __name__ == "__main__":
    main()
