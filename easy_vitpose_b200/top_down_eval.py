"""keypoints_from_heatmaps on the GPU (the branch VitInference takes), same call shape as the
reference function at easy_ViTPose/vit_utils/top_down_eval.py:493-641.

`decode_heatmaps` is the fast form of the branch VitInference takes (unbiased=True, use_udp=True: DARK/UDP with
centre = scale // 2, easy_ViTPose/inference.py:200-203).  `keypoints_from_heatmaps` covers every GaussianHeatmap
branch of the reference function (SURVEY.md section 8 row f4) with general centre / scale; `decode_topdown` is
TopdownHeatmapBaseHead.decode on top of it, including modulation kernels 1..35 and target_type='CombinedTarget'.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

__all__ = ["keypoints_from_heatmaps", "decode_heatmaps", "decode_topdown"]


def decode_heatmaps(heatmaps: torch.Tensor, org_wh: torch.Tensor, wrap_batch: bool = False):
    """heatmaps f32 CUDA [N,K,64,48], org_wh i32 [N,2] (crop width,height) -> (kpts [N,K,3] rows (y,x,score), idx [N,K])."""
    if not heatmaps.is_cuda:
        raise RuntimeError("decode_heatmaps needs a CUDA tensor: there is no CPU path")
    if heatmaps.dim() != 4 or tuple(heatmaps.shape[2:]) != (64, 48):
        raise ValueError(f"expected [N,K,64,48], got {tuple(heatmaps.shape)}")
    hm = heatmaps.to(torch.float32).contiguous()
    N, K = hm.shape[:2]
    org = torch.as_tensor(org_wh).to(device=hm.device, dtype=torch.int32).contiguous()
    if tuple(org.shape) != (N, 2):
        raise ValueError(f"org_wh must be [N,2], got {tuple(org.shape)}")
    kp = torch.empty((N, K, 3), dtype=torch.float32, device=hm.device)
    idx = torch.empty((N, K), dtype=torch.int32, device=hm.device)
    with torch.cuda.device(hm.device):
        st = C.c_void_p(torch.cuda.current_stream(hm.device).cuda_stream)
        _lib.check(_lib.lib().vpb_decode(C.c_void_p(hm.data_ptr()), N, K, C.c_void_p(org.data_ptr()), C.c_void_p(kp.data_ptr()),
                                         C.c_void_p(idx.data_ptr()), 1 if wrap_batch else 0, st))
    return kp, idx


_MODES = {None: 0, "default": 1, "unbiased": 2, "megvii": 3}


def _centre_scale(center, scale, n: int, device):
    """-> (cs32 | None, cs64 | None): [n,4] (cx, cy, sx, sy) in the dtype numpy's transform_preds arithmetic would run in
    (numpy >= 2: two float32 arrays stay float32; int64 / float64 promote to float64)."""
    center = np.asarray(center); scale = np.asarray(scale)
    if center.shape != (n, 2) or scale.shape != (n, 2):
        raise ValueError("center and scale must be [N,2]")
    if center.dtype == np.float32 and scale.dtype == np.float32:
        return torch.from_numpy(np.ascontiguousarray(np.concatenate([center, scale], 1))).to(device), None
    cs = np.concatenate([center.astype(np.float64), scale.astype(np.float64)], 1)
    return None, torch.from_numpy(np.ascontiguousarray(cs)).to(device)


def keypoints_from_heatmaps(heatmaps, center, scale, unbiased=False, post_process="default", kernel=11,
                            valid_radius_factor=0.0546875, use_udp=False, target_type="GaussianHeatmap", return_idx=False):
    """Reference signature and semantics (vit_utils/top_down_eval.py:493-641) on the GPU; returns
    (preds [N,K,2] (x,y) float32, maxvals [N,K,1] float32) as numpy arrays.  `heatmaps` may be a numpy array or a CUDA tensor
    [N,K,64,48] and is never modified (the reference works on a copy, :545).

    Every branch is built: post_process None / 'default' / 'unbiased' / 'megvii' with use_udp=False, the DARK/UDP branch
    (use_udp=True; the one VitInference.postprocess takes) and use_udp=True with target_type='CombinedTarget' (:580-593, heatmaps
    [N,3K,64,48] -> K keypoints).  `kernel` is any odd size 1..35 (cv2's fixed tables below 11, its small-kernel summation order
    for 3 and 5 taps and the scalar tail of its column filter for 5 and 7 are reproduced bit for bit); CombinedTarget blurs the
    response maps with 2*kernel+1, so kernel <= 17 there; kernel = 1 with post_process 'unbiased' / 'megvii' raises ValueError as
    the reference's `_gaussian_blur` does (a zero-width border, :453).  Like the reference, CombinedTarget only accepts N = 1: its
    index arithmetic (:589) does not broadcast for larger N.  Also like the reference, use_udp=True on one-keypoint maps
    [N,1,64,48] raises ValueError for N > 1 (post_dark_udp's squeeze, :414); vpb_decode_modes mode 4 and the engine's affine
    calls decode that case with the formula's intended shape."""
    # the reference's conflict checks (:548-553) and config normalisation (:556-579), deprecation warnings dropped
    if unbiased:
        assert post_process not in [False, None, "megvii"]
    if post_process in ["megvii", "unbiased"]:
        assert kernel > 0
    if use_udp:
        assert not post_process == "megvii"
    if post_process is False:
        post_process = None
    elif post_process is True:
        post_process = "unbiased" if unbiased is True else "default"
    elif post_process == "default" and unbiased is True:
        post_process = "unbiased"
    combined = bool(use_udp) and str(target_type).lower() == "combinedtarget"
    if use_udp and not combined and str(target_type).lower() != "gaussianheatmap":
        raise ValueError("target_type should be either 'GaussianHeatmap' or 'CombinedTarget'")
    if post_process not in _MODES:
        raise ValueError(f"unknown post_process {post_process!r}")
    blurs = use_udp or post_process in ("unbiased", "megvii")
    if blurs and (int(kernel) != kernel or kernel % 2 == 0 or not 1 <= kernel <= (17 if combined else 35)):
        raise NotImplementedError(f"modulation kernel {kernel}: odd sizes 1..{17 if combined else 35} are built")
    if kernel == 1 and not use_udp and post_process in ("unbiased", "megvii"):
        raise ValueError("could not broadcast input array from shape (64,48) into shape (0,0)")       # the reference's :453 with border = 0

    if len(heatmaps.shape) != 4 or tuple(heatmaps.shape[2:]) != (64, 48):
        raise ValueError(f"expected [N,K,64,48], got {tuple(heatmaps.shape)}")
    N, K = (int(v) for v in heatmaps.shape[:2])
    valid_radius = 0.0
    if combined:
        if N != 1 or K % 3:
            # the reference adds an arange of N*K/3 plane offsets to an [N, K/3] index array (:589) and reshapes to K // 3 (:590)
            raise ValueError(f"CombinedTarget: operands could not be broadcast together for N={N}, K={K} (reference :589-590)")
        K //= 3
        valid_radius = float(np.float32(valid_radius_factor * heatmaps.shape[2]))
    elif use_udp and N > 1 and K == 1:
        # post_dark_udp's `.squeeze()` (:414) drops the K = 1 axis of its [N, 1, 2] offsets, which then do not broadcast
        raise ValueError(f"use_udp with one keypoint: non-broadcastable output operand for N={N}, K=1 (reference :414)")
    hm = heatmaps if isinstance(heatmaps, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(heatmaps, np.float32))
    if not hm.is_cuda:
        hm = hm.cuda()
    hm = hm.to(torch.float32).contiguous()
    cs32, cs64 = _centre_scale(center, scale, N, hm.device)
    kp = torch.empty((N, K, 3), dtype=torch.float32, device=hm.device)
    idx = torch.empty((N, K), dtype=torch.int32, device=hm.device)
    mode = (5 if combined else 4) if use_udp else _MODES[post_process]
    with torch.cuda.device(hm.device):
        st = C.c_void_p(torch.cuda.current_stream(hm.device).cuda_stream)
        _lib.check(_lib.lib().vpb_decode_modes_ex(C.c_void_p(hm.data_ptr()), N, K, mode, int(kernel) if blurs else 11, valid_radius,
                                                  C.c_void_p(cs32.data_ptr()) if cs32 is not None else None,
                                                  C.c_void_p(cs64.data_ptr()) if cs64 is not None else None,
                                                  C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), st))
    kp = kp.cpu().numpy()
    out = (np.ascontiguousarray(kp[:, :, 1::-1]), kp[:, :, 2:3].copy())
    return out + (idx.cpu().numpy(),) if return_idx else out


def decode_topdown(img_metas, output, test_cfg: "dict | None" = None) -> dict:
    """TopdownHeatmapBaseHead.decode (vit_models/head/topdown_heatmap_base_head.py:40-103): per-image centre / scale /
    bbox score from `img_metas`, keypoints_from_heatmaps configured by `test_cfg` (configs/ViTPose_common.py:123-129), and the
    mmpose result dict: preds [N,K,3] (x, y, score), boxes [N,6] (centre, scale, area = prod(scale * 200), score),
    image_paths, bbox_ids."""
    cfg = test_cfg or {}
    n = len(img_metas)
    c = np.zeros((n, 2), np.float32); s = np.zeros((n, 2), np.float32)
    score = np.ones(n)
    for i, meta in enumerate(img_metas):
        c[i, :] = meta["center"]; s[i, :] = meta["scale"]
        if "bbox_score" in meta:
            score[i] = np.array(meta["bbox_score"]).reshape(-1)[0]
    preds, maxvals = keypoints_from_heatmaps(
        output, c, s, unbiased=cfg.get("unbiased_decoding", False), post_process=cfg.get("post_process", "default"),
        kernel=cfg.get("modulate_kernel", 11), valid_radius_factor=cfg.get("valid_radius_factor", 0.0546875),
        use_udp=cfg.get("use_udp", False), target_type=cfg.get("target_type", "GaussianHeatmap"))
    all_preds = np.zeros((n, preds.shape[1], 3), np.float32)
    all_preds[:, :, 0:2] = preds; all_preds[:, :, 2:3] = maxvals
    boxes = np.zeros((n, 6), np.float32)
    boxes[:, 0:2] = c; boxes[:, 2:4] = s; boxes[:, 4] = np.prod(s * 200.0, axis=1); boxes[:, 5] = score
    return {"preds": all_preds, "boxes": boxes, "image_paths": [m["image_file"] for m in img_metas],
            "bbox_ids": [m["bbox_id"] for m in img_metas] if n and "bbox_id" in img_metas[0] else None}
