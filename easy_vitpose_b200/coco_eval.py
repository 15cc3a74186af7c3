"""COCO keypoint AP on the device: pycocotools' `COCOeval(cocoGt, cocoDt, 'keypoints')` evaluate, accumulate and summarize for
category 1 (OKS matching at maxDets 20, the 101-point precision, the ten summary numbers) over a whole evaluation set in one
`vpb_coco_eval` enqueue.  oracle/coco_oks_eval.py states the algorithm; the device equals it bit for bit wherever no OKS lies
within an ulp of a threshold or of another OKS it is compared with (CUDA's exp is not numpy's).

- `coco_eval_device(...)` takes device tensors and returns a `CocoEvalResult` of device tensors with no synchronisation;
  with `out=` and `workspace=` it can be captured in a CUDA graph.  `check(result)` raises on its status bits.
- `DeviceCocoEval(gt_annotations, image_ids, sigmas)` uploads the ground truth once; `add(results)` takes the result records
  `COCO.loadRes` takes, `add_device(...)` the engine's kept poses straight from device memory (e.g. what
  `B200PoseBackend.inference_topdown_eval(..., evaluator=)` passes), and `evaluate()` reads back only the ten numbers.
- `evaluate(gt_annotations, results, image_ids, sigmas)` is the host drop-in for the evaluate / accumulate / summarize calls.

Where pycocotools and a reader's expectations part:
- images are evaluated in ascending image id (COCOeval's `np.unique(imgIds)`), which decides ties among equal scores of
  different images; within an image, detections keep the order in which they were added;
- a ground truth's `ignore` field is overwritten by `iscrowd` in pycocotools' `_prepare`, so it is not read here;
- ground-truth ids must be non-zero: COCOeval stores a match as the ground truth's id, so an id of 0 reads as unmatched;
- detections of images outside `image_ids` or of another category are dropped by `add` and rejected by `add_device`.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np

from . import _lib

MAX_GTS = 256                         # VPB_COCO_MAX_GTS: ground truths per image
MAX_ROWS = 1024                       # VPB_COCO_MAX_ROWS: detection rows per image before the truncation to 20
MAX_K = 144                           # VPB_COCO_MAX_K
MAX_IMAGES = 1000000                  # VPB_COCO_MAX_IMAGES
STATUS_TOO_MANY_GTS = 1               # VPB_COCO_TOO_MANY_GTS
STATUS_TOO_MANY_ROWS = 2              # VPB_COCO_TOO_MANY_ROWS
STATUS_BAD_INPUT = 4                  # VPB_COCO_BAD_INPUT
STAT_NAMES = ("AP", "AP50", "AP75", "AP_medium", "AP_large", "AR", "AR50", "AR75", "AR_medium", "AR_large")

__all__ = ["CocoEvalResult", "coco_eval_device", "workspace_bytes", "check", "DeviceCocoEval", "evaluate", "pack_ground_truth",
           "pack_results", "STAT_NAMES"]


class CocoEvalResult(NamedTuple):
    """stats float64 [10] (STAT_NAMES order), precision float64 [3, 10, 101] (area all / medium / large, OKS threshold, recall
    threshold), recall float64 [3, 10], status int32 [1]."""
    stats: "object"
    precision: "object"
    recall: "object"
    status: "object"


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _check_tensor(name, t, dtype, shape, dev):
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and tuple(t.shape) == tuple(shape) and t.is_contiguous()
            and t.device == dev):
        raise ValueError(f"{name} must be a contiguous {dtype} {list(shape)} tensor on {dev}")


def _sigmas(sigmas, k):
    if sigmas is None:
        if k != 17:
            raise ValueError(f"{k} keypoints need sigmas (the default table is COCO's 17)")
        return None
    s = np.ascontiguousarray(np.asarray(sigmas, np.float64).reshape(-1))
    if s.size != k:
        raise ValueError(f"{s.size} sigmas for {k} keypoints")
    return s


def workspace_bytes(num_images: int, num_frames: int) -> int:
    """Bytes of device workspace coco_eval_device needs for this many images and detection frames."""
    b = _lib.lib().vpb_coco_eval_workspace_bytes(int(num_images), int(num_frames))
    if b < 0:
        raise ValueError(f"{num_images} images (1..{MAX_IMAGES}), {num_frames} frames")
    return b


def coco_eval_device(gt_offsets, gt_kpts, gt_area, gt_bbox, gt_iscrowd, gt_num_keypoints, dt_kpts, dt_scores, counts, frame_image,
                     keep=None, keep_counts=None, sigmas=None, workspace=None, out=None) -> CocoEvalResult:
    """COCOeval over I images in one enqueue on the current stream, no synchronisation.
    Ground truths, CSR by image in ascending image id: gt_offsets int32 [I + 1], gt_kpts float64 [G, K, 3] (x, y, v), gt_area
    float64 [G], gt_bbox float64 [G, 4] (x, y, w, h), gt_iscrowd and gt_num_keypoints int32 [G].
    Detections as frames: frame f holds the next counts[f] (int32 [F]) rows of dt_kpts float64 [n, K, 2] (x, y) and dt_scores
    float64 [n] and belongs to image index frame_image[f] (int32 [F], 0..I-1); keep / keep_counts (int32 [n] / [F]): the
    kept-row layout oks_nms_device writes, or None for every row.
    sigmas: K values, None = the COCO-17 table.  workspace: a uint8 CUDA tensor of at least workspace_bytes(I, F) bytes
    (allocated when None).  out: a CocoEvalResult of preallocated tensors (its status is OR-ed into, not cleared)."""
    import torch
    if not (isinstance(gt_offsets, torch.Tensor) and gt_offsets.dim() == 1 and gt_offsets.is_cuda):
        raise ValueError("gt_offsets must be a CUDA int32 [I + 1] tensor")
    dev = gt_offsets.device
    I = gt_offsets.shape[0] - 1
    if not 1 <= I <= MAX_IMAGES:
        raise ValueError(f"{I} images (1..{MAX_IMAGES})")
    if not (isinstance(gt_kpts, torch.Tensor) and gt_kpts.dim() == 3):
        raise ValueError("gt_kpts must be a CUDA float64 [G, K, 3] tensor")
    G, K = gt_kpts.shape[0], gt_kpts.shape[1]
    if not 1 <= K <= MAX_K:
        raise ValueError(f"{K} keypoints (1..{MAX_K})")
    _check_tensor("gt_offsets", gt_offsets, torch.int32, (I + 1,), dev)
    _check_tensor("gt_kpts", gt_kpts, torch.float64, (G, K, 3), dev)
    _check_tensor("gt_area", gt_area, torch.float64, (G,), dev)
    _check_tensor("gt_bbox", gt_bbox, torch.float64, (G, 4), dev)
    _check_tensor("gt_iscrowd", gt_iscrowd, torch.int32, (G,), dev)
    _check_tensor("gt_num_keypoints", gt_num_keypoints, torch.int32, (G,), dev)
    if not (isinstance(dt_kpts, torch.Tensor) and dt_kpts.dim() == 3):
        raise ValueError("dt_kpts must be a CUDA float64 [n, K, 2] tensor")
    n = dt_kpts.shape[0]
    if not (isinstance(counts, torch.Tensor) and counts.dim() == 1):
        raise ValueError("counts must be a CUDA int32 [F] tensor")
    F = counts.shape[0]
    _check_tensor("dt_kpts", dt_kpts, torch.float64, (n, K, 2), dev)
    _check_tensor("dt_scores", dt_scores, torch.float64, (n,), dev)
    _check_tensor("counts", counts, torch.int32, (F,), dev)
    _check_tensor("frame_image", frame_image, torch.int32, (F,), dev)
    if (keep is None) != (keep_counts is None):
        raise ValueError("keep and keep_counts go together")
    if keep is not None:
        _check_tensor("keep", keep, torch.int32, (n,), dev)
        _check_tensor("keep_counts", keep_counts, torch.int32, (F,), dev)
    sig = _sigmas(sigmas, K)
    need = workspace_bytes(I, F)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.uint8, device=dev)
    elif not (isinstance(workspace, torch.Tensor) and workspace.is_cuda and workspace.device == dev and workspace.is_contiguous()
              and workspace.numel() * workspace.element_size() >= need and workspace.data_ptr() % 256 == 0):
        raise ValueError(f"workspace must be a contiguous 256-byte aligned CUDA tensor of at least {need} bytes on {dev}")
    if out is None:
        out = CocoEvalResult(torch.empty(10, dtype=torch.float64, device=dev), torch.empty((3, 10, 101), dtype=torch.float64, device=dev),
                             torch.empty((3, 10), dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
    else:
        out = CocoEvalResult(*out)
        _check_tensor("out.stats", out.stats, torch.float64, (10,), dev)
        _check_tensor("out.precision", out.precision, torch.float64, (3, 10, 101), dev)
        _check_tensor("out.recall", out.recall, torch.float64, (3, 10), dev)
        _check_tensor("out.status", out.status, torch.int32, (1,), dev)
    gts = _lib.VpbCocoGts(_ptr(gt_offsets), _ptr(gt_kpts), _ptr(gt_area), _ptr(gt_bbox), _ptr(gt_iscrowd), _ptr(gt_num_keypoints), I, G)
    dts = _lib.VpbCocoDets(_ptr(dt_kpts), _ptr(dt_scores), _ptr(counts), _ptr(frame_image), _ptr(keep), _ptr(keep_counts), n, F)
    with torch.cuda.device(dev):
        _lib.check_value(_lib.lib().vpb_coco_eval(
            K, None if sig is None else sig.ctypes.data_as(C.c_void_p), C.byref(gts), C.byref(dts), _ptr(workspace),
            workspace.numel() * workspace.element_size(), _ptr(out.stats), _ptr(out.precision), _ptr(out.recall), _ptr(out.status),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out


def check(result) -> None:
    """Raises ValueError if the call that wrote `result` (a CocoEvalResult, its status tensor or the status value) met an image
    over a limit or malformed input; its stats are then NaN.  Synchronises on a device status."""
    st = result.status if isinstance(result, CocoEvalResult) else result
    st = int(st.item()) if hasattr(st, "item") else int(st)
    if st:
        why = []
        if st & STATUS_TOO_MANY_GTS:
            why.append(f"an image has more than {MAX_GTS} ground truths")
        if st & STATUS_TOO_MANY_ROWS:
            why.append(f"an image has more than {MAX_ROWS} detections")
        if st & STATUS_BAD_INPUT:
            why.append("a frame's count, keep list or image index is out of range, or the ground-truth offsets are out of order")
        raise ValueError("COCO evaluation refused its input: " + "; ".join(why))


def pack_ground_truth(gt_annotations, index: dict, K: int) -> dict:
    """The ground-truth arrays vpb_coco_eval reads (numpy): annotations of category 1 whose image is a key of `index` (image id
    -> position in ascending id order), stably ordered by that position, as CSR offsets int32 [I + 1], kpts float64 [G, K, 3],
    area, bbox [G, 4], iscrowd and num_keypoints int32 (absent: 0 and 1, as the oracle reads them)."""
    gts = [g for g in gt_annotations if g.get("category_id", 1) == 1 and int(g["image_id"]) in index]
    img = np.array([index[int(g["image_id"])] for g in gts], np.int64)
    gts = [gts[j] for j in np.argsort(img, kind="stable")]
    G = len(gts)
    kp = np.zeros((G, 3 * K), np.float64)
    for j, g in enumerate(gts):
        v = np.asarray(g["keypoints"], np.float64).reshape(-1)
        if v.size != 3 * K:
            raise ValueError(f"ground-truth keypoints of {v.size} values for {K} keypoints")
        kp[j] = v
    return {"offsets": np.concatenate([[0], np.cumsum(np.bincount(img, minlength=len(index)))]).astype(np.int32),
            "kpts": kp.reshape(G, K, 3), "area": np.array([float(g["area"]) for g in gts], np.float64),
            "bbox": np.array([np.asarray(g["bbox"], np.float64).reshape(4) for g in gts], np.float64).reshape(G, 4),
            "iscrowd": np.array([int(g.get("iscrowd", 0)) for g in gts], np.int32),
            "num_keypoints": np.array([int(g.get("num_keypoints", 1)) for g in gts], np.int32)}


def pack_results(results, index: dict, K: int) -> dict:
    """Result records as detection frames (numpy): records of category 1 whose image is a key of `index`, one frame per image
    in ascending position, each frame's records in list order -> kpts float64 [n, K, 2] (x, y), scores float64 [n], counts and
    frame_image (the image's position) int32 [F], keep int32 [n] (every row of each frame, in order)."""
    recs = [r for r in results if r.get("category_id", 1) == 1 and int(r["image_id"]) in index]
    n = len(recs)
    kp = np.zeros((n, 3 * K), np.float64)
    for j, r in enumerate(recs):
        v = np.asarray(r["keypoints"], np.float64).reshape(-1)
        if v.size != 3 * K:
            raise ValueError(f"result keypoints of {v.size} values for {K} keypoints")
        kp[j] = v
    img = np.array([index[int(r["image_id"])] for r in recs], np.int64)
    order = np.argsort(img, kind="stable")
    frames, counts = np.unique(img, return_counts=True)
    return {"kpts": np.ascontiguousarray(kp.reshape(n, K, 3)[order][..., :2]),
            "scores": np.array([float(recs[j]["score"]) for j in order], np.float64),
            "counts": counts.astype(np.int32), "frame_image": frames.astype(np.int32),
            "keep": (np.arange(n) - np.repeat(np.cumsum(counts) - counts, counts)).astype(np.int32)}


class DeviceCocoEval:
    """COCOeval for one ground-truth set whose detections accumulate on the device.  gt_annotations: COCO annotation dicts
    (image_id, id, keypoints [3K], area, bbox, iscrowd, num_keypoints, category_id; those of other categories or images are
    left out); image_ids: the images evaluated (cocoGt.getImgIds(), or a subset); sigmas: K values, None = COCO's 17."""

    def __init__(self, gt_annotations, image_ids, sigmas=None, device=None):
        import torch
        ids = np.unique(np.asarray(list(image_ids), np.int64))
        if not 1 <= len(ids) <= MAX_IMAGES:
            raise ValueError(f"{len(ids)} images (1..{MAX_IMAGES})")
        self.image_ids = ids
        self._index = {int(v): i for i, v in enumerate(ids)}
        gts = [g for g in gt_annotations if g.get("category_id", 1) == 1 and int(g["image_id"]) in self._index]
        if any(g.get("id", 1) == 0 for g in gts):
            raise ValueError("ground-truth ids must be non-zero (COCOeval reads a match to id 0 as no match)")
        if sigmas is not None:
            K = len(np.asarray(sigmas).reshape(-1))
        elif gts:
            K = len(gts[0]["keypoints"]) // 3
        else:
            K = 17
        self.k = K
        self.sigmas = _sigmas(sigmas, K)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        p = pack_ground_truth(gts, self._index, K)
        G, I = len(p["area"]), len(ids)
        d = torch.from_numpy(np.concatenate([p["kpts"].reshape(-1), p["area"], p["bbox"].reshape(-1)])).to(self.device)
        w = torch.from_numpy(np.concatenate([p["offsets"], p["iscrowd"], p["num_keypoints"]])).to(self.device)
        nk = G * K * 3
        self._gt = (w[:I + 1], d[:nk].view(G, K, 3), d[nk:nk + G], d[nk + G:].view(G, 4), w[I + 1:I + 1 + G], w[I + 1 + G:])
        self._chunks = []

    def add(self, results) -> None:
        """Appends result records ({image_id, category_id, keypoints [x, y, v] * K, score}, what COCO.loadRes takes); records of
        other images or categories are dropped, as COCOeval drops them."""
        import torch
        p = pack_results(results, self._index, self.k)
        n, F, K = len(p["scores"]), len(p["counts"]), self.k
        if n == 0:
            return
        d = torch.from_numpy(np.concatenate([p["kpts"].reshape(-1), p["scores"]])).to(self.device)
        w = torch.from_numpy(np.concatenate([p["counts"], p["frame_image"], p["keep"], p["counts"]])).to(self.device)
        self._chunks.append((d[:n * K * 2].view(n, K, 2), d[n * K * 2:], w[:F], w[F:2 * F], w[2 * F:2 * F + n], w[2 * F + n:], None))

    def add_device(self, kpts, scores, counts, image_ids, keep=None, keep_counts=None) -> None:
        """Appends detections from device memory without a synchronisation: kpts CUDA float32 [n, K, 3] (y, x, score, the
        engine's rows), scores CUDA float64 [n], counts CUDA int32 [F] (frame f holds the next counts[f] rows; they must add up
        to n), image_ids the F frames' image ids (host; an id outside the evaluated images raises), keep / keep_counts the
        kept-row layout oks_nms_device writes (None: every row).  The rows are copied, so the caller may reuse its buffers."""
        import torch
        dev = self.device
        if not (isinstance(kpts, torch.Tensor) and kpts.dim() == 3 and kpts.shape[1:] == (self.k, 3)):
            raise ValueError(f"kpts must be a CUDA float32 [n, {self.k}, 3] tensor")
        n = kpts.shape[0]
        _check_tensor("kpts", kpts.contiguous(), torch.float32, (n, self.k, 3), dev)
        if not (isinstance(counts, torch.Tensor) and counts.dim() == 1):
            raise ValueError("counts must be a CUDA int32 [F] tensor")
        F = counts.shape[0]
        _check_tensor("scores", scores, torch.float64, (n,), dev)
        _check_tensor("counts", counts, torch.int32, (F,), dev)
        ids = [int(v) for v in np.asarray(image_ids).reshape(-1)]
        if len(ids) != F:
            raise ValueError(f"{len(ids)} image ids for {F} frames")
        unknown = [v for v in ids if v not in self._index]
        if unknown:
            raise ValueError(f"image ids {unknown[:5]} are not among the evaluated images")
        if (keep is None) != (keep_counts is None):
            raise ValueError("keep and keep_counts go together")
        xy = torch.stack((kpts[..., 1], kpts[..., 0]), -1).to(torch.float64).contiguous()
        fimg = torch.tensor([self._index[v] for v in ids], dtype=torch.int32).to(dev)
        cnt = counts.clone()
        # a frame table that does not add up to n would shift every later chunk's rows: checked on the device, at evaluate()
        bad = (cnt.clamp(min=0).sum() != n).to(torch.int32) * STATUS_BAD_INPUT
        if keep is None:                                      # every row of each frame, in order
            ends = torch.cumsum(cnt.clamp(min=0).to(torch.int64), 0)
            rows = torch.arange(n, dtype=torch.int64, device=dev)
            f = torch.searchsorted(ends, rows, right=True).clamp(max=max(F - 1, 0))
            local = (rows - (ends - cnt.clamp(min=0).to(torch.int64))[f] if F else rows).to(torch.int32)
            kc = cnt.clone()
        else:
            _check_tensor("keep", keep, torch.int32, (n,), dev)
            _check_tensor("keep_counts", keep_counts, torch.int32, (F,), dev)
            local, kc = keep.clone(), keep_counts.clone()
        self._chunks.append((xy, scores.clone(), cnt, fimg, local, kc, bad))

    def evaluate_device(self, workspace=None, out=None) -> CocoEvalResult:
        """Everything added so far, evaluated on the device with no synchronisation."""
        import torch
        dev, K = self.device, self.k
        ch = self._chunks
        if ch:
            cat = [torch.cat([c[j] for c in ch]) for j in range(6)]
        else:
            e32 = torch.zeros(0, dtype=torch.int32, device=dev)
            cat = [torch.zeros((0, K, 2), dtype=torch.float64, device=dev), torch.zeros(0, dtype=torch.float64, device=dev)] + [e32] * 4
        if out is None:
            out = CocoEvalResult(torch.empty(10, dtype=torch.float64, device=dev), torch.empty((3, 10, 101), dtype=torch.float64, device=dev),
                                 torch.empty((3, 10), dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        for c in ch:
            if c[6] is not None:
                out.status.bitwise_or_(c[6])
        return coco_eval_device(*self._gt, cat[0], cat[1], cat[2], cat[3], cat[4], cat[5], sigmas=self.sigmas, workspace=workspace, out=out)

    def evaluate(self) -> dict:
        """The ten summary numbers under the oracle's names (floats), plus "precision" [3, 10, 101] and "recall" [3, 10] as
        device tensors.  Reads back only the stats and the status; raises ValueError on a status bit."""
        import torch
        res = self.evaluate_device()
        h = torch.cat([res.stats, res.status.to(torch.float64)]).cpu().numpy()
        check(int(h[10]))
        out = {k: float(v) for k, v in zip(STAT_NAMES, h[:10])}
        out["precision"], out["recall"] = res.precision, res.recall
        return out


def evaluate(gt_annotations, results, image_ids, sigmas=None, device=None) -> dict:
    """Host drop-in for COCOeval(cocoGt, cocoGt.loadRes(results), 'keypoints').evaluate(); accumulate(); summarize() for category
    1 (and for oracle/coco_oks_eval.evaluate): the ten summary numbers under their usual names."""
    ev = DeviceCocoEval(gt_annotations, image_ids, sigmas, device)
    ev.add(results)
    r = ev.evaluate()
    return {k: r[k] for k in STAT_NAMES}
