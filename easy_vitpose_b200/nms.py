"""OKS NMS on the device: the reference's `oks_iou`, `oks_nms` and `soft_oks_nms` (vit_utils/post_processing/nms.py) for
many frames in one `vpb_oks_nms` launch, with HRNet's evaluation rescoring (box score x mean keypoint score above
`in_vis_thr`) as an option.  oracle/oks_nms_oracle.py states the contract.

`oks_nms_device(kpts, counts, areas, scores, thr, ...)` takes the concatenated tensors `infer_frames` / `infer_affine` return
and keeps everything on the device (no synchronisation); `check(result)` raises on its status bits.  `oks_nms` and
`soft_oks_nms` are host drop-ins with the reference's signatures and return values (exact for float32 keypoints, float64 or
Python-float scores and Python-float thresholds; see their docstrings); `oks_nms_frames` is the batched host form, one array
per frame.  Ties among equal scores follow the reference's `scores.argsort()[::-1]` evaluated with a stable
argsort (later index first); the reference's own default sort is unstable there.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import numpy as np

from . import _lib

MAX_PEOPLE = 256                      # VPB_NMS_MAX_PEOPLE: people per frame
MAX_K = 144                           # VPB_NMS_MAX_K
MAX_DETS = 256                        # VPB_NMS_MAX_DETS: soft NMS's max_dets
STATUS_TOO_MANY_PEOPLE = 1            # VPB_NMS_TOO_MANY_PEOPLE: a frame with more than MAX_PEOPLE people
STATUS_BAD_ROWS = 2                   # VPB_NMS_BAD_ROWS: a negative count, or a frame's rows run past the keypoints

__all__ = ["OksNmsResult", "oks_nms_device", "oks_iou_device", "check", "oks_nms", "soft_oks_nms", "oks_nms_frames"]


class OksNmsResult(NamedTuple):
    """keep int32 [n]: over each frame's rows its kept frame-local indices in the reference's order, then -1;
    keep_counts int32 [F]; scores float64 [n]: the score each row was sorted by (rescored when asked); status int32 [1]."""
    keep: "object"
    keep_counts: "object"
    scores: "object"
    status: "object"


def _nan(v):
    return math.nan if v is None else float(v)


def _sigmas(sigmas, k):
    if sigmas is None:
        if k != 17:
            raise ValueError(f"{k} keypoints need sigmas (the default table is COCO's 17)")
        return None
    s = np.ascontiguousarray(np.asarray(sigmas, np.float64).reshape(-1))
    if s.size != k:
        raise ValueError(f"{s.size} sigmas for {k} keypoints")
    return s


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(dev):
    import torch
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _check_tensor(name, t, dtype, shape, dev):
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and tuple(t.shape) == tuple(shape) and t.is_contiguous()
            and t.device == dev):
        raise ValueError(f"{name} must be a contiguous {dtype} {list(shape)} tensor on {dev}")


def _inputs(kpts, counts, areas, scores):
    import torch
    if not (isinstance(kpts, torch.Tensor) and kpts.dim() == 3 and kpts.is_cuda):
        raise ValueError("kpts must be a CUDA float32 [n, K, 3] tensor")
    n, k = kpts.shape[0], kpts.shape[1]
    if not 1 <= k <= MAX_K:
        raise ValueError(f"{k} keypoints (1..{MAX_K})")
    dev = kpts.device
    _check_tensor("kpts", kpts, torch.float32, (n, k, 3), dev)
    if not (isinstance(counts, torch.Tensor) and counts.dim() == 1):
        raise ValueError("counts must be a CUDA int32 [F] tensor")
    _check_tensor("counts", counts, torch.int32, (counts.shape[0],), dev)
    _check_tensor("areas", areas, torch.float64, (n,), dev)
    if scores is not None:
        _check_tensor("scores", scores, torch.float64, (n,), dev)
    return n, k, counts.shape[0], dev


def oks_nms_device(kpts, counts, areas, scores, thr, sigmas=None, vis_thr=None, soft=False, max_dets=20, rescore_vis_thr=None,
                   out=None) -> OksNmsResult:
    """OKS NMS of F frames in one launch.  kpts CUDA float32 [n, K, 3] (y, x, score; the reference's (x, y, score) gives the
    same result), the rows of every frame concatenated, frame f holding the next counts[f] (CUDA int32 [F]); areas and scores
    CUDA float64 [n].  thr, sigmas (K values; None = the COCO-17 table), vis_thr (None = every keypoint) and max_dets as the
    reference's oks_nms / soft_oks_nms (soft=True) take them.  rescore_vis_thr: HRNet's in_vis_thr; the scores are then box
    scores and each becomes box x mean keypoint score above it before the sort.  `out`: an OksNmsResult of preallocated
    tensors to write (needed to capture the call in a CUDA graph); its status is OR-ed into, not cleared.  Enqueued on the
    current stream with no synchronisation."""
    import torch
    n, k, F, dev = _inputs(kpts, counts, areas, scores)
    sig = _sigmas(sigmas, k)
    if soft and not 0 <= int(max_dets) <= MAX_DETS:
        raise ValueError(f"max_dets {max_dets} (0..{MAX_DETS})")
    if out is None:
        out = OksNmsResult(torch.empty(n, dtype=torch.int32, device=dev), torch.empty(F, dtype=torch.int32, device=dev),
                           torch.empty(n, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
    else:
        out = OksNmsResult(*out)
        _check_tensor("out.keep", out.keep, torch.int32, (n,), dev)
        _check_tensor("out.keep_counts", out.keep_counts, torch.int32, (F,), dev)
        _check_tensor("out.scores", out.scores, torch.float64, (n,), dev)
        _check_tensor("out.status", out.status, torch.int32, (1,), dev)
    p = _lib.VpbOksNmsParams(float(thr), _nan(vis_thr), _nan(rescore_vis_thr), 1 if soft else 0, int(max_dets))
    with torch.cuda.device(dev):
        _lib.check_value(_lib.lib().vpb_oks_nms(
            _ptr(kpts), n, k, _ptr(counts), F, _ptr(areas), _ptr(scores), None if sig is None else sig.ctypes.data_as(C.c_void_p),
            C.byref(p), _ptr(out.keep), _ptr(out.keep_counts), _ptr(out.scores), _ptr(out.status), _stream(dev)))
    return out


def oks_iou_device(kpts, counts, areas, sigmas=None, vis_thr=None):
    """Every frame's OKS matrix on the device -> (oks float32 [n, MAX_PEOPLE], status int32 [1]): row r (frame f's row i),
    column j < counts[f] = the reference's oks_iou(g = person i, d = person j).  Other columns are NaN."""
    import torch
    n, k, F, dev = _inputs(kpts, counts, areas, None)
    sig = _sigmas(sigmas, k)
    oks = torch.full((n, MAX_PEOPLE), float("nan"), dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check_value(_lib.lib().vpb_oks_iou(
            _ptr(kpts), n, k, _ptr(counts), F, _ptr(areas), None if sig is None else sig.ctypes.data_as(C.c_void_p), _nan(vis_thr),
            _ptr(oks), _ptr(status), _stream(dev)))
    return oks, status


def check(result) -> None:
    """Raises ValueError if a frame of the call that wrote `result` (an OksNmsResult, its status tensor or the status value)
    was skipped.  Synchronises on a device status."""
    st = result.status if isinstance(result, OksNmsResult) else result
    st = int(st.item()) if hasattr(st, "item") else int(st)
    if st:
        why = []
        if st & STATUS_TOO_MANY_PEOPLE:
            why.append(f"a frame has more than {MAX_PEOPLE} people")
        if st & STATUS_BAD_ROWS:
            why.append("a frame's count is negative or its rows run past the keypoints")
        raise ValueError("OKS NMS skipped a frame: " + "; ".join(why))


# ------------------------------------------------------------------------------------------------------------- host forms
def oks_nms_frames(kpts_list, areas_list, scores_list, thr, sigmas=None, vis_thr=None, soft=False, max_dets=20,
                   rescore_vis_thr=None, device=None, return_scores=False):
    """Batched host form: per frame keypoints [n_f, K, 3] (taken as float32), areas [n_f] and scores [n_f] (float64) -> per
    frame the kept indices (int64), in one upload, one launch and one read-back; with return_scores also per frame the
    float64 scores the sort used.  A frame over a limit raises ValueError."""
    import torch
    F = len(kpts_list)
    if len(areas_list) != F or len(scores_list) != F:
        raise ValueError(f"{F} keypoint arrays, {len(areas_list)} area arrays, {len(scores_list)} score arrays")
    kps = [np.asarray(k, np.float32) for k in kpts_list]
    K = next((k.shape[1] for k in kps if k.ndim == 3 and k.shape[0]), None)
    if K is None:
        K = len(sigmas) if sigmas is not None else 17
    for f, k in enumerate(kps):
        if k.size == 0:
            kps[f] = k.reshape(0, K, 3)
        elif k.ndim != 3 or k.shape[1:] != (K, 3):
            raise ValueError(f"frame {f}: keypoints must be [n, {K}, 3], not {list(k.shape)}")
        if len(kps[f]) > MAX_PEOPLE:
            raise ValueError(f"frame {f}: {len(kps[f])} people (at most {MAX_PEOPLE})")
    counts = [len(k) for k in kps]
    ar = [np.asarray(a, np.float64).reshape(-1) for a in areas_list]
    sc = [np.asarray(s, np.float64).reshape(-1) for s in scores_list]
    for f in range(F):
        if len(ar[f]) != counts[f] or len(sc[f]) != counts[f]:
            raise ValueError(f"frame {f}: {counts[f]} people, {len(ar[f])} areas, {len(sc[f])} scores")
    if F == 0:
        return ([], []) if return_scores else []
    n = sum(counts)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    # one upload: areas f64 [n] | scores f64 [n] | kpts f32 [n, K, 3] | counts i32 [F] (as float64 words)
    nk = n * K * 3
    buf = np.zeros(2 * n + (nk + F + 1) // 2, np.float64)
    buf[:n] = np.concatenate(ar) if n else []
    buf[n:2 * n] = np.concatenate(sc) if n else []
    words = buf[2 * n:].view(np.int32)
    words[:nk].view(np.float32)[:] = np.concatenate(kps).reshape(-1) if n else []
    words[nk:nk + F] = counts
    d = torch.from_numpy(buf).to(dev)
    dw = d[2 * n:].view(torch.int32)
    kp = dw[:nk].view(torch.float32).view(n, K, 3)
    res = oks_nms_device(kp, dw[nk:nk + F], d[:n], d[n:2 * n], thr, sigmas, vis_thr, soft, max_dets, rescore_vis_thr)
    # one read-back: scores f64 [n] | keep i32 [n] | keep_counts i32 [F] | status i32 [1]
    back = torch.empty(n + (n + F + 2) // 2, dtype=torch.float64, device=dev)
    back[:n] = res.scores
    bw = back[n:].view(torch.int32)
    bw[:n] = res.keep
    bw[n:n + F] = res.keep_counts
    bw[n + F] = res.status[0]
    h = back.cpu().numpy()
    hw = h[n:].view(np.int32)
    check(hw[n + F])
    offs = np.cumsum([0] + counts)
    keep = [hw[offs[f]:offs[f] + hw[n + f]].astype(np.int64) for f in range(F)]
    if return_scores:
        return keep, [h[offs[f]:offs[f + 1]].copy() for f in range(F)]
    return keep


def _db_arrays(kpts_db, score_per_joint):
    if score_per_joint:
        scores = np.array([k["score"].mean() for k in kpts_db])         # per-joint means computed with numpy, as the reference
    else:
        scores = np.array([k["score"] for k in kpts_db])
    kpts = np.array([np.asarray(k["keypoints"], np.float32).reshape(-1, 3) for k in kpts_db])
    areas = np.array([k["area"] for k in kpts_db], np.float64)
    return kpts, areas, scores.astype(np.float64)


def oks_nms(kpts_db, thr, sigmas=None, vis_thr=None, score_per_joint=False):
    """The reference's oks_nms on the device: kpts_db a list of {'keypoints' [K, 3], 'area', 'score'} -> np.ndarray of the
    kept indices ([] for an empty list).
    The device computes in fixed types: keypoints are rounded to float32, scores (and per-joint means) widened to float64,
    areas taken as float64, and thr, vis_thr used as float32, which is what the reference does with float32 keypoints,
    Python-float or float64 scores and Python-float thresholds.  Other inputs make the reference compute in other types,
    where the result can differ from it: float64 keypoints (its dx, dy in float64), float32 scores (soft NMS then rescales
    in float32, e.g. score_per_joint with float32 per-joint scores) or a np.float64 thr (numpy 2 then compares in float64)."""
    if len(kpts_db) == 0:
        return []
    kpts, areas, scores = _db_arrays(kpts_db, score_per_joint)
    return oks_nms_frames([kpts], [areas], [scores], thr, sigmas, vis_thr)[0]


def soft_oks_nms(kpts_db, thr, max_dets=20, sigmas=None, vis_thr=None, score_per_joint=False):
    """The reference's soft_oks_nms on the device: kpts_db as oks_nms -> np.ndarray of at most max_dets kept indices.
    Computation types as oks_nms."""
    if len(kpts_db) == 0:
        return []
    kpts, areas, scores = _db_arrays(kpts_db, score_per_joint)
    return oks_nms_frames([kpts], [areas], [scores], thr, sigmas, vis_thr, soft=True, max_dets=max_dets)[0]
