"""ViTPose(cfg): the reference's model object (easy_ViTPose/vit_models/model.py:10-24) backed by the
sm_90a engine.  Same constructor argument, same state_dict key contract, same forward signature;
the arithmetic runs in libvitpose_b200.so (bf16 tensor-core GEMMs, fp32 residual stream/softmax/LN).

torch is used for what it is good at here: owning device memory and the current stream.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .configs import VITPOSE_PLUS_HEADS

__all__ = ["ViTPose", "plan_frame_chunks", "nv12_planes", "yuv_planes", "split_vitpose_plus", "merge_split_state_dicts", "group_by_head", "head_flip_permutations",
           "plan_head_calls"]

IMG_H, IMG_W, HM_H, HM_W = 256, 192, 64, 48
_EMPTY_BOX = "a box is empty after padding and clipping to its frame"     # check=True of the multi-frame calls: status bit 0
_BAD_AFFINE = "a matrix entry is not finite or a scale is <= 0"             # and of the affine calls: status bit 1


def plan_frame_chunks(counts, limit: int, max_frames: int = _lib.MAX_FRAMES) -> "list[list[tuple[int, int, int]]]":
    """Splits the boxes of several frames (counts[j] boxes in frame j) into engine calls of at most `limit` boxes from at most
    `max_frames` frames.  Returns the calls in order; each is a list of (frame, first, stop): boxes first..stop-1 of that
    frame.  Every box lands in exactly one call, in frame order; frames without boxes appear in none, and a frame's boxes
    may continue in the next call."""
    if limit < 1 or max_frames < 1:
        raise ValueError(f"limit {limit} and max_frames {max_frames} must be >= 1")
    chunks, cur, used = [], [], 0
    for f, c in enumerate(counts):
        c = int(c)
        if c < 0:
            raise ValueError(f"frame {f} has {c} boxes")
        s = 0
        while s < c:
            if used == limit or len(cur) == max_frames:
                chunks.append(cur)
                cur, used = [], 0
            take = min(c - s, limit - used)
            cur.append((f, s, s + take))
            used += take
            s += take
    if cur:
        chunks.append(cur)
    return chunks


def _rotations(rotate, num_frames: int) -> "list[int]":
    """The `rotate` argument of the frame methods -> one rotation per frame.  `rotate` is one int for all frames or a sequence
    of num_frames ints, each 0, 90, 180 or 270: degrees counter-clockwise, the reference's `--rotate`.  A rotated frame is seen
    as cv2.rotate(frame, ...) would turn it (its view), and its boxes, matrices and keypoints are in view pixels.  Raises
    ValueError for anything else, before any launch."""
    r = np.asarray(rotate.cpu() if isinstance(rotate, torch.Tensor) else rotate)
    if r.ndim == 0:
        r = np.full(num_frames, r)
    if r.ndim != 1 or r.size != num_frames:
        raise ValueError(f"rotate: one value or one per frame expected ({num_frames} frames), got shape {r.shape}")
    if r.size and (r.dtype.kind not in "iu" or not np.isin(r, _lib.ROTATIONS).all()):
        raise ValueError(f"rotate: 0, 90, 180 or 270 (degrees counter-clockwise) expected, got {r.tolist()}")
    return [int(v) for v in r]


def _frame_array(frames, chunk, struct=_lib.VpbFrame, rot=None):
    """vpb_frame array for one planned call: entries 0..last frame of the call, so that the engine's messages name the
    caller's frame index; frames outside the call get 0 boxes (skipped).  `frames` holds (data pointer, h, w, pitch), or
    for struct=VpbFrameNv12 (y pointer, y pitch, uv pointer, uv pitch, h, w), or for struct=VpbFrameYuv ViTPose._yuv_row;
    rot[f] is frame f's rotation (_rotations; None: all upright)."""
    arr = (struct * (chunk[-1][0] + 1))()
    for f, s, e in chunk:
        arr[f] = struct(*frames[f], e - s, 0 if rot is None else rot[f])
    return arr


def nv12_planes(frame, what: str = "frame"):
    """One NV12 frame -> its (y [H,W], uv [H/2,W]) planes as views, for numpy arrays and torch tensors alike.  A frame is
    either a uint8 [3H/2, W] array with the planes stacked (what cv2 and ffmpeg's `-pix_fmt nv12` produce) or a pair
    (y, uv) (what a decoder surface is: two planes, any row pitch).  Raises ValueError for odd or mismatched sizes."""
    if isinstance(frame, (tuple, list)):
        if len(frame) != 2:
            raise ValueError(f"{what}: an NV12 (y, uv) pair expected, got {len(frame)} planes")
        y, uv = frame
    else:
        if getattr(frame, "ndim", 0) != 2 or frame.shape[0] % 3:
            raise ValueError(f"{what}: NV12 [3H/2, W] with the planes stacked expected, got shape {tuple(getattr(frame, 'shape', ()))}")
        h = frame.shape[0] // 3 * 2
        y, uv = frame[:h], frame[h:]
    for p in (y, uv):
        if getattr(p, "ndim", 0) != 2 or str(p.dtype) not in ("uint8", "torch.uint8"):
            raise ValueError(f"{what}: NV12 planes must be 2-D uint8, got {getattr(p, 'dtype', type(p))} {tuple(getattr(p, 'shape', ()))}")
    if type(y) is not type(uv):
        raise ValueError(f"{what}: the y and uv planes must both be numpy arrays or both tensors")
    h, w = y.shape
    if h < 2 or w < 2 or h % 2 or w % 2:
        raise ValueError(f"{what}: NV12 needs an even height and width >= 2, got {h}x{w} (h x w)")
    if tuple(uv.shape) != (h // 2, w):
        raise ValueError(f"{what}: uv plane {tuple(uv.shape)} does not match the {h}x{w} y plane ([H/2, W] expected)")
    return y, uv


def _yuv_matrix(matrix: str) -> int:
    try:
        return _lib.YUV_MATRICES[str(matrix).lower()]
    except KeyError:
        raise ValueError(f"unknown YUV matrix {matrix!r}: one of {sorted(_lib.YUV_MATRICES)}") from None


def _yuv_format(layout: str, matrix: str, full_range: bool) -> "tuple[int, int, int]":
    """(layout, matrix, range) names -> the C constants of the _yuv calls; ValueError for an unknown name."""
    try:
        lay = _lib.YUV_LAYOUTS[str(layout).lower()]
    except KeyError:
        raise ValueError(f"unknown YUV layout {layout!r}: one of {sorted(_lib.YUV_LAYOUTS)}") from None
    return lay, _yuv_matrix(matrix), _lib.YUV_RANGES["full" if full_range else "limited"]


def _is_u8_2d(p) -> bool:
    return getattr(p, "ndim", 0) == 2 and str(getattr(p, "dtype", "")) in ("uint8", "torch.uint8")


def yuv_planes(frame, layout: str, what: str = "frame") -> "tuple[tuple, int, int]":
    """One YUV frame -> (its planes in the layout's storage order, as vpb_frame_yuv takes them, height, width), as views
    where the memory allows, for numpy arrays and torch tensors alike.  Accepted forms:
      nv12, nv21   uint8 [3H/2, W] with the planes stacked, or a (y [H,W], uv [H/2,W]) pair (uv: vu for nv21)
      i420, yv12   uint8 [3H/2, W] as cv2 and ffmpeg write it (each chroma plane H/2 x W/2 bytes, packed after the luma), or a
                   (y [H,W], u [H/2,W/2], v [H/2,W/2]) triple named by content for both layouts
      yuyv, uyvy   uint8 [H, W, 2] (what cv2.VideoCapture returns with CAP_PROP_CONVERT_RGB = 0) or [H, 2W]
    Planes may have any row pitch with contiguous rows.  Raises ValueError for unknown layouts, odd or mismatched sizes."""
    lay = _yuv_format(layout, "bt601", False)[0]
    name = str(layout).lower()
    if lay >= _lib.YUV_LAYOUTS["yuyv"]:                      # packed 4:2:2: one [H, 2W] plane
        if isinstance(frame, (tuple, list)) or getattr(frame, "ndim", 0) not in (2, 3):
            raise ValueError(f"{what}: {name} [H, W, 2] or [H, 2W] expected, got {type(frame).__name__} "
                             f"{tuple(getattr(frame, 'shape', ()))}")
        if frame.ndim == 3:
            if frame.shape[2] != 2:
                raise ValueError(f"{what}: {name} [H, W, 2] expected, got shape {tuple(frame.shape)}")
            frame = frame.reshape(frame.shape[0], 2 * frame.shape[1])
        if not _is_u8_2d(frame):
            raise ValueError(f"{what}: {name} frames must be uint8, got {getattr(frame, 'dtype', type(frame))}")
        h, w = frame.shape[0], frame.shape[1] // 2
        if h < 1 or w < 2 or frame.shape[1] % 4:
            raise ValueError(f"{what}: {name} needs an even width >= 2, got {frame.shape[1] / 2:g}x{h} (w x h)")
        return (frame,), h, w
    if lay <= _lib.YUV_LAYOUTS["nv21"]:                       # semi-planar: the NV12 forms, for NV21 with the chroma bytes swapped
        y, c = nv12_planes(frame, what)
        return (y, c), y.shape[0], y.shape[1]
    if isinstance(frame, (tuple, list)):                      # planar: (y, u, v) by content
        if len(frame) != 3:
            raise ValueError(f"{what}: an {name} (y, u, v) triple expected, got {len(frame)} planes")
        y, u, v = frame
    else:
        if not _is_u8_2d(frame) or frame.shape[0] % 3:
            raise ValueError(f"{what}: {name} [3H/2, W] with the planes stacked expected, got shape {tuple(getattr(frame, 'shape', ()))}")
        h, w = frame.shape[0] // 3 * 2, frame.shape[1]
        if h < 2 or w < 2 or w % 2:
            raise ValueError(f"{what}: {name} needs an even height and width >= 2, got {h}x{w} (h x w)")
        y, c = frame[:h], frame[h:]
        c = c.contiguous() if isinstance(c, torch.Tensor) else np.ascontiguousarray(c)
        flat, q = c.reshape(-1), (h // 2) * (w // 2)          # each chroma plane is H/2 x W/2 packed bytes
        first, second = flat[:q].reshape(h // 2, w // 2), flat[q:].reshape(h // 2, w // 2)
        u, v = (first, second) if name == "i420" else (second, first)
    for p in (y, u, v):
        if not _is_u8_2d(p):
            raise ValueError(f"{what}: {name} planes must be 2-D uint8, got {getattr(p, 'dtype', type(p))} {tuple(getattr(p, 'shape', ()))}")
    if not (type(y) is type(u) is type(v)):
        raise ValueError(f"{what}: the planes must all be numpy arrays or all tensors")
    h, w = y.shape
    if h < 2 or w < 2 or h % 2 or w % 2:
        raise ValueError(f"{what}: {name} needs an even height and width >= 2, got {h}x{w} (h x w)")
    if tuple(u.shape) != (h // 2, w // 2) or tuple(v.shape) != (h // 2, w // 2):
        raise ValueError(f"{what}: chroma planes {tuple(u.shape)} / {tuple(v.shape)} do not match the {h}x{w} y plane "
                         "([H/2, W/2] expected)")
    return ((y, u, v) if name == "i420" else (y, v, u)), h, w


def group_by_head(heads, num_heads: int) -> "tuple[np.ndarray, list[int]]":
    """Per-box head indices -> (order, counts): `order` lists the boxes grouped by head, stable inside a head (box order[i]
    goes to position i of the grouped call), counts[h] = boxes of head h.  Raises ValueError for an index outside
    0..num_heads-1."""
    h = np.asarray(heads).reshape(-1)
    if h.size and (h.dtype.kind not in "iu" or h.min() < 0 or h.max() >= num_heads):
        raise ValueError(f"head indices must be integers in 0..{num_heads - 1}")
    h = h.astype(np.int64)
    return np.argsort(h, kind="stable"), [int(c) for c in np.bincount(h, minlength=num_heads)]


def head_flip_permutations(head_keypoints, flip_pairs_per_head) -> np.ndarray:
    """The permutation of every head (ViTPose.flip_permutation of its pairs), concatenated in head order: what
    vpb_set_flip_test_heads takes.  Raises ValueError when the pair lists do not match the heads or a pair index lies outside
    its head's 0..K_j-1."""
    ks = [int(k) for k in head_keypoints]
    pairs = list(flip_pairs_per_head)
    if len(pairs) != len(ks):
        raise ValueError(f"{len(pairs)} flip pair lists for {len(ks)} heads")
    out = []
    for j, (K, pp) in enumerate(zip(ks, pairs)):
        pp = [(int(a), int(b)) for a, b in pp]
        if any(not 0 <= i < K for pair in pp for i in pair):
            raise ValueError(f"head {j}: flip pairs {pp} index outside 0..{K - 1}")
        out += ViTPose.flip_permutation(K, pp)
    return np.array(out, np.int32)


def plan_head_calls(counts, heads, num_heads: int, limit: int, max_frames: int = _lib.MAX_FRAMES):
    """The boxes of several frames (counts[j] boxes in frame j, heads[j] = their head indices) grouped by head for the
    multi-head frame / affine calls -> (entries, order, chunks):
      entries  [(frame, box indices within the frame, head)], head-major, frame order inside a head: a frame appears once
               per head it uses;
      order    the flat index (frames concatenated) of each box in call order;
      chunks   plan_frame_chunks over the entries: calls of at most `limit` boxes from at most `max_frames` entries.
    The one planner of infer_frames_heads(_host) and infer_affine_heads(_host).  heads[j] may be a list, array or tensor."""
    if len(counts) != len(heads):
        raise ValueError(f"{len(counts)} frames but {len(heads)} head arrays")
    hs = []
    for j, (c, h) in enumerate(zip(counts, heads)):
        h = np.asarray(h.cpu() if isinstance(h, torch.Tensor) else h).reshape(-1)
        if h.size != int(c):
            raise ValueError(f"{int(c)} boxes but {h.size} head indices in frame {j}")
        group_by_head(h, num_heads)                         # range check
        hs.append(h.astype(np.int64))
    entries = [(j, np.nonzero(h == k)[0], k) for k in range(num_heads) for j, h in enumerate(hs) if (h == k).any()]
    first = np.concatenate([[0], np.cumsum([int(c) for c in counts])]).astype(np.int64)
    order = np.concatenate([first[j] + sel for j, sel, _ in entries]) if entries else np.zeros((0,), np.int64)
    return entries, order, plan_frame_chunks([len(sel) for _, sel, _ in entries], limit, max_frames)


def _inverse(order: np.ndarray) -> np.ndarray:
    inv = np.empty_like(order)
    inv[order] = np.arange(order.size)
    return inv


# the head tensors model_split.py moves (:35-48), relative to the head's prefix
_HEAD_PARTS = ("deconv_layers.0.weight", "deconv_layers.1.weight", "deconv_layers.1.bias", "deconv_layers.1.running_mean",
               "deconv_layers.1.running_var", "deconv_layers.1.num_batches_tracked", "deconv_layers.3.weight",
               "deconv_layers.4.weight", "deconv_layers.4.bias", "deconv_layers.4.running_mean", "deconv_layers.4.running_var",
               "deconv_layers.4.num_batches_tracked", "final_layer.weight", "final_layer.bias")


def _head_prefix(j: int) -> str:
    return "keypoint_head." if j == 0 else f"associate_keypoint_heads.{j - 1}."


def _unwrap(sd):
    return sd["state_dict"] if "state_dict" in sd and not any(k.startswith("backbone.") for k in sd) else sd


def split_vitpose_plus(sd, names=None, keypoints=None) -> "OrderedDict[str, OrderedDict[str, torch.Tensor]]":
    """model_split.py in torch on the CPU: an unsplit ViTPose+ state_dict -> {dataset: single-dataset state_dict}.  Head i
    (names[i], default the VITPOSE_PLUS_HEADS order) gets fc2 = cat([fc2, experts.i]) in every block (:53-57, :83-92) and,
    for i >= 1, associate_keypoint_heads.{i-1} as keypoint_head with final_layer cut to keypoints[i] rows (:97-102); the
    expert and associate tensors are dropped (:59-69, :104-114).  A checkpoint without experts (a frozen-backbone fine-tune
    merged with P = 0) keeps its fc2 as is."""
    sd = _unwrap(sd)
    table = dict(VITPOSE_PLUS_HEADS)
    names = [n for n, _ in VITPOSE_PLUS_HEADS] if names is None else list(names)
    keypoints = [table[n] for n in names] if keypoints is None else [int(k) for k in keypoints]
    if len(names) != len(keypoints):
        raise ValueError(f"{len(names)} names but {len(keypoints)} keypoint counts")
    experts = any(".mlp.experts." in k for k in sd)
    out: "OrderedDict[str, OrderedDict[str, torch.Tensor]]" = OrderedDict()
    for i, (name, K) in enumerate(zip(names, keypoints)):
        d: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        for k, v in sd.items():
            if "expert" in k or k.startswith("associate_keypoint_heads."):
                continue
            if "mlp.fc2" in k and experts:
                ek = k.replace("fc2.", f"experts.{i}.")
                if ek not in sd:
                    raise KeyError(f"{ek}: the checkpoint has no expert {i} for {name!r}")
                v = torch.cat([torch.as_tensor(v), torch.as_tensor(sd[ek])], 0)
            d[k] = v
        if i > 0:
            for part in _HEAD_PARTS:
                src = _head_prefix(i) + part
                if src in sd:
                    d["keypoint_head." + part] = sd[src]
                elif not part.endswith("num_batches_tracked"):
                    raise KeyError(f"{src} missing")
            for part in ("final_layer.weight", "final_layer.bias"):
                d["keypoint_head." + part] = d["keypoint_head." + part][:K]
        out[name] = d
    return out


def merge_split_state_dicts(sds, part_features: int) -> "OrderedDict[str, torch.Tensor]":
    """The inverse of split_vitpose_plus: {dataset: state_dict} (split ViTPose+ checkpoints, or frozen-backbone fine-tunes with
    part_features = 0) -> one state_dict under ViTPose+ keys for a multi-head ViTPose, heads in the dict's order: each
    block's fc2 is split into the shared rows (mlp.fc2) and the last part_features rows of checkpoint j (mlp.experts.{j}),
    checkpoint 0's head is keypoint_head and checkpoint j's is associate_keypoint_heads.{j-1}.  Every other backbone tensor,
    and the shared rows of fc2, must be equal in all checkpoints: ValueError names the first key whose shared part differs."""
    items = [(str(n), {k: torch.as_tensor(v) for k, v in _unwrap(sd).items()}) for n, sd in sds.items()]
    if not items:
        raise ValueError("no checkpoints to merge")
    P = int(part_features)
    base_name, base = items[0]
    for name, sd in items[1:]:
        for k in sd:
            if not k.startswith("keypoint_head.") and k not in base:
                raise ValueError(f"{k}: in {name!r} but not in {base_name!r}")
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for k, v in base.items():
        if k.startswith("keypoint_head."):
            continue
        split = P > 0 and "mlp.fc2" in k
        shared = v[: v.shape[0] - P] if split else v
        for name, sd in items[1:]:
            w = sd.get(k)
            ws = None if w is None else (w[: w.shape[0] - P] if split else w)
            if ws is None or ws.shape != shared.shape or not torch.equal(ws, shared):
                raise ValueError(f"{k}: the shared part of {name!r} differs from {base_name!r}")
        out[k] = shared
        if split:
            for j, (_, sd) in enumerate(items):
                out[k.replace("fc2.", f"experts.{j}.")] = sd[k][sd[k].shape[0] - P:]
    for j, (_, sd) in enumerate(items):
        for k, v in sd.items():
            if k.startswith("keypoint_head."):
                out[_head_prefix(j) + k[len("keypoint_head."):]] = v
    return out


def _expected_shapes(D: int, depth: int, K: int, head_keypoints=None, P: int = 0) -> "OrderedDict[str, tuple]":
    """state_dict contract of the reference ViTPose (SURVEY.md section 8b); with head_keypoints / P the ViTPose+ key set of a
    multi-head engine (vpb_create_heads)."""
    s: "OrderedDict[str, tuple]" = OrderedDict()
    s["backbone.pos_embed"] = (1, 193, D)
    s["backbone.patch_embed.proj.weight"] = (D, 3, 16, 16)
    s["backbone.patch_embed.proj.bias"] = (D,)
    for i in range(depth):
        p = f"backbone.blocks.{i}."
        s[p + "norm1.weight"] = (D,); s[p + "norm1.bias"] = (D,)
        s[p + "attn.qkv.weight"] = (3 * D, D); s[p + "attn.qkv.bias"] = (3 * D,)
        s[p + "attn.proj.weight"] = (D, D); s[p + "attn.proj.bias"] = (D,)
        s[p + "norm2.weight"] = (D,); s[p + "norm2.bias"] = (D,)
        s[p + "mlp.fc1.weight"] = (4 * D, D); s[p + "mlp.fc1.bias"] = (4 * D,)
        s[p + "mlp.fc2.weight"] = (D - P, 4 * D); s[p + "mlp.fc2.bias"] = (D - P,)
        for j in range(len(head_keypoints) if P else 0):
            s[p + f"mlp.experts.{j}.weight"] = (P, 4 * D); s[p + f"mlp.experts.{j}.bias"] = (P,)
    s["backbone.last_norm.weight"] = (D,); s["backbone.last_norm.bias"] = (D,)
    for j, Kj in enumerate(head_keypoints or [K]):
        hp = _head_prefix(j)
        cin = D
        for li in (0, 3):
            s[f"{hp}deconv_layers.{li}.weight"] = (cin, 256, 4, 4)
            for n in ("weight", "bias", "running_mean", "running_var"):
                s[f"{hp}deconv_layers.{li + 1}.{n}"] = (256,)
            s[f"{hp}deconv_layers.{li + 1}.num_batches_tracked"] = ()
            cin = 256
        s[hp + "final_layer.weight"] = (Kj, 256, 1, 1)
        s[hp + "final_layer.bias"] = (Kj,)
    return s


class _Backbone:
    """`model.backbone` of the reference ViTPose (vit_models/model.py:14): callable, [B,3,256,192] -> [B,D,16,12]."""

    def __init__(self, owner):
        self._owner = owner
        self.num_heads = owner.num_heads if hasattr(owner, "num_heads") else None

    def __call__(self, x):
        return self._owner.forward_features(x)

    forward = __call__


class _Head:
    """`model.keypoint_head` (vit_models/model.py:15, head/topdown_heatmap_simple_head.py): forward and inference_model."""

    def __init__(self, owner):
        self._owner = owner
        self.target_type = "GaussianHeatmap"
        self.test_cfg = {}

    def __call__(self, features):
        return self._owner.head_forward(features)

    forward = __call__

    def inference_model(self, x, flip_pairs=None):
        """head/topdown_heatmap_simple_head.py:195-218: numpy heatmaps, flipped back (and shifted by one pixel when
        test_cfg['shift_heatmap']) if flip_pairs is given."""
        out = self._owner.head_forward(x)
        if flip_pairs is not None:
            out = self._owner.flip_back(out, flip_pairs, bool(self.test_cfg.get("shift_heatmap", False)))
        return out.cpu().numpy()


class ViTPose:
    """Drop-in for the reference `ViTPose(cfg)` on the inference path.

    cfg is the reference's model dict (cfg['backbone'], cfg['keypoint_head']; 'type' keys ignored,
    model.py:14-15).  Only the configurations the reference ships are accepted: patch 16, 256x192,
    mlp_ratio 4, qkv_bias, two 4x4 deconvs of 256 filters and a 1x1 final conv.
    """

    def __init__(self, cfg: dict, max_batch: int = 64, device: "int | str | torch.device | None" = None, *, heads=None,
                 expert_rows: int = 0) -> None:
        bb = {k: v for k, v in cfg["backbone"].items() if k != "type"}
        hd = {k: v for k, v in cfg["keypoint_head"].items() if k != "type"}
        if tuple(bb.get("img_size", (256, 192))) != (256, 192) or bb.get("patch_size", 16) != 16 or bb.get("ratio", 1) != 1:
            raise ValueError("only img_size=(256,192), patch_size=16, ratio=1 (the reference's configs) are built")
        if bb.get("mlp_ratio", 4) != 4 or not bb.get("qkv_bias", False):
            raise ValueError("only mlp_ratio=4, qkv_bias=True (the reference's configs) are built")
        if hd.get("num_deconv_layers", 3) != 2 or tuple(hd.get("num_deconv_filters", ())) != (256, 256) \
                or tuple(hd.get("num_deconv_kernels", ())) != (4, 4) or (hd.get("extra") or {}).get("final_conv_kernel", 1) != 1:
            raise ValueError("only the 2x deconv(256,4x4) + 1x1 conv head of the reference's configs is built")
        self.embed_dim = int(bb["embed_dim"]); self.depth = int(bb["depth"]); self.num_heads = int(bb["num_heads"])
        self.num_keypoints = int(hd["out_channels"])
        # several keypoint heads on one backbone (ViTPose+ / frozen-backbone fine-tunes): `heads` = keypoint counts or
        # (dataset, keypoints) pairs, head j using fc2 expert j of width expert_rows (0 = a fully shared backbone)
        self.head_names = None
        self.head_keypoints = [self.num_keypoints]
        self.expert_rows = int(expert_rows)
        self._multi = heads is not None
        if self._multi:
            heads = list(heads)
            if not 1 <= len(heads) <= _lib.MAX_HEADS:
                raise ValueError(f"{len(heads)} heads: 1..{_lib.MAX_HEADS} expected")
            if all(isinstance(h, (tuple, list)) for h in heads):
                self.head_names = [str(n) for n, _ in heads]
                heads = [k for _, k in heads]
            self.head_keypoints = [int(k) for k in heads]
            if any(not 1 <= k <= 144 for k in self.head_keypoints):
                raise ValueError(f"keypoint counts {self.head_keypoints}: 1..144 each")
            if self.expert_rows and not (0 < self.expert_rows < self.embed_dim and self.expert_rows % 32 == 0):
                raise ValueError(f"expert_rows={self.expert_rows}: 0 or a multiple of 32 below embed_dim={self.embed_dim}")
            self.num_keypoints = self.head_keypoints[0]
        elif self.expert_rows:
            raise ValueError("expert_rows needs heads=")
        self.num_keypoints_max = max(self.head_keypoints)
        if int(hd["in_channels"]) != self.embed_dim:
            raise ValueError("keypoint_head.in_channels must equal backbone.embed_dim")
        self.max_batch = int(max_batch)
        self.training = False
        self._cfg = cfg
        self._handle = C.c_void_p()
        self._loaded = False
        self._state: "OrderedDict[str, torch.Tensor] | None" = None
        self._device = None
        self._side = None
        self._flip = False
        self.backbone = _Backbone(self)              # model.backbone(x) / model.keypoint_head(f), as on the reference module
        self.keypoint_head = _Head(self)
        if device is not None:
            self.to(device)

    # ---------------------------------------------------------------- nn.Module-like surface
    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError("the engine is inference-only (eval mode); training stays with the reference")
        return self

    def to(self, device):
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise RuntimeError(f"ViTPose has no {dev.type} path: it needs a CUDA sm_90 (H100) device")
        index = dev.index if dev.index is not None else torch.cuda.current_device()
        if self._device is not None and self._device != index and self._handle:
            raise RuntimeError("engine already lives on another device")
        self._device = index
        if self._state is not None and not self._loaded:
            self._upload()
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def state_dict(self):
        if self._state is None:
            raise RuntimeError("no weights loaded")
        return OrderedDict((k, v.clone()) for k, v in self._state.items())

    def load_state_dict(self, state_dict, strict: bool = True):
        """Same contract as nn.Module.load_state_dict(strict=True): missing / unexpected keys and
        shape mismatches raise (easy_ViTPose/inference.py:162-166 calls it exactly like this)."""
        if "state_dict" in state_dict and not any(k.startswith("backbone.") for k in state_dict):
            state_dict = state_dict["state_dict"]
        exp = _expected_shapes(self.embed_dim, self.depth, self.num_keypoints, self.head_keypoints if self._multi else None,
                               self.expert_rows)
        missing = [k for k in exp if k not in state_dict and not k.endswith("num_batches_tracked")]
        unexpected = [k for k in state_dict if k not in exp]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for ViTPose: missing keys {missing[:5]}"
                               f"{'...' if len(missing) > 5 else ''}, unexpected keys {unexpected[:5]}")
        st: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        for k, shape in exp.items():
            if k not in state_dict:
                if k.endswith("num_batches_tracked"):
                    st[k] = torch.zeros((), dtype=torch.int64)
                    continue
                raise RuntimeError(f"missing key {k}")
            v = state_dict[k]
            v = torch.as_tensor(np.asarray(v)) if not isinstance(v, torch.Tensor) else v
            if tuple(v.shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {k}: copying a param with shape {tuple(v.shape)}, expected {tuple(shape)}")
            st[k] = v.detach().to("cpu").contiguous()
        if self._loaded:
            raise RuntimeError("weights already packed on the device; create a new ViTPose to load another checkpoint")
        self._state = st
        if self._device is not None:
            self._upload()
        return self

    # ---------------------------------------------------------------- engine plumbing
    def _ensure(self):
        if not self._loaded:
            if self._state is None:
                raise RuntimeError("load_state_dict() before forward()")
            if self._device is None:
                self.to("cuda")
            else:
                self._upload()

    def _upload(self):
        L = _lib.lib()
        cfg = _lib.VpbConfig(self.embed_dim, self.depth, self.num_heads, self.num_keypoints, self.max_batch, self._device)
        with torch.cuda.device(self._device):
            if self._multi:
                ks = (C.c_int32 * len(self.head_keypoints))(*self.head_keypoints)
                _lib.check(L.vpb_create_heads(C.byref(cfg), len(ks), ks, self.expert_rows, C.byref(self._handle)))
            else:
                _lib.check(L.vpb_create(C.byref(cfg), C.byref(self._handle)))
            for k, v in self._state.items():
                if k.endswith("num_batches_tracked"):
                    continue
                a = v.to(torch.float32).contiguous().numpy()
                _lib.check(L.vpb_load_tensor(self._handle, k.encode(), a.ctypes.data_as(C.c_void_p), a.size))
            _lib.check(L.vpb_finalize(self._handle))
        self._loaded = True

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self._device).cuda_stream)

    @property
    def flip_test(self) -> bool:
        """Whether the keypoint calls run the flip test (set_flip_test)."""
        return self._flip

    @property
    def batch_limit(self) -> int:
        """Most crops / boxes one keypoint call takes: max_batch, or max_batch // 2 with flip test on (each crop and its
        mirror image share the workspace)."""
        return self.max_batch // 2 if self._flip else self.max_batch

    @staticmethod
    def flip_permutation(num_keypoints: int, flip_pairs) -> "list[int]":
        """The keypoint permutation the (left, right) pairs induce, built sequentially (a later pair overrides an earlier
        one), like the loop of flip_back (post_processing/post_transforms.py:110-147)."""
        perm = list(range(num_keypoints))
        for left, right in flip_pairs:
            perm[left], perm[right] = right, left
        return perm

    def set_flip_test(self, flip_pairs, shift_heatmap: bool = False) -> None:
        """Flip test on every keypoint call (infer_crops, infer_host, submit_host, infer_frame, infer_frame_host,
        submit_frame_host, infer_frames, infer_frames_host, submit_frames_host, infer_affine, infer_affine_host): heatmaps of each crop and of its mirror image (flipped back, pairs swapped, shifted by one pixel
        when shift_heatmap) averaged before the decode -- the test_cfg flip_test=True of the reference configs
        (configs/ViTPose_common.py:124).  Keypoints and returned heatmaps are then bit-identical to forward_flip_test
        followed by decode_heatmaps.  A call then takes at most max_batch // 2 crops.  `None` turns it off.  Synchronises
        the engine's pending work."""
        self._ensure()
        if flip_pairs is None:
            _lib.check(_lib.lib().vpb_set_flip_test(self._handle, None, self.num_keypoints, 0))
            self._flip = False
            return
        flip_pairs = [(int(a), int(b)) for a, b in flip_pairs]
        if any(not (0 <= i < self.num_keypoints) for pair in flip_pairs for i in pair):
            raise ValueError(f"flip pairs {flip_pairs} index outside 0..{self.num_keypoints - 1}")
        perm = np.array(self.flip_permutation(self.num_keypoints, flip_pairs), np.int32)
        _lib.check_value(_lib.lib().vpb_set_flip_test(self._handle, perm.ctypes.data_as(C.c_void_p), perm.size, 1 if shift_heatmap else 0))
        self._flip = True

    def set_flip_test_heads(self, flip_pairs_per_head, shift_heatmap: bool = False) -> None:
        """Flip test on every keypoint call of a multi-head engine (also valid with one head): flip_pairs_per_head holds the
        (left, right) pairs of every head, in head order (the reference defines pairs for COCO only, so the caller names them
        for the other datasets; an empty list for a head without pairs).  The multi-head calls (infer_crops_heads,
        infer_frames_heads(_host), infer_affine_heads(_host)) then average each crop's maps with those of its mirror image
        under its head's pairs; the single-head calls run head 0 with head 0's pairs.  One shift for all heads.  A call then
        takes at most max_batch // 2 crops.  `None` turns it off.  Replaces a setting made by set_flip_test, and the other
        way round.  Synchronises the engine's pending work."""
        self._ensure()
        L = _lib.lib()
        if flip_pairs_per_head is None:
            _lib.check(L.vpb_set_flip_test_heads(self._handle, None, 0, 0))
            self._flip = False
            return
        perms = head_flip_permutations(self.head_keypoints, flip_pairs_per_head)
        _lib.check_value(L.vpb_set_flip_test_heads(self._handle, perms.ctypes.data_as(C.c_void_p), perms.size, 1 if shift_heatmap else 0))
        self._flip = True

    def _check_input(self, x: torch.Tensor, limit: "int | None" = None) -> torch.Tensor:
        if not isinstance(x, torch.Tensor):
            raise TypeError("expected a torch.Tensor [B,3,256,192]")
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, IMG_H, IMG_W):
            raise ValueError(f"expected [B,3,256,192], got {tuple(x.shape)}")
        limit = self.max_batch if limit is None else limit
        if x.shape[0] < 1 or x.shape[0] > limit:
            raise ValueError(f"batch {x.shape[0]} outside 1..{limit} (max_batch={self.max_batch}, flip test {'on' if self._flip else 'off'})")
        self._ensure()
        if not x.is_cuda:
            x = x.to(torch.device("cuda", self._device), non_blocking=True)
        if x.device.index != self._device:
            raise ValueError("input lives on another GPU than the engine")
        return x.to(torch.float32).contiguous()

    # ---------------------------------------------------------------- forward paths
    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """[B,3,256,192] float32 -> heatmaps [B,K,64,48] float32 (model.py:23-24)."""
        x = self._check_input(x)
        out = torch.empty((x.shape[0], self.num_keypoints, HM_H, HM_W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().vpb_forward(self._handle, C.c_void_p(x.data_ptr()), x.shape[0], C.c_void_p(out.data_ptr()), self._stream()))
        return out

    __call__ = forward

    @torch.no_grad()
    def forward_features(self, x: torch.Tensor) -> torch.Tensor:
        """[B,3,256,192] -> backbone features [B,D,16,12] (model.py:20-21, vit.py:375-389)."""
        x = self._check_input(x)
        out = torch.empty((x.shape[0], self.embed_dim, 16, 12), dtype=torch.float32, device=x.device)
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().vpb_forward_features(self._handle, C.c_void_p(x.data_ptr()), x.shape[0], C.c_void_p(out.data_ptr()), self._stream()))
        return out

    @torch.no_grad()
    def head_forward(self, features: torch.Tensor) -> torch.Tensor:
        """Backbone features [B,D,16,12] -> heatmaps [B,K,64,48]: TopdownHeatmapSimpleHead.forward
        (head/topdown_heatmap_simple_head.py:188-193).  The engine's head consumes bf16 features; those returned by
        forward_features are bf16 values already, so backbone -> head in two calls equals forward()."""
        self._ensure()
        if not isinstance(features, torch.Tensor) or features.dim() != 4 or tuple(features.shape[1:]) != (self.embed_dim, 16, 12):
            raise ValueError(f"expected features [B,{self.embed_dim},16,12]")
        if features.shape[0] < 1 or features.shape[0] > self.max_batch:
            raise ValueError(f"batch {features.shape[0]} outside 1..max_batch={self.max_batch}")
        f = features.to(device=torch.device("cuda", self._device), dtype=torch.float32).contiguous()
        out = torch.empty((f.shape[0], self.num_keypoints, HM_H, HM_W), dtype=torch.float32, device=f.device)
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().vpb_head(self._handle, C.c_void_p(f.data_ptr()), f.shape[0], C.c_void_p(out.data_ptr()), self._stream()))
        return out

    @torch.no_grad()
    def flip_back(self, heatmaps: torch.Tensor, flip_pairs, shift_heatmap: bool = False) -> torch.Tensor:
        """flip_back (post_processing/post_transforms.py:110-147) + the optional shift of inference_model (:210-212) on the GPU."""
        hm = heatmaps.to(device=torch.device("cuda", self._device if self._device is not None else torch.cuda.current_device()),
                         dtype=torch.float32).contiguous()
        if hm.dim() != 4 or tuple(hm.shape[2:]) != (HM_H, HM_W):
            raise ValueError(f"expected [N,K,64,48], got {tuple(hm.shape)}")
        K = hm.shape[1]
        pt = torch.tensor(self.flip_permutation(K, flip_pairs), dtype=torch.int32, device=hm.device)
        out = torch.empty_like(hm)
        with torch.cuda.device(hm.device):
            _lib.check(_lib.lib().vpb_flip_back(C.c_void_p(hm.data_ptr()), hm.shape[0], K, C.c_void_p(pt.data_ptr()), 1 if shift_heatmap else 0,
                                                C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream(hm.device).cuda_stream)))
        return out

    @torch.no_grad()
    def forward_flip_test(self, x: torch.Tensor, flip_pairs, shift_heatmap: bool = False) -> torch.Tensor:
        """mmpose's flip test (the `flip_test=True` of the reference configs, configs/ViTPose_common.py:124): heatmaps of the
        image and of its mirror image (flipped back, keypoint pairs swapped) averaged -- the published-AP protocol."""
        x = self._check_input(x)
        hm = self.forward(x)
        hm_f = self.flip_back(self.forward(torch.flip(x, dims=[3])), flip_pairs, shift_heatmap)
        return (hm + hm_f) * 0.5

    def _call_on_stream(self, tensors, call) -> None:
        """Runs `call(stream)` on the caller's current stream; on the legacy default stream (which cannot be captured into a
        CUDA graph) on a side stream ordered after / before it by two event waits, so small batches get graph replay."""
        with torch.cuda.device(self._device):
            cur = torch.cuda.current_stream(self._device)
            if cur.cuda_stream == 0:
                if self._side is None:
                    self._side = torch.cuda.Stream(self._device)
                self._side.wait_stream(cur)
                for t in tensors:
                    if t is not None:
                        t.record_stream(self._side)
                _lib.check(call(C.c_void_p(self._side.cuda_stream)))
                cur.wait_stream(self._side)
            else:
                _lib.check(call(C.c_void_p(cur.cuda_stream)))

    @torch.no_grad()
    def infer_crops(self, x: torch.Tensor, org_wh: torch.Tensor, return_heatmaps: bool = False):
        """Batched crops -> keypoints [B,K,3] (y, x, score) in crop pixels + flat argmax [B,K].
        org_wh int32 [B,2] = each crop's (width, height) before the resize to 192x256.  With flip test on (set_flip_test)
        the keypoints and the returned heatmaps are those of the flip-test average; B <= max_batch // 2."""
        x = self._check_input(x, self.batch_limit)
        B = x.shape[0]
        org = torch.as_tensor(org_wh).to(device=x.device, dtype=torch.int32).contiguous()
        if tuple(org.shape) != (B, 2):
            raise ValueError(f"org_wh must be [B,2], got {tuple(org.shape)}")
        kp = torch.empty((B, self.num_keypoints, 3), dtype=torch.float32, device=x.device)
        idx = torch.empty((B, self.num_keypoints), dtype=torch.int32, device=x.device)
        hm = torch.empty((B, self.num_keypoints, HM_H, HM_W), dtype=torch.float32, device=x.device) if return_heatmaps else None
        self._call_on_stream((x, org, kp, idx, hm), lambda st: _lib.lib().vpb_infer(
            self._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), B, C.c_void_p(kp.data_ptr()),
            C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()) if hm is not None else None, st))
        return (kp, idx, hm) if return_heatmaps else (kp, idx)

    def infer_host(self, crops: np.ndarray, org_wh: np.ndarray, kpts_out: np.ndarray | None = None,
                   idx_out: np.ndarray | None = None):
        """HOST buffers in, HOST keypoints out through the C ABI (vpb_infer_host): H2D + path + D2H + sync."""
        self._ensure()
        crops = np.ascontiguousarray(crops, np.float32)
        org = np.ascontiguousarray(org_wh, np.int32)
        B = crops.shape[0]
        if crops.shape[1:] != (3, IMG_H, IMG_W) or org.shape != (B, 2):
            raise ValueError("crops [B,3,256,192] float32 and org_wh [B,2] int32 expected")
        kp = kpts_out if kpts_out is not None else np.empty((B, self.num_keypoints, 3), np.float32)
        idx = idx_out if idx_out is not None else np.empty((B, self.num_keypoints), np.int32)
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().vpb_infer_host(self._handle, crops.ctypes.data_as(C.c_void_p), org.ctypes.data_as(C.c_void_p), B,
                                                 kp.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p), self._stream()))
        return kp, idx

    def submit_host(self, crops: np.ndarray, org_wh: np.ndarray, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int) -> None:
        """Asynchronous vpb_submit_host: the arrays must be C-contiguous float32 / int32, stay alive and unmodified until
        wait_host(slot); pinned memory (torch.Tensor.pin_memory().numpy()) gives real copy/compute overlap."""
        self._ensure()
        B = crops.shape[0]
        if crops.dtype != np.float32 or org_wh.dtype != np.int32 or kpts_out.dtype != np.float32 or idx_out.dtype != np.int32:
            raise TypeError("submit_host takes float32 crops / keypoints and int32 org_wh / idx")
        if crops.shape[1:] != (3, IMG_H, IMG_W) or org_wh.shape != (B, 2) or kpts_out.shape != (B, self.num_keypoints, 3) \
                or idx_out.shape != (B, self.num_keypoints) or not all(a.flags.c_contiguous for a in (crops, org_wh, kpts_out, idx_out)):
            raise ValueError("submit_host: wrong shapes or non-contiguous arrays")
        with torch.cuda.device(self._device):
            _lib.check(_lib.lib().vpb_submit_host(self._handle, crops.ctypes.data_as(C.c_void_p), org_wh.ctypes.data_as(C.c_void_p), B,
                                                  kpts_out.ctypes.data_as(C.c_void_p), idx_out.ctypes.data_as(C.c_void_p), int(slot)))

    # ---------------------------------------------------------------------------------------- frame-level calls (SURVEY 8 f1/f2)
    def _check_frame(self, frame: torch.Tensor, bboxes, limit: "int | None" = None) -> "tuple[torch.Tensor, torch.Tensor]":
        self._ensure()
        if not isinstance(frame, torch.Tensor) or frame.dtype != torch.uint8 or frame.dim() != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be a uint8 RGB tensor [H,W,3]")
        dev = torch.device("cuda", self._device)
        if not frame.is_cuda:
            frame = frame.to(dev, non_blocking=True)
        if frame.device.index != self._device:
            raise ValueError(f"frame lives on {frame.device}, the engine on cuda:{self._device}")
        bb = torch.as_tensor(bboxes)
        if bb.is_floating_point():
            bb = bb.round()                                  # easy_ViTPose/inference.py:253 (round half to even, like numpy)
        bb = bb.to(device=dev, dtype=torch.int32).reshape(-1, 4).contiguous()
        limit = self.max_batch if limit is None else limit
        if bb.shape[0] > limit:
            raise ValueError(f"{bb.shape[0]} boxes exceed {limit} (max_batch={self.max_batch}, flip test {'on' if self._flip else 'off'})")
        return frame.contiguous(), bb

    def preprocess(self, frame: torch.Tensor, bboxes, pad_bbox: int = 10):
        """uint8 RGB frame [H,W,3] (CUDA) + boxes [n,4] (x0,y0,x1,y1) -> (crops f32 [n,3,256,192], org_wh i32 [n,2],
        offs_yx i32 [n,2]): box padding/clipping, pad_image and pre_img of the reference in one kernel
        (easy_ViTPose/inference.py:259-265,314-318).  Raises ValueError for a box that is empty after clipping."""
        frame, bb = self._check_frame(frame, bboxes)
        n = bb.shape[0]
        dev = frame.device
        crops = torch.empty((n, 3, IMG_H, IMG_W), dtype=torch.float32, device=dev)
        org = torch.empty((n, 2), dtype=torch.int32, device=dev)
        offs = torch.empty((n, 2), dtype=torch.int32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        if n:
            with torch.cuda.device(self._device):
                _lib.check(_lib.lib().vpb_preprocess(C.c_void_p(frame.data_ptr()), frame.shape[0], frame.shape[1], 0,
                                                     C.c_void_p(bb.data_ptr()), n, int(pad_bbox), C.c_void_p(crops.data_ptr()),
                                                     C.c_void_p(org.data_ptr()), C.c_void_p(offs.data_ptr()),
                                                     C.c_void_p(status.data_ptr()), self._stream()))
            if int(status.item()) & 1:
                raise ValueError("a box is empty after padding and clipping to the frame")
        return crops, org, offs

    def frame_status(self) -> int:
        """Status word of the device-side frame calls since the last query (bit 0: a box was empty after padding and
        clipping).  Synchronises the device and clears the word (vpb_frame_status)."""
        self._ensure()
        st = C.c_int32(0)
        _lib.check(_lib.lib().vpb_frame_status(self._handle, C.byref(st)))
        return int(st.value)

    def infer_frame(self, frame: torch.Tensor, bboxes, check: bool = False):
        """uint8 RGB frame [H,W,3] (CUDA) + boxes [n,4] -> (kpts f32 [n,K,3] (y, x, score) in FRAME pixels, idx i32 [n,K]):
        the whole per-person loop of VitInference.inference (easy_ViTPose/inference.py:258-272) as one enqueue, no host sync.
        A box that is empty after clipping only sets the engine's status word (frame_status()); `check=True` synchronises
        and raises ValueError like the reference does (pad_image / cv2.resize on an empty crop).  Honours the flip test
        (set_flip_test): then n <= max_batch // 2."""
        frame, bb = self._check_frame(frame, bboxes, self.batch_limit)
        n = bb.shape[0]
        kp = torch.empty((n, self.num_keypoints, 3), dtype=torch.float32, device=frame.device)
        idx = torch.empty((n, self.num_keypoints), dtype=torch.int32, device=frame.device)
        if n:
            self._call_on_stream((frame, bb, kp, idx), lambda st: _lib.lib().vpb_infer_frame(
                self._handle, C.c_void_p(frame.data_ptr()), frame.shape[0], frame.shape[1], C.c_void_p(bb.data_ptr()), n,
                C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), st))
            if check and self.frame_status() & 1:
                raise ValueError("a box is empty after padding and clipping to the frame")
        return kp, idx

    @staticmethod
    def _host_frame_args(frame: np.ndarray, bboxes: np.ndarray):
        if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be a uint8 RGB array [H,W,3]")
        bb = np.asarray(bboxes)
        if bb.dtype.kind == "f":
            bb = bb.round()
        return np.ascontiguousarray(frame), np.ascontiguousarray(bb.reshape(-1, 4), np.int32)

    def infer_frame_host(self, frame: np.ndarray, bboxes: np.ndarray):
        """HOST frame + boxes in, HOST keypoints out (vpb_infer_frame_host): H2D of the uint8 frame, the path, D2H, sync.
        More than batch_limit boxes (max_batch, or max_batch // 2 with flip test on) are processed in chunks."""
        self._ensure()
        frame, bb = self._host_frame_args(frame, bboxes)
        n = bb.shape[0]
        kp = np.empty((n, self.num_keypoints, 3), np.float32)
        idx = np.empty((n, self.num_keypoints), np.int32)
        with torch.cuda.device(self._device):
            for s in range(0, n, self.batch_limit):
                m = min(self.batch_limit, n - s)
                _lib.check_value(_lib.lib().vpb_infer_frame_host(
                    self._handle, frame.ctypes.data_as(C.c_void_p), frame.shape[0], frame.shape[1], bb[s:s + m].ctypes.data_as(C.c_void_p), m,
                    kp[s:s + m].ctypes.data_as(C.c_void_p), idx[s:s + m].ctypes.data_as(C.c_void_p), self._stream()))
        return kp, idx

    def submit_frame_host(self, frame: np.ndarray, bboxes: np.ndarray, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int) -> None:
        """Asynchronous vpb_submit_frame_host (wait with wait_host(slot)): uint8 frame [H,W,3], int32 boxes [n,4] (already
        rounded), float32 kpts_out [n,K,3], int32 idx_out [n,K]; all C-contiguous, alive and unmodified until the wait."""
        self._ensure()
        n = bboxes.shape[0]
        if frame.dtype != np.uint8 or bboxes.dtype != np.int32 or kpts_out.dtype != np.float32 or idx_out.dtype != np.int32:
            raise TypeError("submit_frame_host takes a uint8 frame, int32 boxes / idx and float32 keypoints")
        if frame.ndim != 3 or frame.shape[2] != 3 or bboxes.shape != (n, 4) or kpts_out.shape != (n, self.num_keypoints, 3) \
                or idx_out.shape != (n, self.num_keypoints) or not all(a.flags.c_contiguous for a in (frame, bboxes, kpts_out, idx_out)):
            raise ValueError("submit_frame_host: wrong shapes or non-contiguous arrays")
        with torch.cuda.device(self._device):
            _lib.check_value(_lib.lib().vpb_submit_frame_host(
                self._handle, frame.ctypes.data_as(C.c_void_p), frame.shape[0], frame.shape[1], bboxes.ctypes.data_as(C.c_void_p), n,
                kpts_out.ctypes.data_as(C.c_void_p), idx_out.ctypes.data_as(C.c_void_p), int(slot)))

    # ---------------------------------------------------------------------------------------- multi-frame calls
    def _device_frame(self, j: int, frame: torch.Tensor) -> torch.Tensor:
        if not isinstance(frame, torch.Tensor) or frame.dtype != torch.uint8 or frame.dim() != 3 or frame.shape[2] != 3:
            raise ValueError(f"frame {j} must be a uint8 RGB tensor [H,W,3]")
        if not frame.is_cuda:
            frame = frame.to(torch.device("cuda", self._device), non_blocking=True)
        if frame.device.index != self._device:
            raise ValueError(f"frame {j} lives on {frame.device}, the engine on cuda:{self._device}")
        if frame.stride(2) != 1 or frame.stride(1) != 3 or frame.stride(0) < 3 * frame.shape[1]:
            frame = frame.contiguous()                       # rows of packed pixels at any pitch are read in place
        return frame

    @staticmethod
    def _host_frame(j: int, frame: np.ndarray) -> np.ndarray:
        if not isinstance(frame, np.ndarray) or frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError(f"frame {j} must be a uint8 RGB array [H,W,3]")
        if frame.strides[2] != 1 or frame.strides[1] != 3 or frame.strides[0] < 3 * frame.shape[1]:
            frame = np.ascontiguousarray(frame)
        return frame

    @staticmethod
    def _round_boxes(bboxes) -> np.ndarray:
        bb = np.asarray(bboxes)
        if bb.dtype.kind == "f":
            bb = bb.round()                                  # easy_ViTPose/inference.py:253 (round half to even)
        return np.ascontiguousarray(bb.reshape(-1, 4), np.int32)

    def _device_boxes(self, bboxes) -> "list[torch.Tensor]":
        dev = torch.device("cuda", self._device)
        boxes = []
        for b in bboxes:                                     # rounded as _check_frame does; device boxes stay on the device
            b = torch.as_tensor(b)
            if b.is_floating_point():
                b = b.round()
            boxes.append(b.to(device=dev, dtype=torch.int32).reshape(-1, 4))
        return boxes

    def _frame_table(self, frames, struct, layout, host: bool):
        """-> (the frames or planes to keep alive, every frame's `struct` fields before num_boxes), as numpy arrays for the
        host forms and as device tensors otherwise; `layout` names the layout of VpbFrameYuv frames."""
        if struct is _lib.VpbFrameYuv:
            return self._yuv_host_table(frames, layout) if host else self._yuv_device_table(frames, layout)
        if struct is _lib.VpbFrameNv12:                      # the YUV tables' nv12 planes ("NV12" as the messages spell it)
            keep, rows = self._yuv_host_table(frames, "NV12") if host else self._yuv_device_table(frames, "NV12")
            return keep, [(p[0], y_pitch, p[1], uv_pitch, h, w) for p, y_pitch, uv_pitch, h, w in rows]
        if host:
            frames = [self._host_frame(j, f) for j, f in enumerate(frames)]
            return frames, [(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in frames]
        frames = [self._device_frame(j, f) for j, f in enumerate(frames)]
        return frames, [(f.data_ptr(), f.shape[0], f.shape[1], f.stride(0)) for f in frames]

    def _frames_call(self, name: str, fmt: tuple, frames, bboxes=None, affine=None, heads=None, *, host: bool, rotate,
                     check: bool = False, status: int = 0, message: str = "", struct=_lib.VpbFrame, layout=None):
        """The body of the multi-frame calls: entry point `name` with format ints `fmt` over `struct` frames and per-frame
        `bboxes` or `affine` = (matrices, centres, scales), grouped by `heads` (plan_head_calls) when given.  The host forms
        stage numpy arrays and run synchronously; on the device, `check` turns bit `status` into ValueError(message)."""
        named = [(bboxes, "box arrays")] if affine is None else list(zip(affine, ("matrix arrays", "centre arrays", "scale arrays")))
        named = [(frames, "frames")] + named + ([] if heads is None else [(heads, "head arrays")])
        if any(len(a) != len(frames) for a, _ in named):
            sizes = [f"{len(a)} {what}" for a, what in named]
            raise ValueError(" but ".join(sizes) if len(sizes) == 2 else ", ".join(sizes))
        rot = _rotations(rotate, len(frames))
        keep, table = self._frame_table(frames, struct, layout, host)
        if affine is not None:
            counts, M, CS = self._affine_args(*affine, validate=not host)   # the engine checks host values
            staged = [M.cpu().numpy(), CS.cpu().numpy()] if host else [M, CS]
        else:
            boxes = [self._round_boxes(b) for b in bboxes] if host else self._device_boxes(bboxes)
            counts = [len(b) for b in boxes]
            staged = [np.concatenate(boxes) if boxes else np.zeros((0, 4), np.int32)] if host else \
                [torch.cat(boxes) if boxes else torch.zeros((0, 4), dtype=torch.int32, device=torch.device("cuda", self._device))]
        if heads is None:
            chunks, K = plan_frame_chunks(counts, self.batch_limit), self.num_keypoints
        else:
            ents, order, chunks = plan_head_calls(counts, heads, len(self.head_keypoints), self.batch_limit)
            rot, table = [rot[j] for j, _, _ in ents], [table[j] for j, _, _ in ents]   # one row per entry: its frame's
            hv, K = np.array([k for _, _, k in ents], np.int32), self.num_keypoints_max
        n = len(staged[0])
        if host:
            staged = [np.ascontiguousarray(a if heads is None else a[order]) for a in staged]
            new = np.empty if heads is None else np.zeros
            kp, idx = new((n, K, 3), np.float32), new((n, K), np.int32)
        else:
            dev = torch.device("cuda", self._device)
            staged = [(a if heads is None else a.index_select(0, torch.as_tensor(order, device=a.device))).to(dev) for a in staged]
            new = torch.empty if heads is None else torch.zeros
            kp, idx = new((n, K, 3), dtype=torch.float32, device=dev), new((n, K), dtype=torch.int32, device=dev)
        ptr = (lambda a: a.ctypes.data_as(C.c_void_p)) if host else (lambda t: C.c_void_p(t.data_ptr()))
        s = 0                                                # first box of the current call
        with torch.cuda.device(self._device) if host else contextlib.nullcontext():
            for chunk in chunks:
                arr = _frame_array(table, chunk, struct, rot)
                ha = [] if heads is None else [np.ascontiguousarray(hv[:len(arr)])]
                args = (self._handle, arr, len(arr), *fmt, *(h.ctypes.data_as(C.c_void_p) for h in ha),
                        *(ptr(a[s:]) for a in staged + [kp, idx]))
                if host:
                    _lib.check_value(getattr(_lib.lib(), name)(*args, self._stream()))
                else:
                    self._call_on_stream(keep + staged + [kp, idx], lambda st: getattr(_lib.lib(), name)(*args, st))
                s += sum(e - b for _, b, e in chunk)
        if check and n and self.frame_status() & status:
            raise ValueError(message)
        if heads is not None:
            if not host:
                return self._per_frame(ents, counts, kp, idx)
            k_t, i_t = self._per_frame(ents, counts, torch.from_numpy(kp), torch.from_numpy(idx))
            return [k.numpy() for k in k_t], [i.numpy() for i in i_t]
        if not counts:
            return [], []
        if host:
            split = np.cumsum(counts)[:-1]
            return np.split(kp, split), np.split(idx, split)
        return list(kp.split(counts)), list(idx.split(counts))

    @staticmethod
    def _per_frame(ents, counts, kp, idx):
        outs_k = [kp.new_zeros((c,) + tuple(kp.shape[1:])) for c in counts]
        outs_i = [idx.new_zeros((c,) + tuple(idx.shape[1:])) for c in counts]
        s = 0
        for j, sel, _ in ents:
            outs_k[j][sel] = kp[s:s + len(sel)]
            outs_i[j][sel] = idx[s:s + len(sel)]
            s += len(sel)
        return outs_k, outs_i

    def _submit_frames(self, name: str, fmt: tuple, frames, bboxes, table, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int,
                       rotate, struct) -> None:
        """The body of the submit_frames*_host calls: the length and `rotate` checks, table() (the method's own frame and box
        checks -> (the arrays to keep alive, every frame's `struct` fields before num_boxes)), the outputs check and ONE
        asynchronous call of engine entry point `name` over all frames, with the format ints `fmt`."""
        if len(frames) != len(bboxes):
            raise ValueError(f"{len(frames)} frames but {len(bboxes)} box arrays")
        rot = _rotations(rotate, len(frames))
        keep, rows = table()                                 # keep: what the rows point into, alive over the call
        bb = np.ascontiguousarray(np.concatenate(bboxes, 0) if len(bboxes) else np.zeros((0, 4), np.int32))
        n = bb.shape[0]
        if kpts_out.dtype != np.float32 or idx_out.dtype != np.int32 or kpts_out.shape != (n, self.num_keypoints, 3) \
                or idx_out.shape != (n, self.num_keypoints) or not (kpts_out.flags.c_contiguous and idx_out.flags.c_contiguous):
            raise ValueError(f"{name[len('vpb_'):]}: outputs must be C-contiguous float32 [n,K,3] and int32 [n,K]")
        arr = (struct * len(rows))(*[struct(*row, len(b), r) for row, b, r in zip(rows, bboxes, rot)])
        with torch.cuda.device(self._device):
            _lib.check_value(getattr(_lib.lib(), name)(
                self._handle, arr, len(arr), *fmt, bb.ctypes.data_as(C.c_void_p), kpts_out.ctypes.data_as(C.c_void_p),
                idx_out.ctypes.data_as(C.c_void_p), int(slot)))

    def infer_frames(self, frames, bboxes, check: bool = False, rotate=0):
        """The people of several frames in as few engine calls as the limits allow: uint8 RGB frames [H_j,W_j,3] (CUDA) and
        per-frame boxes [n_j,4] -> (list of kpts f32 [n_j,K,3] (y, x, score) in frame j's pixels, list of idx i32 [n_j,K]).
        Bit-identical to one infer_frame per frame.  Calls hold at most batch_limit boxes from at most 64 frames with boxes; a
        frame's boxes may be split over two calls.  A frame whose rows are packed pixels at a larger pitch (a column slice
        of a wider image) is read in place.  Empty boxes set the status word; `check=True` synchronises and raises.
        `rotate` (every frame method takes it): 0, 90, 180 or 270 degrees counter-clockwise for all frames or one per frame
        (_rotations); frame j is then seen as cv2.rotate turns it, and its boxes and keypoints are in that view's pixels."""
        self._ensure()
        return self._frames_call("vpb_infer_frames", (), frames, bboxes, host=False, rotate=rotate, check=check, status=1,
                                 message=_EMPTY_BOX)

    def infer_frames_host(self, frames, bboxes, rotate=0):
        """HOST form of infer_frames (vpb_infer_frames_host, synchronous): numpy frames [H_j,W_j,3] uint8 and per-frame boxes
        -> (list of kpts [n_j,K,3], list of idx [n_j,K]) numpy arrays, chunked as infer_frames.  A box that is empty after
        padding and clipping raises ValueError naming its frame."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_host", (), frames, bboxes, host=True, rotate=rotate)

    def submit_frames_host(self, frames, bboxes, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int, rotate=0) -> None:
        """Asynchronous vpb_submit_frames_host, ONE engine call (wait with wait_host(slot)): uint8 frames [H_j,W_j,3] whose
        rows are packed pixels (any row pitch), per-frame int32 boxes [n_j,4] (already rounded), and the concatenated outputs
        float32 kpts_out [n,K,3] / int32 idx_out [n,K], n = sum n_j <= batch_limit, at most 64 frames with boxes.  Frames and
        outputs must stay alive and unmodified until the wait (pinned memory: real copy / compute overlap).  `rotate` as
        infer_frames."""
        self._ensure()

        def table():
            for j, (f, b) in enumerate(zip(frames, bboxes)):
                if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 \
                        or f.strides[2] != 1 or f.strides[1] != 3 or f.strides[0] < 3 * f.shape[1]:
                    raise ValueError(f"frame {j}: uint8 [H,W,3] with packed pixels in each row expected")
                if b.dtype != np.int32 or b.ndim != 2 or b.shape[1] != 4:
                    raise TypeError(f"boxes of frame {j}: int32 [n,4] expected")
            return frames, [(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in frames]
        self._submit_frames("vpb_submit_frames_host", (), frames, bboxes, table, kpts_out, idx_out, slot, rotate, _lib.VpbFrame)

    # ---------------------------------------------------------------------------------------- affine top-down crops
    @staticmethod
    def _affine_args(mats, centers=None, scales=None, validate: bool = True):
        """Per-frame matrices [n_j,2,3] | [n_j,6] and (optionally) centres / scales [n_j,2] -> (counts, mats f64 [n,6],
        cs f32 [n,4] or None), concatenated in frame order on the device they came from.  With `validate`, host-side values
        are checked here (a CUDA tensor is left to the engine's status word: checking it would synchronise)."""
        if centers is not None and not (len(centers) == len(scales) == len(mats)):
            raise ValueError(f"{len(mats)} matrix arrays, {len(centers)} centre arrays, {len(scales)} scale arrays")
        counts, ms, css = [], [], []
        for j, m in enumerate(mats):
            m = torch.as_tensor(m)
            if not ((m.dim() == 3 and tuple(m.shape[1:]) == (2, 3)) or (m.dim() == 2 and m.shape[1] == 6)):
                raise ValueError(f"matrices of frame {j}: [n,2,3] or [n,6] expected, got {tuple(m.shape)}")
            m = m.reshape(-1, 6).to(torch.float64)
            if validate and not m.is_cuda and not bool(torch.isfinite(m).all()):
                raise ValueError(f"matrices of frame {j}: non-finite entries")
            counts.append(m.shape[0])
            ms.append(m)
            if centers is None:
                continue
            c = torch.as_tensor(centers[j]).to(device=m.device, dtype=torch.float32).reshape(-1, 2)
            s = torch.as_tensor(scales[j]).to(device=m.device, dtype=torch.float32).reshape(-1, 2)
            if c.shape[0] != m.shape[0] or s.shape[0] != m.shape[0]:
                raise ValueError(f"frame {j}: {m.shape[0]} matrices, {c.shape[0]} centres, {s.shape[0]} scales")
            if validate and not m.is_cuda and not (bool(torch.isfinite(c).all()) and bool(torch.isfinite(s).all()) and bool((s > 0).all())):
                raise ValueError(f"frame {j}: finite centres and scales > 0 expected")
            css.append(torch.cat([c, s], 1))
        if not ms:
            return [], torch.zeros((0, 6), dtype=torch.float64), None if centers is None else torch.zeros((0, 4))
        return counts, torch.cat(ms).contiguous(), None if centers is None else torch.cat(css).contiguous()

    def preprocess_affine(self, frames, mats, rotate=0) -> torch.Tensor:
        """Affine top-down crops: uint8 RGB frames [H_j,W_j,3] and per-frame matrices [n_j,2,3] (what cv2.warpAffine takes,
        image -> 192x256 crop) -> crops f32 [n,3,256,192] on the device, boxes in frame order.  Bit-exact with
        cv2.warpAffine(frame, M, (192, 256), INTER_LINEAR) + torchvision ToTensor / Normalize (datasets/COCO.py:289-302)."""
        self._ensure()
        if len(frames) != len(mats):
            raise ValueError(f"{len(frames)} frames but {len(mats)} matrix arrays")
        rot = _rotations(rotate, len(frames))
        frames, table = self._frame_table(frames, _lib.VpbFrame, None, host=False)
        dev = torch.device("cuda", self._device)
        counts, M, _ = self._affine_args(mats)
        M = M.to(dev)
        n = M.shape[0]
        crops = torch.empty((n, 3, IMG_H, IMG_W), dtype=torch.float32, device=dev)
        s = 0
        with torch.cuda.device(self._device):
            for chunk in plan_frame_chunks(counts, max(n, 1)):       # only the 64-frame table limits a call
                arr = _frame_array(table, chunk, rot=rot)
                _lib.check(_lib.lib().vpb_preprocess_affine(arr, len(arr), C.c_void_p(M[s:].data_ptr()),
                                                            C.c_void_p(crops[s:].data_ptr()), self._stream()))
                s += sum(e - b for _, b, e in chunk)
        return crops

    def infer_affine(self, frames, mats, centers, scales, check: bool = False, rotate=0):
        """The top-down path of mmpose-style evaluation on the device: frames [H_j,W_j,3] uint8 (CUDA), per-frame matrices
        [n_j,2,3], centres [n_j,2] and scales [n_j,2] in PIXELS (topdown_args gives all three) -> (list of kpts f32 [n_j,K,3]
        (y, x, score), list of idx i32 [n_j,K]): the warp fused into the patch gather, the forward and
        keypoints_from_heatmaps(c, s, use_udp=True), in the coordinates transform_preds gives (image pixels for unrotated
        matrices).  Chunked like infer_frames; honours the flip test.  Host-side matrices / scales are checked here; CUDA
        ones set bit 1 of the status word, which `check=True` turns into a ValueError."""
        self._ensure()
        return self._frames_call("vpb_infer_affine", (), frames, affine=(mats, centers, scales), host=False, rotate=rotate,
                                 check=check, status=2, message=_BAD_AFFINE)

    def infer_affine_host(self, frames, mats, centers, scales, rotate=0):
        """HOST form of infer_affine (vpb_infer_affine_host, synchronous): numpy frames and per-frame matrices / centres /
        scales -> (list of kpts [n_j,K,3], list of idx [n_j,K]) numpy arrays.  A non-finite matrix entry or a scale <= 0
        raises ValueError naming the box."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_host", (), frames, affine=(mats, centers, scales), host=True, rotate=rotate)

    # ---------------------------------------------------------------------------------------- NV12 video frames
    # Each frame is a uint8 [3H/2, W] array with the planes stacked or a (y [H,W], uv [H/2,W]) pair (nv12_planes); matrix is
    # "bt601" (cv2's COLOR_YUV2RGB_NV12) or "bt709", both limited range.  Every call is bit-identical to its RGB twin on the
    # converted frames (oracle/nv12_oracle.py: nv12_to_rgb); only the pixels under the boxes are converted, on the fly.
    def _device_plane(self, j: int, p) -> torch.Tensor:
        if not isinstance(p, torch.Tensor):
            p = torch.from_numpy(np.ascontiguousarray(p))
        if not p.is_cuda:
            p = p.to(torch.device("cuda", self._device), non_blocking=True)
        if p.device.index != self._device:
            raise ValueError(f"frame {j} lives on {p.device}, the engine on cuda:{self._device}")
        if p.stride(1) != 1 or p.stride(0) < p.shape[1]:
            p = p.contiguous()                               # rows of bytes at any pitch are read in place
        return p

    def infer_frames_nv12(self, frames, bboxes, matrix: str = "bt601", check: bool = False, rotate=0):
        """infer_frames on NV12 frames (vpb_infer_frames_nv12): CUDA (or host, copied over) NV12 frames and per-frame boxes
        [n_j,4] -> (list of kpts f32 [n_j,K,3], list of idx i32 [n_j,K]).  Chunked, flip test and status word as infer_frames."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_nv12", (_yuv_matrix(matrix),), frames, bboxes, host=False, rotate=rotate,
                                 check=check, status=1, message=_EMPTY_BOX, struct=_lib.VpbFrameNv12)

    def infer_frames_nv12_host(self, frames, bboxes, matrix: str = "bt601", rotate=0):
        """HOST form of infer_frames_nv12 (vpb_infer_frames_nv12_host, synchronous): numpy NV12 frames, per-frame boxes ->
        numpy (kpts, idx) lists.  Each frame is staged packed at 1.5 B per pixel; an empty box raises ValueError."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_nv12_host", (_yuv_matrix(matrix),), frames, bboxes, host=True, rotate=rotate,
                                 struct=_lib.VpbFrameNv12)

    def submit_frames_nv12_host(self, frames, bboxes, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int,
                                matrix: str = "bt601", rotate=0) -> None:
        """Asynchronous vpb_submit_frames_nv12_host, ONE engine call (wait with wait_host(slot)): the pipelined video form of
        submit_frames_host for numpy NV12 frames whose rows are contiguous bytes (any row pitch).  Frames, boxes (int32
        [n_j,4], already rounded) and outputs must stay alive and unmodified until the wait."""
        self._ensure()
        mat = _yuv_matrix(matrix)

        def table():
            planes = []
            for j, (f, b) in enumerate(zip(frames, bboxes)):
                y, uv = nv12_planes(f, f"frame {j}")
                if not isinstance(y, np.ndarray) or y.strides[1] != 1 or uv.strides[1] != 1 or y.strides[0] < y.shape[1] \
                        or uv.strides[0] < uv.shape[1]:
                    raise ValueError(f"frame {j}: numpy NV12 planes with contiguous bytes in each row expected")
                if b.dtype != np.int32 or b.ndim != 2 or b.shape[1] != 4:
                    raise TypeError(f"boxes of frame {j}: int32 [n,4] expected")
                planes.append((y, uv))
            return planes, [(y.ctypes.data, y.strides[0], uv.ctypes.data, uv.strides[0], y.shape[0], y.shape[1]) for y, uv in planes]
        self._submit_frames("vpb_submit_frames_nv12_host", (mat,), frames, bboxes, table, kpts_out, idx_out, slot, rotate,
                            _lib.VpbFrameNv12)

    def infer_affine_nv12(self, frames, mats, centers, scales, matrix: str = "bt601", check: bool = False, rotate=0):
        """infer_affine on NV12 frames (vpb_infer_affine_nv12): the warp reads the NV12 planes and converts each tap."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_nv12", (_yuv_matrix(matrix),), frames, affine=(mats, centers, scales),
                                 host=False, rotate=rotate, check=check, status=2, message=_BAD_AFFINE, struct=_lib.VpbFrameNv12)

    def infer_affine_nv12_host(self, frames, mats, centers, scales, matrix: str = "bt601", rotate=0):
        """HOST form of infer_affine_nv12 (vpb_infer_affine_nv12_host, synchronous), checked as infer_affine_host."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_nv12_host", (_yuv_matrix(matrix),), frames, affine=(mats, centers, scales),
                                 host=True, rotate=rotate, struct=_lib.VpbFrameNv12)

    # ---------------------------------------------------------------------------------------- YUV video frames
    # Every call takes layout = "i420" | "yv12" | "nv12" | "nv21" | "yuyv" | "uyvy" (the frame forms of yuv_planes), matrix =
    # "bt601" | "bt709" and full_range (False: limited range as cv2's COLOR_YUV2RGB_*; True: JPEG range as COLOR_YCrCb2RGB).
    # Every call is bit-identical to its RGB twin on the converted frames (oracle/yuv_oracle.py: yuv_to_rgb); only the pixels
    # under the boxes are converted, on the fly.
    @staticmethod
    def _yuv_row(planes, h: int, w: int):
        """-> the vpb_frame_yuv fields before num_boxes: ((plane pointers), y pitch, chroma pitch, h, w)"""
        dev = isinstance(planes[0], torch.Tensor)
        ptr = (lambda p: p.data_ptr()) if dev else (lambda p: p.ctypes.data)
        pitch = (lambda p: p.stride(0)) if dev else (lambda p: p.strides[0])
        ptrs = tuple(ptr(p) for p in planes) + (None,) * (3 - len(planes))
        return ptrs, pitch(planes[0]), pitch(planes[1]) if len(planes) > 1 else 0, h, w

    def _yuv_device_table(self, frames, layout: str):
        """-> (the plane tensors to keep alive, the _yuv_row of every frame)"""
        keep, table = [], []
        for j, f in enumerate(frames):
            planes, h, w = yuv_planes(f, layout, f"frame {j}")
            planes = [self._device_plane(j, p) for p in planes]
            if len(planes) == 3 and planes[1].stride(0) != planes[2].stride(0):
                planes[1:] = [p.contiguous() for p in planes[1:]]    # U and V share one pitch
            keep += planes
            table.append(self._yuv_row(planes, h, w))
        return keep, table

    @staticmethod
    def _yuv_host_table(frames, layout: str, copy: bool = True):
        """-> (the numpy planes to keep alive, the _yuv_row of every frame).  Planes whose rows are not contiguous bytes, and
        U / V planes of different pitches, are copied packed; with copy=False (the pipelined form) they raise ValueError."""
        keep, table = [], []
        for j, f in enumerate(frames):
            planes, h, w = yuv_planes(f, layout, f"frame {j}")
            if not isinstance(planes[0], np.ndarray):
                raise ValueError(f"frame {j}: numpy {layout} planes expected")
            planes = list(planes)
            for i, p in enumerate(planes):
                if p.strides[1] != 1 or p.strides[0] < p.shape[1]:
                    if not copy:
                        raise ValueError(f"frame {j}: numpy {layout} planes with contiguous bytes in each row expected")
                    planes[i] = np.ascontiguousarray(p)
            if len(planes) == 3 and planes[1].strides[0] != planes[2].strides[0]:
                if not copy:
                    raise ValueError(f"frame {j}: the U and V planes must share one row pitch")
                planes[1:] = [np.ascontiguousarray(p) for p in planes[1:]]
            keep += planes
            table.append(ViTPose._yuv_row(planes, h, w))
        return keep, table

    def infer_frames_yuv(self, frames, bboxes, layout: str = "i420", matrix: str = "bt601", full_range: bool = False,
                         check: bool = False, rotate=0):
        """infer_frames on YUV frames (vpb_infer_frames_yuv): CUDA (or host, copied over) frames and per-frame boxes [n_j,4] ->
        (list of kpts f32 [n_j,K,3], list of idx i32 [n_j,K]).  Chunked, flip test and status word as infer_frames."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_yuv", _yuv_format(layout, matrix, full_range), frames, bboxes, host=False,
                                 rotate=rotate, check=check, status=1, message=_EMPTY_BOX, struct=_lib.VpbFrameYuv, layout=layout)

    def infer_frames_yuv_host(self, frames, bboxes, layout: str = "i420", matrix: str = "bt601", full_range: bool = False, rotate=0):
        """HOST form of infer_frames_yuv (vpb_infer_frames_yuv_host, synchronous): numpy frames, per-frame boxes -> numpy
        (kpts, idx) lists.  Each frame is staged packed (1.5 B per pixel for 4:2:0, 2 B for 4:2:2); an empty box raises
        ValueError."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_yuv_host", _yuv_format(layout, matrix, full_range), frames, bboxes, host=True,
                                 rotate=rotate, struct=_lib.VpbFrameYuv, layout=layout)

    def submit_frames_yuv_host(self, frames, bboxes, kpts_out: np.ndarray, idx_out: np.ndarray, slot: int, layout: str = "i420",
                               matrix: str = "bt601", full_range: bool = False, rotate=0) -> None:
        """Asynchronous vpb_submit_frames_yuv_host, ONE engine call (wait with wait_host(slot)): the pipelined video form of
        submit_frames_host for numpy YUV frames whose planes have contiguous bytes in each row (any row pitch; U and V of one
        pitch).  Frames, boxes (int32 [n_j,4], already rounded) and outputs must stay alive and unmodified until the wait."""
        self._ensure()
        fmt = _yuv_format(layout, matrix, full_range)

        def table():
            for j, b in enumerate(bboxes):
                if b.dtype != np.int32 or b.ndim != 2 or b.shape[1] != 4:
                    raise TypeError(f"boxes of frame {j}: int32 [n,4] expected")
            return self._yuv_host_table(frames, layout, copy=False)
        self._submit_frames("vpb_submit_frames_yuv_host", fmt, frames, bboxes, table, kpts_out, idx_out, slot, rotate,
                            _lib.VpbFrameYuv)

    def infer_affine_yuv(self, frames, mats, centers, scales, layout: str = "i420", matrix: str = "bt601", full_range: bool = False,
                         check: bool = False, rotate=0):
        """infer_affine on YUV frames (vpb_infer_affine_yuv): the warp reads the planes and converts each tap."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_yuv", _yuv_format(layout, matrix, full_range), frames,
                                 affine=(mats, centers, scales), host=False, rotate=rotate, check=check, status=2,
                                 message=_BAD_AFFINE, struct=_lib.VpbFrameYuv, layout=layout)

    def infer_affine_yuv_host(self, frames, mats, centers, scales, layout: str = "i420", matrix: str = "bt601",
                              full_range: bool = False, rotate=0):
        """HOST form of infer_affine_yuv (vpb_infer_affine_yuv_host, synchronous), checked as infer_affine_host."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_yuv_host", _yuv_format(layout, matrix, full_range), frames,
                                 affine=(mats, centers, scales), host=True, rotate=rotate, struct=_lib.VpbFrameYuv, layout=layout)

    # ---------------------------------------------------------------------------------------- several heads (datasets)
    @staticmethod
    def _segments(chunk):
        return (_lib.VpbSegment * len(chunk))(*[_lib.VpbSegment(h, e - s) for h, s, e in chunk])

    def _head_indices(self, j: "int | None", heads, n: int) -> np.ndarray:
        h = np.asarray(heads.cpu() if isinstance(heads, torch.Tensor) else heads).reshape(-1)
        if h.size != n:
            raise ValueError(f"{n} boxes but {h.size} head indices" + ("" if j is None else f" in frame {j}"))
        group_by_head(h, len(self.head_keypoints))           # range check
        return h.astype(np.int64)

    @torch.no_grad()
    def infer_crops_heads(self, x: torch.Tensor, org_wh: torch.Tensor, heads, return_heatmaps: bool = False):
        """infer_crops with a keypoint head per crop (heads [B] ints, 0..H-1): the crops are grouped by head (stable) and run
        in as few vpb_infer_heads calls as batch_limit allows, each with one backbone pass.  Returns (kpts [B,K_max,3],
        idx [B,K_max][, heatmaps [B,K_max,64,48]]) in the caller's crop order; crop c of head j fills rows 0..K_j-1, the rest
        are zeros.  Bit-identical to infer_crops on single-head engines loaded with split_vitpose_plus's checkpoints."""
        x = self._check_input(x, 1 << 30)                  # any batch: the calls are chunked below
        n = x.shape[0]
        h = self._head_indices(None, heads, n)
        org = torch.as_tensor(org_wh).to(device=x.device, dtype=torch.int32).contiguous()
        if tuple(org.shape) != (n, 2):
            raise ValueError(f"org_wh must be [B,2], got {tuple(org.shape)}")
        order, counts = group_by_head(h, len(self.head_keypoints))
        perm = torch.as_tensor(order, device=x.device)
        xs, org = x.index_select(0, perm).contiguous(), org.index_select(0, perm).contiguous()
        Km = self.num_keypoints_max
        kp = torch.zeros((n, Km, 3), dtype=torch.float32, device=x.device)
        idx = torch.zeros((n, Km), dtype=torch.int32, device=x.device)
        hm = torch.zeros((n, Km, HM_H, HM_W), dtype=torch.float32, device=x.device) if return_heatmaps else None
        s = 0
        for chunk in plan_frame_chunks(counts, self.batch_limit):
            segs = self._segments(chunk)
            self._call_on_stream((xs, org, kp, idx, hm), lambda st: _lib.lib().vpb_infer_heads(
                self._handle, C.c_void_p(xs[s:].data_ptr()), C.c_void_p(org[s:].data_ptr()), segs, len(segs),
                C.c_void_p(kp[s:].data_ptr()), C.c_void_p(idx[s:].data_ptr()), C.c_void_p(hm[s:].data_ptr()) if hm is not None else None, st))
            s += sum(e - b for _, b, e in chunk)
        inv = torch.as_tensor(_inverse(order), device=x.device)
        out = (kp.index_select(0, inv), idx.index_select(0, inv))
        return out + (hm.index_select(0, inv),) if return_heatmaps else out

    def infer_frames_heads(self, frames, bboxes, heads, check: bool = False, rotate=0):
        """infer_frames with a keypoint head per box (heads: per frame an int array [n_j]): the boxes are grouped by head
        (stable; a frame appears once per head it uses) and run through vpb_infer_frames_heads in calls of at most batch_limit
        boxes and 64 entries.  Returns per frame kpts f32 [n_j,K_max,3] (y, x, score) in that frame's pixels and idx i32
        [n_j,K_max], rows K_j.. of a head-j box zero."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_heads", (), frames, bboxes, heads=heads, host=False, rotate=rotate, check=check,
                                 status=1, message=_EMPTY_BOX)

    def infer_frames_heads_host(self, frames, bboxes, heads, rotate=0):
        """HOST form of infer_frames_heads (vpb_infer_frames_heads_host, synchronous): numpy frames, per-frame boxes and
        head indices -> (list of kpts [n_j,K_max,3], list of idx [n_j,K_max]) numpy arrays.  An empty box raises ValueError."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_heads_host", (), frames, bboxes, heads=heads, host=True, rotate=rotate)

    def infer_affine_heads(self, frames, mats, centers, scales, heads, check: bool = False, rotate=0):
        """infer_affine with a keypoint head per box (heads: per frame an int array [n_j]): the boxes are grouped by head (stable;
        a frame appears once per head it uses) and run through vpb_infer_affine_heads in calls of at most batch_limit boxes and
        64 entries (plan_head_calls).  Each call decodes a segment (a run of one head) as one keypoints_from_heatmaps(c, s,
        use_udp=True) call.  Returns per frame kpts f32 [n_j,K_max,3] (y, x, score) and idx i32 [n_j,K_max], rows K_j.. of a
        head-j box zero.  Honours the flip test set by set_flip_test_heads."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_heads", (), frames, affine=(mats, centers, scales), heads=heads, host=False,
                                 rotate=rotate, check=check, status=2, message=_BAD_AFFINE)

    def infer_affine_heads_host(self, frames, mats, centers, scales, heads, rotate=0):
        """HOST form of infer_affine_heads (vpb_infer_affine_heads_host, synchronous): numpy frames and per-frame matrices /
        centres / scales / head indices -> (list of kpts [n_j,K_max,3], list of idx [n_j,K_max]) numpy arrays.  A non-finite
        matrix entry or a scale <= 0 raises ValueError."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_heads_host", (), frames, affine=(mats, centers, scales), heads=heads, host=True,
                                 rotate=rotate)

    # the multi-head calls on YUV frames: frames as the _yuv calls take them, everything else as their RGB twins above
    def infer_frames_heads_yuv(self, frames, bboxes, heads, layout: str = "i420", matrix: str = "bt601", full_range: bool = False,
                               check: bool = False, rotate=0):
        """infer_frames_heads on YUV frames (vpb_infer_frames_heads_yuv)."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_heads_yuv", _yuv_format(layout, matrix, full_range), frames, bboxes, heads=heads,
                                 host=False, rotate=rotate, check=check, status=1, message=_EMPTY_BOX, struct=_lib.VpbFrameYuv,
                                 layout=layout)

    def infer_frames_heads_yuv_host(self, frames, bboxes, heads, layout: str = "i420", matrix: str = "bt601", full_range: bool = False, rotate=0):
        """HOST form of infer_frames_heads_yuv (vpb_infer_frames_heads_yuv_host, synchronous)."""
        self._ensure()
        return self._frames_call("vpb_infer_frames_heads_yuv_host", _yuv_format(layout, matrix, full_range), frames, bboxes, heads=heads,
                                 host=True, rotate=rotate, struct=_lib.VpbFrameYuv, layout=layout)

    def infer_affine_heads_yuv(self, frames, mats, centers, scales, heads, layout: str = "i420", matrix: str = "bt601",
                               full_range: bool = False, check: bool = False, rotate=0):
        """infer_affine_heads on YUV frames (vpb_infer_affine_heads_yuv)."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_heads_yuv", _yuv_format(layout, matrix, full_range), frames,
                                 affine=(mats, centers, scales), heads=heads, host=False, rotate=rotate, check=check, status=2,
                                 message=_BAD_AFFINE, struct=_lib.VpbFrameYuv, layout=layout)

    def infer_affine_heads_yuv_host(self, frames, mats, centers, scales, heads, layout: str = "i420", matrix: str = "bt601",
                                    full_range: bool = False, rotate=0):
        """HOST form of infer_affine_heads_yuv (vpb_infer_affine_heads_yuv_host, synchronous)."""
        self._ensure()
        return self._frames_call("vpb_infer_affine_heads_yuv_host", _yuv_format(layout, matrix, full_range), frames,
                                 affine=(mats, centers, scales), heads=heads, host=True, rotate=rotate, struct=_lib.VpbFrameYuv,
                                 layout=layout)

    def wait_host(self, slot: int) -> None:
        _lib.check(_lib.lib().vpb_wait_host(self._handle, int(slot)))

    def kernel_launches(self, batch: int) -> int:
        self._ensure()
        return int(_lib.lib().vpb_kernel_launches(self._handle, batch))

    def cached_graphs(self, mixed: bool = False) -> "tuple[int, int]":
        """(layouts kept, of which captured) of the engine's CUDA-graph cache: the single-head calls', or with `mixed` the
        multi-head calls' (vpb_cached_graphs)."""
        self._ensure()
        n, c = C.c_int32(0), C.c_int32(0)
        _lib.check(_lib.lib().vpb_cached_graphs(self._handle, 1 if mixed else 0, C.byref(n), C.byref(c)))
        return int(n.value), int(c.value)

    def device_bytes(self) -> int:
        """Device memory the engine holds: packed weights, workspace and staging buffers (vpb_device_bytes)."""
        self._ensure()
        return int(_lib.lib().vpb_device_bytes(self._handle))

    def set_option(self, name: str, value: int) -> None:
        self._ensure()
        _lib.check(_lib.lib().vpb_set_option(self._handle, name.encode(), int(value)))

    def profile_collect(self) -> dict:
        """{kernel class: (total ms, launches)} since the last call; needs set_option('profile', 1)."""
        self._ensure()
        L = _lib.lib()
        n = L.vpb_profile_classes()
        ms = (C.c_float * n)()
        cnt = (C.c_int32 * n)()
        _lib.check(L.vpb_profile_collect(self._handle, ms, cnt))
        return {L.vpb_profile_class_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n)}

    def read_buffer(self, name: str, shape, dtype) -> torch.Tensor:
        """Debug: synchronous copy of an internal activation buffer (see vpb_read_buffer)."""
        self._ensure()
        tdtype = torch.bfloat16 if dtype == "bf16" else torch.float32
        out = torch.empty(tuple(shape), dtype=tdtype)
        _lib.check(_lib.lib().vpb_read_buffer(self._handle, name.encode(), C.c_void_p(out.data_ptr()), out.numel() * out.element_size()))
        return out

    def __del__(self):
        try:
            if self._handle:
                _lib.lib().vpb_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
