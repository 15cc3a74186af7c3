"""Pose overlay on the device: the pose layer of `VitInference.draw()` (easy_ViTPose/inference.py:283-312,
vit_utils/visualization.py:360-481) for the people of many frames in one `vpb_draw_poses` call, bit-exact with cv2.

`draw_poses` draws in place on CUDA uint8 [H, W, 3] frames, on the current stream, with a workspace torch allocates;
`plan` checks and packs the host-side arguments (no GPU needed); `reference_palettes` gives the two BGR colour tables
`draw()` passes ('gist_rainbow' sampled at 10 points for the keypoints, 'jet' at 8 for the limbs).
"""
from __future__ import annotations

import ctypes as C
import functools
from typing import NamedTuple

import numpy as np

from . import _lib

MAX_LIMBS = 128                      # vpb_draw_poses table limits
MAX_COLORS = 64
MAX_RADIUS = 1023

# matplotlib's published segment data (matplotlib/_cm.py) for the two colormaps draw() uses.  'jet' is given per channel as
# (x, y0, y1) rows; 'gist_rainbow' as (x, colour) stops, which LinearSegmentedColormap.from_list turns into rows (x, c, c).
_JET = {
    "red": ((0.00, 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1.00, 0.5, 0.5)),
    "green": ((0.000, 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.640, 1, 1), (0.910, 0, 0), (1.000, 0, 0)),
    "blue": ((0.00, 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1.00, 0, 0)),
}
_GIST_RAINBOW = ((0.000, (1.00, 0.00, 0.16)), (0.030, (1.00, 0.00, 0.00)), (0.215, (1.00, 1.00, 0.00)), (0.400, (0.00, 1.00, 0.00)),
                 (0.586, (0.00, 1.00, 1.00)), (0.770, (0.00, 0.00, 1.00)), (0.954, (1.00, 0.00, 1.00)), (1.000, (1.00, 0.00, 0.75)))
_LUTSIZE = 256


def _segment_lut(rows) -> np.ndarray:
    """matplotlib.colors._create_lookup_table(256, rows, gamma=1)."""
    a = np.asarray(rows, np.float64)
    x, y0, y1 = a[:, 0], a[:, 1], a[:, 2]
    xind = np.linspace(0, 1, _LUTSIZE)
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


class RestatedColormap:
    """A 256-entry LinearSegmentedColormap called on floats in [0, 1], as matplotlib evaluates it: RGBA rows of the LUT at
    index int(x * 256), with 1.0 mapped to 255.  Has no `.colors`, like the segment-data colormaps it restates."""

    def __init__(self, name: str):
        if name == "jet":
            data = _JET
        elif name == "gist_rainbow":
            data = {c: [(v, col[i], col[i]) for v, col in _GIST_RAINBOW] for i, c in enumerate(("red", "green", "blue"))}
        else:
            raise ValueError(f"no restatement of colormap {name!r}")
        self.name = name
        self._lut = np.ones((_LUTSIZE, 4))
        for i, c in enumerate(("red", "green", "blue")):
            self._lut[:, i] = _segment_lut(data[c])

    def __call__(self, x):
        xa = np.array(x, np.float64) * _LUTSIZE
        xa[xa == _LUTSIZE] = _LUTSIZE - 1
        xa = np.clip(xa, -1, _LUTSIZE).astype(int)
        return self._lut[np.clip(xa, 0, _LUTSIZE - 1)]


def get_cmap(name: str):
    """matplotlib's colormap when matplotlib is importable, else the restatement."""
    try:
        import matplotlib
        return matplotlib.colormaps[name]
    except ImportError:
        return RestatedColormap(name)


def palette(name: str, samples: int) -> np.ndarray:
    """The reference's `except AttributeError` branch (visualization.py:383-385, 424-426): u8 [samples, 3] BGR."""
    return np.round(np.array(get_cmap(name)(np.linspace(0, 1, samples))) * 255).astype(np.uint8)[:, -2::-1].copy()


@functools.lru_cache(maxsize=None)
def reference_palettes():
    """(point_bgr u8 [10, 3], limb_bgr u8 [8, 3]): the tables VitInference.draw() passes to draw_points_and_skeleton
    (computed once; read-only)."""
    out = palette("gist_rainbow", 10), palette("jet", 8)
    for t in out:
        t.setflags(write=False)
    return out


class DrawPlan(NamedTuple):
    canvases: object                 # (VpbCanvas * num_frames) with data pointers to fill in
    channel_order: int
    k: int
    limbs: np.ndarray                # i32 [E, 2]
    point_bgr: np.ndarray            # u8 [P, 3]
    limb_bgr: np.ndarray             # u8 [L, 3]
    n: int
    radius: int
    threshold: float


def plan(shapes, pitches, n: int, k: int, counts, skeleton, point_colors=None, limb_colors=None, confidence_threshold: float = 0.5,
         channel_order: str = "rgb", radius: int = 0) -> DrawPlan:
    """Checks and packs what vpb_draw_poses takes from the host.  `shapes` are the frames' (H, W), `pitches` their row
    pitches in bytes, kpts are [n, k, 3], frame j owns the next counts[j] people.  Raises ValueError where the call would fail."""
    if channel_order not in _lib.DRAW_CHANNEL_ORDERS:
        raise ValueError(f"channel_order must be one of {sorted(_lib.DRAW_CHANNEL_ORDERS)}, not {channel_order!r}")
    counts = [int(c) for c in counts]
    if len(counts) != len(shapes) or len(pitches) != len(shapes):
        raise ValueError(f"{len(shapes)} frames, {len(counts)} counts and {len(pitches)} pitches")
    if any(c < 0 for c in counts) or sum(counts) != n:
        raise ValueError(f"counts {counts} must be >= 0 and add up to the {n} keypoint rows")
    if k < 1:
        raise ValueError(f"keypoints per person must be >= 1, not {k}")
    limbs = np.asarray(skeleton, np.int64).reshape(-1, 2) if len(skeleton) else np.zeros((0, 2), np.int64)
    if len(limbs) > MAX_LIMBS or (limbs.size and (limbs.min() < 0 or limbs.max() >= k)):
        raise ValueError(f"skeleton: at most {MAX_LIMBS} limbs with indices in [0, {k})")
    if point_colors is None or limb_colors is None:
        pts, lms = reference_palettes()
        point_colors = pts if point_colors is None else point_colors
        limb_colors = lms if limb_colors is None else limb_colors
    tabs = []
    for name, t in (("point_colors", point_colors), ("limb_colors", limb_colors)):
        t = np.asarray(t)
        if t.ndim != 2 or t.shape[1] != 3 or not 1 <= len(t) <= MAX_COLORS or t.min(initial=0) < 0 or t.max(initial=0) > 255:
            raise ValueError(f"{name}: 1..{MAX_COLORS} BGR rows of 0..255, got shape {t.shape}")
        tabs.append(np.ascontiguousarray(t, np.uint8))
    if radius > MAX_RADIUS:
        raise ValueError(f"radius {radius} above {MAX_RADIUS}")
    frames_with_people = sum(c > 0 for c in counts)
    if frames_with_people > _lib.MAX_FRAMES:
        raise ValueError(f"{frames_with_people} frames with people; at most {_lib.MAX_FRAMES} per call")
    canv = (_lib.VpbCanvas * max(len(shapes), 1))()
    for j, ((h, w), pitch, c) in enumerate(zip(shapes, pitches, counts)):
        if c and (h < 1 or w < 1 or pitch < 3 * w):
            raise ValueError(f"frame {j}: {h} x {w} with row pitch {pitch}")
        canv[j].height, canv[j].width, canv[j].pitch_bytes, canv[j].num_people = int(h), int(w), int(pitch), c
    return DrawPlan(canv, _lib.DRAW_CHANNEL_ORDERS[channel_order], int(k), np.ascontiguousarray(limbs, np.int32), tabs[0], tabs[1], int(n),
                    int(radius), float(confidence_threshold))


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def draw_poses(frames, kpts, counts, skeleton, person_index=None, point_colors=None, limb_colors=None, confidence_threshold: float = 0.5,
               channel_order: str = "rgb", radius: int = 0):
    """Draws, in place on CUDA uint8 [H, W, 3] tensors (any row pitch, packed pixels), the skeleton and keypoints of every
    person: kpts f32 [n, K, 3] (y, x, score) in frame pixels on the same device, frame j owning the next counts[j] rows;
    person_index [n] colour index per person (None = position within its frame, as draw() without a tracker); colours BGR
    (None = reference_palettes()); channel_order "rgb" or "bgr" is the frames' layout.  Enqueued on the current stream;
    returns the frames."""
    import torch
    if not isinstance(kpts, torch.Tensor) or not kpts.is_cuda or kpts.dtype != torch.float32 or kpts.dim() != 3 or kpts.shape[2] != 3:
        raise ValueError("kpts must be a CUDA float32 tensor [n, K, 3]")
    kpts = kpts.contiguous()
    for j, f in enumerate(frames):
        if (not isinstance(f, torch.Tensor) or f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3 or f.stride(2) != 1
                or f.stride(1) != 3 or f.device != kpts.device):
            raise ValueError(f"frame {j} must be a uint8 [H, W, 3] tensor with packed pixels on {kpts.device}")
    p = plan([tuple(f.shape[:2]) for f in frames], [f.stride(0) for f in frames], kpts.shape[0], kpts.shape[1], counts, skeleton,
             point_colors, limb_colors, confidence_threshold, channel_order, radius)
    if p.n == 0:
        return frames
    for j, f in enumerate(frames):
        p.canvases[j].data = f.data_ptr()
    pidx = None
    if person_index is not None:
        pidx = torch.as_tensor(person_index, dtype=torch.int32, device=kpts.device).contiguous()
        if pidx.shape != (p.n,):
            raise ValueError(f"person_index must have {p.n} entries, not shape {tuple(pidx.shape)}")
    lib = _lib.lib()
    with torch.cuda.device(kpts.device):
        _launch(lib, p, kpts, pidx, len(frames))
    return frames


def _launch(lib, p: DrawPlan, kpts, pidx, num_frames: int):
    import torch
    ws = torch.empty(max(int(lib.vpb_draw_workspace_bytes(p.n, p.k, len(p.limbs))), 16), dtype=torch.uint8, device=kpts.device)
    _lib.check_value(lib.vpb_draw_poses(p.canvases, num_frames, p.channel_order, C.c_void_p(kpts.data_ptr()), p.k,
                                        C.c_void_p(pidx.data_ptr()) if pidx is not None else None, _ptr(p.limbs), len(p.limbs),
                                        _ptr(p.point_bgr), len(p.point_bgr), _ptr(p.limb_bgr), len(p.limb_bgr), p.radius,
                                        p.threshold, C.c_void_p(ws.data_ptr()),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
