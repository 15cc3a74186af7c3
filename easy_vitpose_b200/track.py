"""SORT on the device: easy_ViTPose/sort.py's `Sort` for many video streams in one `vpb_tracker_update` step, with the
reference's ids and boxes (equal as float64 values; oracle/sort_oracle.py states the contract).

`DeviceSort(S, max_age, min_hits, iou_threshold)` holds S streams, each one reference `Sort`.  `update(dets_list)` takes one
[n, 5] detection array per stream (numpy or CUDA, float32 or float64) and returns what each stream's `Sort.update` returns;
`update_device(dets, counts)` keeps everything on the device (no synchronisation) and also returns the rows' int32 boxes,
the input `ViTPose.infer_frames` takes.  Ids come from one counter per tracker (`next_id`, the reference's class-wide
`KalmanBoxTracker.count`): within an update new tracks take ids in stream order, within a stream in creation order.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

TRACK_MAX = 128                      # VPB_TRACK_MAX: detections and live tracks per stream
STATUS_BAD_ROW = 1                   # VPB_TRACK_BAD_ROW: a non-finite row, or x2 <= x1 or y2 <= y1
STATUS_OVER_CAPACITY = 2             # VPB_TRACK_OVER_CAPACITY: more than TRACK_MAX detections or live tracks


class DeviceSort:
    """S reference `Sort(max_age, min_hits, iou_threshold)` objects on one CUDA device.  Calls run on the device's current
    torch stream."""

    def __init__(self, num_streams: int, max_age: int = 1, min_hits: int = 3, iou_threshold: float = 0.3, device=None):
        import torch
        self.num_streams = int(num_streams)
        self.max_age, self.min_hits, self.iou_threshold = int(max_age), int(min_hits), float(iou_threshold)
        dev = torch.device("cuda") if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ValueError(f"DeviceSort runs on a CUDA device, not {dev}")
        self.device = torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)
        self._handle = None
        h = C.c_void_p()
        _lib.check_value(_lib.lib().vpb_tracker_create(self.num_streams, self.max_age, self.min_hits, self.iou_threshold,
                                                       self.device.index, C.byref(h)))
        self._handle = h

    def __del__(self):
        if getattr(self, "_handle", None) is not None and _lib._lib is not None:
            _lib._lib.vpb_tracker_destroy(self._handle)
            self._handle = None

    def _stream(self):
        import torch
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ---------------------------------------------------------------------------------------------------- device form
    def update_device(self, dets, counts):
        """dets CUDA float64 [S, 128, 5] (stream s's first counts[s] rows), counts CUDA int32 [S] -> (rows f64 [S, 128, 6],
        boxes i32 [S, 128, 4], out_counts i32 [S]) CUDA tensors: stream s's first out_counts[s] rows are its Sort.update
        result.  Enqueued on the current stream with no synchronisation (and can be captured in a CUDA graph)."""
        import torch
        S = self.num_streams
        if not (isinstance(dets, torch.Tensor) and dets.is_cuda and dets.dtype == torch.float64 and tuple(dets.shape) == (S, TRACK_MAX, 5)
                and dets.is_contiguous() and dets.device == self.device):
            raise ValueError(f"dets must be a contiguous float64 [{S}, {TRACK_MAX}, 5] tensor on {self.device}")
        if not (isinstance(counts, torch.Tensor) and counts.is_cuda and counts.dtype == torch.int32 and tuple(counts.shape) == (S,)
                and counts.is_contiguous() and counts.device == self.device):
            raise ValueError(f"counts must be a contiguous int32 [{S}] tensor on {self.device}")
        rows, boxes, oc = self._views(self._out_buffer())
        self._update(dets, counts, rows, boxes, oc)
        return rows, boxes, oc

    def _out_buffer(self):
        import torch
        return torch.empty(self.num_streams * (TRACK_MAX * (12 + 4) + 1), dtype=torch.int32, device=self.device)

    def _views(self, out):
        """One int32 buffer as (rows f64 [S,128,6], boxes i32 [S,128,4], counts i32 [S]): one allocation, one read-back."""
        import torch
        S = self.num_streams
        r, b = S * TRACK_MAX * 12, S * TRACK_MAX * 4
        return out[:r].view(torch.float64).view(S, TRACK_MAX, 6), out[r:r + b].view(S, TRACK_MAX, 4), out[r + b:]

    def _update(self, dets, counts, rows, boxes, oc):
        _lib.check_value(_lib.lib().vpb_tracker_update(self._handle, C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()),
                                                       C.c_void_p(rows.data_ptr()), C.c_void_p(boxes.data_ptr()),
                                                       C.c_void_p(oc.data_ptr()), self._stream()))

    # ---------------------------------------------------------------------------------------------------- host form
    def pack(self, dets_list):
        """Per-stream [n_s, 5] arrays (numpy or CUDA, float32 or float64) -> (dets f64 [S, 128, 5], counts i32 [S]) on the
        device, with one upload for host arrays.  A stream with more than 128 rows keeps its true count (the update then
        skips it and sets STATUS_OVER_CAPACITY)."""
        import torch
        S = self.num_streams
        if len(dets_list) != S:
            raise ValueError(f"{len(dets_list)} detection arrays for {S} streams")
        shapes = []
        for s, d in enumerate(dets_list):
            shp = tuple(d.shape)
            if not ((len(shp) == 2 and shp[1] == 5) or (len(shp) in (1, 2) and shp[0] == 0)):
                raise ValueError(f"stream {s}: detections must be [n, 5], not {shp}")
            shapes.append(shp[0])
        buf = torch.zeros(S * TRACK_MAX * 5 * 2 + S, dtype=torch.int32)
        dets_h = buf[:S * TRACK_MAX * 10].view(torch.float64).view(S, TRACK_MAX, 5)
        counts_h = buf[S * TRACK_MAX * 10:]
        on_device = []
        for s, d in enumerate(dets_list):
            n = shapes[s]
            counts_h[s] = n
            if n == 0:
                continue
            if isinstance(d, torch.Tensor) and d.is_cuda:
                on_device.append((s, d))
                continue
            a = d.cpu().numpy() if isinstance(d, torch.Tensor) else np.asarray(d)
            if a.dtype not in (np.float32, np.float64):
                raise ValueError(f"stream {s}: detections must be float32 or float64, not {a.dtype}")
            m = min(n, TRACK_MAX)
            dets_h[s, :m] = torch.from_numpy(np.ascontiguousarray(a[:m], np.float64))
        dev = buf.to(self.device, non_blocking=False)
        dets = dev[:S * TRACK_MAX * 10].view(torch.float64).view(S, TRACK_MAX, 5)
        for s, d in on_device:
            if d.dtype not in (torch.float32, torch.float64):
                raise ValueError(f"stream {s}: detections must be float32 or float64, not {d.dtype}")
            m = min(d.shape[0], TRACK_MAX)
            dets[s, :m] = d[:m].to(device=self.device, dtype=torch.float64)
        return dets, dev[S * TRACK_MAX * 10:]

    def update(self, dets_list):
        """One Sort.update per stream: dets_list[s] [n_s, 5] (x1, y1, x2, y2, score), numpy or CUDA, float32 or float64 ->
        list of float64 numpy [m_s, 6] (x1, y1, x2, y2, score, id + 1).  One upload, one update, one read-back."""
        dets, counts = self.pack(dets_list)
        out = self._out_buffer()
        self._update(dets, counts, *self._views(out))
        rows, _, oc = self._views(out.cpu())
        rows = rows.numpy()
        return [rows[s, :c].copy() for s, c in enumerate(oc.tolist())]

    # ---------------------------------------------------------------------------------------------------- state
    def reset(self, stream=None):
        """Forget the tracks of one stream (None: every stream), as a new reference Sort; the id counter carries on."""
        s = -1 if stream is None else int(stream)
        _lib.check_value(_lib.lib().vpb_tracker_reset(self._handle, s, self._stream()))

    @property
    def next_id(self) -> int:
        """The id the next new track takes (KalmanBoxTracker.count); reading or setting it synchronises the device."""
        v = C.c_int64(0)
        _lib.check(_lib.lib().vpb_tracker_next_id(self._handle, C.byref(v)))
        return int(v.value)

    @next_id.setter
    def next_id(self, value: int) -> None:
        _lib.check_value(_lib.lib().vpb_tracker_set_next_id(self._handle, int(value)))

    def status(self) -> int:
        """The STATUS_* bits raised since the last query (synchronises, then clears them)."""
        v = C.c_int32(0)
        _lib.check(_lib.lib().vpb_tracker_status(self._handle, C.byref(v)))
        return int(v.value)

    def check(self) -> None:
        """Raises ValueError if an update since the last query skipped a stream (see STATUS_*)."""
        st = self.status()
        if st:
            why = []
            if st & STATUS_BAD_ROW:
                why.append("a detection row is not finite or has x2 <= x1 or y2 <= y1")
            if st & STATUS_OVER_CAPACITY:
                why.append(f"a stream has more than {TRACK_MAX} detections or live tracks")
            raise ValueError("tracker skipped a stream: " + "; ".join(why))
