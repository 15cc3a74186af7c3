"""Keypoint smoothing on the device: the reference's `OneEuroFilter` (vit_utils/post_processing/one_euro_filter.py) kept per
track id, for many video streams in one `vpb_smoother_update` step, equal to the reference class composed per id as
float64 values (oracle/one_euro_oracle.py states the composition).

`DeviceOneEuro(S, K, ...)` holds S streams, each a map track id -> filter.  `update(kpts_list, ids_list)` takes one [n, K, 3]
keypoint array and n ids per stream and returns what the filters return, float64 [n, K, 2] (y, x); `update_device(kpts,
counts, ids)` keeps everything on the device (no synchronisation) and smooths the (y, x) columns of the concatenated
float32 [n, K, 3] keypoints in place, the tensor `draw.draw_poses` takes.  With `fps` given, the clock defaults to each
stream's update count, so t_e counts frames since an id was last seen; with `fps=None` (realtime) every update needs a clock
in seconds, which stands in for the reference's `time()`.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

SMOOTH_MAX = 128                     # VPB_SMOOTH_MAX: rows and live ids per stream
STATUS_DUPLICATE_ID = 1              # VPB_SMOOTH_DUPLICATE_ID: an id twice in one stream's update
STATUS_OVER_CAPACITY = 2             # VPB_SMOOTH_OVER_CAPACITY: more than SMOOTH_MAX rows or live ids, or rows past n


class DeviceOneEuro:
    """S streams of reference `OneEuroFilter(x0, dx0, min_cutoff, beta, d_cutoff, fps)` objects, one per track id, on one
    CUDA device.  An id absent from more than `max_gap` updates in a row is forgotten and starts a new filter when it comes
    back.  Calls run on the device's current torch stream."""

    def __init__(self, num_streams: int, num_keypoints: int, min_cutoff: float = 1.7, beta: float = 0.3, d_cutoff: float = 30.0,
                 fps=None, dx0: float = 0.0, max_gap: int = 30, device=None):
        import torch
        self.num_streams, self.num_keypoints, self.max_gap = int(num_streams), int(num_keypoints), int(max_gap)
        self.min_cutoff, self.beta, self.d_cutoff, self.dx0 = float(min_cutoff), float(beta), float(d_cutoff), float(dx0)
        self.fps = None if fps is None else float(fps)
        if self.fps is not None and not self.fps > 0:
            raise ValueError(f"fps must be > 0 (None for realtime mode), not {fps}")
        dev = torch.device("cuda") if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ValueError(f"DeviceOneEuro runs on a CUDA device, not {dev}")
        self.device = torch.device("cuda", torch.cuda.current_device() if dev.index is None else dev.index)
        self._handle = None
        h = C.c_void_p()
        _lib.check_value(_lib.lib().vpb_smoother_create(self.num_streams, self.num_keypoints, self.min_cutoff, self.beta,
                                                        self.d_cutoff, self.fps if self.fps is not None else 0.0, self.dx0,
                                                        self.max_gap, self.device.index, C.byref(h)))
        self._handle = h

    def __del__(self):
        if getattr(self, "_handle", None) is not None and _lib._lib is not None:
            _lib._lib.vpb_smoother_destroy(self._handle)
            self._handle = None

    @property
    def realtime(self) -> bool:
        return self.fps is None

    def _stream(self):
        import torch
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check(self, name, t, dtype, shape):
        import torch
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and tuple(t.shape) == shape and t.is_contiguous()
                and t.device == self.device):
            raise ValueError(f"{name} must be a contiguous {dtype} {list(shape)} tensor on {self.device}")

    # ---------------------------------------------------------------------------------------------------- device form
    def update_device(self, kpts, counts, ids, clock=None, out=None):
        """kpts CUDA float32 [n, K, 3] (y, x, score), the rows of every stream concatenated, stream s holding the next
        counts[s] (CUDA int32 [S]); ids CUDA int32 [n], each row's track id; clock CUDA float64 [S] (required in realtime
        mode; in fps mode None = each stream's update count); out CUDA float64 [n, K, 2] or None.  Smooths kpts' (y, x) in
        place (rounded to float32, scores untouched) and, when given, writes the float64 result to `out`, which it returns.
        Enqueued on the current stream with no synchronisation (and can be captured in a CUDA graph)."""
        import torch
        S, K = self.num_streams, self.num_keypoints
        n = kpts.shape[0] if isinstance(kpts, torch.Tensor) and kpts.dim() == 3 else -1
        self._check("kpts", kpts, torch.float32, (n, K, 3))
        self._check("counts", counts, torch.int32, (S,))
        self._check("ids", ids, torch.int32, (n,))
        if clock is None:
            if self.realtime:
                raise ValueError("realtime mode (fps=None) needs a clock")
        else:
            self._check("clock", clock, torch.float64, (S,))
        if out is not None:
            self._check("out", out, torch.float64, (n, K, 2))
        self._update(kpts, n, counts, ids, clock, out)
        return out

    def _update(self, kpts, n, counts, ids, clock, out):
        ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())           # noqa: E731
        _lib.check_value(_lib.lib().vpb_smoother_update(self._handle, ptr(kpts), n, ptr(counts), ptr(ids), ptr(clock), ptr(out),
                                                        self._stream()))

    # ---------------------------------------------------------------------------------------------------- host form
    def update(self, kpts_list, ids_list, clock=None):
        """One update of every stream: kpts_list[s] [n_s, K, 3] (y, x, score) float32 (numpy or CUDA), ids_list[s] n_s track
        ids, clock None or one value per stream (seconds; required in realtime mode) -> list of float64 numpy [n_s, K, 2],
        what the stream's filters return.  One upload, one update, one read-back.  A stream the update skips (see
        STATUS_*) comes back as NaN rows; check() raises for it."""
        import torch
        S, K = self.num_streams, self.num_keypoints
        if len(kpts_list) != S or len(ids_list) != S:
            raise ValueError(f"{len(kpts_list)} keypoint arrays and {len(ids_list)} id lists for {S} streams")
        if clock is None and self.realtime:
            raise ValueError("realtime mode (fps=None) needs a clock")
        if clock is not None and len(clock) != S:
            raise ValueError(f"{len(clock)} clock values for {S} streams")
        kps, ids = [], []
        for s, (k, i) in enumerate(zip(kpts_list, ids_list)):
            a = k.detach().cpu().numpy() if isinstance(k, torch.Tensor) else np.asarray(k)
            if a.size == 0:
                a = a.reshape(0, K, 3)
            if a.dtype != np.float32 or a.ndim != 3 or a.shape[1:] != (K, 3):
                raise ValueError(f"stream {s}: keypoints must be float32 [n, {K}, 3], not {a.dtype} {list(a.shape)}")
            i = np.asarray(i.cpu() if isinstance(i, torch.Tensor) else i).reshape(-1)
            if len(i) != len(a):
                raise ValueError(f"stream {s}: {len(i)} ids for {len(a)} keypoint rows")
            if len(i) and (i.dtype.kind not in "iu" or i.min() < -2 ** 31 or i.max() >= 2 ** 31):
                raise ValueError(f"stream {s}: ids must be int32 integers")
            kps.append(a)
            ids.append(i.astype(np.int32))
        n = sum(len(a) for a in kps)
        # one int32 host buffer: kpts f32 [n, K, 3] | ids [n] | counts [S] | clock f64 [S] (8-byte aligned)
        nk, pad = n * K * 3, (n * K * 3 + n + S) % 2
        buf = np.zeros(nk + n + S + pad + 2 * S, np.int32)
        buf[:nk].view(np.float32)[:] = np.concatenate(kps).reshape(-1) if n else []
        buf[nk:nk + n] = np.concatenate(ids) if n else []
        buf[nk + n:nk + n + S] = [len(a) for a in kps]
        if clock is not None:
            buf[nk + n + S + pad:].view(np.float64)[:] = np.asarray(clock, np.float64)
        dev = torch.from_numpy(buf).to(self.device)
        kpts = dev[:nk].view(torch.float32).view(n, K, 3)
        out = torch.full((n, K, 2), float("nan"), dtype=torch.float64, device=self.device)
        self._update(kpts, n, dev[nk + n:nk + n + S], dev[nk:nk + n], None if clock is None else dev[nk + n + S + pad:].view(torch.float64),
                     out)
        res = out.cpu().numpy()
        offs = np.cumsum([0] + [len(a) for a in kps])
        return [res[offs[s]:offs[s + 1]] for s in range(S)]

    # ---------------------------------------------------------------------------------------------------- state
    def reset(self, stream=None):
        """Forget the filters and the update count of one stream (None: every stream)."""
        s = -1 if stream is None else int(stream)
        _lib.check_value(_lib.lib().vpb_smoother_reset(self._handle, s, self._stream()))

    def status(self) -> int:
        """The STATUS_* bits raised since the last query (synchronises, then clears them)."""
        v = C.c_int32(0)
        _lib.check(_lib.lib().vpb_smoother_status(self._handle, C.byref(v)))
        return int(v.value)

    def check(self) -> None:
        """Raises ValueError if an update since the last query skipped a stream (see STATUS_*)."""
        st = self.status()
        if st:
            why = []
            if st & STATUS_DUPLICATE_ID:
                why.append("a stream names a track id twice in one update")
            if st & STATUS_OVER_CAPACITY:
                why.append(f"a stream has more than {SMOOTH_MAX} rows or live ids, or its rows run past the keypoints")
            raise ValueError("smoother skipped a stream: " + "; ".join(why))
