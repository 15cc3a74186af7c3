"""The contract vpb_smoother_update is held to: the reference's `OneEuroFilter`
(easy_ViTPose/vit_utils/post_processing/one_euro_filter.py) kept per track id, for S streams.

The reference class is a single filter; nothing in the reference composes it per person.  `SmoothOracle` states the
composition, taking the filter class as an argument so that the same code runs the unmodified class
(`load_reference_one_euro()`) or `OneEuroNumpy`, the numpy restatement of its arithmetic written here.  Per stream there is
a map id -> (filter, c_last, u_last); update u (the stream's count of accepted updates, from 0) at clock c with rows
(id_i, x_i), x_i the float32 [K, 2] (y, x) columns of the engine's [K, 3] keypoints:

  1. forget every id absent from more than `max_gap` updates in a row (u - u_last - 1 > max_gap), so it starts a new filter
     if it comes back; max_gap = 0 drops an id on its first absence;
  2. a known id outputs filter(x_i, t_e).  fps mode (`fps` given): t_e = c - c_last as a Python float, c being the update
     count unless the caller gives a clock, so t_e counts frames since the id was last seen (the reference docstring's
     "skip frame count").  Realtime mode (fps=None): c is the caller's timestamp in seconds; the filter module's `time` is
     patched to return it, so the reference computes t_e = (c - c_last) * d_cutoff itself;
  3. a new id constructs filter(x_i, dx0, min_cutoff, beta, d_cutoff, fps) at clock c and outputs x_i unchanged;
  4. every id of the update takes c_last = c, u_last = u.

limit=True adds the device's rules: a stream whose count is above 128, that names an id twice, or that would hold more than
128 ids is left unchanged (no rows, update count kept) and raises `status` bits 1 (duplicate id) / 2 (over capacity).
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np

SMOOTH_MAX = 128
STATUS_DUPLICATE_ID = 1
STATUS_OVER_CAPACITY = 2

_NOW = [0.0]                      # the clock both filter classes read in realtime mode


def now() -> float:
    return _NOW[0]


class OneEuroNumpy:
    """The reference filter's arithmetic restated with numpy's promotion rules spelled out: x_prev starts as float32 (so the
    first x - x_prev is a float32 subtraction), every other quantity is float64, and each expression is evaluated in the
    reference's order.  Coordinates with x <= 0 give -10 (NaN is not masked)."""

    def __init__(self, x0, dx0=0.0, min_cutoff=1.7, beta=0.3, d_cutoff=30.0, fps=None):
        x0 = np.asarray(x0)
        self.shape = x0.shape
        self.min_cutoff, self.beta = float(min_cutoff), float(beta)
        self.realtime = fps is None
        self.deriv_cutoff = float(d_cutoff) if self.realtime else float(fps)
        self.skip = float(d_cutoff)
        self.x_prev = x0.astype(np.float32)
        self.dx_prev = np.full(self.shape, float(dx0))
        self.t_prev = now()

    @staticmethod
    def _factor(te, cutoff):
        r = (np.float64(2.0 * np.pi) * cutoff) * te
        return r / (r + 1.0)

    def __call__(self, x, t_e=1.0):
        x = np.asarray(x)
        assert x.shape == self.shape
        if self.realtime:
            t = now()
            t_e = (t - self.t_prev) * self.skip
            self.t_prev = t
        te = np.full(self.shape, float(t_e))
        a_d = self._factor(te, np.full(self.shape, self.deriv_cutoff))
        dx = np.subtract(x, self.x_prev) / te                 # float32 - float32 on the first call, float64 after
        dx_hat = a_d * dx + (1.0 - a_d) * self.dx_prev
        cutoff = self.min_cutoff + self.beta * np.abs(dx_hat)
        a = self._factor(te, cutoff)
        x_hat = a * x.astype(np.float64) + (1.0 - a) * self.x_prev.astype(np.float64)
        x_hat[x <= 0] = -10.0
        self.x_prev, self.dx_prev = x_hat, dx_hat
        return x_hat


def load_reference_one_euro():
    """The UNMODIFIED reference `OneEuroFilter` class, loaded from its file with the module's `time` replaced by `now`.
    Test infrastructure only; raises RuntimeError without the reference tree."""
    from oracle import ref_import
    path = os.path.join(ref_import.REF_PKG, "vit_utils", "post_processing", "one_euro_filter.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"reference one_euro_filter.py not found at {path}")
    sys.dont_write_bytecode = True
    spec = importlib.util.spec_from_file_location("_reference_one_euro_filter", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.time = now
    return mod.OneEuroFilter


class _Stream:
    def __init__(self):
        self.filters = {}             # id -> [filter, c_last, u_last]
        self.updates = 0


class SmoothOracle:
    """S streams of per-id filters of class `filter_cls` (default OneEuroNumpy), as the module docstring states."""

    def __init__(self, num_streams: int, min_cutoff: float = 1.7, beta: float = 0.3, d_cutoff: float = 30.0, fps=None,
                 dx0: float = 0.0, max_gap: int = 30, filter_cls=None, limit: bool = False):
        self.params = dict(dx0=float(dx0), min_cutoff=float(min_cutoff), beta=float(beta), d_cutoff=float(d_cutoff),
                           fps=None if fps is None else float(fps))
        self.max_gap = int(max_gap)
        self.cls = OneEuroNumpy if filter_cls is None else filter_cls
        self.streams = [_Stream() for _ in range(num_streams)]
        self.limit = limit
        self.status = 0

    @property
    def realtime(self) -> bool:
        return self.params["fps"] is None

    def reset(self, stream=None):
        for s in range(len(self.streams)) if stream is None else [stream]:
            self.streams[s] = _Stream()

    def update(self, kpts_list, ids_list, clock=None):
        """kpts_list: per stream float32 [n, K, 3] or [n, K, 2] (y, x[, score]); ids_list: per stream n ids; clock: None or
        one value per stream (required in realtime mode) -> per stream float64 [n, K, 2] (None for a skipped stream)."""
        S = len(self.streams)
        if len(kpts_list) != S or len(ids_list) != S:
            raise ValueError(f"{len(kpts_list)} keypoint arrays and {len(ids_list)} id lists for {S} streams")
        if self.realtime and clock is None:
            raise ValueError("realtime mode needs a clock")
        return [self._update(st, np.asarray(k), [int(i) for i in ids], None if clock is None else float(clock[s]))
                for s, (st, k, ids) in enumerate(zip(self.streams, kpts_list, ids_list))]

    def _update(self, st: _Stream, kpts, ids, clock):
        u = st.updates
        live = {i: v for i, v in st.filters.items() if u - v[2] - 1 <= self.max_gap}
        if self.limit:
            if len(ids) > SMOOTH_MAX:
                self.status |= STATUS_OVER_CAPACITY
                return None
            if len(set(ids)) != len(ids):
                self.status |= STATUS_DUPLICATE_ID
                return None
            if len(live) + sum(i not in live for i in ids) > SMOOTH_MAX:
                self.status |= STATUS_OVER_CAPACITY
                return None
        c = float(u) if clock is None else clock
        _NOW[0] = c
        K = kpts.shape[1] if kpts.ndim == 3 else 0
        out = np.zeros((len(ids), K, 2))
        for r, i in enumerate(ids):
            x = np.ascontiguousarray(kpts[r, :, :2], np.float32)
            if i in live:
                f, c_last, _ = live[i]
                out[r] = f(x) if self.realtime else f(x, float(c - c_last))
            else:
                f = self.cls(x, self.params["dx0"], self.params["min_cutoff"], self.params["beta"], self.params["d_cutoff"],
                             self.params["fps"])
                out[r] = x
            live[i] = [f, c, u]
        st.filters = live
        st.updates = u + 1
        return out
