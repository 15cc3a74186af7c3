"""SORT (easy_ViTPose/sort.py) for S streams in numpy: the contract `DeviceSort` / `vpb_tracker_update` is held to.

`SortOracle(S, max_age, min_hits, iou_threshold).update(dets_list)` returns, per stream, what S reference `Sort` objects updated
round-robin in one process return (`KalmanBoxTracker.count` is one class-wide counter: within one update new tracks take ids in
stream order, within a stream in creation order).  Per stream and frame (sort.py:223-266):

  1. frame_count += 1;
  2. predict every track in list order: the `x[6] + x[2] <= 0` guard (:141), x = Fx, P = 1.0 (F P F^T) + Q, age / hit_streak /
     time_since_update as KalmanBoxTracker.predict;
  3. drop the tracks whose predicted box has a NaN, keeping the order of the rest;
  4. associate (:158-200): iou_batch, the one-to-one shortcut `a.sum(1).max() == 1 and a.sum(0).max() == 1` with np.where order,
     else scipy's linear_sum_assignment on -iou (the reference environment has scipy and no `lap`);
  5. unmatched detections: the never-assigned ones ascending, then the pairs filtered out for IoU < threshold in matched order;
  6. Kalman update of the matched tracks (filterpy 1.4.5, Joseph form), 7. new tracks in the order of step 5;
  8. rows from the reversed track list, with the `frame_count <= min_hits` rule, the death rule and the empty-detections branch.

Why exact equality is reachable: P keeps its block structure exactly.  (x, vx), (y, vy), (s, vs) form 2 x 2 blocks and r is a
scalar; off-block entries start at 0 and stay +-0, S = H P H^T + R is diagonal so inv(S) is exactly 1 / d, and every sum in
the filterpy products has at most two nonzero terms, one of them a product with 1.  So the dense np.dot / np.linalg.inv filter
and the per-element formulas below give the same float64 values; the block entries P[p, v] and P[v, p] are NOT equal in
general (the Joseph form rounds them differently), so a track carries 13 doubles: 4 per block, row-major, and P[3, 3].

The Kalman steps here are written per element in a fixed order, vectorised over tracks (no np.dot, no linalg): each numpy
ufunc rounds once, as `__dadd_rn` / `__dmul_rn` do on the device.

`lsap` restates scipy's rectangular shortest-augmenting-path solver (Crouse 2016, scipy/optimize/rectangular_lsap) with its
tie rule; `KalmanFilter` restates filterpy 1.4.5's class for oracle/make_golden_track.py, which runs the unmodified sort.py.
That restatement is NOT pinned against the real filterpy, which is not installed where the fixture was made.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np

TRACK_MAX = 128                      # VPB_TRACK_MAX: detections and live tracks per stream

# KalmanBoxTracker.__init__ (sort.py:105-116) on filterpy's defaults (eye for P, Q, R)
R_DIAG = np.array([1.0, 1.0, 10.0, 10.0])
Q_POS = np.array([1.0, 1.0, 1.0, 1.0])
Q_VEL = np.array([1.0 * 0.01, 1.0 * 0.01, (1.0 * 0.01) * 0.01])      # Q[4:, 4:] *= 0.01 after Q[-1, -1] *= 0.01
P0_POS = 1.0 * 10.0
P0_VEL = (1.0 * 1000.0) * 10.0


# ------------------------------------------------------------------------------------------------ box conversions
def bbox_to_z(d: np.ndarray) -> np.ndarray:
    """convert_bbox_to_z (sort.py:66-78), rows [n, >=4] -> [n, 4] (x, y, s, r)."""
    w = d[:, 2] - d[:, 0]
    h = d[:, 3] - d[:, 1]
    return np.stack([d[:, 0] + w / 2., d[:, 1] + h / 2., w * h, w / h], 1)


def x_to_bbox(x: np.ndarray) -> np.ndarray:
    """convert_x_to_bbox (sort.py:81-91), states [n, >=4] -> [n, 4] (x1, y1, x2, y2)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.sqrt(x[:, 2] * x[:, 3])
        h = x[:, 2] / w
    return np.stack([x[:, 0] - w / 2., x[:, 1] - h / 2., x[:, 0] + w / 2., x[:, 1] + h / 2.], 1)


def iou_batch(dets: np.ndarray, trks: np.ndarray) -> np.ndarray:
    """iou_batch (sort.py:47-63): [n, >=4] x [m, >=4] -> [n, m]."""
    t = dets[:, None, :]
    g = trks[None, :, :]
    xx1 = np.maximum(t[..., 0], g[..., 0])
    yy1 = np.maximum(t[..., 1], g[..., 1])
    xx2 = np.minimum(t[..., 2], g[..., 2])
    yy2 = np.minimum(t[..., 3], g[..., 3])
    w = np.maximum(0., xx2 - xx1)
    h = np.maximum(0., yy2 - yy1)
    wh = w * h
    with np.errstate(invalid="ignore", divide="ignore"):
        return wh / ((t[..., 2] - t[..., 0]) * (t[..., 3] - t[..., 1]) + (g[..., 2] - g[..., 0]) * (g[..., 3] - g[..., 1]) - wh)


# ------------------------------------------------------------------------------------------------ assignment
def lsap(cost):
    """scipy.optimize.linear_sum_assignment (minimise) as scipy's C++ solver computes it, ties included: a tall matrix is
    transposed and the pairs returned sorted by row; each row starts its remaining-column list in descending column order and
    removes a picked column by swapping in the last one; r = ((minVal + c[i, j]) - u[i]) - v[j]; the scan keeps the first
    strict minimum, but an equal value in an unassigned column replaces it -- as a reduction: the last unassigned column with
    the minimum, else the first column with it.  Returns (rows, cols) int64 arrays."""
    c = np.asarray(cost, np.float64)
    nr, nc = c.shape
    if nr == 0 or nc == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    transpose = nc < nr
    if transpose:
        c = c.T
        nr, nc = nc, nr
    u, v = np.zeros(nr), np.zeros(nc)
    path = np.full(nc, -1, np.int64)
    col4row = np.full(nr, -1, np.int64)
    row4col = np.full(nc, -1, np.int64)
    for cur in range(nr):
        remaining = np.arange(nc - 1, -1, -1)
        num = nc
        sr = np.zeros(nr, bool)
        sc = np.zeros(nc, bool)
        spc = np.full(nc, np.inf)
        i, min_val, sink = cur, 0.0, -1
        while sink == -1:
            sr[i] = True
            js = remaining[:num]
            r = ((min_val + c[i, js]) - u[i]) - v[js]
            better = r < spc[js]
            path[js[better]] = i
            spc[js[better]] = r[better]
            vals = spc[js]
            min_val = vals.min()
            at = np.flatnonzero(vals == min_val)
            free = at[row4col[js[at]] == -1]
            index = int(free[-1]) if len(free) else int(at[0])
            j = int(remaining[index])
            if row4col[j] == -1:
                sink = j
            else:
                i = int(row4col[j])
            sc[j] = True
            num -= 1
            remaining[index] = remaining[num]
        u[cur] += min_val
        others = sr.copy()
        others[cur] = False
        u[others] += min_val - spc[col4row[others]]
        v[sc] -= min_val - spc[sc]
        j = sink
        while True:
            i = int(path[j])
            row4col[j] = i
            col4row[i], j = j, int(col4row[i])
            if i == cur:
                break
    if transpose:
        order = np.argsort(col4row)
        return col4row[order], order
    return np.arange(nr), col4row


def associate(dets: np.ndarray, trks: np.ndarray, iou_threshold: float):
    """associate_detections_to_trackers (sort.py:158-200) -> (matches [k, 2] (det, trk), unmatched dets in reference order)."""
    if len(trks) == 0:
        return np.zeros((0, 2), np.int64), list(range(len(dets)))
    iou = iou_batch(dets, trks)
    if min(iou.shape) > 0:
        a = (iou > iou_threshold).astype(np.int32)
        if a.sum(1).max() == 1 and a.sum(0).max() == 1:
            matched = np.stack(np.where(a), axis=1)
        else:
            from scipy.optimize import linear_sum_assignment
            matched = np.stack(linear_sum_assignment(-iou), axis=1)
    else:
        matched = np.zeros((0, 2), np.int64)
    unmatched = [d for d in range(len(dets)) if d not in matched[:, 0]]
    keep = []
    for m in matched:
        if iou[m[0], m[1]] < iou_threshold:
            unmatched.append(int(m[0]))
        else:
            keep.append(m)
    return (np.array(keep, np.int64).reshape(-1, 2)), unmatched


# ------------------------------------------------------------------------------------------------ Kalman steps
def predict(X: np.ndarray, P: np.ndarray) -> None:
    """KalmanBoxTracker.predict's filter part, in place on X [n, 7], P [n, 13]: the guard, x = Fx, P = 1.0 (F P F^T) + Q."""
    g = (X[:, 6] + X[:, 2]) <= 0
    X[g, 6] *= 0.0
    for b in range(3):
        X[:, b] = X[:, b] + X[:, b + 4]
        a, u, c, d = (P[:, 4 * b + k].copy() for k in range(4))
        P[:, 4 * b] = ((a + c) + (u + d)) + Q_POS[b]
        P[:, 4 * b + 1] = u + d
        P[:, 4 * b + 2] = c + d
        P[:, 4 * b + 3] = d + Q_VEL[b]
    P[:, 12] = P[:, 12] + Q_POS[3]


def kalman_update(X: np.ndarray, P: np.ndarray, z: np.ndarray) -> None:
    """filterpy 1.4.5 KalmanFilter.update on H = [I4 0], R = diag(1, 1, 10, 10), in place on X [n, 7], P [n, 13], z [n, 4]:
    y = z - Hx, S = H P H^T + R, K = P H^T inv(S), x += K y, P = (I - KH) P (I - KH)^T + K R K^T."""
    for b in range(3):
        a, u, c, d = (P[:, 4 * b + k].copy() for k in range(4))
        y = z[:, b] - X[:, b]
        si = 1.0 / (a + R_DIAG[b])
        kp, kv = a * si, c * si
        X[:, b] = X[:, b] + kp * y
        X[:, b + 4] = X[:, b + 4] + kv * y
        ik = 1.0 - kp
        a00, a01 = ik * a, ik * u                 # (I - KH) P
        a10, a11 = (-kv) * a + c, (-kv) * u + d
        kr_p, kr_v = kp * R_DIAG[b], kv * R_DIAG[b]
        P[:, 4 * b] = a00 * ik + kr_p * kp
        P[:, 4 * b + 1] = (a00 * (-kv) + a01) + kr_p * kv
        P[:, 4 * b + 2] = a10 * ik + kr_v * kp
        P[:, 4 * b + 3] = (a10 * (-kv) + a11) + kr_v * kv
    p = P[:, 12].copy()
    y = z[:, 3] - X[:, 3]
    k = p * (1.0 / (p + R_DIAG[3]))
    X[:, 3] = X[:, 3] + k * y
    ik = 1.0 - k
    P[:, 12] = (ik * p) * ik + (k * R_DIAG[3]) * k


# ------------------------------------------------------------------------------------------------ the tracker
class _Stream:
    def __init__(self):
        self.X = np.zeros((0, 7))
        self.P = np.zeros((0, 13))
        self.score = np.zeros(0)
        self.id = np.zeros(0, np.int64)
        self.tsu = np.zeros(0, np.int64)            # time_since_update
        self.hs = np.zeros(0, np.int64)             # hit_streak
        self.frame_count = 0

    def take(self, keep):
        for k in ("X", "P", "score", "id", "tsu", "hs"):
            setattr(self, k, getattr(self, k)[keep])


class SortOracle:
    """S reference `Sort(max_age, min_hits, iou_threshold)` objects sharing one id counter (`next_id`, KalmanBoxTracker.count).

    limit=None is the reference.  limit=TRACK_MAX adds the device's rule: a stream with more than `limit` detections, a row
    that is not finite or has x2 <= x1 or y2 <= y1, or more than `limit` tracks after association is left as it was and
    returns no rows; `status` collects the bits (1: bad row, 2: over capacity) as vpb_tracker_status reports them."""

    def __init__(self, num_streams: int, max_age: int = 1, min_hits: int = 3, iou_threshold: float = 0.3, next_id: int = 0,
                 limit=None):
        self.max_age, self.min_hits, self.iou_threshold = int(max_age), int(min_hits), float(iou_threshold)
        self.streams = [_Stream() for _ in range(num_streams)]
        self.next_id = int(next_id)
        self.limit = limit
        self.status = 0

    def reset(self, stream=None):
        for s in range(len(self.streams)) if stream is None else [stream]:
            self.streams[s] = _Stream()

    def update(self, dets_list):
        """dets_list: per stream [n, 5] (x1, y1, x2, y2, score) -> per stream float64 [m, 6] (x1, y1, x2, y2, score, id + 1)."""
        if len(dets_list) != len(self.streams):
            raise ValueError(f"{len(dets_list)} detection arrays for {len(self.streams)} streams")
        return [self._update(st, np.asarray(d, np.float64).reshape(-1, 5)) for st, d in zip(self.streams, dets_list)]

    def _update(self, st: _Stream, dets: np.ndarray) -> np.ndarray:
        if self.limit is not None:
            if len(dets) > self.limit:
                self.status |= 2
                return np.zeros((0, 6))
            if not np.isfinite(dets).all() or (dets[:, 2] <= dets[:, 0]).any() or (dets[:, 3] <= dets[:, 1]).any():
                self.status |= 1
                return np.zeros((0, 6))
            saved = {k: v.copy() if isinstance(v, np.ndarray) else v for k, v in st.__dict__.items()}
        st.frame_count += 1
        predict(st.X, st.P)
        st.hs[st.tsu > 0] = 0
        st.tsu += 1
        box = x_to_bbox(st.X)
        keep = ~np.isnan(box).any(1)
        st.take(keep)
        box = box[keep]
        matches, unmatched = associate(dets, box, self.iou_threshold)
        if self.limit is not None and len(st.X) + len(unmatched) > self.limit:
            st.__dict__.update(saved)
            self.status |= 2
            return np.zeros((0, 6))
        if len(matches):
            t, d = matches[:, 1], matches[:, 0]
            X, P = st.X[t], st.P[t]
            kalman_update(X, P, bbox_to_z(dets[d]))
            st.X[t], st.P[t] = X, P
            st.tsu[t] = 0
            st.hs[t] += 1
            st.score[t] = dets[d, 4]
        n_new = len(unmatched)
        if n_new:
            nd = dets[np.array(unmatched, np.int64)]
            Xn = np.zeros((n_new, 7))
            Xn[:, :4] = bbox_to_z(nd)
            Pn = np.zeros((n_new, 13))
            Pn[:, [0, 4, 8]] = P0_POS
            Pn[:, [3, 7, 11]] = P0_VEL
            Pn[:, 12] = P0_POS
            st.X = np.concatenate([st.X, Xn])
            st.P = np.concatenate([st.P, Pn])
            st.score = np.concatenate([st.score, nd[:, 4]])
            st.id = np.concatenate([st.id, self.next_id + np.arange(n_new, dtype=np.int64)])
            st.tsu = np.concatenate([st.tsu, np.zeros(n_new, np.int64)])
            st.hs = np.concatenate([st.hs, np.zeros(n_new, np.int64)])
            self.next_id += n_new
        rows = np.concatenate([x_to_bbox(st.X), st.score[:, None], (st.id + 1)[:, None].astype(np.float64)], 1)[::-1]
        rev_tsu, rev_hs = st.tsu[::-1], st.hs[::-1]
        emit = (rev_tsu < 1) & ((rev_hs >= self.min_hits) | (st.frame_count <= self.min_hits))
        st.take(st.tsu <= self.max_age)
        if emit.any():
            return np.ascontiguousarray(rows[emit])
        if len(dets) == 0:
            return np.ascontiguousarray(rows)
        return np.zeros((0, 6))


# ------------------------------------------------------------------------------------------------ the reference itself
class KalmanFilter:
    """filterpy 1.4.5 `filterpy.kalman.KalmanFilter` as far as sort.py uses it (defaults, predict(), update(z)), restated from
    its published formulas with np.dot and np.linalg.inv.  Not pinned against the real package, which is not installed."""

    def __init__(self, dim_x, dim_z, dim_u=0):
        self.dim_x, self.dim_z = dim_x, dim_z
        self.x = np.zeros((dim_x, 1))
        self.P = np.eye(dim_x)
        self.Q = np.eye(dim_x)
        self.B = None
        self.F = np.eye(dim_x)
        self.H = np.zeros((dim_z, dim_x))
        self.R = np.eye(dim_z)
        self._alpha_sq = 1.
        self._I = np.eye(dim_x)
        self.inv = np.linalg.inv

    def predict(self):
        self.x = np.dot(self.F, self.x)
        self.P = self._alpha_sq * np.dot(np.dot(self.F, self.P), self.F.T) + self.Q

    def update(self, z):
        z = np.asarray(z, np.float64).reshape(self.dim_z, 1)
        y = z - np.dot(self.H, self.x)
        PHT = np.dot(self.P, self.H.T)
        S = np.dot(self.H, PHT) + self.R
        SI = self.inv(S)
        K = np.dot(PHT, SI)
        self.x = self.x + np.dot(K, y)
        I_KH = self._I - np.dot(K, self.H)
        self.P = np.dot(np.dot(I_KH, self.P), I_KH.T) + np.dot(np.dot(K, self.R), K.T)


def load_reference_sort():
    """The UNMODIFIED easy_ViTPose/sort.py as a module, importable without its plotting dependencies: matplotlib and skimage
    are empty stubs, filterpy.kalman.KalmanFilter is the restatement above, and `import lap` raises ImportError so that
    linear_assignment takes scipy's branch, as in the reference environment (a permissive stub would raise TypeError instead).
    Test infrastructure only; raises RuntimeError without the reference tree."""
    from oracle import ref_import
    path = os.path.join(ref_import.REF_PKG, "sort.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"reference sort.py not found at {path}")
    for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.patches", "skimage", "skimage.io"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
    fp = types.ModuleType("filterpy")
    fpk = types.ModuleType("filterpy.kalman")
    fpk.KalmanFilter = KalmanFilter
    fp.kalman = fpk
    saved = {k: sys.modules.get(k) for k in ("filterpy", "filterpy.kalman", "lap")}
    sys.modules.update({"filterpy": fp, "filterpy.kalman": fpk, "lap": None})
    try:
        import importlib.util
        spec = importlib.util.spec_from_file_location("_reference_sort", path)
        mod = importlib.util.module_from_spec(spec)
        sys.dont_write_bytecode = True
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if k != "lap":
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
    sys.modules["lap"] = None          # linear_assignment imports lap on every call
    return mod


# ------------------------------------------------------------------------------------------------ sequences
def make_sequence(seed: int, frames: int, people: int, kind: str = "walk", width: float = 1920., height: float = 1080.):
    """Seeded detection frames [n, 5] float64 for one stream.  kind: 'walk' (people moving with noise, some missed
    detections), 'crowd' (40-100 heavily overlapping boxes, crossings), 'jump' (everyone teleports on some frames: all-zero
    IoU), 'dup' (identical duplicate detections), 'shrink' (boxes shrinking fast, which hits the x[6] + x[2] <= 0 guard),
    'occlude' (each person hidden for 6 frames in every 24), 'empty' (no detections after a few frames)."""
    rng = np.random.default_rng(seed)
    n = people
    cx, cy = rng.uniform(0, width, n), rng.uniform(0, height, n)
    bw, bh = rng.uniform(40, 160, n), rng.uniform(90, 320, n)
    vx, vy = rng.normal(0, 6, n), rng.normal(0, 4, n)
    out = []
    for f in range(frames):
        cx, cy = cx + vx + rng.normal(0, 1.5, n), cy + vy + rng.normal(0, 1.5, n)
        if kind == "shrink":
            bw, bh = bw * 0.8, bh * 0.8
            if f % 7 == 6:
                bw, bh = rng.uniform(40, 160, n), rng.uniform(90, 320, n)
        if kind == "jump" and f % 5 == 4:
            cx, cy = rng.uniform(0, width, n), rng.uniform(0, height, n)
        w = np.maximum(bw * rng.uniform(0.95, 1.05, n), 1.0)
        h = np.maximum(bh * rng.uniform(0.95, 1.05, n), 1.0)
        d = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, rng.uniform(0.36, 1.0, n)], 1)
        keep = rng.uniform(size=n) > (0.1 if kind in ("walk", "crowd") else 0.0)
        if kind == "occlude":
            keep &= (f // 6 + np.arange(n)) % 4 != 0
        d = d[keep]
        if kind == "dup" and len(d):
            d = np.concatenate([d, d[: max(1, len(d) // 3)]])
        if kind == "empty" and f >= 3:
            d = d[:0]
        if kind == "crowd":
            d = d[rng.permutation(len(d))]
        out.append(np.round(d, 2) if f % 2 else d)
    return out
