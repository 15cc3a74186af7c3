"""CPU: oracle/sort_oracle.py, the contract vpb_tracker_update is held to, reproduces the unmodified sort.py exactly
(tests/golden/track_sort.npz, oracle/make_golden_track.py, and the live reference where its tree is present); its LSAP
restatement equals scipy's linear_sum_assignment, ties included; the tracker kernels contain no FMA contraction; the
install() tracker adapter, the re-bound reset() and the id interleaving with KalmanBoxTracker.count."""
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

from oracle import sort_oracle as SO
from oracle.make_golden_track import CASES, RAW_FRAMES, case_inputs, crc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "track_sort.npz"))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference_fixture(golden_dir, case):
    g = _golden(golden_dir)
    name, max_age, min_hits = case[:3]
    o = SO.SortOracle(len(case[5]), max_age, min_hits, 0.3)
    first = []
    for f, dl in enumerate(case_inputs(case)):
        outs = o.update(dl)
        assert [len(r) for r in outs] == g[f"{name}_counts"][f].tolist(), f
        assert [crc(r) for r in outs] == g[f"{name}_crc32"][f].tolist(), f
        if f < RAW_FRAMES:
            first.append(outs[0])
    assert np.array_equal(np.concatenate(first), g[f"{name}_stream0_rows"])
    assert o.next_id == int(g[f"{name}_next_id"])


def _reference_or_skip():
    try:
        return SO.load_reference_sort()
    except RuntimeError as exc:
        pytest.skip(str(exc))


@pytest.mark.parametrize("max_age,min_hits", [(1, 3), (3, 1), (5, 1)])
def test_oracle_equals_live_reference(max_age, min_hits):
    """Further seeds against the unmodified sort.py itself, three streams round-robin, every row compared as float64."""
    ref = _reference_or_skip()
    kinds = [("walk", 9, 1920., 1080.), ("crowd", 70, 800., 600.), ("jump", 8, 1920., 1080.)]
    seqs = [SO.make_sequence(100 * max_age + s, 40, p, k, w, h) for s, (k, p, w, h) in enumerate(kinds)]
    ref.KalmanBoxTracker.count = 7
    sorts = [ref.Sort(max_age, min_hits, 0.3) for _ in kinds]
    o = SO.SortOracle(len(kinds), max_age, min_hits, 0.3, next_id=7)
    for f in range(40):
        dl = [sq[f] if (max_age == 1 or f < 3 or f % max_age == 0) else np.empty((0, 5)) for sq in seqs]
        want = [s.update(d) for s, d in zip(sorts, dl)]
        for w, g in zip(want, o.update(dl)):
            assert w.shape == g.shape and np.array_equal(w, g), f
    assert o.next_id == ref.KalmanBoxTracker.count


def test_lsap_restatement_equals_scipy_on_ties():
    """20 000 tie-heavy cost matrices (costs from {0, -0.25, -0.5, -1}, mostly 0), 1..8 on a side and every 200th up to 128."""
    from scipy.optimize import linear_sum_assignment
    rng = np.random.default_rng(1)
    for t in range(20000):
        nr, nc = (int(v) for v in (rng.integers(1, 9, 2) if t % 200 else rng.integers(1, 129, 2)))
        c = -rng.choice([0.0, 0.0, 0.0, 0.25, 0.5, 1.0], size=(nr, nc))
        a, b = SO.lsap(c), linear_sum_assignment(c)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (t, c)


def test_block_formulas_equal_dense_filter():
    """The per-element Kalman steps equal the dense np.dot / np.linalg.inv restatement of filterpy on random tracks."""
    rng = np.random.default_rng(3)
    n = 200
    X = np.zeros((n, 7))
    X[:, :4] = SO.bbox_to_z(np.stack([rng.uniform(0, 500, n), rng.uniform(0, 500, n), rng.uniform(600, 900, n), rng.uniform(600, 900, n)], 1))
    P = np.zeros((n, 13))
    P[:, [0, 4, 8, 12]] = SO.P0_POS
    P[:, [3, 7, 11]] = SO.P0_VEL
    kfs = []
    for i in range(n):
        kf = SO.KalmanFilter(7, 4)
        kf.F = np.eye(7) + np.eye(7, k=4)
        kf.H = np.eye(4, 7)
        kf.R[2:, 2:] *= 10.
        kf.P[4:, 4:] *= 1000.
        kf.P *= 10.
        kf.Q[-1, -1] *= 0.01
        kf.Q[4:, 4:] *= 0.01
        kf.x[:4, 0] = X[i, :4]
        kfs.append(kf)
    pairs = [(r, c) for b in range(3) for r, c in ((b, b), (b, b + 4), (b + 4, b), (b + 4, b + 4))] + [(3, 3)]
    for step in range(12):
        SO.predict(X, P)
        z = X[:, :4] + rng.normal(0, 3, (n, 4)) * [1, 1, 50, 0.01]
        if step % 3 != 2:
            SO.kalman_update(X, P, z)
        for i, kf in enumerate(kfs):
            if (kf.x[6] + kf.x[2]) <= 0:
                kf.x[6] *= 0.0
            kf.predict()
            if step % 3 != 2:
                kf.update(z[i])
            assert np.array_equal(kf.x[:, 0], X[i]), (step, i)
            assert np.array_equal([kf.P[r, c] for r, c in pairs], P[i]), (step, i)


def test_tracker_sass_has_no_fma_contraction(tmp_path):
    """The tracker kernels compile to the same SASS with and without -fmad: every multiply and add rounds on its own.  The
    DFMAs the SASS does contain belong to the correctly rounded division and square root sequences."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("no CUDA toolkit")
    src = tmp_path / "track_only.cu"
    src.write_text('#include "track.cuh"\n')
    sass = {}
    for fmad in ("true", "false"):
        cubin = tmp_path / f"track_{fmad}.cubin"
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", f"-fmad={fmad}",
                        "-I", os.path.join(ROOT, "easy_vitpose_b200", "csrc"), "-cubin", "-o", str(cubin), str(src)], check=True)
        out = subprocess.run([cuobjdump, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
        sass[fmad] = [re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ln).strip() for ln in out.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", ln)]
    assert sass["true"] and sass["true"] == sass["false"]
    assert any("track_associate" in ln for ln in out.splitlines()) and any("track_emit" in ln for ln in out.splitlines())


def test_header_declares_the_tracker_calls():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.track import STATUS_BAD_ROW, STATUS_OVER_CAPACITY, TRACK_MAX
    hdr = open(os.path.join(ROOT, "include", "vitpose_b200.h")).read()
    names = {"vpb_tracker_create", "vpb_tracker_destroy", "vpb_tracker_update", "vpb_tracker_reset", "vpb_tracker_next_id",
             "vpb_tracker_set_next_id", "vpb_tracker_status"}
    assert names <= set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr)) <= set(_lib.EXPORTS)
    assert f"#define VPB_TRACK_MAX {TRACK_MAX}" in hdr and TRACK_MAX == SO.TRACK_MAX
    assert f"#define VPB_TRACK_BAD_ROW {STATUS_BAD_ROW}" in hdr and f"#define VPB_TRACK_OVER_CAPACITY {STATUS_OVER_CAPACITY}" in hdr


# ------------------------------------------------------------------------------------------------ install() adapter
class OracleDeviceSort:
    """Stand-in for track.DeviceSort backed by the oracle (the adapter's logic without a GPU)."""
    made = []

    def __init__(self, num_streams, max_age=1, min_hits=3, iou_threshold=0.3, device=None):
        self.args = (num_streams, max_age, min_hits, iou_threshold, device)
        self.o = SO.SortOracle(num_streams, max_age, min_hits, iou_threshold)
        OracleDeviceSort.made.append(self)

    def update(self, dets_list):
        return self.o.update(dets_list)

    def check(self):
        pass

    @property
    def next_id(self):
        return self.o.next_id

    @next_id.setter
    def next_id(self, v):
        self.o.next_id = int(v)


@pytest.fixture
def oracle_device_sort(monkeypatch):
    from easy_vitpose_b200 import track
    OracleDeviceSort.made = []
    monkeypatch.setattr(track, "DeviceSort", OracleDeviceSort)
    return OracleDeviceSort


def test_reset_rebinding_builds_the_reference_tracker(oracle_device_sort):
    from easy_vitpose_b200.inference import DeviceTracker, _reference_reset
    b200 = types.SimpleNamespace(model=types.SimpleNamespace(_device=2))
    for step, video, single, want in [(1, True, False, (1, 1, 3, 0.3, 2)), (4, True, False, (1, 4, 1, 0.3, 2)),
                                      (1, False, False, None), (3, True, True, None)]:
        vi = types.SimpleNamespace(yolo_step=step, is_video=video, single_pose=single, tracker="old", frame_counter=9, _b200=b200)
        _reference_reset(vi)
        assert vi.frame_counter == 0
        if want is None:
            assert vi.tracker is None
        else:
            assert isinstance(vi.tracker, DeviceTracker) and vi.tracker.sort.args == want


def test_adapter_returns_reference_rows_and_interleaves_ids(oracle_device_sort, monkeypatch):
    """Two CPU reference Sorts and one adapter in one process, updated round-robin, give the ids and rows of three reference
    Sorts: the adapter reads KalmanBoxTracker.count before its update and writes the next id back."""
    ref = _reference_or_skip()
    from easy_vitpose_b200.inference import DeviceTracker
    monkeypatch.setitem(sys.modules, "easy_ViTPose.sort", ref)
    seqs = [SO.make_sequence(40 + s, 30, 6, "jump") for s in range(3)]
    ref.KalmanBoxTracker.count = 0
    want_sorts = [ref.Sort(1, 3, 0.3) for _ in range(3)]
    want = [[s.update(sq[f]) for s, sq in zip(want_sorts, seqs)] for f in range(30)]
    ref.KalmanBoxTracker.count = 0
    got_sorts = [ref.Sort(1, 3, 0.3), DeviceTracker(1, 3, 0.3), ref.Sort(1, 3, 0.3)]
    for f in range(30):
        for j, (s, sq) in enumerate(zip(got_sorts, seqs)):
            r = s.update(sq[f])
            assert r.dtype == np.float64 and np.array_equal(r, want[f][j]), (f, j)
    monkeypatch.delitem(sys.modules, "easy_ViTPose.sort")
    t = DeviceTracker(1, 3, 0.3)                      # without the reference module: its own counter from 0
    assert t.update(seqs[0][0])[:, 5].tolist() == list(range(len(seqs[0][0]), 0, -1))       # reversed track list
