"""CPU: oracle/one_euro_oracle.py, the contract vpb_smoother_update is held to.  Its numpy restatement of the filter equals
the unmodified reference `OneEuroFilter` bit for bit (where the reference tree is present); the composition reproduces
tests/golden/smooth_one_euro.npz; the per-id rules (forget after max_gap, new ids, the device's limits); the smoothing
kernels contain no FMA contraction; the header, the ctypes table and the Python argument checks."""
import os
import re
import shutil
import subprocess
import types
import warnings

import numpy as np
import pytest

from oracle import make_golden_smooth as MG
from oracle import one_euro_oracle as OE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _reference_or_skip():
    try:
        return OE.load_reference_one_euro()
    except RuntimeError as exc:
        pytest.skip(str(exc))


def _sequence(seed, steps, K):
    """float32 [K, 2] inputs with jitter, jumps, coordinates at or below 0 and a NaN; clocks with repeats (t_e = 0)."""
    rng = np.random.default_rng(seed)
    base = rng.uniform(1, 600, (K, 2))
    xs = []
    for t in range(steps):
        x = base + rng.normal(0, 2.0, (K, 2)) + (rng.uniform(-80, 80, (K, 2)) if t % 5 == 4 else 0.0)
        x[rng.uniform(size=(K, 2)) < 0.08] = rng.choice([0.0, -0.5, -20.0])
        if t == 6:
            x[0, 1] = np.nan
        xs.append(x.astype(np.float32))
    clocks = 100.0 + np.cumsum(rng.choice([0.0, 1 / 30, 1 / 29, 2 / 30, 0.5], steps, p=[0.05, 0.5, 0.3, 0.1, 0.05]))
    return xs, clocks


@pytest.mark.parametrize("params", [dict(fps=30.0), dict(fps=None), dict(fps=None, min_cutoff=0.3, beta=2.0, d_cutoff=12.0, dx0=3.0),
                                    dict(fps=7, min_cutoff=4.0, beta=0.0, dx0=-0.5)], ids=["fps", "realtime", "realtime_custom", "fps_custom"])
@pytest.mark.parametrize("K", [1, 17, 133])
def test_restatement_equals_live_reference(params, K):
    ref = _reference_or_skip()
    xs, clocks = _sequence(K + len(params), 40, K)
    p = {**dict(dx0=0.0, min_cutoff=1.7, beta=0.3, d_cutoff=30.0), **params}
    args = (p["dx0"], p["min_cutoff"], p["beta"], p["d_cutoff"], p["fps"])
    OE._NOW[0] = clocks[0]
    a, b = ref(xs[0], *args), OE.OneEuroNumpy(xs[0], *args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for t in range(1, len(xs)):
            OE._NOW[0] = clocks[t]
            te = float(1 + t % 3)
            want, got = a(xs[t], te), b(xs[t], te)
            assert want.dtype == got.dtype == np.float64
            assert np.array_equal(want, got, equal_nan=True), t
            assert np.array_equal(np.signbit(want), np.signbit(got)) or np.isnan(want).any(), t


def test_reference_float32_first_call():
    """The first call's x - x_prev is a float32 subtraction: the case the device's first-call flag exists for."""
    ref = _reference_or_skip()
    x0 = np.array([[1.1, 3.0]], np.float32)
    x1 = np.array([[16777216.0, 3.5]], np.float32)                  # 16777216 - 1.1 rounds to 16777215 in float32
    want = ref(x0, fps=1.0)(x1, 1.0)
    assert np.array_equal(OE.OneEuroNumpy(x0, fps=1.0)(x1, 1.0), want)
    f64 = OE.OneEuroNumpy(x0, fps=1.0)
    f64.x_prev = f64.x_prev.astype(np.float64)
    assert not np.array_equal(f64(x1, 1.0), want)


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_oracle_equals_reference_fixture(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "smooth_one_euro.npz"))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        counts, crcs, first = MG.run(case)
    name = case[0]
    assert np.array_equal(counts, g[f"{name}_counts"]) and np.array_equal(crcs, g[f"{name}_crc32"])
    assert np.array_equal(first, g[f"{name}_stream0_rows"])


def test_composition_forgets_after_max_gap():
    """fps mode: t_e counts the updates since an id was last seen; an id absent from more than max_gap updates in a row
    starts a new filter (its row comes back unchanged)."""
    x = [np.full((1, 2, 3), v, np.float32) for v in (10.0, 12.0, 14.0, 16.0, 18.0)]
    for max_gap, restart in ((0, True), (1, False), (30, False)):
        o = OE.SmoothOracle(1, fps=30.0, max_gap=max_gap)
        o.update([x[0]], [[5]])
        o.update([x[1]], [[5]])
        o.update([x[2][:0]], [[]])                                 # absent once
        out = o.update([x[3]], [[5]])[0]
        assert np.array_equal(out[0], x[3][0, :, :2]) == restart, max_gap
        f = OE.OneEuroNumpy(x[0][0, :, :2], fps=30.0)
        f(x[1][0, :, :2], 1.0)
        if not restart:
            assert np.array_equal(out[0], f(x[3][0, :, :2], 2.0))   # t_e = 2: two updates since the id was seen


def test_oracle_limits():
    o = OE.SmoothOracle(3, fps=30.0, max_gap=0, limit=True)
    k = lambda n: np.ones((n, 1, 3), np.float32)                   # noqa: E731
    out = o.update([k(2), k(129), k(128)], [[1, 1], list(range(129)), list(range(128))])
    assert out[0] is None and out[1] is None and out[2] is not None
    assert o.status == OE.STATUS_DUPLICATE_ID | OE.STATUS_OVER_CAPACITY
    assert [s.updates for s in o.streams] == [0, 0, 1]
    o.status = 0
    assert o.update([k(0), k(0), k(1)], [[], [], [1000]], None)[2] is None and o.status == OE.STATUS_OVER_CAPACITY   # 128 + 1


def test_smoothing_sass_has_no_fma_contraction(tmp_path):
    """The smoothing kernels compile to the same SASS with and without -fmad: every multiply and add rounds on its own.  The
    DFMAs the SASS does contain belong to the correctly rounded division sequences."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("no CUDA toolkit")
    src = tmp_path / "smooth_only.cu"
    src.write_text('#include "smooth.cuh"\n')
    sass = {}
    for fmad in ("true", "false"):
        cubin = tmp_path / f"smooth_{fmad}.cubin"
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", f"-fmad={fmad}",
                        "-I", os.path.join(ROOT, "easy_vitpose_b200", "csrc"), "-cubin", "-o", str(cubin), str(src)], check=True)
        out = subprocess.run([cuobjdump, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
        sass[fmad] = [re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ln).strip() for ln in out.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", ln)]
    assert sass["true"] and sass["true"] == sass["false"]
    assert any("smooth_assign" in ln for ln in out.splitlines()) and any("smooth_apply" in ln for ln in out.splitlines())


def test_header_declares_the_smoother_calls():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.smooth import SMOOTH_MAX, STATUS_DUPLICATE_ID, STATUS_OVER_CAPACITY
    hdr = open(os.path.join(ROOT, "include", "vitpose_b200.h")).read()
    names = {"vpb_smoother_create", "vpb_smoother_destroy", "vpb_smoother_update", "vpb_smoother_reset", "vpb_smoother_status"}
    assert names <= set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr)) <= set(_lib.EXPORTS)
    assert f"#define VPB_SMOOTH_MAX {SMOOTH_MAX}" in hdr and SMOOTH_MAX == OE.SMOOTH_MAX
    assert f"#define VPB_SMOOTH_DUPLICATE_ID {STATUS_DUPLICATE_ID}" in hdr and STATUS_DUPLICATE_ID == OE.STATUS_DUPLICATE_ID
    assert f"#define VPB_SMOOTH_OVER_CAPACITY {STATUS_OVER_CAPACITY}" in hdr and STATUS_OVER_CAPACITY == OE.STATUS_OVER_CAPACITY


def test_python_argument_checks():
    """What raises ValueError before any device work: the constructor's fps and device, install()'s smoothing option, and
    update_device's tensor checks."""
    import torch

    from easy_vitpose_b200 import install
    from easy_vitpose_b200.smooth import DeviceOneEuro
    with pytest.raises(ValueError):
        DeviceOneEuro(1, 17, fps=0.0)
    with pytest.raises(ValueError):
        DeviceOneEuro(1, 17, device="cpu")
    with pytest.raises(ValueError):
        install(types.SimpleNamespace(), smoothing={})                         # needs batched=True
    with pytest.raises(ValueError):
        install(types.SimpleNamespace(), batched=True, smoothing={"min_cutof": 1.0})
    s = object.__new__(DeviceOneEuro)
    s.num_streams, s.num_keypoints, s.fps, s.device, s._handle = 2, 17, None, torch.device("cuda", 0), None
    k, c, i = torch.zeros((3, 17, 3)), torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.int32)
    with pytest.raises(ValueError):
        s.update_device(k, c, i, torch.zeros(2, dtype=torch.float64))      # host tensors
    with pytest.raises(ValueError):
        s.update([k.numpy()], [[0, 1, 2]], clock=[0.0])                     # one array for two streams
    with pytest.raises(ValueError):
        s.update([k.numpy(), k.numpy()], [[0, 1, 2], [0, 1, 2]])             # realtime without a clock
    s.fps = 30.0
    with pytest.raises(ValueError):
        s.update([k.numpy().astype(np.float64), k.numpy()], [[0, 1, 2], [0, 1, 2]])
    with pytest.raises(ValueError):
        s.update([k.numpy(), k.numpy()], [[0, 1], [0, 1, 2]])
