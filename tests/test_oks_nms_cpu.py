"""CPU: oracle/oks_nms_oracle.py, the contract vpb_oks_nms / vpb_oks_iou are held to.  Its numpy restatement equals the
unmodified reference oks_iou / oks_nms / soft_oks_nms bit for bit on tie-free inputs (where the reference tree is present);
known answers pin the candidate-only mask, the float32 threshold, numpy's pairwise sum order and NaN ordering; the fixture
is reproduced; the kernels compile without spills, stack frames or FMA contraction; the header, the ctypes table and the
host-side argument checks."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import make_golden_oks_nms as MG
from oracle import oks_nms_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "easy_vitpose_b200", "csrc")


def _reference_or_skip():
    try:
        return O.load_reference_nms()
    except RuntimeError as exc:
        pytest.skip(str(exc))


def _database(rng, n, K, dup):
    people = max(1, n // 3) if dup else n
    base = rng.uniform(0, 500, (people, K, 2))
    src = rng.integers(0, people, n) if dup else np.arange(n)
    kp = np.zeros((n, K, 3), np.float32)
    kp[:, :, :2] = base[src] + rng.normal(0, rng.choice([0.5, 3.0, 20.0]), (n, K, 2))
    kp[:, :, 2] = rng.uniform(0, 1, (n, K))
    return kp, rng.uniform(1e3, 5e4, n), rng.uniform(0, 1, n)


@pytest.mark.parametrize("vis", [None, 0.2], ids=["all", "vis"])
@pytest.mark.parametrize("K", [1, 17, 133, 144])
def test_restatement_equals_live_reference(K, vis):
    R = _reference_or_skip()
    rng = np.random.default_rng(K + (vis is None))
    sig = None if K == 17 else rng.uniform(0.02, 0.1, K)
    for trial in range(12):
        kp, areas, scores = _database(rng, int(rng.integers(1, 30)), K, trial % 2 == 1)
        db = O.kpts_db(kp, areas, scores)
        flat = kp.reshape(len(kp), -1)
        for i in range(len(kp)):
            want = R.oks_iou(flat[i], flat, areas[i], areas, sig, vis)
            assert want.dtype == np.float32 and np.array_equal(want, O.oks_iou(kp[i], kp, areas[i], areas, sig, vis)), (trial, i)
        for thr in (0.5, 0.9):
            assert np.array_equal(R.oks_nms(db, thr, sig, vis), O.oks_nms(kp, areas, scores, thr, sig, vis, tie="numpy"))
            assert np.array_equal(O.oks_nms(kp, areas, scores, thr, sig, vis, tie="numpy"), O.oks_nms(kp, areas, scores, thr, sig, vis))
            for md in (1, 20):
                want = R.soft_oks_nms(db, thr, md, sig, vis)
                assert np.array_equal(want, O.soft_oks_nms(kp, areas, scores, thr, md, sig, vis, tie="numpy"))
                assert np.array_equal(want, O.soft_oks_nms(kp, areas, scores, thr, md, sig, vis))


def test_candidate_mask_alone():
    """`list(vg > t) and list(vd > t)` is the candidate's mask: a kept person with every score below the threshold still
    gives a nonzero OKS, and a candidate with none visible gives 0."""
    R = _reference_or_skip()
    g = np.zeros((17, 3), np.float32)
    g[:, :2] = np.arange(34).reshape(17, 2)
    d = g.copy()
    d[:, 2] = 0.9
    d[:9, 2] = 0.1
    d[:, 0] += 3
    ref = R.oks_iou(g.flatten(), d.reshape(1, -1), 4000.0, np.array([4000.0]), None, 0.2)
    assert ref[0] > 0 and np.array_equal(ref, O.oks_iou(g, d[None], 4000.0, [4000.0], None, 0.2))
    full = O.oks_iou(g, d[None], 4000.0, [4000.0], None, None)
    assert full[0] != ref[0]
    d[:, 2] = 0.1
    assert R.oks_iou(g.flatten(), d.reshape(1, -1), 4000.0, np.array([4000.0]), None, 0.2)[0] == 0.0
    assert O.oks_iou(g, d[None], 4000.0, [4000.0], None, 0.2)[0] == 0.0


def test_threshold_compares_in_float32():
    """`oks <= thr` with a float32 OKS rounds thr to float32: f32(0.1) <= 0.1 although f32(0.1) > 0.1."""
    assert float(np.float32(0.1)) > 0.1 and bool(np.array([0.1], np.float32) <= 0.1)
    R = _reference_or_skip()
    g = np.zeros((1, 3), np.float32)
    d = np.array([[1.0, 0.0, 1.0]], np.float32)
    sig = np.array([0.1])
    o = O.oks_iou(g, d[None], 50.0, [50.0], sig)[0]
    db = O.kpts_db(np.stack([g, d]), [50.0, 50.0], [0.9, 0.8])
    assert len(R.oks_nms(db, float(o), sig)) == 2 == len(O.oks_nms(np.stack([g, d]), [50.0, 50.0], [0.9, 0.8], float(o), sig))
    below = float(np.nextafter(o, np.float32(0)))
    assert len(R.oks_nms(db, below, sig)) == 1 == len(O.oks_nms(np.stack([g, d]), [50.0, 50.0], [0.9, 0.8], below, sig))


def test_pairwise_sum_order_equals_np_sum():
    rng = np.random.default_rng(3)
    for n in range(0, 145):
        for _ in range(40):
            a = rng.exponential(size=n) * 10.0 ** rng.uniform(-6, 6, n)
            assert O.pairwise_sum(a) == np.sum(a), n
    a = np.array([1.0] + [2.0 ** -53] * 15)       # pairwise: the small terms meet each other first; sequential loses them
    assert O.pairwise_sum(a) == np.sum(a) != sum(a.tolist())


def test_order_rule_and_nan():
    s = np.array([0.5, np.nan, 0.7, 0.5, np.inf, np.nan, -np.inf, 0.7])
    assert O.order_desc(s).tolist() == [5, 1, 4, 7, 2, 3, 0, 6]
    assert O.order_desc(s).tolist() == np.argsort(s, kind="stable")[::-1].tolist()
    assert O.order_desc(np.array([0.0, -0.0, 0.0])).tolist() == [2, 1, 0]


def test_rescore_known_answers():
    kp = np.zeros((3, 4, 3), np.float32)
    kp[0, :, 2] = [0.1, 0.3, 0.5, 0.2]                    # 0.2 is not > 0.2
    kp[1, :, 2] = [0.1, 0.0, 0.2, 0.15]                   # none: 0
    kp[2, :, 2] = [0.9, np.nan, 0.7, 0.3]                 # NaN is not > 0.2
    got = O.rescore(kp, [0.8, 0.9, -0.5], 0.2)
    want0 = np.float32(np.float32(np.float32(0.3) + np.float32(0.5)) / np.float32(2)) * np.float32(0.8)
    want2 = np.float32(np.float32(np.float32(np.float32(0.9) + np.float32(0.7)) + np.float32(0.3)) / np.float32(3)) * np.float32(-0.5)
    assert got[0] == np.float64(want0) and got[1] == 0.0 and got[2] == np.float64(want2)


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_fixture_is_reproduced(golden_dir, case):
    _reference_or_skip()
    g = np.load(os.path.join(golden_dir, "oks_nms.npz"))
    K = case[1]
    for k, v in MG.inputs_for(K).items():
        assert np.array_equal(v, g[f"k{K}_{k}"]), k
    for k, v in MG.make_case(case).items():
        assert np.array_equal(v, g[f"{case[0]}_{k}"]), k


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_restatement_equals_fixture(golden_dir, case):
    """Without the reference tree: the restatement on the fixture's inputs gives its kept lists and OKS, and no frame is
    ambiguous."""
    g = np.load(os.path.join(golden_dir, "oks_nms.npz"))
    name, K, soft, vis, thr, rsc = case
    kp, ar, counts = g[f"k{K}_kpts"], g[f"k{K}_areas"], g[f"k{K}_counts"]
    sig = g[f"k{K}_sigmas"] if len(g[f"k{K}_sigmas"]) else None
    box, keep, kc, oks = g[f"{name}_box_scores"], g[f"{name}_keep"], g[f"{name}_keep_counts"], g[f"{name}_oks"]
    r = ko = oo = 0
    for f, n in enumerate(counts):
        sl = slice(r, r + n)
        k, s = O.run_frame(kp[sl], ar[sl], box[sl], thr, sig, vis, soft, 20, rsc)
        assert np.array_equal(k, keep[ko:ko + kc[f]]) and np.array_equal(s, g[f"{name}_scores"][sl]), f
        assert np.array_equal(O.oks_matrix(kp[sl], ar[sl], sig, vis).reshape(-1), oks[oo:oo + n * n]), f
        assert not O.flag_ambiguous(kp[sl], ar[sl], box[sl], thr, sig, vis, soft, 20, rsc), f
        r, ko, oo = r + n, ko + kc[f], oo + n * n


def _compile(tmp_path, fmad, verbose=False):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no CUDA toolkit")
    src = tmp_path / "nms_only.cu"
    src.write_text('#include "oks_nms.cuh"\n')
    cubin = tmp_path / f"nms_{fmad}.cubin"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", f"-fmad={fmad}", "-I", CSRC, "-cubin", "-o",
           str(cubin), str(src)] + (["-Xptxas", "-v"] if verbose else [])
    res = subprocess.run(cmd, check=True, capture_output=True, text=True)
    return cubin, res.stderr + res.stdout, os.path.join(os.path.dirname(nvcc), "cuobjdump")


def test_kernels_have_no_spills_or_stack(tmp_path):
    _, log, _ = _compile(tmp_path, "true", verbose=True)
    props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    names = {p[0] for p in props}
    assert any("oks_nms_kernel" in x for x in names) and any("oks_iou_kernel" in x for x in names), log
    for name, stack, st, ld in props:
        assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)


def test_sass_has_no_fma_contraction(tmp_path):
    """Same SASS with and without -fmad: every multiply and add before exp rounds on its own."""
    sass = {}
    for fmad in ("true", "false"):
        cubin, _, cuobjdump = _compile(tmp_path, fmad)
        if not os.path.exists(cuobjdump):
            pytest.skip("no cuobjdump")
        out = subprocess.run([cuobjdump, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
        sass[fmad] = [re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ln).strip() for ln in out.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", ln)]
    assert sass["true"] and sass["true"] == sass["false"]


def test_header_and_ctypes_agree():
    import ctypes as C

    from easy_vitpose_b200 import _lib, nms
    hdr = open(os.path.join(ROOT, "include", "vitpose_b200.h")).read()
    assert {"vpb_oks_nms", "vpb_oks_iou"} <= set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr)) <= set(_lib.EXPORTS)
    for name, val in (("MAX_PEOPLE", nms.MAX_PEOPLE), ("MAX_K", nms.MAX_K), ("MAX_DETS", nms.MAX_DETS),
                      ("TOO_MANY_PEOPLE", nms.STATUS_TOO_MANY_PEOPLE), ("BAD_ROWS", nms.STATUS_BAD_ROWS)):
        assert f"#define VPB_NMS_{name} {val}\n" in hdr, name
    assert (nms.MAX_PEOPLE, nms.MAX_K, nms.MAX_DETS) == (O.MAX_PEOPLE, O.MAX_K, O.MAX_DETS)
    assert (nms.STATUS_TOO_MANY_PEOPLE, nms.STATUS_BAD_ROWS) == (O.STATUS_TOO_MANY_PEOPLE, O.STATUS_BAD_ROWS)
    body = re.search(r"typedef struct vpb_oks_nms_params \{(.*?)\} vpb_oks_nms_params;", hdr, re.S).group(1)
    fields = re.findall(r"(double|int32_t)\s+(\w+);", body)
    ctype = {"double": C.c_double, "int32_t": C.c_int32}
    assert [(n, ctype[t]) for t, n in fields] == list(_lib.VpbOksNmsParams._fields_)
    src = open(os.path.join(CSRC, "oks_nms.cuh")).read()
    for name, val in (("NMS_MAX_PEOPLE", 256), ("NMS_MAX_K", 144), ("NMS_MAX_DETS", 256), ("NMS_TOO_MANY_PEOPLE", 1), ("NMS_BAD_ROWS", 2)):
        assert re.search(rf"constexpr int {name} = {val};", src), name


def test_host_argument_errors():
    """What raises ValueError before any device work."""
    import torch

    from easy_vitpose_b200 import nms
    k = torch.zeros((3, 17, 3))
    c, a = torch.zeros(1, dtype=torch.int32), torch.zeros(3, dtype=torch.float64)
    with pytest.raises(ValueError):
        nms.oks_nms_device(k, c, a, a, 0.9)                               # host tensors
    with pytest.raises(ValueError):
        nms._sigmas(None, 133)                                             # no default table for K != 17
    with pytest.raises(ValueError):
        nms._sigmas(np.ones(16), 17)
    kp = np.zeros((2, 17, 3), np.float32)
    with pytest.raises(ValueError):
        nms.oks_nms_frames([kp], [np.ones(2)], [np.ones(3)], 0.9)          # three scores for two people
    with pytest.raises(ValueError):
        nms.oks_nms_frames([kp], [np.ones(2)], [], 0.9)
    with pytest.raises(ValueError):
        nms.oks_nms_frames([kp, np.zeros((1, 5, 3))], [np.ones(2), np.ones(1)], [np.ones(2), np.ones(1)], 0.9)
    with pytest.raises(ValueError):
        nms.oks_nms_frames([np.zeros((257, 17, 3))], [np.ones(257)], [np.ones(257)], 0.9)
    assert nms.oks_nms([], 0.9) == [] and nms.soft_oks_nms([], 0.9) == []
    with pytest.raises(ValueError):
        nms.check(1)
    with pytest.raises(ValueError):
        nms.check(torch.tensor([2], dtype=torch.int32))
    nms.check(0)
