"""CPU: the host side of vpb_coco_eval (easy_vitpose_b200.coco_eval) and its oracle.  The ground truth packs as CSR in ascending
image id; records become one frame per image in list order; the kernel's loadRes area rule (extent of the packed x, y)
equals oracle/coco_oks_eval.load_results'; the threshold tables equal np.linspace's; the kernels compile without spills or
stack frames and without FMA contraction; the header, the ctypes table and the constants agree; the array form of the oracle
(oracle/coco_eval_oracle.py) gives evaluate's numbers."""
import os
import re
import shutil
import subprocess
import warnings

import numpy as np
import pytest

from oracle import coco_eval_oracle as CO
from oracle import coco_oks_eval as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "easy_vitpose_b200", "csrc")


def test_ground_truth_packs_as_csr_by_sorted_image_id():
    from easy_vitpose_b200 import coco_eval as CE
    gts = [{"id": 1, "image_id": 30, "keypoints": [1, 2, 2] * 2, "area": 5.0, "bbox": [0, 0, 1, 1]},
           {"id": 2, "image_id": 10, "keypoints": [3, 4, 1] * 2, "area": 6.0, "bbox": [1, 1, 2, 2], "iscrowd": 1},
           {"id": 3, "image_id": 30, "keypoints": [5, 6, 0] * 2, "area": 7.0, "bbox": [2, 2, 3, 3], "num_keypoints": 0},
           {"id": 4, "image_id": 99, "keypoints": [0, 0, 0] * 2, "area": 8.0, "bbox": [0, 0, 0, 0]},          # not evaluated
           {"id": 5, "image_id": 10, "category_id": 2, "keypoints": [0, 0, 0] * 2, "area": 9.0, "bbox": [0, 0, 0, 0]}]
    index = {10: 0, 20: 1, 30: 2}
    p = CE.pack_ground_truth(gts, index, 2)
    assert p["offsets"].tolist() == [0, 1, 1, 3] and p["offsets"].dtype == np.int32
    assert p["area"].tolist() == [6.0, 5.0, 7.0]
    assert p["kpts"].shape == (3, 2, 3) and p["kpts"][0, 0].tolist() == [3, 4, 1] and p["kpts"][2, 1].tolist() == [5, 6, 0]
    assert p["bbox"][1].tolist() == [0, 0, 1, 1]
    assert p["iscrowd"].tolist() == [1, 0, 0] and p["num_keypoints"].tolist() == [1, 1, 0]
    with pytest.raises(ValueError):
        CE.pack_ground_truth(gts, index, 3)
    assert CE.pack_ground_truth([], index, 17)["offsets"].tolist() == [0, 0, 0, 0]


def test_records_become_frames_in_list_order():
    from easy_vitpose_b200 import coco_eval as CE
    recs = [{"image_id": 30, "score": 0.5, "keypoints": [1, 2, 0, 3, 4, 0]},
            {"image_id": 10, "score": 0.6, "keypoints": [5, 6, 0, 7, 8, 0]},
            {"image_id": 30, "score": 0.7, "keypoints": [9, 10, 0, 11, 12, 0]},
            {"image_id": 55, "score": 0.8, "keypoints": [0, 0, 0, 0, 0, 0]},                 # not evaluated: dropped
            {"image_id": 10, "category_id": 3, "score": 0.9, "keypoints": [0, 0, 0, 0, 0, 0]}]
    p = CE.pack_results(recs, {10: 0, 30: 1}, 2)
    assert p["counts"].tolist() == [1, 2] and p["frame_image"].tolist() == [0, 1]
    assert p["scores"].tolist() == [0.6, 0.5, 0.7] and p["keep"].tolist() == [0, 0, 1]
    assert p["kpts"].tolist() == [[[5, 6], [7, 8]], [[1, 2], [3, 4]], [[9, 10], [11, 12]]]
    assert CE.pack_results([], {10: 0}, 17)["kpts"].shape == (0, 17, 2)


def _device_area(xy):
    """coco_image_kernel's loadRes area: (max x - min x) * (max y - min y) over the keypoints, NaN propagating."""
    x, y = xy[:, 0], xy[:, 1]
    return (np.max(x) - np.min(x)) * (np.max(y) - np.min(y))


def test_loadres_area_rule():
    from easy_vitpose_b200 import coco_eval as CE
    gts, recs, image_ids, _ = CO.random_set(7, 17, n_img=10)
    index = {v: i for i, v in enumerate(image_ids)}
    p = CE.pack_results(recs, index, 17)
    want = {}
    for d in E.load_results(recs):
        want.setdefault(d["image_id"], []).append(d["area"])
    r = 0
    for f, c in zip(p["frame_image"], p["counts"]):
        got = [_device_area(p["kpts"][r + j]) for j in range(c)]
        assert np.array_equal(got, want[image_ids[f]])
        r += c
    rec = {"image_id": 1, "score": 1.0, "keypoints": [3.0, 1.0, 0, -2.5, 7.25, 0, 10.0, 2.0, 0]}
    assert E.load_results([rec])[0]["area"] == 12.5 * 6.25 == _device_area(CE.pack_results([rec], {1: 0}, 3)["kpts"][0])


def test_threshold_tables_equal_linspace():
    src = open(os.path.join(CSRC, "coco_eval.cuh")).read()
    body = re.search(r"kCocoIouThrs\[COCO_T\] = \{(.*?)\};", src, re.S).group(1)
    vals = [float.fromhex(v.strip()) for v in body.split(",")]
    assert np.array_equal(vals, E.IOU_THRS)
    assert "r == COCO_R - 1 ? 1.0 : __dmul_rn(static_cast<double>(r), 0.01)" in src
    assert np.array_equal([1.0 if r == 100 else r * 0.01 for r in range(101)], E.REC_THRS)
    assert (E.MAX_DETS, len(E.IOU_THRS), len(E.REC_THRS)) == (20, 10, 101)
    assert E.AREA_RNG == {"all": (0, 1e10), "medium": (1024, 9216), "large": (9216, 1e10)}


def test_pairwise_depths_cover_the_sums():
    """pairwise_sum<1> for the OKS (K <= 144 terms) and pairwise_sum<4> for the means (<= 1010 terms) reach numpy's blocks."""
    def depth(m):
        if m <= 128:
            return 0
        h = m // 2 - (m // 2) % 8
        return 1 + max(depth(h), depth(m - h))
    assert max(depth(m) for m in range(1, 145)) == 1 and max(depth(m) for m in range(1, 1011)) == 4
    from oracle import oks_nms_oracle as O
    rng = np.random.default_rng(0)
    for n in (1, 7, 8, 101, 129, 303, 505, 1010):
        a = rng.uniform(0, 1, n)
        assert O.pairwise_sum(a) == np.sum(a) and O.pairwise_sum(a) / n == np.mean(a), n


def _compile(tmp_path, fmad, verbose=False):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no CUDA toolkit")
    src = tmp_path / "coco_only.cu"
    src.write_text('#include "coco_eval.cuh"\n')
    cubin = tmp_path / f"coco_{fmad}.cubin"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", f"-fmad={fmad}", "-I", CSRC, "-cubin", "-o",
           str(cubin), str(src)] + (["-Xptxas", "-v"] if verbose else [])
    res = subprocess.run(cmd, check=True, capture_output=True, text=True)
    return cubin, res.stderr + res.stdout, os.path.join(os.path.dirname(nvcc), "cuobjdump")


def test_kernels_have_no_spills_or_stack(tmp_path):
    _, log, _ = _compile(tmp_path, "true", verbose=True)
    props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    names = {p[0] for p in props}
    for k in ("coco_frames_kernel", "coco_image_kernel", "coco_merge_kernel", "coco_accumulate_kernel", "coco_summarize_kernel"):
        assert any(k in x for x in names), (k, log)
    for name, stack, st, ld in props:
        assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)


def test_sass_has_no_fma_contraction(tmp_path):
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

    from easy_vitpose_b200 import _lib, coco_eval as CE
    hdr = open(os.path.join(ROOT, "include", "vitpose_b200.h")).read()
    assert {"vpb_coco_eval", "vpb_coco_eval_workspace_bytes"} <= set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr)) <= set(_lib.EXPORTS)
    for name, val in (("MAX_GTS", CE.MAX_GTS), ("MAX_ROWS", CE.MAX_ROWS), ("MAX_K", CE.MAX_K), ("MAX_IMAGES", CE.MAX_IMAGES),
                      ("TOO_MANY_GTS", CE.STATUS_TOO_MANY_GTS), ("TOO_MANY_ROWS", CE.STATUS_TOO_MANY_ROWS), ("BAD_INPUT", CE.STATUS_BAD_INPUT)):
        assert f"#define VPB_COCO_{name} {val}\n" in hdr, name
    ctype = {"double": C.c_void_p, "int32_t": C.c_void_p}
    for struct, cls in (("vpb_coco_gts", _lib.VpbCocoGts), ("vpb_coco_dets", _lib.VpbCocoDets)):
        body = re.search(rf"typedef struct {struct} \{{(.*?)\}} {struct};", hdr, re.S).group(1)
        fields = re.findall(r"(const )?(double|int32_t)(\*?)\s+(\w+);", body)
        want = [(n, ctype[t] if star else C.c_int32) for _, t, star, n in fields]
        assert want == list(cls._fields_), struct
    src = open(os.path.join(CSRC, "coco_eval.cuh")).read()
    for name, val in (("COCO_MAX_GTS", 256), ("COCO_MAX_ROWS", 1024), ("COCO_MAX_K", 144), ("COCO_TOO_MANY_GTS", 1),
                      ("COCO_TOO_MANY_ROWS", 2), ("COCO_BAD_INPUT", 4)):
        assert re.search(rf"constexpr int {name} = {val};", src), name
    assert CE.STAT_NAMES == CO.STAT_NAMES


def test_host_argument_errors():
    import torch

    from easy_vitpose_b200 import coco_eval as CE
    z = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(ValueError):
        CE.coco_eval_device(z, None, None, None, None, None, None, None, None, None)          # host tensors
    with pytest.raises(ValueError):
        CE._sigmas(None, 133)
    with pytest.raises(ValueError):
        CE.check(1)
    with pytest.raises(ValueError, match="out of range"):
        CE.check(torch.tensor([4], dtype=torch.int32))
    CE.check(0)


@pytest.mark.parametrize("K,seed", [(1, 1), (17, 2), (133, 5)])
def test_array_oracle_gives_evaluates_numbers(K, seed):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        gts, recs, image_ids, sig = CO.random_set(seed, K)
        s = E.KPT_OKS_SIGMAS if sig is None else sig
        full = CO.evaluate_full(gts, recs, image_ids, s)
        assert full["stats"] == E.evaluate(gts, recs, image_ids, s)
        assert full["precision"].shape == (3, 10, 101) and full["recall"].shape == (3, 10)
        assert full["stats"]["AP"] == np.mean(full["precision"][0]) and full["stats"]["AR_large"] == np.mean(full["recall"][2])
        assert not CO.flag_ambiguous(gts, recs, image_ids, s)
        # two OKS of one detection an ulp apart are flagged; equal ones (a duplicate ground truth) are not
        g = dict(gts[0], keypoints=[0.0, 0.0, 2.0] * K, area=100.0, iscrowd=0, num_keypoints=K)
        d = {"image_id": g["image_id"], "score": 1.0, "keypoints": [0.5, 0.0, 0.0] * K}
        assert 0.5 < E.compute_oks([g], E.load_results([d]), s)[0, 0] < 1.0
        assert not CO.flag_ambiguous([g, dict(g, id=g["id"] + 1)], [d], [g["image_id"]], s)
        flagged = 0
        for m in range(1, 9):                             # an area a few ulps away moves the OKS by about an ulp
            g2 = dict(g, area=100.0 * (1 + m * 2.0 ** -52))
            o1, o2 = E.compute_oks([g, g2], E.load_results([d]), s)[0]
            if o1 != o2:
                flagged += bool(CO.flag_ambiguous([g, g2], [d], [g["image_id"]], s))
        assert flagged
