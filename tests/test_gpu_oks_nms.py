"""-m gpu: vpb_oks_nms / vpb_oks_iou (easy_vitpose_b200.nms) against the unmodified reference's fixture and
oracle/oks_nms_oracle.py: identical kept lists (except frames the oracle flags as ambiguous), OKS within one float32 ulp,
bit-exact rescored scores; 1 / 16 / 64 frames of 0 to 256 people, max_dets 1 / 20 / 256, K = 17 / 133; tie-heavy inputs
and NaN; multi-frame equals per-frame; rows outside the written range; graph replays; status bits; C-ABI argument errors;
B200PoseBackend.inference_topdown_eval against inference_topdown followed by the oracle, and the COCO keypoint AP of its
records on tests/golden/coco_ap.npz with duplicated detector boxes; the INTEGRATION.md video example as written."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import make_golden_oks_nms as MG
from oracle import oks_nms_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _quiet_numpy():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def _upload(kps, areas, scores):
    dev = torch.device("cuda", 0)
    K = kps[0].shape[1] if kps else 17
    kp = torch.from_numpy(np.concatenate(kps).astype(np.float32).reshape(-1, K, 3)).to(dev)
    cnt = torch.tensor([len(k) for k in kps], dtype=torch.int32, device=dev)
    ar = torch.from_numpy(np.concatenate(areas).astype(np.float64)).to(dev)
    sc = torch.from_numpy(np.concatenate(scores).astype(np.float64)).to(dev)
    return kp, cnt, ar, sc


def _kept(res, counts):
    keep, kc = res.keep.cpu().numpy(), res.keep_counts.cpu().numpy()
    out, r = [], 0
    for f, n in enumerate(counts):
        assert kc[f] <= max(n, 0)
        assert (keep[r + kc[f]:r + n] == -1).all()
        out.append(keep[r:r + kc[f]].astype(np.int64))
        r += n
    return out


def _ulp_close(a, b):
    """float32 arrays within one ulp (NaN equal to NaN)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (np.abs(ia - ib) <= 1)))


def _compare(kps, areas, scores, thr, sigmas=None, vis=None, soft=False, max_dets=20, rsc=None):
    from easy_vitpose_b200.nms import check, oks_nms_device
    res = oks_nms_device(*_upload(kps, areas, scores), thr, sigmas, vis, soft, max_dets, rsc)
    check(res)
    got = _kept(res, [len(k) for k in kps])
    sc = res.scores.cpu().numpy()
    r = 0
    for f, (kp, ar, s) in enumerate(zip(kps, areas, scores)):
        want, used = O.run_frame(kp, ar, s, thr, sigmas, vis, soft, max_dets, rsc)
        assert np.array_equal(sc[r:r + len(kp)], used, equal_nan=True), f
        if not np.array_equal(got[f], want):
            assert O.flag_ambiguous(kp, ar, s, thr, sigmas, vis, soft, max_dets, rsc), (f, got[f], want)
        r += len(kp)
    return got


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_device_equals_reference_fixture(golden_dir, case):
    from easy_vitpose_b200.nms import check, oks_iou_device, oks_nms_device
    g = np.load(os.path.join(golden_dir, "oks_nms.npz"))
    name, K, soft, vis, thr, rsc = case
    counts = g[f"k{K}_counts"]
    sig = g[f"k{K}_sigmas"] if len(g[f"k{K}_sigmas"]) else None
    dev = torch.device("cuda", 0)
    kp = torch.from_numpy(g[f"k{K}_kpts"]).to(dev)
    cnt = torch.from_numpy(counts).to(dev)
    ar = torch.from_numpy(g[f"k{K}_areas"]).to(dev)
    box = torch.from_numpy(g[f"{name}_box_scores"]).to(dev)
    res = oks_nms_device(kp, cnt, ar, box, thr, sig, vis, soft, 20, rsc)
    check(res)
    got = _kept(res, counts)
    keep, kc = g[f"{name}_keep"], g[f"{name}_keep_counts"]
    assert np.array_equal(np.concatenate(got), keep) and [len(x) for x in got] == kc.tolist()
    assert np.array_equal(res.scores.cpu().numpy(), g[f"{name}_scores"])           # rescoring is bit-exact
    oks, st = oks_iou_device(kp, cnt, ar, sig, vis)
    oks = oks.cpu().numpy()
    want = g[f"{name}_oks"]
    r = o = 0
    for n in counts:
        assert _ulp_close(oks[r:r + n, :n].reshape(-1), want[o:o + n * n])
        assert np.isnan(oks[r:r + n, n:]).all()
        r, o = r + n, o + n * n
    assert int(st.item()) == 0


def _crowd(rng, n, K, dup=True):
    people = max(1, n // 4) if dup else n
    base = rng.uniform(0, 900, (people, 1, 2)) + rng.normal(0, 30, (people, K, 2))
    src = rng.integers(0, people, n) if dup else np.arange(n)
    kp = np.zeros((n, K, 3), np.float32)
    kp[:, :, :2] = base[src] + rng.choice([0.5, 3.0, 10.0], (n, 1, 1)) * rng.normal(0, 1, (n, K, 2))
    kp[:, :, 2] = rng.uniform(0, 1, (n, K))
    return kp, rng.uniform(2e3, 6e4, people)[src], rng.uniform(0, 1, n)


@pytest.mark.parametrize("frames", [1, 16, 64])
@pytest.mark.parametrize("mode", ["hard", "soft1", "soft20", "soft256"])
def test_device_equals_oracle(frames, mode):
    rng = np.random.default_rng(frames * 7 + len(mode))
    sizes = [0, 1, 2, 17, 100, 256]
    K = 17 if frames != 16 else 133
    sig = None if K == 17 else rng.uniform(0.02, 0.1, K)
    kps, ars, scs = [], [], []
    for f in range(frames):
        n = sizes[(f + frames) % len(sizes)] if frames > 1 else 256
        kp, ar, sc = _crowd(rng, n, K, dup=(f % 3 != 2) or n > 100)
        kps.append(kp); ars.append(ar); scs.append(sc)
    soft = mode != "hard"
    md = int(mode[4:]) if soft else 20
    vis = 0.2 if frames == 16 else None
    _compare(kps, ars, scs, 0.9 if frames % 2 else 0.5, sig, vis, soft, md)
    if mode == "hard":                                      # the OKS values, within one float32 ulp (frames up to 100 people)
        from easy_vitpose_b200.nms import oks_iou_device
        kp, cnt, ar, _ = _upload(kps, ars, scs)
        oks, st = oks_iou_device(kp, cnt, ar, sig, vis)
        oks = oks.cpu().numpy()
        r = 0
        for f, k in enumerate(kps):
            n = len(k)
            if n <= 100:
                assert _ulp_close(oks[r:r + n, :n], O.oks_matrix(k, ars[f], sig, vis)), f
            r += n
        assert int(st.item()) == 0


def test_over_limit_frame_sets_status_and_leaves_others_exact():
    from easy_vitpose_b200.nms import STATUS_TOO_MANY_PEOPLE, oks_nms_device
    rng = np.random.default_rng(5)
    data = [_crowd(rng, n, 17) for n in (20, 257, 30)]
    args = _upload(*map(list, zip(*data)))
    res = oks_nms_device(*args, 0.9)
    assert int(res.status.item()) == STATUS_TOO_MANY_PEOPLE
    got = _kept(res, [20, 257, 30])
    assert len(got[1]) == 0
    for f in (0, 2):
        assert np.array_equal(got[f], O.oks_nms(*data[f], 0.9))


def test_bad_counts_set_status():
    from easy_vitpose_b200.nms import STATUS_BAD_ROWS, oks_nms_device
    rng = np.random.default_rng(6)
    kp0, ar0, sc0 = _crowd(rng, 10, 17)
    kp, _, ar, sc = _upload([kp0], [ar0], [sc0])
    cnt = torch.tensor([4, -3, 4, 5], dtype=torch.int32, device=kp.device)      # -3 holds no rows; 5 runs past 10
    res = oks_nms_device(kp, cnt, ar, sc, 0.9)
    assert int(res.status.item()) == STATUS_BAD_ROWS
    kc = res.keep_counts.cpu().tolist()
    assert kc[1] == 0 and kc[3] == 0
    k = res.keep.cpu().numpy()
    assert np.array_equal(k[:kc[0]], O.oks_nms(kp[:4].cpu().numpy(), ar[:4].cpu().numpy(), sc[:4].cpu().numpy(), 0.9))
    assert np.array_equal(k[4:4 + kc[2]], O.oks_nms(kp[4:8].cpu().numpy(), ar[4:8].cpu().numpy(), sc[4:8].cpu().numpy(), 0.9))
    assert (k[8:] == -1).all()


@pytest.mark.parametrize("soft", [False, True], ids=["hard", "soft"])
def test_ties_follow_the_stable_rule(soft):
    """Quantised scores and exact duplicate people: the restatement with the stable tie rule, exactly."""
    rng = np.random.default_rng(11 + soft)
    kps, ars, scs = [], [], []
    for f in range(24):
        n = int(rng.integers(3, 80))
        kp, ar, _ = _crowd(rng, n, 17)
        dup = rng.integers(0, n, n // 3)
        kp[dup[1:]] = kp[dup[0]]                                   # exact copies of one person
        ar[dup[1:]] = ar[dup[0]]
        sc = np.round(rng.uniform(0, 1, n) * 4) / 4                 # five score values
        kps.append(kp); ars.append(ar); scs.append(sc)
    got = _compare(kps, ars, scs, 0.5, soft=soft, max_dets=30)
    for f in range(24):
        want = O.soft_oks_nms(kps[f], ars[f], scs[f], 0.5, 30) if soft else O.oks_nms(kps[f], ars[f], scs[f], 0.5)
        assert np.array_equal(got[f], want), f


def test_nan_scores_and_keypoints():
    rng = np.random.default_rng(12)
    kps, ars, scs = [], [], []
    for f in range(8):
        kp, ar, sc = _crowd(rng, 40, 17)
        sc[rng.integers(0, 40, 5)] = np.nan
        sc[rng.integers(0, 40, 2)] = np.inf
        kp[rng.integers(0, 40, 4), rng.integers(0, 17, 4), rng.integers(0, 3, 4)] = np.nan
        kps.append(kp); ars.append(ar); scs.append(sc)
    for soft in (False, True):
        for vis in (None, 0.2):
            _compare(kps, ars, scs, 0.9, vis=vis, soft=soft)
    _compare(kps, ars, [np.abs(s) for s in scs], 0.9, rsc=0.2)


def test_multi_frame_equals_per_frame_and_leaves_other_rows():
    from easy_vitpose_b200.nms import OksNmsResult, oks_nms_device
    rng = np.random.default_rng(13)
    data = [_crowd(rng, n, 17) for n in (5, 0, 60, 33, 1)]
    kp, cnt, ar, sc = _upload(*map(list, zip(*data)))
    n = kp.shape[0]
    dev = kp.device
    # three rows of slack after the frames: never written
    keep = torch.full((n + 3,), 0x7eadbeef, dtype=torch.int32, device=dev)
    scores = torch.full((n + 3,), float("nan"), dtype=torch.float64, device=dev)
    kp3 = torch.cat([kp, torch.zeros((3, 17, 3), device=dev)])
    ar3, sc3 = torch.cat([ar, torch.ones(3, dtype=torch.float64, device=dev)]), torch.cat([sc, torch.ones(3, dtype=torch.float64, device=dev)])
    out = OksNmsResult(keep, torch.zeros(5, dtype=torch.int32, device=dev), scores, torch.zeros(1, dtype=torch.int32, device=dev))
    oks_nms_device(kp3, cnt, ar3, sc3, 0.9, soft=True, out=out)
    assert (keep[n:].cpu().numpy() == 0x7eadbeef).all() and torch.isnan(scores[n:]).all()
    got = _kept(OksNmsResult(keep[:n], out.keep_counts, scores[:n], out.status), [len(d[0]) for d in data])
    for f, d in enumerate(data):
        one = oks_nms_device(*_upload([d[0]], [d[1]], [d[2]]), 0.9, soft=True)
        assert np.array_equal(got[f], _kept(one, [len(d[0])])[0]), f


def test_graph_replay_equals_eager():
    from easy_vitpose_b200.nms import OksNmsResult, oks_nms_device
    rng = np.random.default_rng(14)
    data = [_crowd(rng, n, 17) for n in (100, 40, 256, 7)]
    kp, cnt, ar, sc = _upload(*map(list, zip(*data)))
    dev = kp.device
    n, F = kp.shape[0], 4
    outs = [OksNmsResult(torch.empty(n, dtype=torch.int32, device=dev), torch.empty(F, dtype=torch.int32, device=dev),
                         torch.empty(n, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)) for _ in range(2)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        oks_nms_device(kp, cnt, ar, sc, 0.9, rescore_vis_thr=0.2, out=outs[0])            # warm-up
        oks_nms_device(kp, cnt, ar, sc, 0.9, soft=True, out=outs[1])
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        oks_nms_device(kp, cnt, ar, sc, 0.9, rescore_vis_thr=0.2, out=outs[0])
        oks_nms_device(kp, cnt, ar, sc, 0.9, soft=True, out=outs[1])
    for step in range(3):
        sc.copy_(torch.from_numpy(rng.uniform(0, 1, n)).to(dev))
        for o in outs:
            o.keep.fill_(-7)
        graph.replay()
        eager = [oks_nms_device(kp, cnt, ar, sc, 0.9, rescore_vis_thr=0.2), oks_nms_device(kp, cnt, ar, sc, 0.9, soft=True)]
        for o, e in zip(outs, eager):
            assert torch.equal(o.keep, e.keep) and torch.equal(o.keep_counts, e.keep_counts) and torch.equal(o.scores, e.scores)
            assert int(o.status.item()) == 0


def test_c_abi_argument_errors():
    from easy_vitpose_b200 import _lib
    L = _lib.lib()
    dev = torch.device("cuda", 0)
    kp = torch.zeros((4, 17, 3), device=dev)
    cnt = torch.tensor([4], dtype=torch.int32, device=dev)
    ar = torch.ones(4, dtype=torch.float64, device=dev)
    keep, kc, st = torch.empty(4, dtype=torch.int32, device=dev), torch.empty(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr())                                       # noqa: E731
    good = _lib.VpbOksNmsParams(0.9, float("nan"), float("nan"), 0, 20)

    def call(k=17, n=4, frames=1, sig=None, params=good, keep_=keep, status=st):
        return L.vpb_oks_nms(p(kp), n, k, p(cnt), frames, p(ar), p(ar), sig, None if params is None else C.byref(params),
                             None if keep_ is None else p(keep_), p(kc), None, None if status is None else p(status), None)
    assert call() == 0
    torch.cuda.synchronize()
    bad = [dict(k=0), dict(k=145), dict(k=133), dict(n=-1), dict(frames=-1), dict(frames=65536), dict(params=None), dict(keep_=None),
           dict(status=None), dict(params=_lib.VpbOksNmsParams(float("nan"), 0.2, float("nan"), 0, 20)),
           dict(params=_lib.VpbOksNmsParams(0.9, 0.2, float("nan"), 2, 20)), dict(params=_lib.VpbOksNmsParams(0.9, 0.2, float("nan"), 1, 257)),
           dict(params=_lib.VpbOksNmsParams(0.9, 0.2, float("nan"), 1, -1)),
           dict(sig=np.array([np.inf] + [0.05] * 16).ctypes.data_as(C.c_void_p))]
    for b in bad:
        assert call(**b) == 1, b                                                   # VPB_ERR_ARG
        assert L.vpb_last_error().decode().startswith("vpb_oks_nms"), b
    oks = torch.empty((4, 256), device=dev)
    assert L.vpb_oks_iou(p(kp), 4, 17, p(cnt), 1, p(ar), None, float("nan"), None, p(st), None) == 1
    assert L.vpb_oks_iou(p(kp), 4, 18, p(cnt), 1, p(ar), None, float("nan"), p(oks), p(st), None) == 1
    assert L.vpb_oks_iou(p(kp), 4, 17, p(cnt), 1, p(ar), None, float("nan"), p(oks), p(st), None) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------- evaluation
_engines = {}


def _engine():
    from easy_vitpose_b200 import ViTPose, model_cfg
    from oracle import vitpose_oracle as VO
    if "b" not in _engines:
        D, depth, _ = VO.MODEL_DIMS["b"]
        sd = VO.make_state_dict(D, depth, 17, 21, peaky=0.1, bumps=True)
        m = ViTPose(model_cfg("b", 17), max_batch=32)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        _engines["b"] = m.to("cuda:0")
    return _engines["b"]


def _eval_case(seed):
    """Frames with person boxes and duplicated, jittered detector boxes (x, y, w, h) and box scores."""
    from oracle import preproc_oracle as P
    rng = np.random.default_rng(seed)
    frames, boxes, scores = [], [], []
    for j in range(3):
        h, w = int(rng.integers(300, 520)), int(rng.integers(300, 640))
        frames.append(P.make_frame(h, w, seed + j))
        base = np.stack([rng.uniform(0, w * 0.6, 4), rng.uniform(0, h * 0.5, 4), rng.uniform(40, w * 0.4, 4), rng.uniform(60, h * 0.5, 4)], 1)
        src = rng.integers(0, 4, 9)
        b = base[src] + rng.normal(0, 1, (9, 4)) * rng.choice([0.0, 2.0, 10.0], (9, 1))
        b[:, 2:] = np.abs(b[:, 2:]) + 8
        boxes.append(b)
        scores.append(rng.uniform(0.3, 1.0, 9))
    return frames, boxes, scores


@pytest.mark.parametrize("flip", [False, True], ids=["plain", "flip"])
@pytest.mark.parametrize("soft", [False, True], ids=["hard", "soft"])
def test_inference_topdown_eval_equals_composition(flip, soft):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, B200PoseBackend
    from easy_vitpose_b200.topdown import xywh2cs
    m = _engine()
    m.set_flip_test(COCO_FLIP_PAIRS if flip else None)
    try:
        be = B200PoseBackend(m)
        frames, boxes, scores = _eval_case(40 + flip + 2 * soft)
        got = be.inference_topdown_eval(frames, boxes, scores, soft_nms=soft)
        kps = be.inference_topdown(frames, boxes)
    finally:
        m.set_flip_test(None)
    for j, (kp, b, s) in enumerate(zip(kps, boxes, scores)):
        areas = np.array([np.float64(xywh2cs(x)[1][0]) * np.float64(xywh2cs(x)[1][1]) * 200 * 200 for x in b])
        want, used = O.run_frame(kp, areas, s, 0.9, soft=soft, rescore_vis_thr=0.2)
        gk, gs, gi = got[j]
        assert np.array_equal(gs, used[gi]) and np.array_equal(gk, kp[gi]), j
        if not np.array_equal(gi, want):
            assert O.flag_ambiguous(kp, areas, s, 0.9, soft=soft, rescore_vis_thr=0.2), j


def test_coco_ap_of_device_kept_records_equals_oracle_kept(golden_dir):
    """The synthetic COCO set of tests/golden/coco_ap.npz with every detector box duplicated twice, jittered by a few pixels
    and rescored: records built from the people inference_topdown_eval keeps (hard and soft NMS) give exactly the
    oracle/coco_oks_eval.py AP / AR of the records built from the people the oracle keeps on the engine's own keypoints.
    Hard NMS must remove people and change the summary against the records of every box, so the comparison exercises the
    suppression; soft NMS (max_dets 20) keeps every one of these frames' people and is checked for equal records' AP."""
    from easy_vitpose_b200 import B200PoseBackend, ViTPose, model_cfg
    from easy_vitpose_b200.topdown import xywh2cs
    from oracle import coco_oks_eval as E, preproc_oracle as P, vitpose_oracle as VO
    g = np.load(os.path.join(golden_dir, "coco_ap.npz"))
    n_img, fh, fw, fseed, D, depth, heads, K, wseed = (int(v) for v in g["meta"])
    size = next(k for k, v in VO.MODEL_DIMS.items() if v == (D, depth, heads))
    m = ViTPose(model_cfg(size, K), max_batch=32)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in VO.make_state_dict(D, depth, K, wseed, peaky=0.1, bumps=True).items()})
    be = B200PoseBackend(m, "cuda:0")
    gts = [{"id": i + 1, "image_id": int(g["gt_image"][i]), "category_id": 1, "iscrowd": 0, "num_keypoints": int(g["gt_num"][i]),
            "keypoints": g["gt_keypoints"][i].tolist(), "bbox": g["gt_bbox"][i].tolist(), "area": float(g["gt_area"][i])}
           for i in range(len(g["gt_image"]))]
    image_ids = [1000 + i for i in range(n_img)]
    rng = np.random.default_rng(2024)
    frames, boxes, scores = [], [], []
    for i in range(n_img):
        rows = g["rows"][i, :int(g["counts"][i])].astype(np.float64)
        rows = rows[rows[:, 4] > 0.35]                                  # the reference's detector gate
        xywh = np.concatenate([rows[:, :2], rows[:, 2:4] - rows[:, :2]], 1)
        jitter = rng.normal(0, 3, (3 * len(xywh), 4))
        jitter[::3] = 0                                                 # the detector's own box, then two jittered copies
        dup = np.repeat(xywh, 3, 0) + jitter
        frames.append(P.make_frame(fh, fw, fseed + i))
        boxes.append(dup)
        scores.append(np.repeat(rows[:, 4], 3) * rng.uniform(0.8, 1.0, len(dup)))

    def records(i, kp, sc):
        return [{"image_id": image_ids[i], "category_id": 1, "score": float(s), "bbox": [],
                 "keypoints": np.stack([k[:, 1], k[:, 0], k[:, 2]], 1).astype(np.float64).reshape(-1).tolist()} for k, s in zip(kp, sc)]

    kps = be.inference_topdown(frames, boxes)
    all_recs = []
    for i, (kp, b, s) in enumerate(zip(kps, boxes, scores)):
        all_recs += records(i, kp, O.rescore(kp, s, 0.2))
    no_nms = E.evaluate(gts, all_recs, image_ids)
    for soft in (False, True):
        got = be.inference_topdown_eval(frames, boxes, scores, soft_nms=soft)
        dev_recs, ora_recs = [], []
        for i, (kp, b, s) in enumerate(zip(kps, boxes, scores)):
            areas = np.array([np.float64(xywh2cs(x)[1][0]) * np.float64(xywh2cs(x)[1][1]) * 200 * 200 for x in b])
            want, used = O.run_frame(kp, areas, s, 0.9, soft=soft, rescore_vis_thr=0.2)
            gk, gs, gi = got[i]
            assert np.array_equal(gk, kp[gi]) and np.array_equal(gs, used[gi]), i
            if not np.array_equal(gi, want):
                assert O.flag_ambiguous(kp, areas, s, 0.9, soft=soft, rescore_vis_thr=0.2), i
            dev_recs += records(i, gk, gs)
            ora_recs += records(i, kp[want], used[want])
        a, b = E.evaluate(gts, dev_recs, image_ids), E.evaluate(gts, ora_recs, image_ids)
        assert a == b, (soft, a, b)
        if not soft:                      # soft NMS keeps up to 20 people per frame, so here it only reorders them
            assert len(dev_recs) < len(all_recs) and a != no_nms, (a, no_nms)


def test_integration_video_example_runs_as_written():
    """INTEGRATION.md section 3i's video step, executed as written on a small engine: the kept rows are the oracle's, the
    smoother and the overlay ran on them."""
    import re

    from easy_vitpose_b200 import DeviceOneEuro
    from oracle import preproc_oracle as P
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "INTEGRATION.md")).read()
    sec = text[text.index("### 3i."):]
    code = re.search(r"```python\n(.*?)```", sec, re.S).group(1)
    m = _engine()
    rng = np.random.default_rng(77)
    frames, boxes, box_scores, track_ids = [], [], [], []
    for j in range(3):
        frames.append(torch.from_numpy(P.make_frame(360, 480, 500 + j)).cuda())
        base = np.array([[40.0, 30.0, 200.0, 330.0], [260.0, 50.0, 420.0, 340.0]])
        b = np.repeat(base, 3, 0) + rng.normal(0, 2, (6, 4))
        boxes.append(b)
        box_scores.append(rng.uniform(0.5, 1.0, 6))
        track_ids.append(np.arange(6) + 10 * j)
    before = [f.clone() for f in frames]
    ns = dict(model=m, frames=frames, boxes=boxes, box_scores=box_scores, track_ids=track_ids,
              smoother=DeviceOneEuro(3, 17, fps=30.0), skeleton=[(0, 1), (1, 2), (5, 6), (5, 11), (6, 12)])
    exec(compile(code, "INTEGRATION.md#3i", "exec"), ns)
    torch.cuda.synchronize()
    kps = [k.cpu().numpy() for k in m.infer_frames(frames=before, bboxes=boxes)[0]]
    counts = ns["res"].keep_counts.cpu().tolist()
    r = 0
    for j, kp in enumerate(kps):
        b = boxes[j]
        areas = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        want, _ = O.run_frame(kp, areas, box_scores[j], 0.9, rescore_vis_thr=0.2)
        assert counts[j] == len(want) and np.array_equal(ns["rows"].cpu().numpy()[r:r + len(want)] - 6 * j, want), j
        assert not torch.equal(frames[j], before[j])                      # the overlay drew
        r += len(want)
    assert ns["kept"].shape == (sum(counts), 17, 3)
