"""-m gpu: vpb_coco_eval (easy_vitpose_b200.coco_eval) against oracle/coco_oks_eval.py and its array form
oracle/coco_eval_oracle.py, bit for bit in the ten stats, the [3, 10, 101] precision and the [3, 10] recall.
The only allowed difference, CUDA's exp against numpy's moving an OKS by an ulp, is excluded by drawing sets that
oracle/coco_eval_oracle.flag_ambiguous does not flag, and each test asserts that.  Covered: the stored records of
tests/golden/coco_ap.npz; seeded random sets at K = 1, 17, 133 (images with ground truths only or detections only, more than
20 detections, ties within and across images, crowd and num_keypoints == 0 ground truths, all three area ranges, NaN scores,
duplicate ground truths); add in pieces and add_device; inference_topdown_eval(..., evaluator=); graph replay; limits and
argument errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import coco_eval_oracle as CO
from oracle import coco_oks_eval as E

pytestmark = pytest.mark.gpu


def _golden_gts(g):
    return [{"id": i + 1, "image_id": int(g["gt_image"][i]), "category_id": 1, "iscrowd": 0, "num_keypoints": int(g["gt_num"][i]),
             "keypoints": g["gt_keypoints"][i].tolist(), "bbox": g["gt_bbox"][i].tolist(), "area": float(g["gt_area"][i])}
            for i in range(len(g["gt_image"]))]


def _oracle(gts, recs, image_ids, sig):
    return CO.evaluate_full(gts, recs, image_ids, E.KPT_OKS_SIGMAS if sig is None else sig)


def _assert_same(got, want):
    for k in CO.STAT_NAMES:
        assert np.float64(got[k]).tobytes() == np.float64(want["stats"][k]).tobytes(), (k, got[k], want["stats"][k])
    assert np.array_equal(got["precision"].cpu().numpy(), want["precision"])
    assert np.array_equal(got["recall"].cpu().numpy(), want["recall"])


def test_golden_records_give_the_oracle_stats(golden_dir):
    from easy_vitpose_b200 import coco_eval
    g = np.load(os.path.join(golden_dir, "coco_ap.npz"))
    gts = _golden_gts(g)
    image_ids = [1000 + i for i in range(int(g["meta"][0]))]
    recs = [{"image_id": int(im), "category_id": 1, "score": float(s), "bbox": [], "keypoints": kp.tolist()}
            for im, s, kp in zip(g["res_image"], g["res_score"], g["res_keypoints"])]
    assert not CO.flag_ambiguous(gts, recs, image_ids)
    want = _oracle(gts, recs, image_ids, None)
    assert want["stats"] == E.evaluate(gts, recs, image_ids)
    ev = coco_eval.DeviceCocoEval(gts, image_ids)
    ev.add(recs)
    got = ev.evaluate()
    _assert_same(got, want)
    ref = dict(zip(g["stat_names"].tolist(), g["stat_values"].tolist()))
    assert all(abs(got[k] - ref[k]) < 1e-12 for k in ref)
    assert coco_eval.evaluate(gts, recs, image_ids) == E.evaluate(gts, recs, image_ids)


@pytest.mark.parametrize("K,seed", [(1, 1), (17, 2), (17, 3), (17, 4), (133, 5)])
def test_random_sets_equal_the_oracle(K, seed):
    from easy_vitpose_b200 import coco_eval
    gts, recs, image_ids, sig = CO.random_set(seed, K)
    assert not CO.flag_ambiguous(gts, recs, image_ids, E.KPT_OKS_SIGMAS if sig is None else sig)
    want = _oracle(gts, recs, image_ids, sig)
    # the set reaches what it is meant to: > 20 detections, ties, NaN, crowds, every area range with ground truths
    per_img = {}
    for r in recs:
        per_img[r["image_id"]] = per_img.get(r["image_id"], 0) + 1
    assert max(per_img.values()) > 20 and any(np.isnan(r["score"]) for r in recs)
    assert any(g["iscrowd"] for g in gts) and any(g["num_keypoints"] == 0 for g in gts)
    assert (want["precision"] > -1).all() and 0 < want["stats"]["AP"] < 1
    ev = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    ev.add(recs)
    got = ev.evaluate()
    _assert_same(got, want)
    assert {k: got[k] for k in CO.STAT_NAMES} == E.evaluate(gts, recs, image_ids, E.KPT_OKS_SIGMAS if sig is None else sig)


def test_single_image_and_empty_areas():
    """One image (no merge pass); an area range with no ground truth gives -1 precision and recall, as the oracle; no
    detections at all gives recall 0."""
    from easy_vitpose_b200 import coco_eval
    gts, recs, _, _ = CO.random_set(9, 17, n_img=6)
    img = next(g["image_id"] for g in gts)
    g1 = [dict(g, area=500.0) for g in gts if g["image_id"] == img]         # every one small: medium and large empty
    r1 = [r for r in recs if r["image_id"] == img]
    for rr in (r1, []):
        want = _oracle(g1, rr, [img], None)
        ev = coco_eval.DeviceCocoEval(g1, [img])
        ev.add(rr)
        _assert_same(ev.evaluate(), want)


def test_add_in_pieces_and_add_device_equal_one_add():
    from easy_vitpose_b200 import coco_eval
    gts, recs, image_ids, sig = CO.random_set(11, 17)
    one = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    one.add(recs)
    want = one.evaluate()
    pieces = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    for a in range(0, len(recs), 37):
        pieces.add(recs[a:a + 37])
    _assert_same(pieces.evaluate(), {"stats": {k: want[k] for k in CO.STAT_NAMES}, "precision": want["precision"].cpu().numpy(),
                                     "recall": want["recall"].cpu().numpy()})
    # the same records as device frames: float32 (y, x, score) rows, a frame per run of records of one image, plus a keep list
    dev = torch.device("cuda", 0)
    dv = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    kp = np.array([np.array(r["keypoints"]).reshape(17, 3) for r in recs])
    f32 = np.zeros((len(recs), 17, 3), np.float32)
    f32[..., 0], f32[..., 1] = kp[..., 1], kp[..., 0]
    exact = [{**r, "keypoints": np.stack([f32[i, :, 1], f32[i, :, 0], np.zeros(17)], 1).astype(np.float64).reshape(-1).tolist()}
             for i, r in enumerate(recs)]
    ref = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    ref.add(exact)
    want = ref.evaluate()
    runs, start = [], 0
    for i in range(1, len(recs) + 1):
        if i == len(recs) or recs[i]["image_id"] != recs[start]["image_id"]:
            runs.append((start, i))
            start = i
    half = len(runs) // 2
    for part, keep in ((runs[:half], False), (runs[half:], True)):
        rows = [i for a, b in part for i in range(a, b)]
        counts = [b - a for a, b in part]
        ids = [recs[a]["image_id"] for a, _ in part]
        kt = torch.from_numpy(f32[rows]).to(dev)
        st = torch.tensor([recs[i]["score"] for i in rows], dtype=torch.float64).to(dev)
        ct = torch.tensor(counts, dtype=torch.int32).to(dev)
        if not keep:
            dv.add_device(kt, st, ct, ids)
            continue
        # each frame padded with a decoy row the keep list leaves out; the kept rows keep their order
        prow, pkeep, pcounts = [], [], []
        for (a, b) in part:
            n = b - a
            prow += list(range(a, b)) + [a]
            pkeep += list(range(n)) + [-1]
            pcounts.append(n + 1)
        kt = torch.from_numpy(f32[prow]).to(dev)
        sc = np.array([recs[i]["score"] for i in prow], np.float64)
        sc[np.cumsum(pcounts) - 1] = 1e9                  # the decoys would lead every image if they were read
        dv.add_device(kt, torch.from_numpy(sc).to(dev), torch.tensor(pcounts, dtype=torch.int32).to(dev), ids,
                      keep=torch.tensor(pkeep, dtype=torch.int32).to(dev), keep_counts=ct)
    got = dv.evaluate()
    _assert_same(got, {"stats": {k: want[k] for k in CO.STAT_NAMES}, "precision": want["precision"].cpu().numpy(),
                       "recall": want["recall"].cpu().numpy()})


def test_inference_topdown_eval_feeds_the_evaluator():
    from easy_vitpose_b200 import B200PoseBackend, ViTPose, coco_eval, model_cfg
    from oracle import preproc_oracle as P
    from oracle import vitpose_oracle as VO
    D, depth, _ = VO.MODEL_DIMS["s"]
    m = ViTPose(model_cfg("s", 17), max_batch=32)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in VO.make_state_dict(D, depth, 17, 31, peaky=0.1, bumps=True).items()})
    be = B200PoseBackend(m, "cuda:0")
    rng = np.random.default_rng(5)
    frames, boxes, scores, ids = [], [], [], [7, 3, 7, 12]           # two frames of image 7
    for j in range(4):
        h, w = int(rng.integers(300, 480)), int(rng.integers(300, 560))
        frames.append(P.make_frame(h, w, 60 + j))
        b = np.stack([rng.uniform(0, w * 0.5, 6), rng.uniform(0, h * 0.5, 6), rng.uniform(40, w * 0.4, 6), rng.uniform(60, h * 0.5, 6)], 1)
        boxes.append(np.concatenate([b, b[:2] + rng.normal(0, 2, (2, 4))]))
        scores.append(rng.uniform(0.3, 1.0, 8))
    # ground truths near the boxes, so there are matches
    gts, gid = [], 1
    for j, b in enumerate(boxes):
        for x, y, bw, bh in b[:4]:
            kp = np.stack([x + rng.uniform(0, bw, 17), y + rng.uniform(0, bh, 17), np.full(17, 2.0)], 1)
            gts.append({"id": gid, "image_id": ids[j], "category_id": 1, "iscrowd": 0, "num_keypoints": 17, "keypoints": kp.reshape(-1).tolist(),
                        "bbox": [float(x), float(y), float(bw), float(bh)], "area": float(bw * bh)})
            gid += 1
    ev = coco_eval.DeviceCocoEval(gts, sorted(set(ids)))
    plain = be.inference_topdown_eval(frames, boxes, scores)
    got = be.inference_topdown_eval(frames, boxes, scores, evaluator=ev, image_ids=ids)
    for (ak, as_, ai), (bk, bs, bi) in zip(plain, got):
        assert np.array_equal(ak, bk) and np.array_equal(as_, bs) and np.array_equal(ai, bi)
    recs = []
    for j, (kp, sc, _) in enumerate(got):
        recs += [{"image_id": ids[j], "category_id": 1, "score": float(s),
                  "keypoints": np.stack([k[:, 1], k[:, 0], k[:, 2]], 1).astype(np.float64).reshape(-1).tolist()} for k, s in zip(kp, sc)]
    ref = coco_eval.DeviceCocoEval(gts, sorted(set(ids)))
    ref.add(recs)
    a, b = ev.evaluate(), ref.evaluate()
    _assert_same(a, {"stats": {k: b[k] for k in CO.STAT_NAMES}, "precision": b["precision"].cpu().numpy(), "recall": b["recall"].cpu().numpy()})
    assert not CO.flag_ambiguous(gts, recs, sorted(set(ids)))
    want = _oracle(gts, recs, sorted(set(ids)), None)
    _assert_same(a, want)


def test_graph_replay_equals_eager():
    from easy_vitpose_b200 import coco_eval
    gts, recs, image_ids, sig = CO.random_set(21, 17, n_img=60)
    ev = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    ev.add(recs)
    eager = ev.evaluate()
    dev = torch.device("cuda", 0)
    ch = ev._chunks
    args = [torch.cat([c[j] for c in ch]) for j in range(6)]
    ws = torch.empty(coco_eval.workspace_bytes(len(image_ids), args[2].shape[0]), dtype=torch.uint8, device=dev)
    out = coco_eval.CocoEvalResult(torch.full((10,), -7.0, dtype=torch.float64, device=dev), torch.zeros((3, 10, 101), dtype=torch.float64, device=dev),
                                   torch.zeros((3, 10), dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        coco_eval.coco_eval_device(*ev._gt, *args, sigmas=sig, workspace=ws, out=out)      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    out.stats.fill_(-7.0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        coco_eval.coco_eval_device(*ev._gt, *args, sigmas=sig, workspace=ws, out=out)
    for _ in range(3):
        out.stats.fill_(-7.0)
        out.precision.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert int(out.status.item()) == 0
        assert np.array_equal(out.stats.cpu().numpy(), np.array([eager[k] for k in CO.STAT_NAMES]))
        assert torch.equal(out.precision, eager["precision"]) and torch.equal(out.recall, eager["recall"])


def test_limits_and_argument_errors():
    from easy_vitpose_b200 import _lib, coco_eval
    dev = torch.device("cuda", 0)
    gts, recs, image_ids, sig = CO.random_set(31, 17, n_img=10)
    good = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    good.add(recs)
    want = good.evaluate()
    # an image with more than MAX_GTS ground truths
    img = image_ids[0]
    many = gts + [dict(gts[0], id=10 ** 6 + i, image_id=img) for i in range(coco_eval.MAX_GTS + 1)]
    ev = coco_eval.DeviceCocoEval(many, image_ids, sig)
    ev.add(recs)
    with pytest.raises(ValueError, match="ground truths"):
        ev.evaluate()
    res = ev.evaluate_device()
    assert torch.isnan(res.stats).all()
    # an image with more than MAX_ROWS detection rows
    ev = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    ev.add(recs + [dict(recs[0], image_id=img)] * (coco_eval.MAX_ROWS + 1))
    with pytest.raises(ValueError, match="detections"):
        ev.evaluate()
    # frame tables that do not fit the rows, keep entries outside their frame
    ev = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    kt = torch.zeros((4, 17, 3), dtype=torch.float32, device=dev)
    st = torch.ones(4, dtype=torch.float64, device=dev)
    ev.add_device(kt, st, torch.tensor([2, 3], dtype=torch.int32, device=dev), [img, img])
    with pytest.raises(ValueError, match="out of range"):
        ev.evaluate()
    ev = coco_eval.DeviceCocoEval(gts, image_ids, sig)
    ev.add_device(kt, st, torch.tensor([4], dtype=torch.int32, device=dev), [img], keep=torch.tensor([0, 5, -1, -1], dtype=torch.int32, device=dev),
                  keep_counts=torch.tensor([2], dtype=torch.int32, device=dev))
    with pytest.raises(ValueError, match="out of range"):
        ev.evaluate()
    with pytest.raises(ValueError):
        ev.add_device(kt, st, torch.tensor([4], dtype=torch.int32, device=dev), [123456789])      # not an evaluated image
    with pytest.raises(ValueError):
        coco_eval.DeviceCocoEval([dict(gts[0], id=0)], image_ids)
    # VPB_ERR_ARG
    L = _lib.lib()
    ws = torch.empty(coco_eval.workspace_bytes(1, 0), dtype=torch.uint8, device=dev)
    o = torch.zeros(400, dtype=torch.float64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    off = torch.zeros(2, dtype=torch.int32, device=dev)
    P = lambda t: C.c_void_p(t.data_ptr())                                                     # noqa: E731
    g0 = _lib.VpbCocoGts(P(off), None, None, None, None, None, 1, 0)
    d0 = _lib.VpbCocoDets(None, None, None, None, None, None, 0, 0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(k=17, sigmas=None, gts_=g0, dets=d0, wsb=None, stats=o):
        return L.vpb_coco_eval(k, sigmas, C.byref(gts_) if gts_ is not None else None, C.byref(dets) if dets is not None else None, P(ws),
                               ws.numel() if wsb is None else wsb, P(stats) if stats is not None else None, P(o[10:]), P(o[350:]), P(status), stream)
    assert call() == 0
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    bad_sig = (C.c_double * 17)(*([0.05] * 16 + [float("inf")]))
    for kw in (dict(k=0), dict(k=145), dict(k=5), dict(sigmas=C.cast(bad_sig, C.c_void_p)), dict(gts_=None), dict(dets=None),
               dict(wsb=16), dict(stats=None), dict(gts_=_lib.VpbCocoGts(P(off), None, None, None, None, None, 0, 0)),
               dict(gts_=_lib.VpbCocoGts(P(off), None, None, None, None, None, 1, 3)),
               dict(dets=_lib.VpbCocoDets(None, None, None, None, None, None, 5, 0)),
               dict(dets=_lib.VpbCocoDets(P(o), P(o), P(off), P(off), P(off), None, 1, 1))):
        assert call(**kw) == 1, kw
    assert L.vpb_coco_eval_workspace_bytes(0, 0) == -1 and L.vpb_coco_eval_workspace_bytes(1, -1) == -1
    # a later valid call is unaffected
    again = good.evaluate()
    _assert_same(again, {"stats": {k: want[k] for k in CO.STAT_NAMES}, "precision": want["precision"].cpu().numpy(),
                         "recall": want["recall"].cpu().numpy()})
