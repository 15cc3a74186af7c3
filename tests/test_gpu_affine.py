"""-m gpu: affine top-down crops (ViTPose.preprocess_affine / infer_affine / infer_affine_host, vpb_*_affine).

The contract:
    crops = preprocess_affine(frames, mats)         # cv2.warpAffine + ToTensor / Normalize, bit-exact (oracle/affine_oracle.py)
    hm = forward(crops)                             # or forward_flip_test(crops, pairs) with flip test on
    kpts, idx = vpb_decode_modes(hm, mode 4, cs)    # keypoints_from_heatmaps(hm, c, s * 200, use_udp=True)
and infer_affine returns exactly that, bit for bit, with the warp fused into the patch gather.  Against the fp32 reference
(tests/golden/affine_b_coco.npz, oracle/make_golden_affine.py) the tolerances of test_gpu_batch_parity apply."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import affine_oracle as A, preproc_oracle as P, vitpose_oracle as O
from oracle.flip_weights import flip_symmetric_state_dict

pytestmark = pytest.mark.gpu

HEATMAP_TOL = 0.01
KPT_MEAN_PX_TOL = 0.5
MAX_BATCH = 16
_engines = {}


def _engine(flip: bool, seed: int):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, ViTPose, model_cfg
    key = (flip, seed)
    if key not in _engines:
        D, depth, _ = O.MODEL_DIMS["b"]
        sd = (flip_symmetric_state_dict(D, depth, 17, seed, [tuple(p) for p in COCO_FLIP_PAIRS]) if flip
              else O.make_state_dict(D, depth, 17, seed, peaky=0.1, bumps=True))
        m = ViTPose(model_cfg("b", 17), max_batch=MAX_BATCH)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        _engines[key] = m.to("cuda:0")
    return _engines[key]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "affine_b_coco.npz"))


def _frames(g):
    return [P.make_frame(int(h), int(w), int(s)) for h, w, s in g["frames"]]


def _decode_mode4(hm, cs):
    from easy_vitpose_b200 import _lib
    n, K = hm.shape[:2]
    kp = torch.empty((n, K, 3), dtype=torch.float32, device=hm.device)
    idx = torch.empty((n, K), dtype=torch.int32, device=hm.device)
    _lib.check(_lib.lib().vpb_decode_modes(C.c_void_p(hm.data_ptr()), n, K, 4, C.c_void_p(cs.data_ptr()), None,
                                           C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return kp, idx


def test_preprocess_affine_bit_exact(golden):
    g = golden
    m = _engine(False, int(g["meta"][4]))
    frames = _frames(g)
    table = A.normalise_table()
    # the fixture's cases, grouped by frame: crops come back in frame order
    order = np.argsort(g["frame_id"], kind="stable")
    mats = [g["mats"][order][g["frame_id"][order] == f] for f in range(len(frames))]
    crops = m.preprocess_affine([torch.from_numpy(f).cuda() for f in frames], mats).cpu().numpy()
    stored = dict(zip(g["crop_ids"].tolist(), g["crops"]))
    for j, i in enumerate(order):
        want = A.warp_normalise(frames[g["frame_id"][i]], g["mats"][i])
        assert np.array_equal(crops[j], want), i
        if i in stored:
            assert np.array_equal(crops[j], np.stack([table[c][stored[i][..., c]] for c in range(3)], 0)), i
    # random matrices (rotation, shear, up / down scaling, out of frame, singular) on a pitched frame (a column slice)
    wide = P.make_frame(220, 400, 13)
    sl = torch.from_numpy(wide).cuda()[:, 60:320]
    rs = np.random.RandomState(3)
    ms = []
    for i in range(40):
        th, k = np.deg2rad(rs.uniform(-60, 60)), np.exp(rs.uniform(-2, 2))
        mm = np.array([[k * np.cos(th), -k * np.sin(th), rs.uniform(-300, 300)], [k * np.sin(th), k * np.cos(th), rs.uniform(-300, 300)]])
        ms.append(np.zeros((2, 3)) if i == 0 else (np.array([[1.0, 2, 5], [2, 4, 7]]) if i == 1 else mm))
    crops = m.preprocess_affine([sl], [np.stack(ms)]).cpu().numpy()
    host = np.ascontiguousarray(wide[:, 60:320])
    for i, mm in enumerate(ms):
        assert np.array_equal(crops[i], A.warp_normalise(host, mm)), i


def _random_case(n, nframes, seed):
    """n boxes spread over nframes frames of different sizes -> (frames, per-frame boxes xywh)."""
    rs = np.random.RandomState(seed)
    sizes = [(240 + 40 * j, 320 + 56 * j) for j in range(nframes)]
    frames = [P.make_frame(h, w, seed + j) for j, (h, w) in enumerate(sizes)]
    owner = np.sort(np.concatenate([np.arange(nframes), rs.randint(0, nframes, n - nframes)]))   # every frame has a box
    boxes = []
    for j, (h, w) in enumerate(sizes):
        k = int((owner == j).sum())
        bw, bh = rs.uniform(8, w * 0.8, k), rs.uniform(8, h * 0.8, k)
        boxes.append(np.stack([rs.uniform(-0.2 * w, w) - bw / 2, rs.uniform(-0.2 * h, h) - bh / 2, bw, bh], 1))
    return frames, boxes


def _composition(m, frames_d, args, flip_pairs=None):
    mats, cs = [a[0] for a in args], np.concatenate([np.concatenate([a[1], a[2]], 1) for a in args], 0)
    crops = m.preprocess_affine(frames_d, mats)
    hm = m.forward_flip_test(crops, flip_pairs) if flip_pairs else m.forward(crops)
    return _decode_mode4(hm, torch.from_numpy(cs).cuda()), hm


@pytest.mark.parametrize("graph", [1, 0])
def test_infer_affine_bit_identical_to_composition(graph):
    from easy_vitpose_b200 import topdown_args
    m = _engine(False, 131)
    m.set_option("graph", graph)
    try:
        for n in (1, 7, MAX_BATCH):
            for nframes in (1, 3):
                if nframes > n:
                    continue
                frames, boxes = _random_case(n, nframes, 100 * n + nframes)
                frames_d = [torch.from_numpy(f).cuda() for f in frames]
                args = [topdown_args(b) for b in boxes]
                (kp_r, idx_r), _ = _composition(m, frames_d, args)
                for call in range(3):                 # eager, capture, replay (graph on)
                    kp, idx = m.infer_affine(frames_d, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], check=True)
                    assert torch.equal(torch.cat(kp), kp_r) and torch.equal(torch.cat(idx), idx_r), (n, nframes, graph, call)
    finally:
        m.set_option("graph", 1)


def test_infer_affine_host_equals_device_and_chunks():
    from easy_vitpose_b200 import B200PoseBackend, topdown_args
    m = _engine(False, 131)
    frames, boxes = _random_case(2 * MAX_BATCH + 5, 3, 7)          # three engine calls
    args = [topdown_args(b) for b in boxes]
    kp_d, idx_d = m.infer_affine([torch.from_numpy(f).cuda() for f in frames], [a[0] for a in args], [a[1] for a in args],
                                 [a[2] for a in args])
    kp_h, idx_h = m.infer_affine_host(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args])
    for a, b, c, d in zip(kp_d, idx_d, kp_h, idx_h):
        assert np.array_equal(a.cpu().numpy(), c) and np.array_equal(b.cpu().numpy(), d)
    # one call per chunk equals the whole: the decode runs per crop unless a map's maximum is <= 0
    kp_1, _ = m.infer_affine_host(frames[:1], args[0][0:1], args[0][1:2], args[0][2:3])
    assert np.array_equal(kp_1[0], kp_h[0])
    back = B200PoseBackend(m).inference_topdown(frames, boxes)
    for a, b in zip(back, kp_h):
        assert np.array_equal(a, b)


def _check_vs_reference(tag, kp, idx, hm, g, key):
    ref_kp, ref_idx = g[f"kpts_{key}"], g[f"idx_{key}"]
    B, K = idx.shape
    rng = float(g[f"range_{key}"][1] - g[f"range_{key}"][0])
    linf = float(np.abs(hm[g["sample_crops"]][:, g["sample_kps"]] - g[f"sample_hm_{key}"]).max())
    msum = float(np.abs(hm.reshape(B, K, -1).sum(-1, dtype=np.float64) - g[f"map_sum_{key}"]).max() / 3072.0)
    s = g["cs_px"][:, 2:]
    to_model_px = np.stack([256.0 / s[:, 1], 192.0 / s[:, 0]], -1)[:, None, :]          # (y, x): image px -> input px
    dev = np.linalg.norm((kp[..., :2] - ref_kp[..., :2]) * to_model_px, axis=-1)
    vis = ref_kp[..., 2] > 0.3
    cell = np.maximum(np.abs(idx % 48 - ref_idx % 48), np.abs(idx // 48 - ref_idx // 48))
    far = vis & (cell > 1)
    flat = hm.reshape(B, K, -1)
    gap = flat.max(-1) - np.take_along_axis(flat, ref_idx[..., None].astype(np.int64), -1)[..., 0]
    print(tag, f"heatmaps Linf {linf / rng:.3%} of range, mean-per-pixel drift {msum / rng:.4%}; visible {int(vis.sum())}/{vis.size}; "
          f"keypoint deviation (input px) mean {dev[vis].mean():.4f} max {dev[vis].max():.4f}; far arg-max flips {int(far.sum())}")
    assert linf < HEATMAP_TOL * rng
    assert msum < HEATMAP_TOL * rng            # the L-inf bar on every map's mean (black and frame-filling crops drift more)
    assert vis.sum() >= 0.7 * vis.size
    assert dev[vis].mean() < KPT_MEAN_PX_TOL
    assert far.sum() <= 0.01 * vis.sum() + 1
    assert np.all(gap[far] <= 2 * HEATMAP_TOL * rng)
    assert np.array_equal(idx, flat.argmax(-1).astype(np.int32))          # bit-exact integer work on the engine's own maps


def _fixture_inputs(g):
    frames = _frames(g)
    fwd = g["fwd"]
    fid = g["frame_id"][fwd]
    assert np.all(np.diff(fid) >= 0)
    mats = [g["mats"][fwd][fid == f] for f in range(len(frames))]
    cs = g["cs_px"]
    return frames, mats, [cs[fid == f, :2] for f in range(len(frames))], [cs[fid == f, 2:] for f in range(len(frames))]


def test_infer_affine_vs_reference_fixture(golden):
    g = golden
    m = _engine(False, int(g["meta"][4]))
    frames, mats, cs, ss = _fixture_inputs(g)
    frames_d = [torch.from_numpy(f).cuda() for f in frames]
    kp, idx = m.infer_affine(frames_d, mats, cs, ss, check=True)
    hm = m.forward(m.preprocess_affine(frames_d, mats))
    _check_vs_reference("plain", torch.cat(kp).cpu().numpy(), torch.cat(idx).cpu().numpy(), hm.cpu().numpy(), g, "plain")


def test_infer_affine_flip_test(golden):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, topdown_args
    g = golden
    pairs = [tuple(p) for p in COCO_FLIP_PAIRS]
    m = _engine(True, int(g["meta"][5]))
    frames, mats, cs, ss = _fixture_inputs(g)
    frames_d = [torch.from_numpy(f).cuda() for f in frames]
    m.set_flip_test(pairs, False)
    try:
        assert m.batch_limit == MAX_BATCH // 2
        kp, idx = m.infer_affine(frames_d, mats, cs, ss)          # 12 boxes: two calls of 8 and 4
        # the composition, chunk by chunk as infer_affine calls the engine
        crops = m.preprocess_affine(frames_d, mats)
        cs_all = torch.from_numpy(np.concatenate([np.concatenate([c, s], 1) for c, s in zip(cs, ss)], 0)).cuda()
        hms, kps, idxs = [], [], []
        for s in range(0, crops.shape[0], MAX_BATCH // 2):
            hms.append(m.forward_flip_test(crops[s:s + MAX_BATCH // 2], pairs))
            k_, i_ = _decode_mode4(hms[-1], cs_all[s:s + MAX_BATCH // 2].contiguous())
            kps.append(k_); idxs.append(i_)
        assert torch.equal(torch.cat(kp), torch.cat(kps)) and torch.equal(torch.cat(idx), torch.cat(idxs))
        for n in (1, 7, MAX_BATCH // 2):
            for call in range(3):
                fr, boxes = _random_case(n, 3 if n >= 3 else 1, 300 + n)
                fd = [torch.from_numpy(f).cuda() for f in fr]
                a = [topdown_args(b) for b in boxes]
                (kr, ir), _ = _composition(m, fd, a, pairs)
                k2, i2 = m.infer_affine(fd, [x[0] for x in a], [x[1] for x in a], [x[2] for x in a])
                assert torch.equal(torch.cat(k2), kr) and torch.equal(torch.cat(i2), ir), (n, call)
        kp_h, _ = m.infer_affine_host(frames, mats, cs, ss)
        assert np.array_equal(np.concatenate(kp_h), torch.cat(kp).cpu().numpy())
        _check_vs_reference("flip", torch.cat(kp).cpu().numpy(), torch.cat(idx).cpu().numpy(), torch.cat(hms).cpu().numpy(), g, "flip")
    finally:
        m.set_flip_test(None)


def test_affine_errors():
    from easy_vitpose_b200 import _lib
    L = _lib.lib()
    m = _engine(False, 131)
    frame = torch.from_numpy(P.make_frame(64, 80, 1)).cuda()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    eye = np.tile(np.array([1.0, 0, 0, 0, 1, 0]), (MAX_BATCH + 1, 1))
    cs = np.tile(np.array([40.0, 32, 80, 64], np.float32), (MAX_BATCH + 1, 1))
    M, CS = torch.from_numpy(eye).cuda(), torch.from_numpy(cs).cuda()
    kp = torch.empty((MAX_BATCH + 1, 17, 3), device="cuda")

    def frames(count, n_each=1, data=None, h=64, w=80, pitch=0):
        arr = (_lib.VpbFrame * count)()
        for j in range(count):
            arr[j] = _lib.VpbFrame(frame.data_ptr() if data is None else data, h, w, pitch, n_each)
        return arr

    def dev(arr, M=M, CS=CS):
        return L.vpb_infer_affine(m._handle, arr, len(arr), C.c_void_p(M.data_ptr()), C.c_void_p(CS.data_ptr()),
                                  C.c_void_p(kp.data_ptr()), None, st)

    def host(arr, mats=eye, c=cs):
        kh = np.empty((MAX_BATCH + 1, 17, 3), np.float32)
        return L.vpb_infer_affine_host(m._handle, arr, len(arr), mats.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p),
                                       kh.ctypes.data_as(C.c_void_p), None, st)

    frame_np = P.make_frame(64, 80, 1)
    for call in (dev, host):
        hp = None if call is dev else frame_np.ctypes.data
        assert call(frames(1, MAX_BATCH + 1, hp)) == 1                       # above max_batch
        assert call(frames(65, 0, hp)) == 0                                   # frames without boxes are skipped
        assert call(frames(1, -1, hp)) == 1                                   # negative count
        assert call(frames(1, 1, 0)) == 1                                     # NULL frame
        assert call(frames(1, 1, hp, h=0)) == 1                               # bad size
        assert call(frames(1, 1, hp, pitch=100)) == 1                         # pitch < 3 * width
    arr = frames(1, 1)
    assert L.vpb_infer_affine(m._handle, arr, 1, None, C.c_void_p(CS.data_ptr()), C.c_void_p(kp.data_ptr()), None, st) == 1
    assert L.vpb_preprocess_affine(arr, 1, None, C.c_void_p(kp.data_ptr()), st) == 1
    # more than VPB_MAX_FRAMES frames with boxes: 65 boxes exceed this engine's batch limit first, so the engine-free call
    # checks the frame limit; 9 frames with boxes among 65 entries are fine
    big =(_lib.VpbFrame * 65)(*[_lib.VpbFrame(frame.data_ptr(), 64, 80, 0, 1) for _ in range(65)])
    crops = torch.empty((65, 3, 256, 192), device="cuda")
    M65 = torch.from_numpy(np.tile(np.array([1.0, 0, 0, 0, 1, 0]), (65, 1))).cuda()
    assert L.vpb_preprocess_affine(big, 65, C.c_void_p(M65.data_ptr()), C.c_void_p(crops.data_ptr()), st) == 1
    assert L.vpb_preprocess_affine(big, 64, C.c_void_p(M65.data_ptr()), C.c_void_p(crops.data_ptr()), st) == 0
    nine = (_lib.VpbFrame * 65)(*[_lib.VpbFrame(frame.data_ptr(), 64, 80, 0, 1 if j % 8 == 0 else 0) for j in range(65)])
    assert dev(nine) == 0
    # non-finite matrix entries and scales <= 0: VPB_ERR_ARG from the host form, bit 1 of the status word from the device form
    hp = frames(1, 2, frame_np.ctypes.data)
    bad = eye.copy()
    bad[1, 4] = np.inf
    assert host(hp, mats=bad) == 1 and b"matrix entry" in L.vpb_last_error()
    bad_cs = cs.copy()
    bad_cs[1, 3] = 0
    assert host(hp, c=bad_cs) == 1 and b"scale" in L.vpb_last_error()
    assert host(hp) == 0
    m.frame_status()
    assert dev(frames(1, 2), M=torch.from_numpy(bad).cuda()) == 0 and m.frame_status() == 2
    assert dev(frames(1, 2), CS=torch.from_numpy(bad_cs).cuda()) == 0 and m.frame_status() == 2
    assert dev(frames(1, 2)) == 0 and m.frame_status() == 0
    with pytest.raises(ValueError, match="not finite"):
        m.infer_affine([frame], [torch.from_numpy(bad[:2]).cuda()], [cs[:2, :2]], [cs[:2, 2:]], check=True)
    with pytest.raises(ValueError, match="non-finite"):
        m.infer_affine([frame], [bad[:2]], [cs[:2, :2]], [cs[:2, 2:]])
    with pytest.raises(ValueError, match="matrix entry"):
        m.infer_affine_host([frame_np], [bad[:2]], [cs[:2, :2]], [cs[:2, 2:]])
    torch.cuda.synchronize()
