"""-m gpu: flip test on the keypoint paths (ViTPose.set_flip_test / vpb_set_flip_test).

The contract: with flip test on, the keypoint calls return exactly -- bit for bit -- what the composition
    hm = forward_flip_test(x, pairs, shift)      # forward(x), forward(flip(x)), flip_back, (a + b) * 0.5
    kpts, idx = decode_heatmaps(hm, org_wh)      # wrap_batch = 0 (+ frame offsets on the frame path)
returns, while running the crops and their mirror images as ONE batch (the forward is batch-invariant).  Against the fp32
reference (tests/golden/flip_*_coco.npz, oracle/make_golden_flip.py) the tolerances of test_gpu_batch_parity apply."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O
from oracle.flip_weights import flip_symmetric_state_dict

pytestmark = pytest.mark.gpu

HEATMAP_TOL = 0.01
KPT_MEAN_PX_TOL = 0.5
SIZES = {384: "s", 768: "b", 1024: "l", 1280: "h"}


def _coco_pairs():
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    return [tuple(p) for p in COCO_FLIP_PAIRS]


def _synthetic_pairs(K, seed=4):
    """Disjoint random pairs over K keypoints plus one pair that overrides an earlier one (the sequential rule)."""
    order = np.random.RandomState(seed).permutation(K)
    pairs = [(int(order[2 * i]), int(order[2 * i + 1])) for i in range(K // 3)]
    return pairs + [(pairs[0][0], int(order[-1]))]


_engines = {}


def _engine(size, K, depth, seed, max_batch=16, flip_pairs=None):
    from easy_vitpose_b200 import ViTPose, model_cfg
    key = (size, K, depth, seed, max_batch, None if flip_pairs is None else tuple(flip_pairs))
    if key not in _engines:
        cfg = model_cfg(size, K)
        cfg["backbone"]["depth"] = depth
        D = cfg["backbone"]["embed_dim"]
        sd = (O.make_state_dict(D, depth, K, seed, peaky=0.1, bumps=True) if flip_pairs is None
              else flip_symmetric_state_dict(D, depth, K, seed, flip_pairs))
        m = ViTPose(cfg, max_batch=max_batch)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        _engines[key] = m.to("cuda:0")
    return _engines[key]


def _composition(m, x, org, pairs, shift):
    from easy_vitpose_b200 import decode_heatmaps
    hm = m.forward_flip_test(x, pairs, shift)
    kp, idx = decode_heatmaps(hm, org)
    return kp, idx, hm


def _org(n, seed):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(np.stack([rs.randint(64, 513, n), rs.randint(64, 513, n)], 1).astype(np.int32))


# ViT-S/17 and ViT-B/17 at full depth; ViT-H (head_dim 80) with K = 133 at reduced depth: the identity is per kernel, not per layer
@pytest.mark.parametrize("size,K,depth,pairs", [("s", 17, 12, "coco"), ("b", 17, 12, "coco"), ("h", 133, 4, "synthetic")])
def test_flip_infer_crops_bit_identical_to_composition(size, K, depth, pairs):
    m = _engine(size, K, depth, 131)
    pairs = _coco_pairs() if pairs == "coco" else _synthetic_pairs(K)
    launches_off = m.kernel_launches(4)
    try:
        for shift in (False, True):
            m.set_flip_test(pairs, shift)
            assert m.flip_test and m.batch_limit == 8
            assert m.kernel_launches(4) == launches_off + 1
            for n in (1, 7, 8):
                x = torch.from_numpy(O.make_crops(n, 40 + n)).cuda()
                org = _org(n, n)
                kp_r, idx_r, hm_r = _composition(m, x, org, pairs, shift)
                for graph in (1, 0):
                    m.set_option("graph", graph)
                    for call in range(3):                    # graph on: eager, capture, replay
                        if call == 1:                          # the averaged maps stay inside the engine (in place)
                            kp, idx = m.infer_crops(x, org)
                        else:
                            kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
                            assert torch.equal(hm, hm_r), (size, shift, n, graph, call)
                        assert torch.equal(kp, kp_r) and torch.equal(idx, idx_r), (size, shift, n, graph, call)
                m.set_option("graph", 1)
    finally:
        m.set_option("graph", 1)
        m.set_flip_test(None)
    assert not m.flip_test and m.batch_limit == 16 and m.kernel_launches(4) == launches_off


def test_flip_host_paths_match_device_path():
    m = _engine("s", 17, 12, 131)
    pairs = _coco_pairs()
    m.set_flip_test(pairs, True)
    try:
        xs = [O.make_crops(n, 60 + n) for n in (8, 5, 3)]
        orgs = [_org(len(x), 70 + len(x)).numpy() for x in xs]
        want = [[t.cpu().numpy() for t in m.infer_crops(torch.from_numpy(x).cuda(), torch.from_numpy(o))] for x, o in zip(xs, orgs)]
        for (wk, wi), x, o in zip(want, xs, orgs):
            kp, idx = m.infer_host(x, o)
            assert np.array_equal(kp, wk) and np.array_equal(idx, wi)
        pinned = [torch.from_numpy(x).pin_memory().numpy() for x in xs]
        kps = [np.empty((len(x), 17, 3), np.float32) for x in xs]
        ids = [np.empty((len(x), 17), np.int32) for x in xs]
        m.submit_host(pinned[0], orgs[0], kps[0], ids[0], 0)
        for i in range(1, 3):
            m.submit_host(pinned[i], orgs[i], kps[i], ids[i], i % 2)
            m.wait_host((i - 1) % 2)
        m.wait_host(0)
        for (wk, wi), k, i in zip(want, kps, ids):
            assert np.array_equal(k, wk) and np.array_equal(i, wi)
    finally:
        m.set_flip_test(None)


def _frame_case(golden_dir):
    g = np.load(os.path.join(golden_dir, "frame_a.npz"))
    fh, fw, fseed = (int(v) for v in g["meta"][:3])
    rows = g["rows"].astype(np.float64)
    boxes = rows[rows[:, 4] > 0.35, :4].round().astype(np.int32)
    return g, P.make_frame(fh, fw, fseed), boxes


def test_flip_frame_paths_equal_crops_path(golden_dir):
    """infer_frame / infer_frame_host / submit_frame_host with flip test == preprocess -> infer_crops (flip test) -> + offsets."""
    g, frame, boxes = _frame_case(golden_dir)
    D, depth, heads, K, wseed = (int(v) for v in g["meta"][3:8])
    m = _engine(SIZES[D], K, depth, wseed)
    m.set_flip_test(_coco_pairs())
    try:
        fr = torch.from_numpy(frame).cuda()
        crops, org, offs = m.preprocess(fr, boxes)
        kp_c, idx_c = m.infer_crops(crops, org)
        want_kp = P.to_frame_coords(kp_c.cpu().numpy(), offs.cpu().numpy())
        want_idx = idx_c.cpu().numpy()
        for _ in range(3):                                               # eager, capture, replay
            kp, idx = m.infer_frame(fr, boxes)
            assert np.array_equal(kp.cpu().numpy(), want_kp) and np.array_equal(idx.cpu().numpy(), want_idx)
            kp_h, idx_h = m.infer_frame_host(frame, boxes)
            assert np.array_equal(kp_h, want_kp) and np.array_equal(idx_h, want_idx)
        # chunking at batch_limit = max_batch // 2: 14 boxes through a max_batch = 16 engine
        kp_t, _ = m.infer_frame_host(frame, np.tile(boxes, (2, 1)))
        assert np.array_equal(kp_t, np.tile(want_kp, (2, 1, 1)))
        # pipelined frames, different box counts in flight on the two slots
        frames = [torch.from_numpy(P.make_frame(360, 480, 11 + i)).pin_memory().numpy() for i in range(4)]
        bbs = [np.ascontiguousarray(boxes[: 7 - 2 * (i % 3)]) for i in range(4)]
        want = [m.infer_frame_host(f, b) for f, b in zip(frames, bbs)]
        kps = [np.empty((len(b), K, 3), np.float32) for b in bbs]
        ids = [np.empty((len(b), K), np.int32) for b in bbs]
        m.submit_frame_host(frames[0], bbs[0], kps[0], ids[0], 0)
        for i in range(1, 4):
            m.submit_frame_host(frames[i], bbs[i], kps[i], ids[i], i % 2)
            m.wait_host((i - 1) % 2)
        m.wait_host(1)
        for (wk, wi), k, i in zip(want, kps, ids):
            assert np.array_equal(wk, k) and np.array_equal(wi, i)
    finally:
        m.set_flip_test(None)


def test_flip_off_restores_plain_outputs():
    from easy_vitpose_b200 import ViTPose, model_cfg
    m = _engine("b", 17, 12, 131)
    x = torch.from_numpy(O.make_crops(6, 81)).cuda()
    org = _org(6, 82)
    m.set_flip_test(_coco_pairs(), True)
    for _ in range(3):
        m.infer_crops(x, org)
    m.set_flip_test(None)
    fresh = ViTPose(model_cfg("b", 17), max_batch=16)
    fresh.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(768, 12, 17, 131, peaky=0.1, bumps=True).items()})
    fresh.to("cuda:0")
    kp_f, idx_f, hm_f = fresh.infer_crops(x, org, return_heatmaps=True)
    for _ in range(3):
        kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
        assert torch.equal(kp, kp_f) and torch.equal(idx, idx_f) and torch.equal(hm, hm_f)


def _check_vs_reference(name, kp, idx, hm, ref_kp, ref_idx, rng, org):
    B, K = idx.shape
    to_model_px = np.stack([256.0 / org[:, 1], 192.0 / org[:, 0]], -1)[:, None, :]
    dev = np.linalg.norm((kp[..., :2] - ref_kp[..., :2]) * to_model_px, axis=-1)
    vis = ref_kp[..., 2] > 0.3
    cell = np.maximum(np.abs(idx % 48 - ref_idx % 48), np.abs(idx // 48 - ref_idx // 48))
    far = vis & (cell > 1)
    flat = hm.reshape(B, K, -1)
    gap = flat.max(-1) - np.take_along_axis(flat, ref_idx[..., None].astype(np.int64), -1)[..., 0]
    print(name, f"visible {int(vis.sum())}/{vis.size}; keypoint deviation px mean {dev[vis].mean():.4f} max {dev[vis].max():.4f}; "
          f"far arg-max flips {int(far.sum())}")
    assert vis.sum() >= 0.7 * vis.size
    assert dev[vis].mean() < KPT_MEAN_PX_TOL
    assert far.sum() <= 0.01 * vis.sum() + 1
    assert np.all(gap[far] <= 2 * HEATMAP_TOL * rng)
    assert np.array_equal(idx, flat.argmax(-1).astype(np.int32))          # bit-exact integer work on the engine's own maps


@pytest.mark.parametrize("name", ["flip_s_coco", "flip_b_coco"])
def test_flip_vs_reference_fixture(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    D, depth, heads, K, B, wseed, xseed, fh, fw, fseed = (int(v) for v in g["meta"])
    pairs = _coco_pairs()
    m = _engine(SIZES[D], K, depth, wseed, flip_pairs=pairs)
    x = torch.from_numpy(O.make_crops(B, xseed)).cuda()
    try:
        for shift in (0, 1):
            m.set_flip_test(pairs, bool(shift))
            kp, idx, hm = (t.cpu().numpy() for t in m.infer_crops(x, torch.from_numpy(g["org_wh"]), return_heatmaps=True))
            rng = float(g[f"range_{shift}"][1] - g[f"range_{shift}"][0])
            linf = float(np.abs(hm[g["crop_ids"]][:, g["kp_ids"]] - g[f"sample_hm_{shift}"]).max())
            msum = float(np.abs(hm.reshape(B, K, -1).sum(-1, dtype=np.float64) - g[f"map_sum_{shift}"]).max() / 3072.0)
            print(name, f"shift={shift}: sampled heatmaps Linf {linf / rng:.3%} of range (tol {HEATMAP_TOL:.0%}); mean-per-pixel drift {msum / rng:.4%}")
            assert linf < HEATMAP_TOL * rng
            assert msum < 0.25 * HEATMAP_TOL * rng
            _check_vs_reference(f"{name} shift={shift}", kp, idx, hm, g[f"kpts_{shift}"], g[f"idx_{shift}"], rng, g["org_wh"])
        # frame + boxes through the reference's per-person loop
        m.set_flip_test(pairs, False)
        rows = g["frame_rows"].astype(np.float64)
        boxes = rows[rows[:, 4] > 0.35, :4].round().astype(np.int32)
        kp, _ = m.infer_frame_host(P.make_frame(fh, fw, fseed), boxes)
        ref = g["frame_kpts"]
        org = g["frame_org_wh"]
        to_model_px = np.stack([256.0 / org[:, 1], 192.0 / org[:, 0]], -1)[:, None, :]
        dev = np.linalg.norm((kp[..., :2] - ref[..., :2]) * to_model_px, axis=-1)
        vis = ref[..., 2] > 0.3
        print(name, f"frame: visible {int(vis.sum())}/{vis.size}; keypoint deviation px mean {dev[vis].mean():.4f} max {dev[vis].max():.4f}")
        assert vis.sum() >= 0.7 * vis.size and dev[vis].mean() < KPT_MEAN_PX_TOL
    finally:
        m.set_flip_test(None)


def test_install_flip_test_equals_engine_call(golden_dir):
    from easy_vitpose_b200 import install
    g, frame, boxes = _frame_case(golden_dir)
    D, depth, heads, K, wseed = (int(v) for v in g["meta"][3:8])
    sd = O.make_state_dict(D, depth, K, wseed, peaky=0.1, bumps=True)

    class FakeRefModel(torch.nn.Module):           # what install() needs of the reference ViTPose: state_dict() + num_heads
        def __init__(self):
            super().__init__()
            for k, v in sd.items():
                self.register_buffer(k.replace(".", "__"), torch.from_numpy(np.asarray(v)))
            self.backbone = types.SimpleNamespace(blocks=[types.SimpleNamespace(attn=types.SimpleNamespace(num_heads=heads))])

        def state_dict(self, *a, **kw):
            return {k.replace("__", "."): v for k, v in super().state_dict(*a, **kw).items()}

    def yolo(img, **kw):
        data = types.SimpleNamespace(cpu=lambda: types.SimpleNamespace(numpy=lambda: g["rows"]))
        return [types.SimpleNamespace(boxes=types.SimpleNamespace(data=data))]

    vi = types.SimpleNamespace(_vit_pose=FakeRefModel(), _inference=None, postprocess=None, tracker=None, frame_counter=0, yolo_step=1,
                               yolo=yolo, yolo_size=320, device="cuda", yolo_classes=[0], save_state=True, dataset="coco")
    backend = install(vi, max_batch=8, batched=True, flip_test=True)
    assert backend.model.max_batch == 16 and backend.model.batch_limit == 8 and backend.model.flip_test
    out = vi.inference(frame)
    kp = np.stack([out[i] for i in range(len(boxes))], 0)
    m = _engine(SIZES[D], K, depth, wseed)
    m.set_flip_test(_coco_pairs())
    try:
        want, _ = m.infer_frame_host(frame, boxes)
    finally:
        m.set_flip_test(None)
    assert np.array_equal(kp, want)
    vi2 = types.SimpleNamespace(_vit_pose=FakeRefModel(), dataset="ap10k")
    with pytest.raises(ValueError):                                      # no pairs for ap10k: never guessed from K = 17
        install(vi2, max_batch=8, flip_test=True)


def test_flip_errors():
    from easy_vitpose_b200 import _lib
    m = _engine("s", 17, 12, 131)
    pairs = _coco_pairs()
    m.set_flip_test(pairs)
    try:
        x = O.make_crops(9, 91)
        org = _org(9, 92)
        with pytest.raises(ValueError):
            m.infer_crops(torch.from_numpy(x).cuda(), org)
        with pytest.raises(RuntimeError):                                # VPB_ERR_ARG from vpb_infer_host
            m.infer_host(x, org.numpy())
        with pytest.raises(ValueError):
            m.infer_frame(torch.zeros((64, 64, 3), dtype=torch.uint8).cuda(), np.tile([[0, 0, 30, 30]], (9, 1)))
        m.infer_crops(torch.from_numpy(x[:8]).cuda(), org[:8])            # max_batch // 2 is fine
    finally:
        m.set_flip_test(None)
    m.infer_crops(torch.from_numpy(x).cuda(), org)                        # and flip test off: max_batch again
    with pytest.raises(ValueError):
        m.set_flip_test([(0, 17)])
    L = _lib.lib()
    for perm, k in ((np.arange(16, dtype=np.int32), 16), (np.array(list(range(16)) + [17], np.int32), 17),
                    (np.array([-1] + list(range(1, 17)), np.int32), 17)):
        assert L.vpb_set_flip_test(m._handle, perm.ctypes.data_as(C.c_void_p), k, 0) == 1      # VPB_ERR_ARG
    assert not m.flip_test
    assert L.vpb_kernel_launches(m._handle, 4) == m.kernel_launches(4)
