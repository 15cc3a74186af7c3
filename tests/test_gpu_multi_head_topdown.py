"""-m gpu: flip test and affine top-down crops on multi-head engines (ViTPose.set_flip_test_heads, infer_affine_heads and
its host form; vpb_set_flip_test_heads, vpb_infer_affine_heads).

The reference for every case is a single-head engine per head, loaded with the checkpoint split_vitpose_plus makes for
that head, with set_flip_test(that head's pairs) and infer_crops / infer_frames / infer_affine on that segment's crops.  A
flipped mixed call runs its crops and then their mirror images through one backbone pass; the fc2 experts, the heads, the
flip-back average and the decode give every element the same operations as the single-head path, so the results must be
BIT-IDENTICAL."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O
from oracle.multi_head import plus_state_dict

pytestmark = pytest.mark.gpu

CASES = {"s": (("coco", 17), ("aic", 14), ("mpii", 16), ("ap10k", 17), ("apt36k", 17), ("wholebody", 133)),
         "b": (("coco", 17), ("ap10k", 17), ("wholebody", 133))}
EXPERT_ROWS = {"s": 96, "b": 192}
MAX_BATCH = 24
HALF = MAX_BATCH // 2
_cache = {}


def _pairs(name, K):
    """COCO's pairs for the coco head; for the others (the reference defines none) a fixed choice: neighbours from 1 on."""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    if name == "coco":
        return [tuple(int(v) for v in p) for p in COCO_FLIP_PAIRS]
    return [(i, i + 1) for i in range(1, K - 1, 2)]


def _engines(size):
    """(multi-head engine, [single-head engine per head], [pairs per head])"""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus
    if size not in _cache:
        heads, P_ = CASES[size], EXPERT_ROWS[size]
        plus = {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict(size, [k for _, k in heads], P_, 31).items()}
        multi = ViTPose(model_cfg(size, 17), max_batch=MAX_BATCH, heads=heads, expert_rows=P_)
        multi.load_state_dict(plus)
        multi.to("cuda:0")
        singles = []
        for (name, K), sd in zip(heads, split_vitpose_plus(plus, [n for n, _ in heads], [k for _, k in heads]).values()):
            m = ViTPose(model_cfg(size, K), max_batch=MAX_BATCH)
            m.load_state_dict(sd)
            singles.append(m.to("cuda:0"))
        _cache[size] = (multi, singles, [_pairs(n, k) for n, k in heads])
    return _cache[size]


class _Flip:
    """flip test on the multi-head engine and on every single-head engine for the duration of a `with` block"""

    def __init__(self, size, shift):
        self.multi, self.singles, self.pairs = _engines(size)
        self.shift = shift

    def __enter__(self):
        if self.shift is not None:
            self.multi.set_flip_test_heads(self.pairs, self.shift)
            for m, p in zip(self.singles, self.pairs):
                m.set_flip_test(p, self.shift)
        return self

    def __exit__(self, *exc):
        self.multi.set_flip_test_heads(None)
        for m in self.singles:
            m.set_flip_test(None)


def _bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _assert_same(got, want, what):
    for g, w, name in zip(got, want, ("keypoints", "argmax", "heatmaps")):
        assert np.array_equal(_bits(g), _bits(w)), f"{what}: {name} differ"


def _crops(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).cuda()
    org = torch.from_numpy(np.random.RandomState(seed).randint(20, 400, size=(n, 2)).astype(np.int32)).cuda()
    return x, org


def _expected_crops(singles, x, org, heads, Km):
    n = x.shape[0]
    kp, idx, hm = np.zeros((n, Km, 3), np.float32), np.zeros((n, Km), np.int32), np.zeros((n, Km, 64, 48), np.float32)
    heads = np.asarray(heads)
    for j, m in enumerate(singles):
        sel = np.nonzero(heads == j)[0]
        if sel.size == 0:
            continue
        t = torch.as_tensor(sel, device=x.device)
        k, i, h = m.infer_crops(x.index_select(0, t), org.index_select(0, t), return_heatmaps=True)
        K = m.num_keypoints
        kp[sel, :K], idx[sel, :K], hm[sel, :K] = k.cpu().numpy(), i.cpu().numpy(), h.cpu().numpy()
    return kp, idx, hm


def _layouts(H):
    rs = np.random.RandomState(5)
    return [[H - 1], [1, 0, 2 % H, 2 % H, 0, 1, H - 1], list(rs.randint(0, H, size=HALF))]    # 1, 7 and max_batch / 2 crops


@pytest.mark.parametrize("size", ["s", "b"])
@pytest.mark.parametrize("shift", [False, True])
def test_flip_crops_bit_identical_to_single_head_engines(size, shift):
    with _Flip(size, shift) as f:
        for i, heads in enumerate(_layouts(len(f.singles))):
            x, org = _crops(len(heads), 500 + i)
            want = _expected_crops(f.singles, x, org, heads, f.multi.num_keypoints_max)
            for rep in range(3):                          # eager (first use), graph capture, graph replay
                _assert_same(f.multi.infer_crops_heads(x, org, heads, return_heatmaps=True), want, f"heads {heads} rep {rep}")


def _frames_boxes(seed, per_frame, H):
    rs = np.random.RandomState(seed)
    frames = [P.make_frame(h, w, seed + j) for j, (h, w) in enumerate(((480, 640), (720, 1280), (300, 200)))]
    boxes, heads = [], []
    for f, n in zip(frames, per_frame):
        x0, y0 = rs.randint(0, f.shape[1] - 40, n), rs.randint(0, f.shape[0] - 40, n)
        boxes.append(np.stack([x0, y0, rs.randint(20, 200, n), rs.randint(20, 200, n)], 1).astype(np.float64) + 0.3)   # x, y, w, h
        heads.append(rs.randint(0, H, n))
    return frames, boxes, heads


@pytest.mark.parametrize("shift", [False, True])
def test_flip_frames_heads_bit_identical(shift):
    with _Flip("b", shift) as f:
        frames, boxes, heads = _frames_boxes(11, (4, 4, 3), len(f.singles))
        xyxy = [np.concatenate([b[:, :2], b[:, :2] + b[:, 2:]], 1) for b in boxes]
        Km = f.multi.num_keypoints_max
        want_k = [np.zeros((len(b), Km, 3), np.float32) for b in boxes]
        want_i = [np.zeros((len(b), Km), np.int32) for b in boxes]
        for j, m in enumerate(f.singles):
            sel = [np.nonzero(h == j)[0] for h in heads]
            k, i = m.infer_frames([torch.from_numpy(fr).cuda() for fr in frames], [b[s] for b, s in zip(xyxy, sel)])
            for fi, s in enumerate(sel):
                want_k[fi][s, :m.num_keypoints], want_i[fi][s, :m.num_keypoints] = k[fi].cpu().numpy(), i[fi].cpu().numpy()
        for rep in range(3):
            gk, gi = f.multi.infer_frames_heads([torch.from_numpy(fr).cuda() for fr in frames], xyxy, heads)
            for fi in range(len(frames)):
                _assert_same((gk[fi], gi[fi]), (want_k[fi], want_i[fi]), f"frame {fi} rep {rep}")
        hk, hi = f.multi.infer_frames_heads_host(frames, xyxy, heads)
        for fi in range(len(frames)):
            _assert_same((hk[fi], hi[fi]), (want_k[fi], want_i[fi]), f"host frame {fi}")


def _affine_expected(singles, frames, args, heads, Km):
    """each head's boxes (frame order) in ONE single-head infer_affine call: the segment the grouped call makes"""
    want_k = [np.zeros((len(h), Km, 3), np.float32) for h in heads]
    want_i = [np.zeros((len(h), Km), np.int32) for h in heads]
    dframes = [torch.from_numpy(fr).cuda() for fr in frames]
    for j, m in enumerate(singles):
        sel = [np.nonzero(h == j)[0] for h in heads]
        if not sum(len(s) for s in sel):
            continue
        k, i = m.infer_affine(dframes, [a[0][s] for a, s in zip(args, sel)], [a[1][s] for a, s in zip(args, sel)],
                              [a[2][s] for a, s in zip(args, sel)])
        for fi, s in enumerate(sel):
            want_k[fi][s, :m.num_keypoints], want_i[fi][s, :m.num_keypoints] = k[fi].cpu().numpy(), i[fi].cpu().numpy()
    return want_k, want_i


@pytest.mark.parametrize("size", ["s", "b"])
@pytest.mark.parametrize("shift", [None, False, True])           # None: flip test off
def test_affine_heads_bit_identical_to_single_head_engines(size, shift):
    from easy_vitpose_b200 import topdown_args
    with _Flip(size, shift) as f:
        limit = f.multi.batch_limit
        for per_frame in ((1, 0, 0), (3, 2, 2), (limit - 4, 2, 2)):                 # 1, 7 and batch_limit boxes
            frames, boxes, heads = _frames_boxes(40 + sum(per_frame), per_frame, len(f.singles))
            args = [topdown_args(b, 1.25, True) for b in boxes]
            want_k, want_i = _affine_expected(f.singles, frames, args, heads, f.multi.num_keypoints_max)
            for rep in range(3):
                gk, gi = f.multi.infer_affine_heads([torch.from_numpy(fr).cuda() for fr in frames], [a[0] for a in args],
                                                    [a[1] for a in args], [a[2] for a in args], heads)
                for fi in range(len(frames)):
                    _assert_same((gk[fi], gi[fi]), (want_k[fi], want_i[fi]), f"{per_frame} frame {fi} rep {rep}")
            hk, hi = f.multi.infer_affine_heads_host(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], heads)
            for fi in range(len(frames)):
                _assert_same((hk[fi], hi[fi]), (want_k[fi], want_i[fi]), f"{per_frame} host frame {fi}")


def test_interleaved_segments_through_the_c_abi():
    """Segments A, B, A through vpb_infer_heads and vpb_infer_affine_heads with flip test on: each segment equals its own
    single-head call (the affine decode is one reference call per segment)."""
    from easy_vitpose_b200 import _lib, topdown_args
    L = _lib.lib()
    with _Flip("b", False) as f:
        Km = f.multi.num_keypoints_max
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        # crops
        segs = [(1, 2), (0, 3), (1, 1), (2, 1), (0, 1)]
        heads = [h for h, c in segs for _ in range(c)]
        x, org = _crops(len(heads), 77)
        want = _expected_crops(f.singles, x, org, heads, Km)
        n = len(heads)
        kp, idx, hm = torch.zeros((n, Km, 3), device="cuda"), torch.zeros((n, Km), dtype=torch.int32, device="cuda"), \
            torch.zeros((n, Km, 64, 48), device="cuda")
        arr = (_lib.VpbSegment * len(segs))(*[_lib.VpbSegment(h, c) for h, c in segs])
        for rep in range(3):                              # eager, capture, replay
            _lib.check(L.vpb_infer_heads(f.multi._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, len(segs),
                                         C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()),
                                         C.c_void_p(st.cuda_stream)))
            st.synchronize()
            _assert_same((kp, idx, hm), want, f"crops rep {rep}")
        # affine: entries (frame, head) = (0, 1), (1, 0), (0, 1) -> segments A, B, A
        frames, boxes, _ = _frames_boxes(91, (5, 3, 0), 1)
        ents = [(0, slice(0, 3), 1), (1, slice(0, 3), 0), (0, slice(3, 5), 1)]
        args = [topdown_args(boxes[fi][s], 1.25, True) for fi, s, _ in ents]
        dfr = [torch.from_numpy(fr).cuda() for fr in frames]
        M = torch.from_numpy(np.concatenate([a[0].reshape(-1, 6) for a in args])).cuda()
        CS = torch.from_numpy(np.concatenate([np.concatenate([a[1], a[2]], 1) for a in args]).astype(np.float32)).cuda()
        n = M.shape[0]
        farr = (_lib.VpbFrame * len(ents))(*[_lib.VpbFrame(dfr[fi].data_ptr(), dfr[fi].shape[0], dfr[fi].shape[1], dfr[fi].stride(0),
                                                           len(a[0])) for (fi, _, _), a in zip(ents, args)])
        ha = np.array([h for _, _, h in ents], np.int32)
        want_k, want_i = np.zeros((n, Km, 3), np.float32), np.zeros((n, Km), np.int32)
        r = 0
        for (fi, _, h), a in zip(ents, args):            # one single-head call per segment
            m = f.singles[h]
            k, i = m.infer_affine([dfr[fi]], [a[0]], [a[1]], [a[2]])
            want_k[r:r + len(a[0]), :m.num_keypoints], want_i[r:r + len(a[0]), :m.num_keypoints] = k[0].cpu().numpy(), i[0].cpu().numpy()
            r += len(a[0])
        kp, idx = torch.zeros((n, Km, 3), device="cuda"), torch.zeros((n, Km), dtype=torch.int32, device="cuda")
        for rep in range(3):
            _lib.check(L.vpb_infer_affine_heads(f.multi._handle, farr, len(farr), ha.ctypes.data_as(C.c_void_p), C.c_void_p(M.data_ptr()),
                                                C.c_void_p(CS.data_ptr()), C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()),
                                                C.c_void_p(st.cuda_stream)))
            st.synchronize()
            _assert_same((kp, idx), (want_k, want_i), f"affine rep {rep}")


@pytest.mark.parametrize("size", ["s", "b"])
def test_single_head_calls_on_a_flipped_multi_head_engine(size):
    """With set_flip_test_heads the single-head calls run head 0 with head 0's pairs: a head-0 engine with set_flip_test."""
    from easy_vitpose_b200 import topdown_args
    with _Flip(size, True) as f:
        x, org = _crops(HALF, 43)
        for _ in range(3):
            _assert_same(f.multi.infer_crops(x, org, return_heatmaps=True), f.singles[0].infer_crops(x, org, return_heatmaps=True), "crops")
        frames, boxes, _ = _frames_boxes(44, (3, 2, 1), 1)
        args = [topdown_args(b, 1.25, True) for b in boxes]
        dfr = [torch.from_numpy(fr).cuda() for fr in frames]
        a = f.multi.infer_affine(dfr, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args])
        b = f.singles[0].infer_affine(dfr, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args])
        for fi in range(len(frames)):
            _assert_same((a[0][fi], a[1][fi]), (b[0][fi], b[1][fi]), f"affine frame {fi}")


def test_errors_and_setting_rules():
    from easy_vitpose_b200 import _lib
    L = _lib.lib()
    multi, _, pairs = _engines("s")
    h = multi._handle
    from easy_vitpose_b200 import head_flip_permutations
    perms = head_flip_permutations(multi.head_keypoints, pairs)
    ptr = perms.ctypes.data_as(C.c_void_p)
    assert L.vpb_set_flip_test_heads(h, ptr, perms.size - 1, 0) == 1                  # wrong total
    bad = perms.copy()
    bad[17] = 14                                                                        # head 1 (aic) has 14 keypoints
    assert L.vpb_set_flip_test_heads(h, bad.ctypes.data_as(C.c_void_p), bad.size, 0) == 1
    bad = perms.copy()
    bad[0] = -1
    assert L.vpb_set_flip_test_heads(h, bad.ctypes.data_as(C.c_void_p), bad.size, 0) == 1
    assert not multi.flip_test and multi.batch_limit == MAX_BATCH
    with pytest.raises(ValueError):
        multi.set_flip_test_heads(pairs[:-1])
    with pytest.raises(ValueError):
        multi.set_flip_test_heads([[(0, 17)]] + pairs[1:])
    with pytest.raises(RuntimeError, match="error 3"):
        multi.set_flip_test([(1, 2)])                   # vpb_set_flip_test stays refused on a multi-head engine
    try:
        multi.set_flip_test_heads(pairs)
        assert multi.flip_test and multi.batch_limit == HALF
        Km = multi.num_keypoints_max
        xs = torch.zeros((HALF + 1, 3, 256, 192), device="cuda")
        og = torch.full((HALF + 1, 2), 100, dtype=torch.int32, device="cuda")
        kp = torch.empty((HALF + 1, Km, 3), device="cuda")
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        arr = (_lib.VpbSegment * 2)(_lib.VpbSegment(0, HALF), _lib.VpbSegment(1, 1))
        assert L.vpb_infer_heads(h, C.c_void_p(xs.data_ptr()), C.c_void_p(og.data_ptr()), arr, 2, C.c_void_p(kp.data_ptr()), None, None, st) == 1
        assert L.vpb_infer(h, C.c_void_p(xs.data_ptr()), C.c_void_p(og.data_ptr()), HALF + 1, C.c_void_p(kp.data_ptr()), None, None, st) == 1
        # 1-crop segments of alternating heads: the crops and their mirror images make 2 * HALF expert segments
        arr = (_lib.VpbSegment * HALF)(*[_lib.VpbSegment(j % 2, 1) for j in range(HALF)])
        assert L.vpb_infer_heads(h, C.c_void_p(xs.data_ptr()), C.c_void_p(og.data_ptr()), arr, HALF, C.c_void_p(kp.data_ptr()), None, None, st) == 0
        torch.cuda.synchronize()
    finally:
        multi.set_flip_test_heads(None)
    # a single-head engine: vpb_set_flip_test keeps the multi-head calls refused, vpb_set_flip_test_heads (H = 1) opens them
    from easy_vitpose_b200 import ViTPose, model_cfg
    one = ViTPose(model_cfg("s", 17), max_batch=8, heads=[("coco", 17)], expert_rows=0)
    one.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("s", [17], 0, 7).items()})
    one.to("cuda:0")
    x, org = _crops(3, 9)
    one.set_flip_test(pairs[0])
    with pytest.raises(RuntimeError, match="error 3"):
        one.infer_crops_heads(x, org, [0, 0, 0])
    one.set_flip_test_heads([pairs[0]], False)
    got = one.infer_crops_heads(x, org, [0, 0, 0], return_heatmaps=True)
    ref = one.infer_crops(x, org, return_heatmaps=True)
    _assert_same(got, ref, "one head, flip test")
    one.set_flip_test(None)
    assert not one.flip_test


def test_toggling_flip_drops_both_graph_caches():
    multi, singles, pairs = _engines("b")
    x, org = _crops(4, 12)
    heads = [0, 2, 2, 1]
    multi.set_flip_test_heads(None)                       # starts both caches empty
    for _ in range(2):
        multi.infer_crops_heads(x, org, heads)
        multi.infer_crops(x, org)
    assert multi.cached_graphs(mixed=True) == (1, 1) and multi.cached_graphs() == (1, 1)
    multi.set_flip_test_heads(pairs, True)
    try:
        assert multi.cached_graphs(mixed=True) == (0, 0) and multi.cached_graphs() == (0, 0)
        for _ in range(2):
            multi.infer_crops_heads(x, org, heads)
        assert multi.cached_graphs(mixed=True) == (1, 1)
    finally:
        multi.set_flip_test_heads(None)
    assert multi.cached_graphs(mixed=True) == (0, 0) and multi.cached_graphs() == (0, 0)


# ---- against the reference: tests/golden/multi_head_topdown_s.npz (oracle/make_golden_multi_head_topdown.py)
HEATMAP_TOL = 0.01             # DESIGN §2: L_inf as a fraction of the reference heatmap range
KPT_MEAN_PX_TOL = 0.5          # mean keypoint deviation, pixels of the 192x256 model input


@pytest.mark.parametrize("shift", [0, 1])
def test_affine_flip_heads_vs_reference_fixture(golden_dir, shift):
    """One infer_affine_heads call over the boxes of all six heads (ViT-S, P = 96) with each head's flip pairs against the
    unmodified reference on model_split.py's checkpoints: one keypoints_from_heatmaps(c, s, use_udp=True) per head."""
    from easy_vitpose_b200 import ViTPose, model_cfg
    from oracle.multi_head_flip import flip_plus_state_dict
    g = np.load(os.path.join(golden_dir, "multi_head_topdown_s.npz"))
    D, depth, heads, P_, wseed, _ = (int(v) for v in g["meta"])
    names, Ks = [str(h) for h in g["heads"]], [int(k) for k in g["keypoints"]]
    ends = np.cumsum(g["pair_counts"])
    pairs = [[tuple(int(v) for v in p) for p in g["pairs"][e - c:e]] for c, e in zip(g["pair_counts"], ends)]
    key = ("fixture", shift)
    if key not in _cache:
        m = ViTPose(model_cfg("s", 17), max_batch=2 * len(g["crc"]), heads=list(zip(names, Ks)), expert_rows=P_)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in flip_plus_state_dict("s", Ks, P_, wseed, pairs).items()})
        _cache[key] = m.to("cuda:0")
    m = _cache[key]
    m.set_flip_test_heads(pairs, bool(shift))
    try:
        frames = [torch.from_numpy(P.make_frame(int(h), int(w), int(s))).cuda() for h, w, s in g["frames"]]
        per = [np.nonzero(g["frame_id"] == f)[0] for f in range(len(frames))]
        cs = g["cs_px"]
        kp_f, idx_f = m.infer_affine_heads(frames, [g["mats"][s] for s in per], [cs[s, :2] for s in per], [cs[s, 2:] for s in per],
                                           [g["head_id"][s] for s in per], check=True)
        order = np.concatenate(per)
        N, Km = len(order), m.num_keypoints_max
        kp, idx = np.zeros((N, Km, 3), np.float32), np.zeros((N, Km), np.int32)
        kp[order], idx[order] = torch.cat(kp_f).cpu().numpy(), torch.cat(idx_f).cpu().numpy()
        crops = m.preprocess_affine(frames, [g["mats"][s] for s in per])
        hm_f = m.infer_crops_heads(crops, torch.full((N, 2), 100, dtype=torch.int32), g["head_id"][order], return_heatmaps=True)[2]
        hm = np.zeros((N, Km, 64, 48), np.float32)
        hm[order] = hm_f.cpu().numpy()
    finally:
        m.set_flip_test_heads(None)
    for j, (name, K) in enumerate(zip(names, Ks)):
        sel = np.nonzero(g["head_id"] == j)[0]
        n = len(sel)
        h_, k_, i_ = hm[sel, :K], kp[sel, :K], idx[sel, :K]
        ref_kp, ref_idx = g[f"kpts_{shift}"][sel, :K], g[f"idx_{shift}"][sel, :K]
        rng = float(g[f"range_{shift}"][j, 1] - g[f"range_{shift}"][j, 0])
        linf = float(np.abs(h_[0, g["sample_kps"][j]] - g[f"sample_hm_{shift}"][j]).max())
        msum = float(np.abs(h_.reshape(n, K, -1).sum(-1, dtype=np.float64) - g[f"map_sum_{shift}"][sel, :K]).max() / 3072.0)
        s = cs[sel, 2:]
        to_model_px = np.stack([256.0 / s[:, 1], 192.0 / s[:, 0]], -1)[:, None, :]          # (y, x): image px -> input px
        dev = np.linalg.norm((k_[..., :2] - ref_kp[..., :2]) * to_model_px, axis=-1)
        vis = ref_kp[..., 2] > 0.3
        cell = np.maximum(np.abs(i_ % 48 - ref_idx % 48), np.abs(i_ // 48 - ref_idx // 48))
        far = vis & (cell > 1)
        flat = h_.reshape(n, K, -1)
        gap = flat.max(-1) - np.take_along_axis(flat, ref_idx[..., None].astype(np.int64), -1)[..., 0]
        print(name, f"shift={shift}: heatmaps Linf {linf / rng:.3%} of range, drift {msum / rng:.4%}; visible {int(vis.sum())}/{vis.size}; "
              f"keypoint deviation (input px) mean {dev[vis].mean():.4f} max {dev[vis].max():.4f}; far arg-max flips {int(far.sum())}")
        assert linf < HEATMAP_TOL * rng and msum < HEATMAP_TOL * rng
        assert vis.sum() >= 0.7 * vis.size
        assert dev[vis].mean() < KPT_MEAN_PX_TOL
        assert far.sum() <= 0.01 * vis.sum() + 1
        assert np.all(gap[far] <= 2 * HEATMAP_TOL * rng)
        assert np.array_equal(i_, flat.argmax(-1).astype(np.int32))           # the engine's own maps, bit-exact integer work


def test_affine_heads_previous_map_sentinel_in_the_kmax_layout():
    """Keypoint 0 of heads 1 and 2 has an all-negative map (final_layer row 0 zero, bias -1), so the mode-4 decode takes the
    reference's max <= 0 branch and reads the previous map of the segment's array -- for the first crop of a segment the last map
    of its last crop, at its K_max-strided slot.  Bit-identical to single-head engines, flip on and off."""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus, topdown_args
    heads = (("coco", 17), ("aic", 14), ("wholebody", 133))
    if "sentinel" not in _cache:
        sd = plus_state_dict("s", [k for _, k in heads], 96, 51)
        for j in (1, 2):
            p = f"associate_keypoint_heads.{j - 1}.final_layer."
            sd[p + "weight"] = sd[p + "weight"].copy()
            sd[p + "bias"] = sd[p + "bias"].copy()
            sd[p + "weight"][0] = 0.0
            sd[p + "bias"][0] = -1.0
        plus = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
        multi = ViTPose(model_cfg("s", 17), max_batch=16, heads=heads, expert_rows=96)
        multi.load_state_dict(plus)
        singles = []
        for (name, K), part in zip(heads, split_vitpose_plus(plus, [n for n, _ in heads], [k for _, k in heads]).values()):
            s_ = ViTPose(model_cfg("s", K), max_batch=16)
            s_.load_state_dict(part)
            singles.append(s_.to("cuda:0"))
        _cache["sentinel"] = (multi.to("cuda:0"), singles, [_pairs(n, k) for n, k in heads])
    multi, singles, pairs = _cache["sentinel"]
    frames, boxes, _ = _frames_boxes(61, (3, 2, 2), 1)
    hs = [np.array([1, 0, 2]), np.array([2, 1]), np.array([1, 2])]
    args = [topdown_args(b, 1.25, True) for b in boxes]
    for shift in (None, False):
        if shift is not None:
            multi.set_flip_test_heads(pairs, shift)
            for m, p in zip(singles, pairs):
                m.set_flip_test(p, shift)
        try:
            want_k, want_i = _affine_expected(singles, frames, args, hs, multi.num_keypoints_max)
            for rep in range(3):
                gk, gi = multi.infer_affine_heads([torch.from_numpy(fr).cuda() for fr in frames], [a[0] for a in args],
                                                  [a[1] for a in args], [a[2] for a in args], hs)
                for fi in range(len(frames)):
                    _assert_same((gk[fi], gi[fi]), (want_k[fi], want_i[fi]), f"flip {shift} frame {fi} rep {rep}")
            for fi, h in enumerate(hs):
                sent = want_k[fi][h > 0, 0]                    # keypoint 0 of heads 1 and 2: the sentinel branch
                assert np.all(sent[:, 2] <= 0) and np.all(want_i[fi][h > 0, 0] == 0)
        finally:
            multi.set_flip_test_heads(None)
            for m in singles:
                m.set_flip_test(None)
