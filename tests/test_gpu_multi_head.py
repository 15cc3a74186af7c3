"""-m gpu: several keypoint heads on one engine (ViTPose(..., heads=, expert_rows=); vpb_create_heads, vpb_infer_heads,
vpb_infer_frames_heads and its host form).  The reference for every case is a single-head engine loaded with the checkpoint
split_vitpose_plus makes for that head (model_split.py's checkpoint): the fc2 expert columns run in the grouped GEMM, every
element still gets one fp32 add of (acc + bias) in k order, so a mixed call must be BIT-IDENTICAL to the per-head calls."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import vitpose_oracle as O
from oracle.multi_head import plus_state_dict

pytestmark = pytest.mark.gpu

# ViT-S with all six ViTPose+ heads and P = 96 (D - P = 288: padded tiles on both sides); ViT-B with three heads, P = 192
CASES = {"s": (("coco", 17), ("aic", 14), ("mpii", 16), ("ap10k", 17), ("apt36k", 17), ("wholebody", 133)), "b": (("coco", 17), ("ap10k", 17), ("wholebody", 133))}
EXPERT_ROWS = {"s": 96, "b": 192}
MAX_BATCH = 24
_cache = {}


def _torch_sd(sd):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}


def _engines(size, P=None, heads=None):
    """(multi-head engine, [single-head engine per head]) for one size and expert width."""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus
    P = EXPERT_ROWS[size] if P is None else P
    heads = CASES[size] if heads is None else heads
    key = (size, P, heads)
    if key not in _cache:
        plus = _torch_sd(plus_state_dict(size, [k for _, k in heads], P, 31))
        multi = ViTPose(model_cfg(size, 17), max_batch=MAX_BATCH, heads=heads, expert_rows=P)
        multi.load_state_dict(plus)
        multi.to("cuda:0")
        singles = []
        for (name, K), sd in zip(heads, split_vitpose_plus(plus, [n for n, _ in heads], [k for _, k in heads]).values()):
            m = ViTPose(model_cfg(size, K), max_batch=MAX_BATCH)
            m.load_state_dict(sd)
            singles.append(m.to("cuda:0"))
        _cache[key] = (multi, singles)
    return _cache[key]


def _crops(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).cuda()
    org = torch.from_numpy(np.random.RandomState(seed).randint(20, 400, size=(n, 2)).astype(np.int32)).cuda()
    return x, org


def _expected(singles, x, org, heads, Km):
    """per-crop results of the single-head engines, padded to K_max with zeros (what infer_crops_heads returns)"""
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


def _check(multi, singles, heads, seed):
    x, org = _crops(len(heads), seed)
    want = _expected(singles, x, org, heads, multi.num_keypoints_max)
    got = [t.cpu().numpy() for t in multi.infer_crops_heads(x, org, heads, return_heatmaps=True)]
    for g, w, what in zip(got, want, ("keypoints", "argmax", "heatmaps")):
        assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g, w.view(np.uint32) if w.dtype == np.float32 else w), \
            f"{what} differ for heads {list(heads)}"


def _layouts(H):
    rs = np.random.RandomState(3)
    out = [[j] * 3 for j in range(H)]                                         # each head alone
    out += [[0, 0, 1, 1, 1], [H - 1, 0, 0, 1, 1, 1, 1], [1, 1, 0, 0, 0, 1, 1]]  # 2 and 3 heads, interleaved (A, B, A)
    out += [[0, 1, 2 % H, 1], [1], [2 % H, 0, 1, 0, 2 % H, 0, 1]]               # 1-crop segments, odd segment starts, batch 1 and 7
    out += [list(rs.randint(0, H, size=MAX_BATCH))]                           # max_batch
    return out


@pytest.mark.parametrize("size", ["s", "b"])
def test_mixed_calls_bit_identical_to_single_head_engines(size):
    multi, singles = _engines(size)
    for i, heads in enumerate(_layouts(len(singles))):
        for _ in range(3):                        # eager (first use), graph capture, graph replay
            _check(multi, singles, heads, 100 + i)


def test_graph_off_and_cache_eviction():
    multi, singles = _engines("s")
    multi.set_option("graph", 0)
    try:
        _check(multi, singles, [2, 0, 0, 5], 7)
    finally:
        multi.set_option("graph", 1)
    multi.set_option("ln_fused", 0)               # the default; setting an option that captured graphs embed drops them all
    assert multi.cached_graphs(mixed=True) == (0, 0)
    first = [4, 1]
    _check(multi, singles, first, 8)
    assert multi.cached_graphs(mixed=True) == (1, 0)          # seen once: ran eagerly
    _check(multi, singles, first, 8)
    assert multi.cached_graphs(mixed=True) == (1, 1)          # captured
    for j in range(17):                           # 17 new segment lists push the first one out of the 16-entry cache
        _check(multi, singles, [j % 6, (j + 1) % 6, j % 6] + [0] * (j // 6), 9 + j)
        assert multi.cached_graphs(mixed=True) == (min(j + 2, 16), 1 if j < 15 else 0)
    _check(multi, singles, first, 8)              # evicted: eager again (pushes out the least recently used list)
    assert multi.cached_graphs(mixed=True) == (16, 0)
    for _ in range(2):
        _check(multi, singles, first, 8)          # captured again, replayed
        assert multi.cached_graphs(mixed=True) == (16, 1)


def test_frames_heads_bit_identical_to_per_head_infer_frames():
    multi, singles = _engines("b")
    rs = np.random.RandomState(11)
    frames = [rs.randint(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in ((480, 640), (720, 1280), (300, 200))]
    boxes, heads = [], []
    for f in frames:
        n = 5
        x0, y0 = rs.randint(0, f.shape[1] - 40, n), rs.randint(0, f.shape[0] - 40, n)
        boxes.append(np.stack([x0, y0, x0 + rs.randint(20, 200, n), y0 + rs.randint(20, 200, n)], 1).astype(np.float64) + 0.3)
        heads.append(rs.randint(0, len(singles), n))
    Km = multi.num_keypoints_max
    want_k = [np.zeros((len(b), Km, 3), np.float32) for b in boxes]
    want_i = [np.zeros((len(b), Km), np.int32) for b in boxes]
    for j, m in enumerate(singles):
        sel = [np.nonzero(h == j)[0] for h in heads]
        k, i = m.infer_frames([torch.from_numpy(f).cuda() for f in frames], [b[s] for b, s in zip(boxes, sel)])
        for f, s in enumerate(sel):
            want_k[f][s, :m.num_keypoints], want_i[f][s, :m.num_keypoints] = k[f].cpu().numpy(), i[f].cpu().numpy()
    for _ in range(3):
        gk, gi = multi.infer_frames_heads([torch.from_numpy(f).cuda() for f in frames], boxes, heads)
        for f in range(len(frames)):
            assert np.array_equal(gk[f].cpu().numpy().view(np.uint32), want_k[f].view(np.uint32))
            assert np.array_equal(gi[f].cpu().numpy(), want_i[f])
    hk, hi = multi.infer_frames_heads_host(frames, boxes, heads)
    for f in range(len(frames)):
        assert np.array_equal(hk[f].view(np.uint32), want_k[f].view(np.uint32))
        assert np.array_equal(hi[f], want_i[f])


@pytest.mark.parametrize("P", [32, 64, 128])
def test_other_expert_widths(P):
    """P = 32 / 64 / 128 run the 32-, 64- and 128-wide expert GEMM tiles (P = 96 and 192 above: the 96- and 192-wide ones)."""
    multi, singles = _engines("s", P=P, heads=(("coco", 17), ("aic", 14), ("wholebody", 133)))
    for i, heads in enumerate([[0, 1, 2, 1, 0], [2] * 3 + [1] * 10 + [0] * 11, [1, 2]]):
        for _ in range(2):
            _check(multi, singles, heads, 300 + i)


def test_shared_backbone_heads_bit_identical():
    """P = 0 (frozen-backbone fine-tunes): every head shares the whole backbone."""
    multi, singles = _engines("s", P=0)
    for i, heads in enumerate([[0, 5, 5, 1], [3, 3, 2, 0, 4]]):
        for _ in range(2):
            _check(multi, singles, heads, 200 + i)


@pytest.mark.parametrize("size", ["s", "b"])
def test_single_head_calls_run_head_zero(size):
    multi, singles = _engines(size)
    x, org = _crops(5, 41)
    for a, b in zip(multi.infer_crops(x, org, return_heatmaps=True), singles[0].infer_crops(x, org, return_heatmaps=True)):
        assert torch.equal(a, b)


def test_errors():
    from easy_vitpose_b200 import _lib
    multi, _ = _engines("s")
    x, org = _crops(3, 5)
    with pytest.raises(ValueError):
        multi.infer_crops_heads(x, org, [0, 6, 1])
    with pytest.raises(ValueError):
        multi.infer_crops_heads(x, org, [0, 1])
    L = _lib.lib()
    Km = multi.num_keypoints_max
    kp = torch.empty((MAX_BATCH + 1, Km, 3), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    xs = torch.zeros((MAX_BATCH + 1, 3, 256, 192), device="cuda")
    og = torch.full((MAX_BATCH + 1, 2), 100, dtype=torch.int32, device="cuda")

    def call(segs):
        arr = (_lib.VpbSegment * max(len(segs), 1))(*[_lib.VpbSegment(h, c) for h, c in segs])
        return L.vpb_infer_heads(multi._handle, C.c_void_p(xs.data_ptr()), C.c_void_p(og.data_ptr()), arr, len(segs),
                                 C.c_void_p(kp.data_ptr()), None, None, st)
    assert call([(0, 2), (6, 1)]) == 1                   # head out of range
    assert call([(-1, 1)]) == 1
    assert call([(0, 2), (1, -1)]) == 1                  # negative count
    assert call([(j % 2, 1) for j in range(65)]) == 1    # more than VPB_MAX_SEGMENTS
    assert call([(0, MAX_BATCH), (1, 1)]) == 1           # above max_batch
    assert call([]) == 0 and call([(1, 0)]) == 0         # nothing to do
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="error 3"):
        multi.set_flip_test([(1, 2)])


def test_interleaved_segments_through_the_c_abi():
    """vpb_infer_heads with runs the Python grouping never makes: A, B, A and 1-crop runs at odd crops."""
    from easy_vitpose_b200 import _lib
    multi, singles = _engines("b")
    segs = [(1, 2), (0, 3), (1, 1), (2, 1), (0, 1)]
    heads = [h for h, c in segs for _ in range(c)]
    x, org = _crops(len(heads), 77)
    Km = multi.num_keypoints_max
    n = len(heads)
    kp = torch.zeros((n, Km, 3), device="cuda")
    idx = torch.zeros((n, Km), dtype=torch.int32, device="cuda")
    hm = torch.zeros((n, Km, 64, 48), device="cuda")
    arr = (_lib.VpbSegment * len(segs))(*[_lib.VpbSegment(h, c) for h, c in segs])
    st = torch.cuda.Stream()
    want = _expected(singles, x, org, heads, Km)
    st.wait_stream(torch.cuda.current_stream())
    for _ in range(3):                            # eager, capture, replay
        _lib.check(_lib.lib().vpb_infer_heads(multi._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, len(segs),
                                              C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()),
                                              C.c_void_p(st.cuda_stream)))
        st.synchronize()
        for g, w in zip((kp, idx, hm), want):
            g = g.cpu().numpy()
            assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g, w.view(np.uint32) if w.dtype == np.float32 else w)


def test_experts_and_heads_matter():
    """The bit-identity above would also hold if the engine ignored the expert or the head: a swapped expert, and separately a
    swapped head, must move the heatmaps far beyond the 1 % of range the reference comparisons allow."""
    from easy_vitpose_b200 import ViTPose, model_cfg, split_vitpose_plus
    multi, singles = _engines("s")
    plus = _torch_sd(plus_state_dict("s", [k for _, k in CASES["s"]], EXPERT_ROWS["s"], 31))
    parts = list(split_vitpose_plus(plus, [n for n, _ in CASES["s"]], [k for _, k in CASES["s"]]).values())
    x, org = _crops(4, 61)
    ref = singles[3].infer_crops(x, org, return_heatmaps=True)[2]        # ap10k
    rng = float(ref.max() - ref.min())
    for swap in ("expert", "head"):
        sd = dict(parts[3])
        donor = parts[0]                                                    # coco: same K = 17
        keys = [k for k in sd if (".mlp.fc2." in k) == (swap == "expert") and (k.startswith("keypoint_head.") or swap == "expert")]
        for k in keys:
            sd[k] = donor[k]
        m = ViTPose(model_cfg("s", 17), max_batch=4)
        m.load_state_dict(sd)
        hm = m.to("cuda:0").infer_crops(x, org, return_heatmaps=True)[2]
        assert float((hm - ref).abs().max()) > 0.05 * rng, f"a swapped {swap} barely changes the heatmaps"


HEATMAP_TOL = 0.01             # L_inf as a fraction of the reference heatmap range (as test_gpu_batch_parity.py)
KPT_MEAN_PX_TOL = 0.5          # mean keypoint deviation, pixels of the 256x192 model input


@pytest.mark.parametrize("name", ["multi_head_s", "multi_head_b"])
def test_mixed_call_vs_reference_fixture(golden_dir, name):
    """One mixed call over the crops of every served head against the unmodified reference run on model_split.py's
    checkpoints (oracle/make_golden_multi_head.py): heatmaps within 1 % of range, mean keypoint deviation within 0.5 px,
    argmax = np.argmax of the engine's own heatmaps.  ViT-S loads the unsplit ViTPose+ state_dict as is; ViT-B serves three
    of the six heads, merged back from the split checkpoints."""
    import os
    from easy_vitpose_b200 import VITPOSE_PLUS_HEADS, ViTPose, merge_split_state_dicts, model_cfg, split_vitpose_plus
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    D, depth, heads, P, n, wseed, xseed = (int(v) for v in g["meta"])
    size = {384: "s", 768: "b"}[D]
    served = [str(h) for h in g["heads"]]
    plus = _torch_sd(plus_state_dict(size, [k for _, k in VITPOSE_PLUS_HEADS], P, wseed))
    if len(served) < len(VITPOSE_PLUS_HEADS):
        parts = split_vitpose_plus(plus)
        plus = merge_split_state_dicts({h: parts[h] for h in served}, P)
    hk = list(zip(served, (int(k) for k in g["keypoints"])))
    m = ViTPose(model_cfg(size, 17), max_batch=n * len(served), heads=hk, expert_rows=P)
    m.load_state_dict(plus)
    m.to("cuda:0")
    x = torch.from_numpy(np.concatenate([O.make_crops(n, xseed + j) for j in range(len(served))])).cuda()
    org = torch.from_numpy(g["org_wh"].reshape(-1, 2)).cuda()
    hidx = np.repeat(np.arange(len(served)), n)
    perm = np.random.RandomState(0).permutation(hidx.size)                  # interleave the heads in the call
    inv = np.argsort(perm)
    kp, idx, hm = m.infer_crops_heads(x[perm], org[perm], hidx[perm], return_heatmaps=True)
    kp, idx, hm = kp.cpu().numpy()[inv], idx.cpu().numpy()[inv], hm.cpu().numpy()[inv]
    for j, (h, K) in enumerate(hk):
        s = slice(j * n, (j + 1) * n)
        k_, i_, h_ = kp[s, :K], idx[s, :K], hm[s, :K]
        rng = float(g["range"][j, 1] - g["range"][j, 0])
        linf = float(np.abs(h_[0, g["kp_ids"][j]] - g["sample_hm"][j]).max())
        msum = float(np.abs(h_.reshape(n, K, -1).sum(-1, dtype=np.float64) - g["map_sum"][j, :, :K]).max() / 3072.0)
        ref = g["kpts"][j, :, :K]
        o = g["org_wh"][j]
        to_model_px = np.stack([256.0 / o[:, 1], 192.0 / o[:, 0]], -1)[:, None, :]
        dev = np.linalg.norm((k_[..., :2] - ref[..., :2]) * to_model_px, axis=-1)
        vis = ref[..., 2] > 0.3
        print(name, h, f"sampled heatmaps Linf {linf / rng:.3%} of range, mean-per-pixel drift {msum / rng:.4%}, "
              f"keypoint deviation mean {dev[vis].mean():.4f} px over {int(vis.sum())}/{vis.size} visible")
        assert linf <= HEATMAP_TOL * rng and msum <= HEATMAP_TOL * rng
        assert vis.sum() >= 0.7 * vis.size and dev[vis].mean() < KPT_MEAN_PX_TOL
        assert np.array_equal(i_, h_.reshape(n, K, -1).argmax(-1).astype(np.int32))
