"""CPU: the host side of flip test and affine crops on multi-head engines -- the per-head permutations
vpb_set_flip_test_heads takes (head_flip_permutations) and the grouping / chunking of infer_affine_heads (plan_head_calls)."""
import numpy as np
import pytest

from easy_vitpose_b200 import COCO_FLIP_PAIRS, ViTPose, head_flip_permutations, plan_head_calls
from easy_vitpose_b200.model import plan_frame_chunks


def test_permutations_concatenate_in_head_order():
    coco = [tuple(p) for p in COCO_FLIP_PAIRS]
    perms = head_flip_permutations([17, 14, 5], [coco, [(0, 3), (1, 2)], []])
    assert perms.dtype == np.int32 and perms.shape == (17 + 14 + 5,)
    assert perms[:17].tolist() == ViTPose.flip_permutation(17, coco)
    assert perms[17:31].tolist() == [3, 2, 1, 0] + list(range(4, 14))
    assert perms[31:].tolist() == list(range(5))
    for K, off in ((17, 0), (14, 17), (5, 31)):             # every head's entries are a permutation of its own 0..K-1
        assert sorted(perms[off:off + K].tolist()) == list(range(K))


def test_permutations_sequential_like_flip_back():
    """a later pair overrides an earlier one, as the loop of flip_back does (post_transforms.py:110-147)"""
    assert head_flip_permutations([4], [[(0, 1), (1, 2)]]).tolist() == ViTPose.flip_permutation(4, [(0, 1), (1, 2)])


def test_permutation_errors():
    with pytest.raises(ValueError, match="2 flip pair lists for 3 heads"):
        head_flip_permutations([17, 14, 5], [[], []])
    with pytest.raises(ValueError, match="head 1"):
        head_flip_permutations([17, 14], [[], [(0, 14)]])
    with pytest.raises(ValueError, match="head 0"):
        head_flip_permutations([17], [[(-1, 2)]])


def test_plan_groups_by_head_and_keeps_frame_order():
    counts = [3, 0, 4]
    heads = [np.array([2, 0, 2]), np.array([], np.int64), np.array([0, 0, 1, 2])]
    ents, order, chunks = plan_head_calls(counts, heads, 3, 64)
    assert [(j, sel.tolist(), h) for j, sel, h in ents] == [(0, [1], 0), (2, [0, 1], 0), (2, [2], 1), (0, [0, 2], 2), (2, [3], 2)]
    assert order.tolist() == [1, 3, 4, 5, 0, 2, 6]        # flat indices (frames concatenated) in call order
    assert chunks == [[(0, 0, 1), (1, 0, 2), (2, 0, 1), (3, 0, 2), (4, 0, 1)]]


def test_plan_chunks_by_batch_limit_and_entries():
    rs = np.random.RandomState(0)
    counts = [int(c) for c in rs.randint(0, 9, size=40)]
    heads = [rs.randint(0, 6, size=c) for c in counts]
    for limit in (1, 5, 12, 32):
        ents, order, chunks = plan_head_calls(counts, heads, 6, limit, max_frames=7)
        assert sorted(order.tolist()) == list(range(sum(counts)))              # every box exactly once
        assert chunks == plan_frame_chunks([len(sel) for _, sel, _ in ents], limit, 7)
        for ch in chunks:
            assert sum(e - s for _, s, e in ch) <= limit and len(ch) <= 7
        hs = np.concatenate(heads)[order]
        assert np.all(np.diff(hs) >= 0)                     # head-major: every head's boxes form one run


def test_plan_errors():
    with pytest.raises(ValueError, match="2 frames but 1 head arrays"):
        plan_head_calls([1, 1], [np.array([0])], 2, 8)
    with pytest.raises(ValueError, match="frame 1"):
        plan_head_calls([1, 2], [np.array([0]), np.array([1])], 2, 8)
    with pytest.raises(ValueError, match="0..1"):
        plan_head_calls([2], [np.array([0, 2])], 2, 8)


# ---- the numpy oracle against tests/golden/multi_head_topdown_s.npz (oracle/make_golden_multi_head_topdown.py: the unmodified
# reference's ViTPose, inference_model(..., flip_pairs) and keypoints_from_heatmaps on model_split.py's checkpoints)
def _fixture():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multi_head_topdown_s.npz"))


def _pairs(g):
    ends = np.cumsum(g["pair_counts"])
    return [[tuple(int(v) for v in p) for p in g["pairs"][e - c:e]] for c, e in zip(g["pair_counts"], ends)]


def _weights(g):
    from oracle.multi_head_flip import flip_plus_state_dict
    D, depth, heads, P, wseed, _ = (int(v) for v in g["meta"])
    return flip_plus_state_dict("s", [int(k) for k in g["keypoints"]], P, wseed, _pairs(g))


def test_flip_weights_and_split_reproduce_fixture_crcs():
    import zlib
    import torch
    from easy_vitpose_b200 import split_vitpose_plus
    g = _fixture()
    sd = _weights(g)
    assert sorted(sd) == [str(k) for k in g["weight_keys"]]
    assert [zlib.crc32(np.ascontiguousarray(sd[str(k)]).tobytes()) for k in g["weight_keys"]] == g["weight_crc"].tolist()
    parts = split_vitpose_plus({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, [str(h) for h in g["heads"]],
                               [int(k) for k in g["keypoints"]])
    for j, part in enumerate(parts.values()):
        assert [zlib.crc32(np.ascontiguousarray(part[str(k)].numpy()).tobytes()) for k in g["split_keys"]] == g["split_crc"][j].tolist()


def test_flip_weights_leave_plus_state_dict_alone():
    from oracle.multi_head import plus_state_dict
    from oracle.multi_head_flip import flip_plus_state_dict
    a = plus_state_dict("s", [17, 14], 96, 3)
    flip_plus_state_dict("s", [17, 14], 96, 3, [[(1, 2)], []])
    b = plus_state_dict("s", [17, 14], 96, 3)
    assert all(np.array_equal(a[k], b[k]) for k in a)


def test_oracle_matches_fixture():
    """affine crop -> forward -> flip average -> one mode-4 decode per head, numpy, against the reference's numbers"""
    import torch
    from easy_vitpose_b200 import split_vitpose_plus
    from oracle import affine_oracle as A, decode_modes_oracle as DM, preproc_oracle as P, vitpose_oracle as O
    import zlib
    g = _fixture()
    D, depth, heads, _, _, _ = (int(v) for v in g["meta"])
    pairs = _pairs(g)
    names, Ks = [str(h) for h in g["heads"]], [int(k) for k in g["keypoints"]]
    parts = split_vitpose_plus({k: torch.from_numpy(np.asarray(v)) for k, v in _weights(g).items()}, names, Ks)
    frames = [P.make_frame(int(h), int(w), int(s)) for h, w, s in g["frames"]]
    for i in range(len(g["crc"])):
        img = A.warp_affine_u8(frames[g["frame_id"][i]], g["mats"][i])
        assert zlib.crc32(np.ascontiguousarray(img).tobytes()) == int(g["crc"][i]), i
    for j, (name, K) in enumerate(zip(names, Ks)):
        sd = {k: v.numpy() for k, v in parts[name].items()}
        sel = np.nonzero(g["head_id"] == j)[0]
        x = np.stack([A.warp_normalise(frames[g["frame_id"][i]], g["mats"][i]) for i in sel])
        out = O.forward_heatmaps(x, sd, depth, heads)
        out_f = O.forward_heatmaps(np.ascontiguousarray(x[..., ::-1]), sd, depth, heads)
        cs = g["cs_px"][sel]
        for shift in (0, 1):
            hm = ((out + DM.flip_back(out_f, pairs[j], bool(shift))) * np.float32(0.5)).astype(np.float32)
            rng = float(g[f"range_{shift}"][j, 1] - g[f"range_{shift}"][j, 0])
            assert np.abs(hm[0, g["sample_kps"][j]] - g[f"sample_hm_{shift}"][j]).max() < 2e-4 * rng
            assert np.abs(hm.reshape(len(sel), K, -1).sum(-1) - g[f"map_sum_{shift}"][sel, :K]).max() / 3072 < 2e-4 * rng
            assert np.array_equal(hm.reshape(len(sel), K, -1).argmax(-1), g[f"idx_{shift}"][sel, :K])
            pts, prob, _ = DM.keypoints_from_heatmaps(hm, cs[:, :2], cs[:, 2:], post_process="unbiased", use_udp=True)
            ref = g[f"kpts_{shift}"][sel, :K]
            assert np.abs(pts[..., ::-1] - ref[..., :2]).max() < 1e-3, (name, shift)
            assert np.abs(prob[..., 0] - ref[..., 2]).max() < 2e-4 * rng
