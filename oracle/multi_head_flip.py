"""Seeded ViTPose+ state_dicts for flip-test fixtures of several heads  --  TEST INFRASTRUCTURE ONLY.

oracle/multi_head.plus_state_dict gives every head the default bump pathway of vitpose_oracle (keypoint k on channel k), so
the heads' bumps share channels and pos_embed tokens.  A flip test needs each averaged map to have one peak
(oracle/flip_weights.py), and pos_embed is shared by all heads, so here every head owns channels of its own.
"""
from __future__ import annotations

import numpy as np

from oracle import vitpose_oracle as O
from oracle.multi_head import SIZES, plus_state_dict


# the 1x1 conv's weight on a keypoint's own channel: twice _add_bump_pathway's 0.03, because 214 hot channels leak through the
# random deconv weights into every map and one bump must stay well above that cross-talk for the flip average to keep one peak
FINAL_GAIN = 0.06


def _head_prefix(j: int) -> str:
    return "keypoint_head." if j == 0 else f"associate_keypoint_heads.{j - 1}."


def flip_plus_state_dict(size: str, head_keypoints, P: int, seed: int, flip_pairs_per_head) -> "dict[str, np.ndarray]":
    """plus_state_dict with the bump pathway of every head moved to channels of its own and placed flip-symmetrically (the
    placement rule of oracle/flip_weights.py) -- for flip-test fixtures of several heads.  pos_embed is shared by all heads, so
    head j's keypoint k owns channel sum(K_<j) + k (214 channels for the six ViTPose+ heads, within the 256 bump channels of
    every ViT): the default bumps of plus_state_dict are taken out (pos_embed redrawn without them, the head terms subtracted)
    and the new ones added with a separate seeded stream.  plus_state_dict itself is unchanged."""
    D, depth, _ = SIZES[size]
    ks = [int(k) for k in head_keypoints]
    nch = min(D, 256)
    if sum(ks) > nch:
        raise ValueError(f"{sum(ks)} keypoints over all heads need more than the {nch} bump channels")
    sd = plus_state_dict(size, ks, P, seed)
    sd["backbone.pos_embed"] = O.make_state_dict(D, depth, max(ks), seed, peaky=0.1)["backbone.pos_embed"]   # same draws, no bumps
    kern = np.outer([1.0, 2.0, 2.0, 1.0], [1.0, 2.0, 2.0, 1.0]).astype(np.float32) / 4.0
    amp = np.float32(12.0 * depth / 12.0)                          # as _add_bump_pathway
    gw = O.GRID_W
    rs = np.random.RandomState(seed + 7919)
    off = 0
    for j, (K, pairs) in enumerate(zip(ks, flip_pairs_per_head)):
        hp = _head_prefix(j)
        d0, d3, fin = (sd[hp + "deconv_layers.0.weight"].copy(), sd[hp + "deconv_layers.3.weight"].copy(),
                       sd[hp + "final_layer.weight"].copy())
        for k in range(K):                                         # the default pathway: channel k % nch
            c = k % nch
            d0[c, c] -= kern * np.float32(1.5)
            d3[c, c] -= kern * np.float32(1.0)
            fin[k, c, 0, 0] -= np.float32(0.03)
        perm = list(range(K))
        for left, right in pairs:
            perm[left], perm[right] = right, left
        placed: "dict[int, int]" = {}
        for k in range(K):
            c = off + k
            t = int(rs.randint(0, O.TOKENS))
            if perm[k] == k:                                       # self-paired: patch column 5 or 6, its mirror merges
                t = (t // gw) * gw + 5 + t % 2
            elif perm[k] in placed:                                # the partner's mirror token
                t = (placed[perm[k]] // gw) * gw + gw - 1 - placed[perm[k]] % gw
            placed[k] = t
            sd["backbone.pos_embed"][0, 1 + t, c] += amp
            d0[c, c] += kern * np.float32(1.5)
            d3[c, c] += kern * np.float32(1.0)
            fin[k, c, 0, 0] += np.float32(FINAL_GAIN)
        sd[hp + "deconv_layers.0.weight"], sd[hp + "deconv_layers.3.weight"], sd[hp + "final_layer.weight"] = d0, d3, fin
        off += K
    return sd


def topdown_pairs(name: str, K: int):
    """Flip pairs of the multi-head top-down fixture: COCO's for coco (datasets/COCO.py:114); the reference defines none for
    the other datasets, so the fixture takes neighbouring keypoints (1, 2), (3, 4), ... and stores them."""
    if name == "coco":
        return [(1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16)]
    return [(i, i + 1) for i in range(1, K - 1, 2)]
