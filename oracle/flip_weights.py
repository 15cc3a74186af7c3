"""Seeded weights for the flip-test fixtures  --  TEST INFRASTRUCTURE ONLY.

vitpose_oracle._add_bump_pathway puts keypoint k's peak at a token t_k fixed by pos_embed, whatever the image is.  In a flip
test the mirrored crop's map perm[k] therefore also peaks at t_perm[k], and after flip_back the averaged map k has two peaks
of similar height, at t_k and at the mirror of t_perm[k]: the argmax of a bf16 engine and of the fp32 reference would jump
between them.  flip_symmetric_state_dict keeps every weight of make_state_dict(..., bumps=True) and moves only the pos_embed
bumps to a flip-symmetric placement: t_perm[k] is the mirror of t_k (same patch row, px -> 11 - px; token column px peaks at
heatmap column 4 px + 1.5, whose mirror 47 - x is column 4 (11 - px) + 1.5), and a self-paired keypoint sits in patch column
5 or 6, where its two mirrored bumps (4 heatmap columns apart) merge into one maximum.
"""
from __future__ import annotations

import numpy as np

from oracle import vitpose_oracle as O


def flip_symmetric_state_dict(embed_dim: int, depth: int, num_keypoints: int, seed: int, flip_pairs,
                              peaky: float = 0.1) -> dict:
    sd = O.make_state_dict(embed_dim, depth, num_keypoints, seed, peaky=peaky, bumps=True)
    pos = O.make_state_dict(embed_dim, depth, num_keypoints, seed, peaky=peaky)["backbone.pos_embed"]   # the same draws, no bumps
    bumped = sd["backbone.pos_embed"]
    nch = min(embed_dim, 256)
    if num_keypoints > nch:
        raise ValueError("one bump channel per keypoint is needed to find the default placement")
    amp = np.float32(12.0 * depth / 12.0)                         # as _add_bump_pathway
    perm = list(range(num_keypoints))
    for left, right in flip_pairs:
        perm[left], perm[right] = right, left
    placed: dict[int, int] = {}
    out = pos.copy()
    gw = O.GRID_W
    for k in range(num_keypoints):
        c = k % nch
        t = int(np.argmax(bumped[0, 1:, c] - pos[0, 1:, c]))         # the default placement: where the bump was added
        if perm[k] == k:
            t = (t // gw) * gw + 5 + t % 2
        elif perm[k] in placed:
            t = (placed[perm[k]] // gw) * gw + gw - 1 - placed[perm[k]] % gw
        placed[k] = t
        out[0, 1 + t, c] += amp
    sd["backbone.pos_embed"] = out
    return sd
