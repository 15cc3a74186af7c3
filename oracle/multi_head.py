"""Seeded synthetic ViTPose+ state_dicts (several keypoint heads, fc2 experts) that every side can regenerate.

The key set is the one of an unsplit ViTPose+ checkpoint, the input of the reference's model_split.py: each block's
mlp.fc2 holds the D - P shared output rows and mlp.experts.{j} the P rows of dataset j; keypoint_head is head 0 and
associate_keypoint_heads.{j-1} head j.  Every head carries its own bump pathway (vitpose_oracle._add_bump_pathway), so each
has one clear peak per keypoint; the experts are independent random rows, so a swapped expert moves the heatmaps.
"""
from __future__ import annotations

import numpy as np

from oracle import vitpose_oracle as O

SIZES = {"s": (384, 12, 12), "b": (768, 12, 12)}


def plus_state_dict(size: str, head_keypoints, P: int, seed: int) -> "dict[str, np.ndarray]":
    """float32 / int64 numpy arrays under ViTPose+ keys; P = 0 gives a fully shared backbone (no expert keys)."""
    D, depth, _ = SIZES[size]
    base = O.make_state_dict(D, depth, max(head_keypoints), seed, peaky=0.1, bumps=True)
    heads = [O.make_state_dict(D, depth, K, seed + 1000 * (j + 1), peaky=0.1, bumps=True) for j, K in enumerate(head_keypoints)]
    sd: "dict[str, np.ndarray]" = {}
    for k, v in base.items():
        if k.startswith("keypoint_head."):
            continue
        if P and ".mlp.fc2." in k:
            sd[k] = v[: D - P].copy()
            for j, h in enumerate(heads):
                sd[k.replace("fc2.", f"experts.{j}.")] = h[k][D - P:].copy()
        else:
            sd[k] = v
    for j, h in enumerate(heads):
        prefix = "keypoint_head." if j == 0 else f"associate_keypoint_heads.{j - 1}."
        for k, v in h.items():
            if k.startswith("keypoint_head."):
                sd[prefix + k[len("keypoint_head."):]] = v
    return sd
