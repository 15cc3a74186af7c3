"""Random-init weights and inputs of the reference's architecture, for benchmarks and smoke runs where no checkpoint or
dataset can be mounted.  Key names and shapes are the `state_dict()` contract of the reference ViTPose
(vit_models/backbone/vit.py, vit_models/head/topdown_heatmap_simple_head.py; SURVEY.md section 8b).

Random weights alone give noise heatmaps, so `peaks=True` adds a small signal path (position embedding -> one channel per
keypoint -> positive deconv kernels -> 1x1 conv) that puts one clear maximum into every heatmap, as a trained model has.
Throughput does not depend on the values; the decode's work does not either (one warp per map, fixed stencil)."""
from __future__ import annotations

import math

import numpy as np

__all__ = ["random_state_dict", "random_crops"]

_DIMS = {"s": (384, 12, 12), "b": (768, 12, 12), "l": (1024, 24, 16), "h": (1280, 32, 16)}


def random_state_dict(size: str, num_keypoints: int, seed: int = 0, peaks: bool = True, decoder: str = "classic") -> "dict[str, np.ndarray]":
    """float32 arrays under the reference key names for ViT-`size` ('s' | 'b' | 'l' | 'h') with a K-keypoint head: decoder
    "classic" (2 deconvs + 1x1 conv) or "simple" (final_layer [K, D, 3, 3]; its peak pathway reads the hot channel through the
    centre tap)."""
    D, depth, _ = _DIMS[size]
    F, K = 256, int(num_keypoints)
    rs = np.random.RandomState(seed)

    def n(*shape, std, mean=0.0):
        return (rs.standard_normal(shape) * std + mean).astype(np.float32)

    sd = {"backbone.pos_embed": n(1, 193, D, std=0.02),
          "backbone.patch_embed.proj.weight": n(D, 3, 16, 16, std=0.03),
          "backbone.patch_embed.proj.bias": n(D, std=0.02)}
    for i in range(depth):
        p = f"backbone.blocks.{i}."
        for name, shape, std, mean in (("norm1.weight", (D,), 0.05, 1.0), ("norm1.bias", (D,), 0.02, 0.0),
                                       ("attn.qkv.weight", (3 * D, D), 0.04, 0.0), ("attn.qkv.bias", (3 * D,), 0.02, 0.0),
                                       ("attn.proj.weight", (D, D), 0.02, 0.0), ("attn.proj.bias", (D,), 0.02, 0.0),
                                       ("norm2.weight", (D,), 0.05, 1.0), ("norm2.bias", (D,), 0.02, 0.0),
                                       ("mlp.fc1.weight", (4 * D, D), 0.03, 0.0), ("mlp.fc1.bias", (4 * D,), 0.02, 0.0),
                                       ("mlp.fc2.weight", (D, 4 * D), 0.02, 0.0), ("mlp.fc2.bias", (D,), 0.02, 0.0)):
            sd[p + name] = n(*shape, std=std, mean=mean)
    sd["backbone.last_norm.weight"] = n(D, std=0.05, mean=1.0)
    sd["backbone.last_norm.bias"] = n(D, std=0.02)
    if decoder == "simple":
        sd["keypoint_head.final_layer.weight"] = n(K, D, 3, 3, std=(0.002 if peaks else 0.02) / math.sqrt(9 * D / F))
        sd["keypoint_head.final_layer.bias"] = n(K, std=0.01)
        for k in range(K if peaks else 0):
            c, t = k % D, int(rs.randint(0, 192))
            sd["backbone.pos_embed"][0, 1 + t, c] += np.float32(depth)
            sd["keypoint_head.final_layer.weight"][k, c, 1, 1] += np.float32(0.2)
        return sd
    if decoder != "classic":
        raise ValueError(f"decoder {decoder!r}: 'classic' or 'simple'")
    cin = D
    for li in (0, 3):
        sd[f"keypoint_head.deconv_layers.{li}.weight"] = n(cin, F, 4, 4, std=(0.15 if peaks else 1.0) / math.sqrt(cin))
        b = f"keypoint_head.deconv_layers.{li + 1}."
        sd[b + "weight"] = n(F, std=0.1, mean=1.0)
        sd[b + "bias"] = n(F, std=0.1)
        sd[b + "running_mean"] = n(F, std=0.1)
        sd[b + "running_var"] = rs.uniform(0.5, 1.5, size=(F,)).astype(np.float32)
        cin = F
    sd["keypoint_head.final_layer.weight"] = n(K, F, 1, 1, std=0.002 if peaks else 0.02)
    sd["keypoint_head.final_layer.bias"] = n(K, std=0.01)
    if peaks:
        bump = (np.outer([1.0, 2.0, 2.0, 1.0], [1.0, 2.0, 2.0, 1.0]) / 4.0).astype(np.float32)
        for k in range(K):
            c, t = k % min(D, F), int(rs.randint(0, 192))
            sd["backbone.pos_embed"][0, 1 + t, c] += np.float32(depth)        # scaled with depth: the random stream grows too
            sd["keypoint_head.deconv_layers.0.weight"][c, c] += bump * np.float32(1.5)
            sd["keypoint_head.deconv_layers.3.weight"][c, c] += bump
            sd["keypoint_head.final_layer.weight"][k, c, 0, 0] += np.float32(0.03)
    return sd


def random_crops(batch: int, seed: int = 0) -> np.ndarray:
    """float32 [batch,3,256,192] ~ N(0,1): the distribution of (img / 255 - MEAN) / STD (easy_ViTPose/inference.py:314-318)."""
    return np.random.RandomState(seed).standard_normal((batch, 3, 256, 192)).astype(np.float32)
