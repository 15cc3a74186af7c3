"""Model hyper-parameters of the reference configs, in the shape ViTPose(cfg) expects.

Values restate easy_ViTPose/configs/ViTPose_common.py:65-195 (four sizes) and the per-dataset
out_channels patches (configs/ViTPose_<dataset>.py, e.g. ViTPose_coco.py:16-18).  Only the keys the
hot path consumes are kept; `dyn_model_import(dataset, size)` mirrors vit_utils/util.py:37-41.
"""
from __future__ import annotations

import copy

MODEL_ABBR = {"s": "small", "b": "base", "l": "large", "h": "huge"}
_DIMS = {"small": (384, 12, 12), "base": (768, 12, 12), "large": (1024, 24, 16), "huge": (1280, 32, 16)}
_DROP_PATH = {"small": 0.1, "base": 0.3, "large": 0.5, "huge": 0.55}
# dataset -> number of keypoints (configs/ViTPose_<dataset>.py: channel_cfg['num_output_channels'])
DATASET_KEYPOINTS = {"coco": 17, "coco_25": 25, "wholebody": 133, "mpii": 16, "aic": 14, "ap10k": 17, "apt36k": 17, "custom": 18}

# The heads of a ViTPose+ checkpoint in model_split.py's order (:71-74): keypoint_head is COCO, associate_keypoint_heads.{i}
# the others; head j uses fc2 expert j.
VITPOSE_PLUS_HEADS = (("coco", 17), ("aic", 14), ("mpii", 16), ("ap10k", 17), ("apt36k", 17), ("wholebody", 133))

data_cfg = dict(image_size=[192, 256], heatmap_size=[48, 64])   # ViTPose_common.py:29-31

# left/right keypoint pairs for the flip test: eye, ear, shoulder, elbow, wrist, hip, knee, ankle (datasets/COCO.py:114).
# The reference defines pairs for COCO only.
COCO_FLIP_PAIRS = ((1, 2), (3, 4), (5, 6), (7, 8), (9, 10), (11, 12), (13, 14), (15, 16))


def flip_pairs_for(dataset: str, flip_pairs=None) -> "list[tuple[int, int]]":
    """The flip pairs of a dataset: explicit `flip_pairs` win, 'coco' gets COCO_FLIP_PAIRS, any other dataset raises
    ValueError -- the reference gives no pairs for them, and a keypoint count alone does not determine them (ap10k also has
    17 keypoints, with other pairs)."""
    if flip_pairs is not None:
        return [(int(a), int(b)) for a, b in flip_pairs]
    if dataset == "coco":
        return list(COCO_FLIP_PAIRS)
    raise ValueError(f"no flip pairs known for dataset {dataset!r}: pass flip_pairs explicitly")


def model_cfg(size: str, num_keypoints: int, decoder: str = "classic") -> dict:
    """The reference's model dict for ViT-`size` with a K-keypoint head: decoder "classic" = the configs' 2x deconv + 1x1 conv
    head (configs/ViTPose_common.py), "simple" = the paper's simple decoder of the reference's training configs
    (train_configs/ViTPose_{base,large,huge}_simple_coco_256x192.py:60-68: relu, 4x bilinear upsample, 3x3 conv)."""
    name = MODEL_ABBR.get(size, size)
    if name not in _DIMS:
        raise KeyError(f"unknown model size {size!r}")
    if decoder not in ("classic", "simple"):
        raise ValueError(f"decoder {decoder!r}: 'classic' or 'simple'")
    D, depth, heads = _DIMS[name]
    if decoder == "simple":
        head = dict(type="TopdownHeatmapSimpleHead", in_channels=D, num_deconv_layers=0, num_deconv_filters=[],
                    num_deconv_kernels=[], upsample=4, extra=dict(final_conv_kernel=3), out_channels=num_keypoints)
    else:
        head = dict(type="TopdownHeatmapSimpleHead", in_channels=D, num_deconv_layers=2, num_deconv_filters=(256, 256),
                    num_deconv_kernels=(4, 4), extra=dict(final_conv_kernel=1), out_channels=num_keypoints)
    return dict(
        type="TopDown", pretrained=None,
        backbone=dict(type="ViT", img_size=(256, 192), patch_size=16, embed_dim=D, depth=depth, num_heads=heads,
                      ratio=1, use_checkpoint=False, mlp_ratio=4, qkv_bias=True, drop_path_rate=_DROP_PATH[name]),
        keypoint_head=head,
        train_cfg=dict(),
        test_cfg=dict(flip_test=True, post_process="default", shift_heatmap=False,
                      target_type="GaussianHeatmap", modulate_kernel=11, use_udp=True))


def dyn_model_import(dataset: str, model: str, decoder: str = "classic") -> dict:
    """Same call shape as the reference helper: dataset name + size letter -> model cfg dict (decoder: see model_cfg)."""
    if dataset not in DATASET_KEYPOINTS:
        raise KeyError(f"dataset {dataset!r} has no fixed keypoint count here; use model_cfg(size, K)")
    return copy.deepcopy(model_cfg(model, DATASET_KEYPOINTS[dataset], decoder))
