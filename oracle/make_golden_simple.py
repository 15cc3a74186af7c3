"""Goldens of the simple decoder from the reference's own ViTPose  --  TEST INFRASTRUCTURE ONLY.

Run with the reference tree available (oracle/ref_import.py says where it looks):   python oracle/make_golden_simple.py

For each of the reference's simple-decoder training configs (train_configs/ViTPose_{base,large,huge}_simple_coco_256x192.py)
the config file is executed and its `model` dict builds the reference's ViTPose.  The reference's head raises
NotImplementedError in _transform_inputs for upsample > 0 on a tensor input (topdown_heatmap_simple_head.py:269-271), so that
one method is replaced on the instance by the upstream ViTPose line it stands for,
    resize(input=F.relu(inputs), scale_factor=self.upsample, mode='bilinear', align_corners=self.align_corners)
(ReLU first: oracle/simple_head_oracle.py says where that order comes from).  Weights and crops are regenerated from seeds
(simple_head_oracle.make_state_dict(..., bumps=True), make_crops), the forward runs in fp32 on the CPU, and
tests/golden/simple_{b,l,h}_coco.npz get the heatmaps and the keypoints of VitInference.postprocess, one call per crop, in
the layout of the fwd_* goldens (meta = D, depth, heads, K, B, wseed, xseed).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _REPO)

from oracle import ref_import  # noqa: E402
from oracle import simple_head_oracle as S  # noqa: E402
from oracle import vitpose_oracle as O  # noqa: E402

CASES = (("b", "base", 2, 112, 212, [[192, 256], [151, 211]]),
         ("l", "large", 2, 113, 213, [[288, 384], [97, 140]]),
         ("h", "huge", 1, 114, 214, [[333, 444]]))


def config_model(size_name: str) -> dict:
    path = os.path.join(ref_import.REF_PKG, "configs", "train_configs", f"ViTPose_{size_name}_simple_coco_256x192.py")
    ns: dict = {}
    with open(path) as f:
        src = f.read()
    # mmcv substitutes {{_base_.x}} textually before running a config; `model` reads none of them
    src = src.replace("{{_base_.dataset_info}}", "None")
    exec(compile(src, path, "exec"), ns)
    return ns["model"]


def upstream_transform_inputs(self, inputs):
    return F.interpolate(F.relu(inputs), scale_factor=self.upsample, mode="bilinear", align_corners=self.align_corners)


def main() -> None:
    ref = ref_import.load()
    torch.set_grad_enabled(False)
    for size, size_name, B, wseed, xseed, org_wh in CASES:
        cfg = config_model(size_name)
        bb, hd = cfg["backbone"], cfg["keypoint_head"]
        D, depth, heads, K = int(bb["embed_dim"]), int(bb["depth"]), int(bb["num_heads"]), int(hd["out_channels"])
        model = ref.ViTPose(cfg).eval()
        model.keypoint_head._transform_inputs = types.MethodType(upstream_transform_inputs, model.keypoint_head)
        peaky = 0.1
        sd = S.make_state_dict(D, depth, K, wseed, peaky=peaky, bumps=True)
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        x = O.make_crops(B, xseed)
        hm = model(torch.from_numpy(x)).numpy().astype(np.float32)
        org = np.asarray(org_wh, np.int32)
        kpts = np.concatenate([ref_import.postprocess(ref, hm[i:i + 1], int(org[i, 0]), int(org[i, 1])) for i in range(B)], 0)
        out = os.path.join(_REPO, "tests", "golden", f"simple_{size}_coco.npz")
        np.savez_compressed(out, heatmaps=hm, kpts=kpts.astype(np.float32), org_wh=org,
                            meta=np.array([D, depth, heads, K, B, wseed, xseed], np.int64), peaky=np.float64(peaky))
        print(out, hm.shape, float(hm.min()), float(hm.max()), os.path.getsize(out))


if __name__ == "__main__":
    main()
