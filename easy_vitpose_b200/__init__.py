"""easy_vitpose_b200: the ViTPose crop path of JunkyByte/easy_ViTPose on H100 (sm_90a).

    crops [B,3,256,192] -> ViT -> TopdownHeatmapSimpleHead -> heatmaps [B,K,64,48] -> keypoints [B,K,3]

csrc/ holds the hand-written CUDA (wgmma GEMM + attention, LayerNorm, gathers, decode) and the C ABI
(include/vitpose_b200.h); the Python modules mirror the reference's interface for this path:
model.ViTPose, top_down_eval.keypoints_from_heatmaps, inference.install / B200PoseBackend.
"""
from . import distributed  # noqa: F401
from .configs import COCO_FLIP_PAIRS, VITPOSE_PLUS_HEADS, data_cfg, dyn_model_import, flip_pairs_for, model_cfg  # noqa: F401
from .inference import B200PoseBackend, install  # noqa: F401
from .nms import oks_iou_device, oks_nms, oks_nms_device, oks_nms_frames, soft_oks_nms  # noqa: F401
from .model import ViTPose, head_flip_permutations, merge_split_state_dicts, plan_head_calls, split_vitpose_plus  # noqa: F401
from .top_down_eval import decode_heatmaps, decode_topdown, keypoints_from_heatmaps  # noqa: F401
from .topdown import topdown_args  # noqa: F401
from .smooth import DeviceOneEuro  # noqa: F401
from .track import DeviceSort  # noqa: F401
