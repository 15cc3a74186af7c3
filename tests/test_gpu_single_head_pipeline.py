"""-m gpu: the single-head keypoint calls (vpb_infer, vpb_infer_frames, vpb_infer_affine) run the keypoint pipeline as the one
segment {head 0, n}.  With flip test off and on, a call enqueues exactly the launches vpb_kernel_launches counts, class by
class: one gather, the model, and one decode (plus the flip-back average, profiled in the same class).  Its eager, captured
and replayed forms return the same keypoints and argmax indices bit for bit."""
import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P, vitpose_oracle as O

pytestmark = pytest.mark.gpu

MAX_BATCH = 16
_engines = {}


def _engine():
    from easy_vitpose_b200 import ViTPose, model_cfg
    if "s" not in _engines:
        D, depth, _ = O.MODEL_DIMS["s"]
        m = ViTPose(model_cfg("s", 17), max_batch=MAX_BATCH)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, 17, 131, peaky=0.1, bumps=True).items()})
        _engines["s"] = m.to("cuda:0")
    return _engines["s"]


def _calls(m, n, seed):
    """(gather class, call) for crops, frames + boxes and affine crops of n people; call() -> (keypoints, argmax) tensors"""
    from easy_vitpose_b200 import topdown_args
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(O.make_crops(n, seed)).cuda()
    org = torch.from_numpy(rs.randint(64, 513, size=(n, 2)).astype(np.int32)).cuda()
    frames = [torch.from_numpy(P.make_frame(240, 320, seed + j)).cuda() for j in range(2)]
    x0, y0 = rs.randint(0, 200, n), rs.randint(0, 140, n)
    xyxy = np.stack([x0, y0, x0 + rs.randint(30, 120, n), y0 + rs.randint(30, 100, n)], 1).astype(np.int32)
    boxes = [xyxy[: n // 2], xyxy[n // 2:]]                          # n = 1: the first frame has no boxes
    args = [topdown_args(np.concatenate([b[:, :2], b[:, 2:] - b[:, :2]], 1)) for b in boxes]
    cat = lambda out: tuple(torch.cat(t) for t in out)             # noqa: E731
    return [("patch_im2col", lambda: m.infer_crops(x, org)),
            ("crop_preprocess", lambda: cat(m.infer_frames(frames, boxes))),
            ("crop_preprocess", lambda: cat(m.infer_affine(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args])))]


@pytest.mark.parametrize("flip", [False, True])
def test_single_head_calls_launch_what_kernel_launches_counts(flip):
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    m = _engine()
    depth = O.MODEL_DIMS["s"][1]
    if flip:
        m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS])
    try:
        for n in (1, 7):
            for i, (gather, call) in enumerate(_calls(m, n, 10 * n)):
                what = (flip, n, i)
                m.set_option("profile", 1)
                m.profile_collect()
                want_kp, want_idx = call()                           # eager: profiled calls are never captured
                counts = {k: c for k, (_, c) in m.profile_collect().items() if c}
                m.set_option("profile", 0)
                # ViT-S: standalone LayerNorms, and qkv and attention as two launches (head_dim 32 is never fused)
                assert counts == {gather: 1, "gemm_patch_embed": 1, "layernorm": 2 * depth + 1, "gemm_qkv": depth, "attention": depth,
                                  "gemm_proj": depth, "gemm_fc1_gelu": depth, "gemm_fc2": depth, "gemm_deconv": 2, "gemm_final_conv": 1,
                                  "decode": 1 + flip}, what
                assert sum(counts.values()) == m.kernel_launches(n), what
                m.set_option("ln_fused", 0)            # the default; setting it drops the cached graphs
                for state in ((1, 0), (1, 1), (1, 1)):                   # eager, capture, replay
                    kp, idx = call()
                    assert m.cached_graphs() == state, what
                    assert torch.equal(kp, want_kp) and torch.equal(idx, want_idx), what
    finally:
        m.set_option("profile", 0)
        m.set_flip_test(None)
