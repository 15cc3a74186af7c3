"""CPU: the C-ABI library loads and exports every symbol include/vitpose_b200.h declares; host-side
mirror of the reference interface behaves (no GPU compute here)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.build import LIB, build
    build()
    hdr = open(os.path.join(ROOT, "include", "vitpose_b200.h")).read()
    declared = set(re.findall(r"\b(vpb_[a-z_]+)\s*\(", hdr))
    assert declared, "header declares nothing?"
    lib = ctypes.CDLL(LIB)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    _lib.lib()


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from easy_vitpose_b200 import ViTPose, decode_heatmaps, model_cfg
    m = ViTPose(model_cfg("b", 17))
    with pytest.raises(RuntimeError):
        m.to("cpu")
    with pytest.raises(RuntimeError):
        decode_heatmaps(torch.zeros(1, 17, 64, 48), torch.tensor([[192, 256]]))


def test_configs_match_reference_shapes():
    from easy_vitpose_b200 import dyn_model_import
    from easy_vitpose_b200.model import _expected_shapes
    from oracle import vitpose_oracle as O
    for size, ds, K in [("s", "coco", 17), ("b", "ap10k", 17), ("l", "coco_25", 25), ("h", "wholebody", 133)]:
        cfg = dyn_model_import(ds, size)
        D, depth, heads = O.MODEL_DIMS[size]
        assert (cfg["backbone"]["embed_dim"], cfg["backbone"]["depth"], cfg["backbone"]["num_heads"]) == (D, depth, heads)
        assert cfg["keypoint_head"]["out_channels"] == K
        sd = O.make_state_dict(D, 1, K, 0)
        exp = _expected_shapes(D, 1, K)
        assert set(sd) == set(exp)
        for k in sd:
            assert tuple(np.asarray(sd[k]).shape) == tuple(exp[k]), k


def test_state_dict_contract_is_strict():
    import torch
    from easy_vitpose_b200 import ViTPose, model_cfg
    from oracle import vitpose_oracle as O
    m = ViTPose(model_cfg("s", 17))
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(384, 12, 17, 0).items()}
    extra = dict(sd); extra["backbone.cls_token"] = torch.zeros(1)
    with pytest.raises(RuntimeError):
        m.load_state_dict(extra)
    wrong = dict(sd); wrong["backbone.pos_embed"] = torch.zeros(1, 197, 384)
    with pytest.raises(RuntimeError):
        m.load_state_dict(wrong)
    m.load_state_dict({"state_dict": sd})                     # both checkpoint layouts (inference.py:162-166)
    out = m.state_dict()
    assert set(out) == set(sd) and torch.equal(out["backbone.pos_embed"], sd["backbone.pos_embed"])


def test_synthetic_weights_follow_the_state_dict_contract():
    """easy_vitpose_b200.synthetic (what bench.py's GPU arm loads: it must not import oracle/) produces exactly the reference's
    state_dict keys and shapes (SURVEY.md section 8b), and a strict load accepts them without a GPU."""
    import numpy as np
    import torch

    from easy_vitpose_b200 import ViTPose, model_cfg
    from easy_vitpose_b200.synthetic import random_crops, random_state_dict
    from oracle import vitpose_oracle as O
    for size, K in (("s", 17), ("b", 25)):
        D, depth, heads = O.MODEL_DIMS[size]
        mine = random_state_dict(size, K, seed=3)
        ref = {k: v.shape for k, v in O.make_state_dict(D, depth, K, 3).items() if not k.endswith("num_batches_tracked")}
        assert {k: v.shape for k, v in mine.items()} == ref
        assert all(v.dtype == np.float32 for v in mine.values())
        ViTPose(model_cfg(size, K)).load_state_dict({k: torch.from_numpy(v) for k, v in mine.items()})      # strict, CPU side only
    assert random_crops(2, 1).shape == (2, 3, 256, 192) and np.array_equal(random_crops(2, 1), random_crops(2, 1))


def test_decode_api_fails_loudly_without_cuda_and_checks_its_config():
    """No CPU fallback anywhere on the product path: decode entry points refuse CPU tensors; the reference's config conflicts
    (vit_utils/top_down_eval.py:548-553) and the combinations that are not built raise before any device work."""
    import numpy as np
    import pytest
    import torch

    from easy_vitpose_b200 import decode_heatmaps, keypoints_from_heatmaps
    hm = np.zeros((1, 17, 64, 48), np.float32)
    c = np.array([[96, 128]]); s = np.array([[192, 256]])
    with pytest.raises(RuntimeError):
        decode_heatmaps(torch.zeros(1, 17, 64, 48), torch.tensor([[192, 256]]))
    with pytest.raises(AssertionError):
        keypoints_from_heatmaps(hm, c, s, post_process="megvii", use_udp=True)
    with pytest.raises(AssertionError):
        keypoints_from_heatmaps(hm, c, s, unbiased=True, post_process="megvii")
    with pytest.raises(ValueError):                                   # 17 maps are not triples (reference: reshape fails, :590)
        keypoints_from_heatmaps(hm, c, s, use_udp=True, target_type="CombinedTarget")
    with pytest.raises(ValueError):                                   # N > 1: the reference's index arithmetic does not broadcast (:589)
        keypoints_from_heatmaps(np.zeros((2, 18, 64, 48), np.float32), np.tile(c, (2, 1)), np.tile(s, (2, 1)), use_udp=True,
                                target_type="CombinedTarget")
    with pytest.raises(ValueError):
        keypoints_from_heatmaps(hm, c, s, use_udp=True, target_type="nonsense")
    with pytest.raises(NotImplementedError):                          # even / oversized modulation kernels
        keypoints_from_heatmaps(hm, c, s, post_process="unbiased", kernel=8)
    with pytest.raises(NotImplementedError):
        keypoints_from_heatmaps(hm, c, s, post_process="megvii", kernel=37)
    with pytest.raises(ValueError):                                   # kernel = 1: the reference's _gaussian_blur raises (zero-width border)
        keypoints_from_heatmaps(hm, c, s, post_process="unbiased", kernel=1)
    with pytest.raises(NotImplementedError):                          # CombinedTarget blurs with 2 * kernel + 1 <= 35
        keypoints_from_heatmaps(hm[:, :15], c, s, use_udp=True, kernel=19, target_type="CombinedTarget")
    with pytest.raises(ValueError):
        keypoints_from_heatmaps(hm, c, s, post_process="fancy")


def test_gemm_entry_points_reject_what_the_kernels_cannot_serve():
    """vpb_gemm, vpb_expert_gemm, vpb_debug_gemm, vpb_attention and vpb_qkv_attention check their arguments before touching the
    device, so VPB_ERR_ARG (1)
    comes back with or without a GPU.  The device pointers are misaligned dummies that no tensor map accepts."""
    import ctypes as C

    from easy_vitpose_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(8)
    EPI_BF16, EPI_BF16_RELU_UP, EPI_F32_NCHW, EPI_F32_ADD = 0, 2, 4, 5

    def gemm(m, n, k, epi, bias=p, aux=(0, 0, 0, 0)):
        return L.vpb_gemm(p, p, bias, p, m, n, k, epi, None, 0, *aux, None)

    assert gemm(0, 128, 64, EPI_BF16) == 1                                    # M < 1
    assert gemm(-5, 128, 64, EPI_F32_ADD) == 1
    assert gemm(128, 0, 64, EPI_BF16) == 1                                    # N < 1
    assert gemm(128, 128, 64, EPI_BF16, bias=None) == 1                       # epilogues that read a bias
    assert gemm(128, 128, 64, EPI_F32_ADD, bias=None) == 1
    assert gemm(192, 256, 1024, EPI_BF16_RELU_UP, bias=None, aux=(16, 12, 8, (12 << 16) | 256)) == 1
    assert gemm(192, 256, 1024, EPI_BF16_RELU_UP, aux=(0, 12, 8, (12 << 16) | 256)) == 1      # no input grid (was a host / 0)
    assert gemm(3072, 32, 256, EPI_F32_NCHW, aux=(0, 3072, 0, 0)) == 1       # no channels
    assert gemm(3072, 32, 256, EPI_F32_NCHW, aux=(33, 3072, 0, 0)) == 1      # more channels than W rows
    assert gemm(3072, 32, 256, EPI_F32_NCHW, aux=(17, 0, 0, 0)) == 1         # no pixels

    def experts(segs, M=384, D=384, P=64, H=2):
        table = (C.c_int32 * max(1, 3 * len(segs)))(*[v for s in segs for v in s])
        return L.vpb_expert_gemm(p, p, p, p, M, D, P, H, table, len(segs), 1, None)

    for segs in ([(100, 200, 0), (50, 150, 1)], [(10, 10, 0)], [(0, 385, 0)], [(0, 100, 2)], [(0, 100, -1)], [], [(-1, 10, 0)]):
        assert experts(segs) == 1, segs
    assert experts([(i, i + 1, 0) for i in range(129)], M=200) == 1          # more than EXPERT_MAX_SEGMENTS
    for P in (0, 48, 384, 400):
        assert experts([(0, 100, 0)], P=P) == 1, P
    assert experts([(0, 100, 0)], D=400, P=64) == 1                          # D % 32
    assert experts([(0, 100, 0)], H=0) == 1
    # the attention entry points: head_dim not built, non-positive counts, int overflow of 3 D, batch * heads or batch * 192
    big = 2 ** 31 - 1
    for batch, heads, hd in ((1, 12, 48), (1, 12, 0), (0, 12, 64), (1, 0, 64), (-1, 12, 64), (1, big // 64, 64),
                             (1, big // 150 + 1, 80), (big // 100, 200, 32), (big // 192 + 1, 1, 64)):
        assert L.vpb_attention(p, batch, heads, hd, p, None) == 1, (batch, heads, hd)
        assert L.vpb_qkv_attention(p, p, p, batch, heads, hd, p, None) == 1, (batch, heads, hd)
    assert L.vpb_attention(None, 1, 12, 64, p, None) == 1
    assert L.vpb_qkv_attention(p, p, None, 1, 12, 64, p, None) == 1
    assert L.vpb_qkv_attention(p, p, p, 1, 1, 32, p, None) == 1             # D = 32: not a whole 64-wide k-block
    try:
        assert L.vpb_debug_gemm(1, None) == 1                                 # a one-stage ring cannot hold two k-blocks
        assert L.vpb_debug_gemm(1 | (4 << 8), None) == 1
        assert L.vpb_debug_gemm(3 | (4 << 8), None) == 0
    finally:
        L.vpb_debug_gemm(0, None)
