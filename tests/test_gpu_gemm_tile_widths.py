"""Tile widths of the standalone GEMM (128, 192, 256; engine.cu pick_tile).  The accumulation order of an output element is the
k order whatever the tile width, so every width must give the same bits as the 128-wide tiles: kernel by kernel through
vpb_gemm with the width override, and end to end through the engine's own rule."""
import os

import numpy as np
import pytest
import torch

from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

EPI_BF16, EPI_BF16_GELU, EPI_F32_ADD, EPI_BF16_GELU_ERF = 0, 1, 5, 6


def _force_width(width):
    """vpb_debug_gemm flags >> 8 = the tile width every following GEMM launch must use (0 = the rule)"""
    from easy_vitpose_b200 import _lib
    _lib.lib().vpb_debug_gemm((width << 8) << 8, None)


@pytest.fixture
def restore_rule():
    yield
    _force_width(0)


@pytest.mark.parametrize("epi", [EPI_BF16, EPI_BF16_GELU, EPI_BF16_GELU_ERF, EPI_F32_ADD])
@pytest.mark.parametrize("M,N,K", [(1000, 768, 768), (200, 2304, 768), (1000, 3072, 768), (709, 768, 3072), (12288, 768, 768),
                                   (331, 1280, 1280)])
def test_every_width_matches_128_wide_tiles(restore_rule, epi, M, N, K):
    from gpu_util import gemm
    g =torch.Generator(device="cuda").manual_seed(M * 7 + N + K + epi)
    a = (torch.randn(M, K, generator=g, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, generator=g, device="cuda")
    x0 = torch.randn(M, N, generator=g, device="cuda")
    outs = {}
    for width in (128, 192, 256):
        if N % width:
            continue
        _force_width(width)
        out = x0.clone() if epi == EPI_F32_ADD else torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        gemm(a, w, bias, out, epi)
        outs[width] = out
    assert len(outs) >= 2
    for width, out in outs.items():
        assert torch.equal(out.view(torch.int16 if out.dtype == torch.bfloat16 else torch.int32),
                           outs[128].view(torch.int16 if out.dtype == torch.bfloat16 else torch.int32)), f"width {width}"


def test_fused_layernorm_tail_at_every_width(golden_dir, restore_rule):
    """The residual GEMMs' fused LayerNorm tail (engine option ln_fused) counts column tiles from the tile width: the normalised
    rows and the stream must not depend on it (ViT-B at 7 crops: a ragged last row block)."""
    from easy_vitpose_b200 import ViTPose, model_cfg
    g = np.load(os.path.join(golden_dir, "fwd_b_coco.npz"))
    D, depth, heads, K, B, wseed, xseed = (int(v) for v in g["meta"])
    m = ViTPose(model_cfg("b", K), max_batch=7)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, K, wseed, peaky=float(g["peaky"]), bumps=True).items()})
    m.to("cuda:0")
    m.set_option("ln_fused", 1)
    x = torch.from_numpy(O.make_crops(7, 4242)).cuda()
    org = torch.tensor([[200, 300]] * 7, dtype=torch.int32)
    outs = {}
    for width in (128, 192, 256):
        _force_width(width)
        m.set_option("ln_fused", 1)                                      # drops the captured graphs: they embed the tile choice
        outs[width] = [t.cpu().numpy() for t in m.infer_crops(x, org, return_heatmaps=True)]
    for width in (192, 256):
        for u, v in zip(outs[width], outs[128]):
            assert np.array_equal(u, v), f"width {width}"


@pytest.mark.parametrize("name", ["s_coco", "b_coco", "h_wholebody"])
def test_engine_rule_matches_128_wide_tiles(golden_dir, name):
    """infer_crops at 1, 7 and 64 crops: the default width rule and forced 128-wide tiles (debug flag 8) give the same heatmaps,
    keypoints and argmax, bit for bit."""
    from easy_vitpose_b200 import ViTPose, _lib, model_cfg
    g = np.load(os.path.join(golden_dir, f"fwd_{name}.npz"))
    D, depth, heads, K, B, wseed, xseed = (int(v) for v in g["meta"])
    size = {384: "s", 768: "b", 1280: "h"}[D]
    m = ViTPose(model_cfg(size, K), max_batch=64)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, K, wseed, peaky=float(g["peaky"]), bumps=True).items()})
    m.to("cuda:0")
    x = torch.from_numpy(O.make_crops(64, 777)).cuda()
    org = torch.tensor([[190 + i, 260 - i] for i in range(64)], dtype=torch.int32)
    outs = {}
    try:
        for narrow in (0, 1):
            _lib.lib().vpb_debug_gemm((8 << 8) if narrow else 0, None)
            m.set_option("chain", 0)                                      # drops the captured graphs: they embed the tile choice
            outs[narrow] = [[t.cpu().numpy() for t in m.infer_crops(x[:n], org[:n], return_heatmaps=True)] for n in (1, 7, 64)]
    finally:
        _lib.lib().vpb_debug_gemm(0, None)
    for a, b in zip(outs[0], outs[1]):
        for u, v in zip(a, b):
            assert np.array_equal(u, v)
