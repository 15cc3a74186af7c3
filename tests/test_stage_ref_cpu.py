"""CPU: the single-stage fp64 references of oracle/stage_ref.py.

1. Chained on their own outputs, rounded as the engine rounds its buffers, they reproduce the reference's fp32 heatmaps
   (tests/golden/fwd_*.npz) within the 1 % of range the engine tests use: they compute the right model.
2. Their bounds are tight enough to matter: each wiring bug below moves the heatmaps by less than 1 % of the range (every
   end-to-end test passes with it), yet the stage it touches leaves its bound.  The "engine" here is the reference itself,
   rounded as the engine rounds (bf16 buffers): the correct one stays within the bound, the bugged one does not.
"""
import os

import numpy as np
import pytest
import torch

from oracle import stage_ref as S
from oracle import vitpose_oracle as O


def _fixture(golden_dir, name):
    g = np.load(os.path.join(golden_dir, f"fwd_{name}.npz"))
    D, depth, heads, K, B, wseed, xseed = (int(v) for v in g["meta"])
    sd = O.make_state_dict(D, depth, K, wseed, peaky=float(g["peaky"]), bumps=True)
    return g, sd, O.make_crops(B, xseed), depth, heads


@pytest.mark.parametrize("name", ["s_coco", "b_coco"])
def test_chained_stage_references_reproduce_golden_heatmaps(golden_dir, name):
    g, sd, crops, depth, heads = _fixture(golden_dir, name)
    with torch.no_grad():
        hm = S.chained_forward(crops, sd, depth, heads).numpy()
    ref = g["heatmaps"]
    rng = float(ref.max() - ref.min())
    linf = float(np.abs(hm - ref).max())
    print(name, f"chained stage references: heatmap Linf {linf / rng:.3%} of range")
    assert linf < 0.01 * rng


@pytest.fixture(scope="module")
def block0(golden_dir):
    """Block-0 inputs of the b_coco fixture, each stage's input rounded as the engine stores it."""
    _, sd, crops, _, heads = _fixture(golden_dir, "b_coco")
    x0 = S.patch_embed(S.patch_rows(crops), sd)[0].float().double()
    xn1 = S.bf16(S.block_norm(x0, sd, 0, 1)[0].float())
    x1 = S.proj(S.bf16(S.attention(S.bf16(S.qkv(xn1, sd, 0, heads)[0].float()), heads)[0].float()), x0, sd, 0)[0].float().double()
    xn2 = S.bf16(S.block_norm(x1, sd, 0, 2)[0].float())
    return sd, heads, x0, xn1, xn2


def _engine_like(ref):
    return S.bf16(ref.float())


def _check_caught(name, good, bad, ref, bound):
    ok, caught = S.worst_ratio(good, ref, bound), S.worst_ratio(bad, ref, bound)
    n_out = int(((bad - ref).abs() > bound).sum())
    print(f"{name}: correct worst error / bound {ok:.3f}, bugged {caught:.2f} ({n_out} elements outside)")
    assert ok <= 1.0
    assert caught > 1.0


def _bugged(sd, key, fn):
    bad = dict(sd)
    bad[key] = fn(np.array(sd[key]))
    return bad


def test_bound_catches_zero_v_bias_of_one_head(block0):
    sd, heads, _, xn1, _ = block0
    D = xn1.shape[1]
    hd = D // heads

    def zero(b):
        b[2 * D + 3 * hd: 2 * D + 4 * hd] = 0
        return b
    ref, bound = S.qkv(xn1, sd, 0, heads)
    bad = S.qkv(xn1, _bugged(sd, "backbone.blocks.0.attn.qkv.bias", zero), 0, heads)[0]
    _check_caught("v bias of head 3 zero", _engine_like(ref), _engine_like(bad), ref, bound)


def test_bound_catches_qkv_bias_missing_on_last_tile(block0):
    sd, heads, _, xn1, _ = block0

    def drop(b):
        b[-128:] = 0
        return b
    ref, bound = S.qkv(xn1, sd, 0, heads)
    bad = S.qkv(xn1, _bugged(sd, "backbone.blocks.0.attn.qkv.bias", drop), 0, heads)[0]
    _check_caught("qkv bias missing on the last 128 columns", _engine_like(ref), _engine_like(bad), ref, bound)


def test_bound_catches_fc1_bias_missing_on_last_tile(block0):
    sd, _, _, _, xn2 = block0

    def drop(b):
        b[-128:] = 0
        return b
    ref, bound = S.fc1(xn2, sd, 0)
    bad = S.fc1(xn2, _bugged(sd, "backbone.blocks.0.mlp.fc1.bias", drop), 0)[0]
    _check_caught("fc1 bias missing on the last 128 columns", _engine_like(ref), _engine_like(bad), ref, bound)


def test_bound_catches_layernorm_eps(block0):
    sd, _, x0, _, _ = block0
    ref, bound = S.block_norm(x0, sd, 0, 1)
    bad = S.block_norm(x0, sd, 0, 1, eps=1e-2)[0]
    _check_caught("LayerNorm eps 1e-2", _engine_like(ref), _engine_like(bad), ref, bound)


def test_bound_catches_unshifted_batchnorm(golden_dir):
    """pack_deconv writing the BatchNorm shift as beta instead of beta - mean * s."""
    _, sd, _, _, _ = _fixture(golden_dir, "s_coco")
    feat = S.bf16(torch.from_numpy(np.random.RandomState(0).standard_normal((192, 384)).astype(np.float32)))
    ref, bound = S.deconv(feat, sd, 0)
    bad = dict(sd)
    bad["keypoint_head.deconv_layers.1.running_mean"] = np.zeros_like(sd["keypoint_head.deconv_layers.1.running_mean"])
    _check_caught("BatchNorm shift without the mean", _engine_like(ref), _engine_like(S.deconv(feat, bad, 0)[0]), ref, bound)


def test_bf16_helpers():
    x = torch.tensor([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 3.0, -0.75], dtype=torch.float64)
    assert S.bf16(x).tolist() == [1.0, 1.0, 1.0 + 2 ** -6, 3.0, -0.75]               # round to nearest even
    assert S.half_ulp_bf16(x.abs()).tolist() == [2 ** -8, 2 ** -8, 2 ** -8, 2 ** -7, 2 ** -9]
    assert S.q_scale(64) == np.float32(0.125)
