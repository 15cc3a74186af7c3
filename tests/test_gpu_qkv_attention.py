"""-m gpu: the fused qkv + attention launch (csrc/qkv_attention.cuh) against the qkv GEMM followed by the attention kernel.
Both forms round q, k and v to bf16 the same way and run the same attention code, so every output must agree bit for bit:
heatmaps, keypoints, argmax and the last block's attention output.  vpb_debug_attention forces either form (bit 1 fused,
bit 2 the two launches); the engine's own choice (fuse_qkv_attention in engine.cu) must agree with both."""
import os

import numpy as np
import pytest
import torch

from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

FUSED, SEPARATE, DEFAULT = 2, 4, 0
MAX_BATCH = 64
_engines = {}


def _engine(golden_dir, name):
    from easy_vitpose_b200 import ViTPose, model_cfg
    if name not in _engines:
        g = np.load(os.path.join(golden_dir, f"fwd_{name}.npz"))
        D, depth, heads, K, _, wseed, _ = (int(v) for v in g["meta"])
        m = ViTPose(model_cfg({384: "s", 768: "b", 1024: "l", 1280: "h"}[D], K), max_batch=MAX_BATCH)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, K, wseed, peaky=float(g["peaky"]), bumps=True).items()})
        _engines[name] = (m.to("cuda:0"), D)
    return _engines[name]


def _inputs(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).cuda()
    org = torch.from_numpy(np.random.RandomState(seed).randint(64, 513, size=(n, 2)).astype(np.int32))
    return x, org


def _run(m, D, x, org, flags, model_crops=None):
    """keypoints, argmax, heatmaps and the attention buffer of one eager call in the form `flags` selects"""
    from easy_vitpose_b200 import _lib
    rows = (model_crops or x.shape[0]) * 192
    try:
        _lib.lib().vpb_debug_attention(flags)
        m.set_option("graph", 0)
        kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
        torch.cuda.synchronize()
        attn = m.read_buffer("attn", (rows, D), "bf16")
    finally:
        _lib.lib().vpb_debug_attention(-1)
        m.set_option("graph", 1)
    return [t.cpu() for t in (kp, idx, hm)] + [attn]


def _same(a, b, what):
    for u, v, name in zip(a, b, ("keypoints", "argmax", "heatmaps", "attn")):
        assert torch.equal(u.view(torch.int16) if u.dtype == torch.bfloat16 else u, v.view(torch.int16) if v.dtype == torch.bfloat16 else v), \
            f"{name} differ: {what}"


@pytest.mark.parametrize("poly", [0, 1])
@pytest.mark.parametrize("name", ["s_coco", "b_coco", "l_coco_25", "h_wholebody"])
def test_fused_equals_separate(golden_dir, name, poly):
    """Every ViT size (head_dim 32, 64, 64, 80), with and without the polynomial exponentials, at batch sizes on both sides of
    the fusion rule and at max_batch."""
    m, D = _engine(golden_dir, name)
    for n in (1, 5, 17, 24, 47, MAX_BATCH):
        x, org = _inputs(n, 7 * n + poly)
        ref = _run(m, D, x, org, SEPARATE | poly)
        _same(_run(m, D, x, org, FUSED | poly), ref, f"{name} fused, poly {poly}, {n} crops")
        _same(_run(m, D, x, org, DEFAULT | poly), ref, f"{name} engine's choice, poly {poly}, {n} crops")


@pytest.mark.parametrize("cap", [1, 7, 13, 131])
def test_fused_capped_grids(golden_dir, cap):
    """Fewer CTAs than items: a CTA walks many items and the operand ring wraps across item boundaries at odd counts (ViT-S:
    6 k-blocks per item on a 5-stage ring; ViT-B: 12 on 3)."""
    for name, n in (("s_coco", 3), ("b_coco", 5)):
        m, D = _engine(golden_dir, name)
        x, org = _inputs(n, 100 + cap)
        ref = _run(m, D, x, org, SEPARATE)
        _same(_run(m, D, x, org, FUSED | (cap << 8)), ref, f"{name}, {n} crops, grid capped at {cap}")


def test_fused_with_graph_capture(golden_dir):
    """Graph on: eager first call, capture on the second, replay on the third -- each equal to the two-launch form."""
    from easy_vitpose_b200 import _lib
    m, D = _engine(golden_dir, "b_coco")
    n = 48
    x, org = _inputs(n, 5)
    ref = _run(m, D, x, org, SEPARATE)
    try:
        _lib.lib().vpb_debug_attention(FUSED)
        m.set_option("graph", 1)
        for call in range(3):
            kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
            torch.cuda.synchronize()
            attn = m.read_buffer("attn", (n * 192, D), "bf16")
            _same([t.cpu() for t in (kp, idx, hm)] + [attn], ref, f"graph call {call}")
    finally:
        _lib.lib().vpb_debug_attention(-1)


def test_fused_flip_test(golden_dir):
    """Flip test: 2n model crops, the mirror images gathered on the fly."""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    m, D = _engine(golden_dir, "b_coco")
    try:
        m.set_flip_test([tuple(p) for p in COCO_FLIP_PAIRS], True)
        for n in (3, 32):
            x, org = _inputs(n, 11 + n)
            ref = _run(m, D, x, org, SEPARATE, model_crops=2 * n)
            _same(_run(m, D, x, org, FUSED, model_crops=2 * n), ref, f"flip test, {n} crops")
    finally:
        m.set_flip_test(None)


def test_fused_mixed_multi_head_call():
    """A multi-head engine (ViTPose+ experts) on a mixed batch: the fused launch serves every crop whatever its head."""
    from easy_vitpose_b200 import ViTPose, _lib, model_cfg
    from oracle.multi_head import plus_state_dict
    heads = (("coco", 17), ("aic", 14), ("wholebody", 133))
    m = ViTPose(model_cfg("b", 17), max_batch=48, heads=heads, expert_rows=192)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("b", [k for _, k in heads], 192, 31).items()})
    m.to("cuda:0")
    n = 40
    x, org = _inputs(n, 3)
    hidx = np.random.RandomState(3).randint(0, 3, n)
    out = {}
    for flags in (SEPARATE, FUSED):
        try:
            _lib.lib().vpb_debug_attention(flags)
            m.set_option("graph", 0)
            kp, idx, hm = m.infer_crops_heads(x, org.cuda(), hidx, return_heatmaps=True)
            torch.cuda.synchronize()
            out[flags] = [t.cpu() for t in (kp, idx, hm)] + [m.read_buffer("attn", (n * 192, 768), "bf16")]
        finally:
            _lib.lib().vpb_debug_attention(-1)
            m.set_option("graph", 1)
    _same(out[FUSED], out[SEPARATE], "mixed multi-head call")
