"""CPU: the trained-like weights of oracle/trained_like.py carry the statistics they promise, and those statistics expose
bugs the benign weights of make_state_dict hide.

1. The stage references of oracle/stage_ref.py, chained as the engine rounds its buffers (chained_forward, keeping every
   intermediate), on ViT-S at full depth and ViT-B at depth 4: massive stream channels, sink tokens, sharp logits in every
   block and a GELU input tail beyond +-8 must all be present.  If the generator silently turns benign again, this fails.
2. A bug that the benign weights hide, emulated in fp32 as the kernel would compute it, against the stage bound: it prints
   the worst error / bound of the bugged stage on benign and on trained-like inputs, and the trained-like inputs must push
   it outside the bound.  Two other candidates stay inside the bound on these weights, so they have no test here:
     * var = E[x^2] - E[x]^2 in fp32 (block 6 norm1 of ViT-S: 0.999 benign, 0.9996 trained-like).  It cancels only when a
       row's mean is large next to its spread; two massive channels of the same sign give mean^2 / var = 2 / D.
     * the softmax max taken over the first 64 of 192 keys (last block of ViT-S: 0.60 benign, 0.98 trained-like).
       exp(s - max) is shift-invariant; the slip shows only when a later key lies more than 88.7 above the first tile's max.
"""
import math

import numpy as np
import pytest
import torch

from oracle import stage_ref as S
from oracle import trained_like as T
from oracle import vitpose_oracle as O
from test_gelu_fit import _coefficients

SEED = 71
_cache = {}


def _chain(size, depth, benign=False):
    """Per block: the stream into the block, norm1 output, qkv, norm2 output and the fc1 pre-activation z (fp64), each
    stage fed the engine-rounded output of the one before (S.chained_forward, intermediates kept)."""
    key = (size, depth, benign)
    if key not in _cache:
        D, _, heads = O.MODEL_DIMS[size]
        sd = (O.make_state_dict(D, depth, 17, SEED, peaky=0.1, bumps=True) if benign
              else T.trained_like_state_dict(size, depth, 17, SEED))
        blocks = []
        with torch.no_grad():
            x = S.patch_embed(S.patch_rows(O.make_crops(1, 808)), sd)[0].float().double()
            for i in range(depth):
                xn1 = S.bf16(S.block_norm(x, sd, i, 1)[0].float())
                qkv = S.bf16(S.qkv(xn1, sd, i, heads)[0].float())
                a = S.bf16(S.attention(qkv, heads)[0].float())
                x_mid = S.proj(a, x, sd, i)[0].float().double()
                xn2 = S.bf16(S.block_norm(x_mid, sd, i, 2)[0].float())
                w, b = S.linear_weights(sd, f"backbone.blocks.{i}.mlp.fc1", xn2.device)
                z = xn2 @ w.T + b
                blocks.append(dict(x=x, xn1=xn1, qkv=qkv, x_mid=x_mid, xn2=xn2, z=z))
                x = S.fc2(S.bf16(S.gelu_erf(z).float()), x_mid, sd, i)[0].float().double()
        _cache[key] = sd, heads, blocks
    return _cache[key]


def _logits(qkv, heads):
    D = qkv.shape[1] // 3
    t = qkv.reshape(-1, 192, 3, heads, D // heads)
    return torch.einsum("bqhd,bkhd->bhqk", t[:, :, 0], t[:, :, 1])


@pytest.mark.parametrize("size,depth", [("s", 12), ("b", 4)])
def test_planted_statistics_are_present(size, depth):
    sd, heads, blocks = _chain(size, depth)
    mass, _, sink_tok = T.channels(size, SEED)
    tag = f"vit-{size} depth {depth}"
    sink_heads, tail, z_max = 0, [], 0.0
    for i, bl in enumerate(blocks):
        x = bl["x"]
        med = x.abs().median(-1).values
        m = x[:, mass].abs()
        ratio = float((m.min(-1).values / med).median())
        s = _logits(bl["qkv"], heads)[0]
        w = torch.softmax(s, -1)
        sink_w = w[:, :, sink_tok].sum(-1).median(-1).values            # per head: the median query's weight on the sinks
        z = bl["z"]
        frac = float((z.abs() > 8).double().mean())
        print(f"{tag} block {i}: massive channels {float(m.min()):.0f}..{float(m.max()):.0f}, {ratio:.0f} x the row median; "
              f"sink weight of the median query >= 0.5 in {int((sink_w >= 0.5).sum())}/{heads} heads; "
              f"logit std {float(s.std()):.1f}, max |logit| {float(s.abs().max()):.1f}; "
              f"fc1 |z| > 8: {frac:.2%}, max |z| {float(z.abs().max()):.1f}")
        if i > T.MASSIVE_BLOCK:                                          # block 1's fc2 plants them
            assert float(m.min()) > 0.8 * T.MASSIVE[size] and ratio > 100, f"{tag} block {i}: massive channels"
        assert int((sink_w >= 0.5).sum()) > heads // 2, f"{tag} block {i}: sinks in too few heads"
        assert 4.0 < float(s.std()) < 9.0, f"{tag} block {i}: logit std"
        assert float(s.abs().max()) >= 25, f"{tag} block {i}: max |logit|"
        sink_heads += int((sink_w >= 0.5).sum())
        tail.append(frac)
        z_max = max(z_max, float(z.abs().max()))
    print(f"{tag}: sink weight of the median query >= 0.5 in {sink_heads}/{heads * depth} heads")
    assert sink_heads >= 0.75 * heads * depth
    assert min(tail) >= 0.005 and z_max >= 20, f"{tag}: GELU tail {min(tail):.2%}, max |z| {z_max:.1f}"


def test_planted_gammas():
    sd = T.trained_like_state_dict("s", 2, 17, SEED)
    mass, sink_ch, _ = T.channels("s", SEED)
    for name in ("backbone.blocks.0.norm1.weight", "backbone.blocks.1.norm2.weight", "backbone.last_norm.weight"):
        g = sd[name]
        assert np.all(g[mass] == np.float32(0.01))
        other = np.delete(g, np.concatenate([mass, sink_ch]))
        assert other.min() >= 0.01 and other.max() <= 5.0 and other.min() < 0.05 and other.max() > 3.0, name


def test_weights_are_deterministic():
    a, b = T.trained_like_state_dict("s", 2, 17, 5), T.trained_like_state_dict("s", 2, 17, 5)
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


# ------------------------------------------------------------------------------------------------ mutations
def _ratios(name, fn):
    """fn(benign) -> (good, bad, ref, bound): print both worst ratios for benign and trained-like inputs."""
    out = {}
    for benign in (True, False):
        good, bad, ref, bound = fn(benign)
        out[benign] = (S.worst_ratio(good, ref, bound), S.worst_ratio(bad, ref, bound))
    print(f"{name}: correct {out[True][0]:.3f} / {out[False][0]:.3f}, bugged {out[True][1]:.3g} on benign weights, "
          f"{out[False][1]:.3g} on trained-like weights")
    assert out[True][0] <= 1.0 and out[False][0] <= 1.0
    return out[True][1], out[False][1]


def _gelu_fit(z, clamp):
    (c2, c1, c0), _ = _coefficients()
    x = z.float().numpy()
    x2 = np.minimum(x * x, np.float32(clamp))
    p = (c2 * x2 + c1).astype(np.float32)
    p = (p * x2 + c0).astype(np.float32)
    t = np.tanh((x * p).astype(np.float32)).astype(np.float32)
    hx = np.float32(0.5) * x
    return S.bf16(torch.from_numpy((hx * t + hx).astype(np.float32)))


def test_gelu_without_clamp_is_caught():
    """fc1's fitted GELU without the x^2 <= 64 clamp: the polynomial turns over near |x| = 11."""
    def case(benign):
        sd, _, blocks = _chain("s", 12, benign)
        i = 5
        ref, bound = S.fc1(blocks[i]["xn2"], sd, i)
        z = blocks[i]["z"]
        return _gelu_fit(z, 64.0), _gelu_fit(z, math.inf), ref, bound
    benign, trained = _ratios("GELU fit without the clamp", case)
    assert trained > 1.0
