"""Seeded ViTPose weights with the activation statistics reported for trained ViT checkpoints  --  TEST INFRASTRUCTURE ONLY.

make_state_dict (oracle/vitpose_oracle.py) gives benign weights: a unit-scale residual stream, LayerNorm gammas near 1,
near-uniform softmax rows (logit std ~0.0016 D) and fc1 pre-activations inside [-8, 8].  Bugs in the LayerNorm, the
softmax and the GELU clamp are muted there.  The literature on massive activations and on register / high-norm tokens
reports four features of trained ViTs, large ones most of all; trained_like_state_dict plants each of them on top of
make_state_dict(..., peaky=0.1, bumps=True):

  * Massive residual channels.  Two stream channels (same sign) get a large fc2 bias in block 1, so from block 1's
    output on they sit at about MASSIVE[size] on every token (3e2 at ViT-S/B, 1e3 at ViT-L/H) and keep that size through
    the remaining blocks.  Their norm1 / norm2 / last_norm gammas are 1e-2; every other gamma is log-normal (median 0.5, sigma 1.2 in
    log space) clipped to [1e-2, 5].
  * Sink tokens.  Two token positions at or after 64 (in the second and third 64-key tile of a softmax row) get a
    pos_embed component of SINK_FRAC * MASSIVE on four channels.  Those channels keep gamma 1 in norm1, so the sink rows'
    normalised values are large there and small on every other token.  No k row reads those channels except one per head:
    its weight on the four is g, and the matching q row is the constant bias beta (twice the head's q rms), so every query
    gives each sink the same logit boost.  g is set by bisection so that the median query of each head gives the two sinks
    SINK_WEIGHT of its softmax weight on the calibration crop; on other crops the weight varies from head to head.
  * Sharp logits in every block.  The q rows of each block are scaled so that the logits over the ordinary keys have a
    standard deviation of LOGIT_STD.
  * GELU inputs beyond +-8.  The fc1 rows of each block are scaled so that GELU_TAIL of the pre-activations have |z| > 8
    (and the fc2 weights by the inverse, so the stream grows as with the benign weights), and eight fc1 biases per block
    are set to +-12, +-16, +-20 and +-24.

The scale factors are calibrated on a float64 forward of one make_crops crop, block by block, and rounded to three
significant digits, so the weights are a pure function of (size, depth, K, seed).

Measured by tests/test_trained_like_cpu.py on the engine-rounded stage references (ViT-S at depth 12, ViT-B at depth 4,
one crop of another seed), per block:
  ViT-S  massive channels 297-304 from block 2 on, 334-358 x the median |x| of a row; median-query sink weight >= 0.5 in
         129 of 144 heads (8 to 12 of 12 per block); logit std 6.0-7.4, max |logit| 45-129; 1.4-1.6 % of fc1 inputs
         beyond |z| = 8, max |z| 29-106.
  ViT-B  massive channels 295-307, 229-234 x the median; sink weight >= 0.5 in 45 of 48 heads; logit std 6.1-6.5, max
         |logit| 32-69; 1.2-1.3 % beyond 8, max |z| 31-59.
On the GPU, after the last block of the test engines: massive channels 293-309 (ViT-S/B) and 990-1010 (ViT-L/H).
The LayerNorm E[x^2] - E[x]^2 variance stays inside its bound on these weights: two massive channels of the same sign
give mean^2 / var = 2 / D, far from the cancelling regime.  No statistic was changed to expose it.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import vitpose_oracle as O

MASSIVE = {"s": 300.0, "b": 300.0, "l": 1000.0, "h": 1000.0}
MASSIVE_BLOCK = 1
SINK_FRAC = 0.5
SINK_WEIGHT = 0.9
LOGIT_STD = 6.0
GELU_TAIL = 0.01
GELU_BIASES = np.array([12, -12, 16, -16, 20, -20, 24, -24], np.float32)


def _round3(v: float) -> float:
    """three significant digits: the calibrated factors do not depend on the last bits of the BLAS used"""
    return float(f"{v:.3g}")


def _ln(x, g, b):
    c = x - x.mean(-1, keepdims=True)
    return c / np.sqrt((c * c).mean(-1, keepdims=True) + O.LN_EPS) * g + b


def _gelu(z):
    return 0.5 * z * (1.0 + O._erf(z / math.sqrt(2.0)))


def _softmax(s):
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def channels(size: str, seed: int):
    """(massive channels, sink channels, sink tokens) of trained_like_state_dict(size, ..., seed)."""
    D = O.MODEL_DIMS[size][0]
    rs = np.random.RandomState(seed + 7919)
    ch = rs.choice(np.arange(256, D), size=6, replace=False)        # clear of the bump pathway's channels (< K <= 256)
    tok = rs.choice(np.arange(64, O.TOKENS), size=2, replace=False)
    return np.sort(ch[:2]), np.sort(ch[2:]), np.sort(tok)


def _gammas(rs, D):
    return np.clip(np.exp(rs.standard_normal(D) * 1.2 + math.log(0.5)), 1e-2, 5.0).astype(np.float32)


def trained_like_state_dict(size: str, depth: int, K: int, seed: int) -> dict[str, np.ndarray]:
    D, _, heads = O.MODEL_DIMS[size]
    hd = D // heads
    sd = O.make_state_dict(D, depth, K, seed, peaky=0.1, bumps=True)
    sd = {k: np.array(v) for k, v in sd.items()}
    rs = np.random.RandomState(seed + 104729)
    mass, sink_ch, sink_tok = channels(size, seed)
    A = MASSIVE[size]
    sd["backbone.pos_embed"][0, 1 + sink_tok[:, None], sink_ch[None, :]] += np.float32(SINK_FRAC * A)
    for name in [f"backbone.blocks.{i}.norm{w}.weight" for i in range(depth) for w in (1, 2)] + ["backbone.last_norm.weight"]:
        g = _gammas(rs, D)
        g[mass] = 0.01
        if ".norm1." in name:
            g[sink_ch] = 1.0
        sd[name] = g
    sd[f"backbone.blocks.{min(MASSIVE_BLOCK, depth - 1)}.mlp.fc2.bias"][mass] += np.float32(A)

    # calibration forward, float64, one crop
    x = O.patch_rows(O.make_crops(1, seed))[0].astype(np.float64) @ sd["backbone.patch_embed.proj.weight"].reshape(D, -1).T.astype(np.float64)
    pos = sd["backbone.pos_embed"][0].astype(np.float64)
    x += pos[1:] + pos[:1] + sd["backbone.patch_embed.proj.bias"]
    ordinary = np.setdiff1d(np.arange(O.TOKENS), sink_tok)
    for i in range(depth):
        p = f"backbone.blocks.{i}."
        f64 = lambda k: sd[p + k].astype(np.float64)
        xn = _ln(x, f64("norm1.weight"), f64("norm1.bias"))
        W, b = sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]
        W[D:2 * D, sink_ch] = 0.0                                    # the sink channels reach k through the sink row only
        q = (xn @ W[:D].T.astype(np.float64) + b[:D]).reshape(-1, heads, hd).transpose(1, 0, 2)
        k = (xn @ W[D:2 * D].T.astype(np.float64) + b[D:2 * D]).reshape(-1, heads, hd).transpose(1, 0, 2)
        s = q @ k[:, ordinary].transpose(0, 2, 1) / math.sqrt(hd)
        f = np.float32(_round3(LOGIT_STD / float(s.std())))
        W[:D] *= f
        b[:D] *= f
        q *= float(f)
        u = xn[:, sink_ch].sum(-1)                                   # what the sink k row reads
        for h in range(heads):
            r = h * hd                                               # the head's first dimension carries the sink
            beta = np.float32(_round3(2.0 * float(np.sqrt((q[h] ** 2).mean()))))
            W[r] = 0.0                                               # every query has q[r] = beta
            b[r] = beta
            q[h, :, 0] = float(beta)

            def median_sink_weight(g):
                kk = k[h].copy()
                kk[:, 0] += g * u
                w = _softmax(q[h] @ kk.T / math.sqrt(hd))
                return float(np.median(w[:, sink_tok].sum(-1)))
            lo, hi = 0.0, 1.0
            while median_sink_weight(hi) < SINK_WEIGHT:
                hi *= 2.0
            for _ in range(30):
                mid = 0.5 * (lo + hi)
                lo, hi = (mid, hi) if median_sink_weight(mid) < SINK_WEIGHT else (lo, mid)
            g = np.float32(_round3(hi))
            W[D + r, sink_ch] += g
        qkv = xn @ W.T.astype(np.float64) + b
        t = qkv.reshape(-1, 3, heads, hd).transpose(1, 2, 0, 3)
        o = _softmax(t[0] @ t[1].transpose(0, 2, 1) / math.sqrt(hd)) @ t[2]
        x = x + o.transpose(1, 0, 2).reshape(-1, D) @ f64("attn.proj.weight").T + f64("attn.proj.bias")
        xn = _ln(x, f64("norm2.weight"), f64("norm2.bias"))
        W1, b1 = sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]
        z = xn @ W1.T.astype(np.float64) + b1
        f = np.float32(_round3(8.0 / float(np.quantile(np.abs(z), 1.0 - GELU_TAIL))))
        W1 *= f
        b1 *= f
        sd[p + "mlp.fc2.weight"] /= f
        b1[rs.choice(4 * D, size=len(GELU_BIASES), replace=False)] = GELU_BIASES
        z = xn @ W1.T.astype(np.float64) + b1
        x = x + _gelu(z) @ f64("mlp.fc2.weight").T + f64("mlp.fc2.bias")
    return sd
