"""-m gpu: every engine stage against its fp64 reference (oracle/stage_ref.py) on weights with the activation statistics of
trained checkpoints (oracle/trained_like.py): massive residual channels with tiny LayerNorm gammas, sink tokens that take
most of the softmax weight, logit std ~6 in every block and fc1 inputs beyond the GELU fit's +-8.

The machinery is that of tests/test_gpu_stages.py: set_option("stop_after", s) ends a forward after stage s and
read_buffer copies the activations out, so each stage is checked on exactly the input the engine gave it, against the
bounds of stage_ref, unchanged.  Block i of a depth-d engine is fed from a depth-i engine built from the same weights
whose last norm is block i's norm1.  Every check prints its worst error / bound.

The bit-identity tests hold the engine's other paths -- the fused qkv + attention launch, forced GEMM tile widths, captured
and replayed graphs, flip test -- bit-identical, on these weights, to the eager separate-launch path the stage checks cover.
"""
import numpy as np
import pytest
import torch

from oracle import stage_ref as S
from oracle import trained_like as T
from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

# (embed_dim, depth, heads); ViT-H at reduced depth (the kernels are per layer, the depth only repeats them)
DIMS = {"s": (384, 12, 12), "b": (768, 12, 12), "l": (1024, 24, 16), "h": (1280, 8, 16)}
MAX_CROPS = {"s": 64, "b": 64, "l": 64, "h": 32}      # pick_tile chooses other tile widths there than at 1 and 5 crops
SEED = 71
FUSED, SEPARATE = 2, 4                               # vpb_debug_attention bits: force the fused / the two-launch form
_cache = {}


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need an H100"
    return torch.device("cuda", 0)


def _state_dict(size):
    key = ("sd", size)
    if key not in _cache:                                     # kept for every size: the calibration forward takes seconds
        D, depth, heads = DIMS[size]
        _cache[key] = T.trained_like_state_dict(size, depth, 17, SEED)
    return _cache[key]


def _engine(size, sd, depth, max_batch, last_norm_of=None):
    """depth-`depth` engine; with last_norm_of = i its last norm is block i's norm1, so its stage-10 output is the norm1
    output block i computes from the same stream."""
    from easy_vitpose_b200 import ViTPose, model_cfg
    sd = dict(sd)
    if last_norm_of is not None:
        sd["backbone.last_norm.weight"] = sd[f"backbone.blocks.{last_norm_of}.norm1.weight"]
        sd["backbone.last_norm.bias"] = sd[f"backbone.blocks.{last_norm_of}.norm1.bias"]
    cfg = model_cfg(size, 17)
    cfg["backbone"]["depth"] = depth
    m = ViTPose(cfg, max_batch=max_batch)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()
                       if not k.startswith("backbone.blocks.") or int(k.split(".")[2]) < depth})
    return m.to("cuda:0")


def _cached_engine(size, depth, last_norm_of=None, max_batch=None):
    key = ("engine", size, depth, last_norm_of, max_batch or MAX_CROPS[size])
    if key not in _cache:
        for k in [k for k in _cache if k[0] == "engine" and k[1] != size]:     # one size at a time on the device
            del _cache[k]
        _cache[key] = _engine(size, _state_dict(size), depth, key[-1], last_norm_of)
    return _cache[key]


def _run(m, x, stop):
    """forward stopped after `stop` (0: the whole forward, heatmaps returned)."""
    try:
        m.set_option("stop_after", stop)
        out = m(x)
        torch.cuda.synchronize()
    finally:
        m.set_option("stop_after", 0)
    return out


def _buf(m, name, n):
    D = m.embed_dim
    shape = {"patch_rows": (n * 192, 768), "x": (n * 192, D), "xn": (n * 192, D), "qkv": (n * 192, 3 * D),
             "attn": (n * 192, D), "hid": (n * 192, 4 * D), "d1": (n, 32, 24, 256), "d2": (n, 64, 48, 256)}[name]
    return m.read_buffer(name, shape, "f32" if name == "x" else "bf16").to(_dev())


class Checks:
    """Collects worst error / bound ratios, prints each, fails at the end naming every stage outside its bound."""

    def __init__(self, tag):
        self.tag, self.bad = tag, []

    def __call__(self, stage, got, ref_bound):
        ref, bound = ref_bound
        assert got.shape == ref.shape, (stage, got.shape, ref.shape)
        r = S.worst_ratio(got, ref, bound)
        print(f"{self.tag} {stage}: worst error / bound {r:.3f}")
        if not r <= 1.0:
            self.bad.append(f"{stage} ({r:.2f})")

    def done(self):
        assert not self.bad, f"{self.tag}: outside the bound: {', '.join(self.bad)}"


def _check_block0_and_head(m, sd, heads, x, chk):
    n = x.shape[0]
    _run(m, x, 3)
    rows, x0, xn1 = _buf(m, "patch_rows", n), _buf(m, "x", n), _buf(m, "xn", n)
    assert torch.equal(rows.double(), S.patch_rows(x).to(_dev())), f"{chk.tag}: patch rows differ from the bf16 im2col"
    chk("patch embed", x0, S.patch_embed(rows, sd))
    chk("block 0 norm1", xn1, S.block_norm(x0, sd, 0, 1))
    _run(m, x, 7)
    qkv, attn, x1, xn2, hid = (_buf(m, k, n) for k in ("qkv", "attn", "x", "xn", "hid"))
    chk("block 0 qkv", qkv, S.qkv(xn1, sd, 0, heads))
    chk("block 0 attention", attn, S.attention(qkv, heads))
    chk("block 0 proj", x1, S.proj(attn, x0, sd, 0))
    chk("block 0 norm2", xn2, S.block_norm(x1, sd, 0, 2))
    chk("block 0 fc1", hid, S.fc1(xn2, sd, 0))
    _run(m, x, 8)
    chk("block 0 fc2", _buf(m, "x", n), S.fc2(hid, x1, sd, 0))


def _check_block(prev, m, sd, i, heads, x, chk):
    """Block i of engine m, fed from prev (depth i, last norm = block i's norm1).  m stopped after all blocks still holds
    block i's qkv, attention, norm2 output and hidden activations; the stream after its proj is not kept, so norm2 is
    checked against the reference stream (its error carried through the LayerNorm's slope) and the block's output against
    both residual GEMMs at once (as tests/test_gpu_stages.py does)."""
    n = x.shape[0]
    _run(prev, x, 10)
    x_in, xn1 = _buf(prev, "x", n), _buf(prev, "xn", n)
    _run(m, x, 9)
    qkv, attn, xn2, hid, x_out = (_buf(m, k, n) for k in ("qkv", "attn", "xn", "hid", "x"))
    chk(f"block {i} norm1", xn1, S.block_norm(x_in, sd, i, 1))
    chk(f"block {i} qkv", qkv, S.qkv(xn1, sd, i, heads))
    chk(f"block {i} attention", attn, S.attention(qkv, heads))
    x_mid, b_mid = S.proj(attn, x_in, sd, i)
    ref2, b2 = S.block_norm(x_mid, sd, i, 2)
    g = S.t64(sd[f"backbone.blocks.{i}.norm2.weight"], x_mid.device)
    xc = x_mid - x_mid.mean(-1, keepdim=True)
    rstd = ((xc * xc).mean(-1, keepdim=True) + S.LN_EPS).rsqrt()
    e = b_mid.amax(-1, keepdim=True)
    chk(f"block {i} norm2", xn2, (ref2, b2 + g.abs() * rstd * e * (2 + (xc * rstd).abs()) * 1.01))
    chk(f"block {i} fc1", hid, S.fc1(xn2, sd, i))
    ref_out, b_out = S.fc2(hid, x_mid, sd, i)
    chk(f"block {i} proj + fc2", x_out, (ref_out, b_out + b_mid))


def _check_tail(m, sd, x, chk):
    """stage 10 from the stream after all blocks (stage 9), then deconv 1, deconv 2 and the heatmaps."""
    n = x.shape[0]
    heat = _run(m, x, 0)
    xs, xn, d1, d2 = (_buf(m, k, n) for k in ("x", "xn", "d1", "d2"))
    chk("last norm", xn, S.last_norm(xs, sd))
    chk("deconv1", d1, S.deconv(xn, sd, 0))
    chk("deconv2", d2, S.deconv(d1, sd, 1))
    chk("heatmaps", heat, S.final_layer(d2, sd))


@pytest.mark.parametrize("size,n", [(s, n) for s in DIMS for n in (1, 5, MAX_CROPS[s])])
def test_trained_like_stages_against_fp64(size, n):
    """Patch embed, block 0 stage by stage, the middle block, the last block, last norm, both deconvs and the heatmaps."""
    D, depth, heads = DIMS[size]
    sd = _state_dict(size)
    mid = depth // 2
    full = _cached_engine(size, depth)
    x = torch.from_numpy(O.make_crops(n, 300 + n)).to(_dev())
    chk = Checks(f"trained-like vit-{size} {n} crops")
    with torch.no_grad():
        _check_block0_and_head(full, sd, heads, x, chk)
        _check_block(_cached_engine(size, mid, mid), _cached_engine(size, mid + 1), sd, mid, heads, x, chk)
        _check_block(_cached_engine(size, depth - 1, depth - 1), full, sd, depth - 1, heads, x, chk)
        _check_tail(full, sd, x, chk)
    chk.done()


@pytest.mark.parametrize("size", ["s", "b"])
def test_trained_like_every_block(size):
    """Every block of the depth at 5 crops: block i of a depth-(i+1) engine fed from a depth-i engine."""
    D, depth, heads = DIMS[size]
    sd = _state_dict(size)
    n = 5
    x = torch.from_numpy(O.make_crops(n, 600)).to(_dev())
    chk = Checks(f"trained-like vit-{size} every block")
    engines = {d: _engine(size, sd, d, n, d if d < depth else None) for d in range(1, depth + 1)}
    with torch.no_grad():
        _check_block0_and_head(engines[1], sd, heads, x, chk)
        for i in range(1, depth):
            _check_block(engines[i], engines[i + 1], sd, i, heads, x, chk)
    del engines
    chk.done()


# ------------------------------------------------------------------------------------------------ kernel edges
@pytest.mark.parametrize("size", list(DIMS))
def test_layernorm_kernel_on_massive_channel_rows(size):
    """vpb_layernorm on the engine's stream after the last block (every row holds the two massive channels), with the norm1
    gammas and betas of the middle and the last block (1e-2 on the massive channels, log-normal elsewhere)."""
    from gpu_util import layernorm
    D, depth, heads = DIMS[size]
    sd = _state_dict(size)
    m = _cached_engine(size, depth)
    n = MAX_CROPS[size]
    mass, _, _ = T.channels(size, SEED)
    with torch.no_grad():
        _run(m, torch.from_numpy(O.make_crops(n, 700)).to(_dev()), 9)
        xs = _buf(m, "x", n)
        print(f"vit-{size} stream after the last block: massive channels {float(xs[:, mass].abs().min()):.0f}.."
              f"{float(xs[:, mass].abs().max()):.0f}, median |x| {float(xs.abs().median()):.2f}")
        for i in (depth // 2, depth - 1):
            g = torch.from_numpy(sd[f"backbone.blocks.{i}.norm1.weight"]).to(_dev())
            b = torch.from_numpy(sd[f"backbone.blocks.{i}.norm1.bias"]).to(_dev())
            r = S.worst_ratio(layernorm(xs, g, b), *S.layernorm(xs, g, b))
            print(f"vit-{size} layernorm kernel, block {i} norm1 on massive-channel rows: worst error / bound {r:.3f}")
            assert r <= 1.0


@pytest.mark.parametrize("size", ["s", "b", "h"])           # head_dim 32, 64, 80
def test_attention_kernel_on_sink_block(size):
    """vpb_attention on the last block's qkv (sink tokens, sharp logits), all exponentials on the MUFU and every 4th as
    ex2_poly."""
    from easy_vitpose_b200 import _lib
    from gpu_util import attention
    D, depth, heads = DIMS[size]
    m = _cached_engine(size, depth)
    n = 5
    _, _, sink_tok = T.channels(size, SEED)
    with torch.no_grad():
        _run(m, torch.from_numpy(O.make_crops(n, 710)).to(_dev()), 9)
        qkv = _buf(m, "qkv", n)
        t = qkv.double().reshape(n, 192, 3, heads, D // heads)
        w = torch.softmax(torch.einsum("bqhd,bkhd->bhqk", t[:, :, 0], t[:, :, 1]), -1)
        sink_w = w[..., sink_tok].sum(-1).median(-1).values
        print(f"vit-{size} last block: sink weight of the median query >= 0.5 in {int((sink_w >= 0.5).sum())}/{sink_w.numel()} "
              f"(crop, head) pairs")
        ref = S.attention(qkv, heads)
        try:
            for mode in (0, 1):
                _lib.lib().vpb_debug_attention(mode)
                r = S.worst_ratio(attention(qkv, n, heads, D // heads), *ref)
                print(f"vit-{size} attention kernel on the sink block, {'ex2_poly' if mode else 'mufu'}: worst error / bound {r:.3f}")
                assert r <= 1.0
        finally:
            _lib.lib().vpb_debug_attention(-1)


# ------------------------------------------------------------------------------------------------ bit identity
def _infer(m, x, org, attention_flags=SEPARATE, graph=0):
    from easy_vitpose_b200 import _lib
    try:
        _lib.lib().vpb_debug_attention(attention_flags)
        m.set_option("graph", graph)
        kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
        torch.cuda.synchronize()
        return [t.clone() for t in (kp, idx, hm)] + [m.read_buffer("attn", (x.shape[0] * 192, m.embed_dim), "bf16").clone()]
    finally:
        _lib.lib().vpb_debug_attention(-1)
        m.set_option("graph", 1)


def _same(a, b, what):
    for u, v, name in zip(a, b, ("keypoints", "argmax", "heatmaps", "attn")):
        u = u.view(torch.int16) if u.dtype == torch.bfloat16 else u
        v = v.view(torch.int16) if v.dtype == torch.bfloat16 else v
        assert torch.equal(u.to(v.device), v), f"{name} differ: {what}"


def _inputs(n, seed):
    x = torch.from_numpy(O.make_crops(n, seed)).to(_dev())
    org = torch.from_numpy(np.random.RandomState(seed).randint(64, 513, size=(n, 2)).astype(np.int32))
    return x, org


@pytest.mark.parametrize("size", ["b", "l"])
def test_trained_like_fused_tiles_and_graphs_bit_identical(size):
    """At 64 crops, against the eager two-launch qkv + attention path: the fused launch, the engine's own choice, forced
    128/192/256-wide GEMM tiles (those that divide D), and graph calls (eager, capture, replay)."""
    from easy_vitpose_b200 import _lib
    m = _cached_engine(size, DIMS[size][1])
    x, org = _inputs(64, 31)
    ref = _infer(m, x, org, SEPARATE)
    _same(_infer(m, x, org, FUSED), ref, f"vit-{size} fused")
    _same(_infer(m, x, org, 0), ref, f"vit-{size} engine's choice")
    try:
        for width in [w for w in (128, 192, 256) if DIMS[size][0] % w == 0]:     # ViT-L: N = 1024 has no 192-wide tiles
            _lib.lib().vpb_debug_gemm((width << 8) << 8, None)
            m.set_option("chain", 0)                            # drops the captured graphs: they embed the tile choice
            _same(_infer(m, x, org, SEPARATE), ref, f"vit-{size} GEMM tiles {width} wide")
    finally:
        _lib.lib().vpb_debug_gemm(0, None)
        m.set_option("chain", 0)
    for call in ("eager", "capture", "replay"):
        _same(_infer(m, x, org, SEPARATE, graph=1), ref, f"vit-{size} graph call: {call}")
    print(f"vit-{size} trained-like: fused, engine's choice, tile widths 128/192/256 and graph calls bit-identical")


def test_trained_like_flip_test_equals_composition():
    """Flip test on: the keypoint call equals forward_flip_test + decode_heatmaps bit for bit (eager, capture, replay)."""
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, decode_heatmaps
    m = _cached_engine("s", DIMS["s"][1])
    pairs = [tuple(p) for p in COCO_FLIP_PAIRS]
    try:
        for shift in (False, True):
            m.set_flip_test(pairs, shift)
            for n in (1, 7, 32):
                x, org = _inputs(n, 50 + n)
                hm_r = m.forward_flip_test(x, pairs, shift)
                kp_r, idx_r = decode_heatmaps(hm_r, org)
                for call in range(3):                           # graph on: eager, capture, replay
                    if call == 1:                               # the averaged maps stay inside the engine (in place)
                        kp, idx = m.infer_crops(x, org)
                    else:
                        kp, idx, hm = m.infer_crops(x, org, return_heatmaps=True)
                        assert torch.equal(hm, hm_r), (shift, n, call)
                    assert torch.equal(kp, kp_r) and torch.equal(idx, idx_r), (shift, n, call)
    finally:
        m.set_flip_test(None)
