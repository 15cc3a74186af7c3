"""-m gpu: every stage of the engine against its fp64 reference (oracle/stage_ref.py), fed from the engine's own buffers.

set_option("stop_after", s) ends a forward after stage s (engine.cu, above patch_gather) and read_buffer copies the
activations out, so each stage is checked on exactly the input the engine gave it: its error does not accumulate, and a
few bf16 ulps (the derived bounds of stage_ref) replace the 1 % of heatmap range the end-to-end tests can afford.  Every
check prints its worst error / bound ratio.

stop_after disables the CUDA graphs and the fused qkv + attention launch: the qkv and attention checked here are the two
separate launches.  tests/test_gpu_qkv_attention.py holds the fused launch bit-identical to them.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stage_ref as S
from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

# (embed_dim, depth, heads); ViT-H at reduced depth (the kernels are per layer, the depth only repeats them)
DIMS = {"s": (384, 12, 12), "b": (768, 12, 12), "l": (1024, 24, 16), "h": (1280, 8, 16)}
MAX_CROPS = {"s": 64, "b": 64, "l": 64, "h": 32}      # pick_tile chooses other tile widths there than at 1 and 5 crops
SEED = 71
_cache = {}


def _dev():
    assert torch.cuda.is_available(), "-m gpu tests need an H100"
    return torch.device("cuda", 0)


def _state_dict(size, sharp=False):
    key = ("sd", size, sharp)
    if key not in _cache:
        for k in [k for k in _cache if k[1] != size]:           # one size at a time on the device
            del _cache[k]
        D, depth, heads = DIMS[size]
        sd = O.make_state_dict(D, depth, 17, SEED, peaky=0.1, bumps=True)
        if sharp:
            # trained checkpoints reach block-0 logits of about +-30; the synthetic weights give near-uniform softmax rows
            # (logit std ~0.0016 D), where attention bugs are muted: scale the q rows to a logit std of ~6.5
            f = np.float32(6.5 / (0.0016 * D))
            for i in range(depth):
                p = f"backbone.blocks.{i}.attn.qkv."
                sd[p + "weight"] = sd[p + "weight"].copy()
                sd[p + "bias"] = sd[p + "bias"].copy()
                sd[p + "weight"][:D] *= f
                sd[p + "bias"][:D] *= f
        _cache[key] = sd
    return _cache[key]


def _engine(size, sd, depth, max_batch):
    from easy_vitpose_b200 import ViTPose, model_cfg
    cfg = model_cfg(size, 17)
    cfg["backbone"]["depth"] = depth
    m = ViTPose(cfg, max_batch=max_batch)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()
                       if not k.startswith("backbone.blocks.") or int(k.split(".")[2]) < depth})
    return m.to("cuda:0")


def _full_engine(size, sharp=False):
    key = ("engine", size, sharp)
    if key not in _cache:
        _cache[key] = _engine(size, _state_dict(size, sharp), DIMS[size][1], MAX_CROPS[size])
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
    want = S.patch_rows(x).to(_dev())
    assert torch.equal(rows.double(), want), f"{chk.tag}: patch rows differ from the bf16 im2col"
    print(f"{chk.tag} patch rows: bit-exact")
    chk("patch embed", x0, S.patch_embed(rows, sd))
    chk("norm1", xn1, S.block_norm(x0, sd, 0, 1))
    _run(m, x, 7)
    qkv, attn, x1, xn2, hid = (_buf(m, k, n) for k in ("qkv", "attn", "x", "xn", "hid"))
    chk("qkv", qkv, S.qkv(xn1, sd, 0, heads))
    chk("attention", attn, S.attention(qkv, heads))
    chk("proj", x1, S.proj(attn, x0, sd, 0))
    chk("norm2", xn2, S.block_norm(x1, sd, 0, 2))
    chk("fc1", hid, S.fc1(xn2, sd, 0))
    _run(m, x, 8)
    chk("fc2", _buf(m, "x", n), S.fc2(hid, x1, sd, 0))
    return qkv


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
def test_engine_stages_against_fp64(size, n):
    """Block 0 stage by stage, then last norm, the two deconvs and the 1x1 conv, at 1 crop, 5 (a ragged last 128-row
    block) and the largest batch."""
    D, depth, heads = DIMS[size]
    sd = _state_dict(size)
    m = _full_engine(size)
    x = torch.from_numpy(O.make_crops(n, 300 + n)).to(_dev())
    chk = Checks(f"vit-{size} {n} crops")
    with torch.no_grad():
        _check_block0_and_head(m, sd, heads, x, chk)
        _check_tail(m, sd, x, chk)
    chk.done()


@pytest.mark.parametrize("size", list(DIMS))
def test_engine_stages_sharp_attention(size):
    """q rows scaled so that block-0 logits reach about +-30 (trained-checkpoint softmax rows, far from uniform)."""
    D, depth, heads = DIMS[size]
    sd = _state_dict(size, sharp=True)
    m = _full_engine(size, sharp=True)
    x = torch.from_numpy(O.make_crops(5, 77)).to(_dev())
    chk = Checks(f"vit-{size} sharp")
    with torch.no_grad():
        qkv = _check_block0_and_head(m, sd, heads, x, chk)
    t = qkv.double().reshape(5, 192, 3, heads, D // heads)
    logits = torch.einsum("bqhd,bkhd->bhqk", t[:, :, 0], t[:, :, 1])
    print(f"vit-{size} sharp: block-0 logits in [{float(logits.min()):.1f}, {float(logits.max()):.1f}]")
    assert float(logits.abs().max()) > 20
    chk.done()


@pytest.mark.parametrize("size,d", [(s, d) for s in DIMS for d in (2, DIMS[s][1])])
def test_later_blocks_against_fp64(size, d):
    """Block d-1 of a depth-d engine, fed from a depth-(d-1) engine built from the same state dict: same kernels and shapes,
    so that engine's stream after its last block is bit for bit the input of block d-1.  The depth-(d-1) engine's last norm
    is loaded with block d-1's norm1, so its stage-10 output is the norm1 block d-1 computes.  The depth-d engine stopped
    after all blocks still holds block d-1's qkv, attention, norm2 output and hidden activations; the stream after its proj
    is not kept, so norm2 is checked against the reference stream (its error carried through the LayerNorm's slope) and
    the block's output against both residual GEMMs at once."""
    D, depth, heads = DIMS[size]
    sd = dict(_state_dict(size))
    n, i = 5, d - 1
    x = torch.from_numpy(O.make_crops(n, 500 + d)).to(_dev())
    chk = Checks(f"vit-{size} block {i}")
    prev_sd = dict(sd)
    prev_sd["backbone.last_norm.weight"] = sd[f"backbone.blocks.{i}.norm1.weight"]
    prev_sd["backbone.last_norm.bias"] = sd[f"backbone.blocks.{i}.norm1.bias"]
    with torch.no_grad():
        prev = _engine(size, prev_sd, i, n)
        _run(prev, x, 10)
        x_in, xn1 = _buf(prev, "x", n), _buf(prev, "xn", n)
        del prev
        m = _full_engine(size) if d == depth else _engine(size, sd, d, n)
        _run(m, x, 9)
        qkv, attn, xn2, hid, x_out = (_buf(m, k, n) for k in ("qkv", "attn", "xn", "hid", "x"))
        chk("norm1", xn1, S.block_norm(x_in, sd, i, 1))
        chk("qkv", qkv, S.qkv(xn1, sd, i, heads))
        chk("attention", attn, S.attention(qkv, heads))
        x_mid, b_mid = S.proj(attn, x_in, sd, i)
        ref2, b2 = S.block_norm(x_mid, sd, i, 2)
        g = S.t64(sd[f"backbone.blocks.{i}.norm2.weight"], x_mid.device)
        xc = x_mid - x_mid.mean(-1, keepdim=True)
        rstd = ((xc * xc).mean(-1, keepdim=True) + S.LN_EPS).rsqrt()
        e = b_mid.amax(-1, keepdim=True)                   # |stream error| after proj: shifts mean, centring and variance
        chk("norm2", xn2, (ref2, b2 + g.abs() * rstd * e * (2 + (xc * rstd).abs()) * 1.01))
        chk("fc1", hid, S.fc1(xn2, sd, i))
        ref_out, b_out = S.fc2(hid, x_mid, sd, i)
        chk("proj + fc2", x_out, (ref_out, b_out + b_mid))
    chk.done()


def test_multi_head_mixed_call_stages():
    """ViT-B with three heads (coco 17, ap10k 17, wholebody 133) and 192 expert rows, crops in interleaved runs of the
    heads: the stream after block 0 against each crop's own fc2 (shared rows + its head's expert, split_vitpose_plus),
    and each crop's deconvs and heatmaps against its head's layers."""
    from easy_vitpose_b200 import ViTPose, _lib, model_cfg, split_vitpose_plus
    from oracle.multi_head import plus_state_dict
    heads_kp = (("coco", 17), ("ap10k", 17), ("wholebody", 133))
    plus = plus_state_dict("b", [k for _, k in heads_kp], 192, 31)
    split = list(split_vitpose_plus({k: torch.from_numpy(np.asarray(v)) for k, v in plus.items()},
                                    [h for h, _ in heads_kp], [k for _, k in heads_kp]).values())
    m = ViTPose(model_cfg("b", 17), max_batch=16, heads=heads_kp, expert_rows=192).to("cuda:0")
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in plus.items()})
    m._ensure()
    segs = [(0, 2), (1, 3), (0, 1), (2, 2), (1, 1), (2, 1)]
    n, Km = sum(c for _, c in segs), m.num_keypoints_max
    x = torch.from_numpy(O.make_crops(n, 909)).to(_dev())
    org = torch.full((n, 2), 200, dtype=torch.int32, device=_dev())
    kp = torch.zeros((n, Km, 3), device=_dev())
    idx = torch.zeros((n, Km), dtype=torch.int32, device=_dev())
    hm = torch.zeros((n, Km, 64, 48), device=_dev())
    arr = (_lib.VpbSegment * len(segs))(*[_lib.VpbSegment(h, c) for h, c in segs])

    def run(stop):
        try:
            m.set_option("stop_after", stop)
            _lib.check(_lib.lib().vpb_infer_heads(m._handle, C.c_void_p(x.data_ptr()), C.c_void_p(org.data_ptr()), arr, len(segs),
                                                  C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(hm.data_ptr()), None))
            torch.cuda.synchronize()
        finally:
            m.set_option("stop_after", 0)

    chk = Checks("vit-b 3 heads")
    with torch.no_grad():
        run(7)
        x1, hid = _buf(m, "x", n), _buf(m, "hid", n)
        run(8)
        x2 = _buf(m, "x", n)
        run(0)
        xn, d1, d2 = _buf(m, "xn", n), _buf(m, "d1", n), _buf(m, "d2", n)
        c0 = 0
        for j, c in segs:
            r = slice(c0 * 192, (c0 + c) * 192)
            cs = slice(c0, c0 + c)
            name, K = heads_kp[j]
            prefix = "keypoint_head." if j == 0 else f"associate_keypoint_heads.{j - 1}."
            chk(f"crops {c0}..{c0 + c - 1} ({name}) fc2 + expert", x2[r], S.fc2(hid[r], x1[r], split[j], 0))
            chk(f"crops {c0}..{c0 + c - 1} ({name}) deconv1", d1[cs], S.deconv(xn[r], plus, 0, prefix))
            chk(f"crops {c0}..{c0 + c - 1} ({name}) deconv2", d2[cs], S.deconv(d1[cs], plus, 1, prefix))
            chk(f"crops {c0}..{c0 + c - 1} ({name}) heatmaps", hm[cs, :K], S.final_layer(d2[cs], plus, prefix))
            c0 += c
    chk.done()


# ------------------------------------------------------------------------------------------------ kernel-level edges
def _attention_case(case, hd, seed):
    """qkv [2*192, 3D] (q pre-scaled as the engine stores it) whose logits have the named shape."""
    heads = {32: 4, 64: 3, 80: 2}[hd]
    D, B = heads * hd, 2
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, 192, heads, hd, generator=g)
    k = torch.randn(B, 192, heads, hd, generator=g)
    v = torch.randn(B, 192, heads, hd, generator=g)
    star = torch.randint(0, 192, (B, heads), generator=g)         # the special key of every (crop, head)
    if case.startswith("std"):                                    # logit std 10 or 30
        q *= float(case[3:]) / hd ** 0.5
    elif case == "dominant":                                      # one key ~12 above a spread of +-1: weight ~0.999
        q[..., 0], k[..., 0] = 3.5, 0.0
        q[..., 1:] *= 0.5 / hd ** 0.5
        for b in range(B):
            for h in range(heads):
                k[b, star[b, h], h, 0] = 3.5
    elif case == "equal":                                         # every key the same vector: all logits of a row equal
        k = k[:, :1].expand_as(k).clone()
    elif case == "spike100":                                      # one key exactly 100 above all others (which are 0)
        q[:] = 0.0
        k[..., 0] = 0.0
        q[..., 0] = 10.0
        for b in range(B):
            for h in range(heads):
                k[b, star[b, h], h] = 0.0
                k[b, star[b, h], h, 0] = 10.0
    qkv = torch.stack([q, k, v], 2).reshape(B * 192, 3 * D)
    return qkv.bfloat16().to(_dev()), B, heads


@pytest.mark.parametrize("hd", [32, 64, 80])
@pytest.mark.parametrize("case", ["std10", "std30", "dominant", "equal", "spike100"])
def test_attention_kernel_logit_shapes(case, hd):
    """vpb_attention with all exponentials on the MUFU and with every 4th as ex2_poly, against the fp64 reference."""
    from easy_vitpose_b200 import _lib
    from gpu_util import attention
    qkv, B, heads = _attention_case(case, hd, {"std10": 1, "std30": 2, "dominant": 3, "equal": 4, "spike100": 5}[case] * 100 + hd)
    ref = S.attention(qkv, heads)
    try:
        for mode in (0, 1):
            _lib.lib().vpb_debug_attention(mode)
            out = attention(qkv, B, heads, hd)
            r = S.worst_ratio(out, *ref)
            print(f"attention {case} hd {hd} {'ex2_poly' if mode else 'mufu'}: worst error / bound {r:.3f}")
            assert r <= 1.0
    finally:
        _lib.lib().vpb_debug_attention(-1)


@pytest.mark.parametrize("D", [384, 768, 1024, 1280])
@pytest.mark.parametrize("case", ["constant", "offset1e4", "outlier"])
def test_layernorm_kernel_edge_rows(case, D):
    """vpb_layernorm on constant rows, rows offset by 1e4 and rows with one +-100 channel.  A constant row whose sum is exact
    in fp32 must give exactly bf16(beta): the kernel once took the mean as s * fl(1/D), an ulp off for D = 384, 768 and
    1280, and at variance 0 (rstd = 1000) a row of 1024.0 at D = 384 came out as beta - 0.12 gamma."""
    from gpu_util import layernorm
    g = torch.Generator().manual_seed(D + len(case))
    rows = 257
    x = torch.randn(rows, D, generator=g)
    gamma = 1 + 0.1 * torch.randn(D, generator=g)
    beta = 0.1 * torch.randn(D, generator=g)
    exact = None
    if case == "constant":                                        # variance 0: the output is beta
        consts = torch.tensor([0.0, 3.0, -0.5, 1024.0, 0.1, -7.3, 1e4, 1e-3])
        x = consts.repeat_interleave(-(-rows // len(consts)))[:rows, None].expand(rows, D).contiguous()
        exact = torch.isin(x[:, 0], torch.tensor([0.0, 3.0, -0.5, 1024.0]))   # sums exact in fp32: mean exact, output bf16(beta)
    elif case == "offset1e4":
        x = x + 1e4
    else:                                                         # one +-100 channel per row
        ch = torch.randint(0, D, (rows,), generator=g)
        x[torch.arange(rows), ch] = torch.where(torch.rand(rows, generator=g) < 0.5, -100.0, 100.0)
    dev = _dev()
    y = layernorm(x.to(dev), gamma.to(dev), beta.to(dev))
    r = S.worst_ratio(y, *S.layernorm(x.to(dev), gamma.to(dev), beta.to(dev)))
    print(f"layernorm {case} D {D}: worst error / bound {r:.3f}")
    assert r <= 1.0
    if exact is not None:
        assert torch.equal(y[exact.to(dev)].float(), beta.to(dev).bfloat16().float().expand(int(exact.sum()), D))
