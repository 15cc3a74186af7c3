"""The simple decoder (relu -> 4x bilinear upsample -> 3x3 conv) without a GPU: the fp64 oracle against F.interpolate / F.conv2d
and against the reference's own head, the teeth of the per-element bound tests/test_gpu_simple_head.py uses, config
validation, the strict state-dict contract and decoder detection."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ref_import
from oracle import simple_head_oracle as S
from oracle import vitpose_oracle as O

F64 = torch.float64
GOLDEN_SEEDS = {"base": (768, 12, 17, 112), "large": (1024, 24, 17, 113), "huge": (1280, 32, 17, 114)}


def _simple_head_dict(K=17, D=768, **kw):
    hd = dict(type="TopdownHeatmapSimpleHead", in_channels=D, num_deconv_layers=0, num_deconv_filters=[], num_deconv_kernels=[],
              upsample=4, extra=dict(final_conv_kernel=3), out_channels=K)
    hd.update(kw)
    return hd


@pytest.mark.parametrize("n_out,n_in", [(64, 16), (48, 12)])
def test_bilinear_table_equals_interpolate(n_out, n_in):
    x = torch.eye(n_in, dtype=F64).view(1, n_in, n_in, 1)          # channel i = the unit impulse at source row i
    y = F.interpolate(x, scale_factor=(4, 1), mode="bilinear", align_corners=False)[0, :, :, 0].T.numpy()
    assert np.array_equal(S.bilinear_matrix(n_out, n_in), y)
    T = np.zeros((n_out, n_in))
    for o, (i0, i1, w0, w1) in enumerate(S.tap_table(n_out, n_in)):
        T[o, i0] += w0
        T[o, i1] += w1
    assert np.array_equal(T, y)                                       # every row, edges (0, 1, n-2, n-1) included


@pytest.mark.parametrize("D", [384, 768, 1024, 1280])
@pytest.mark.parametrize("K", [1, 17, 133, 144])
def test_tap_form_equals_upsample_then_conv(D, K):
    g = torch.Generator().manual_seed(D * 1000 + K)
    f = torch.randn(2, D, 16, 12, generator=g, dtype=F64)
    w = torch.randn(K, D, 3, 3, generator=g, dtype=F64) / np.sqrt(9 * D)
    b = torch.randn(K, generator=g, dtype=F64)
    d, t = S.direct(f, w, b), S.taps(f, w, b)
    assert (d - t).abs().max().item() <= 1e-12 * max(1.0, d.abs().max().item())


@pytest.mark.skipif(not ref_import.available(), reason="reference tree absent")
@pytest.mark.parametrize("size", sorted(GOLDEN_SEEDS))
def test_oracle_equals_reference_head_fp32(size):
    import types

    from oracle.make_golden_simple import config_model, upstream_transform_inputs
    ref = ref_import.load()
    cfg = config_model(size)
    D, depth, K, wseed = GOLDEN_SEEDS[size]
    assert (cfg["backbone"]["embed_dim"], cfg["backbone"]["depth"], cfg["keypoint_head"]["out_channels"]) == (D, depth, K)
    head_cfg = {k: v for k, v in cfg["keypoint_head"].items() if k not in ("type", "loss_keypoint")}
    head = ref.ViTPose(dict(cfg, backbone=dict(cfg["backbone"], depth=1))).keypoint_head.eval()
    head._transform_inputs = types.MethodType(upstream_transform_inputs, head)
    sd = S.make_state_dict(D, depth, K, wseed, peaky=0.1, bumps=True)
    w, b = torch.from_numpy(sd["keypoint_head.final_layer.weight"]), torch.from_numpy(sd["keypoint_head.final_layer.bias"])
    head.final_layer.weight.data.copy_(w)
    head.final_layer.bias.data.copy_(b)
    assert head_cfg["upsample"] == 4 and head_cfg["extra"]["final_conv_kernel"] == 3
    f = torch.randn(2, D, 16, 12, generator=torch.Generator().manual_seed(wseed))
    with torch.no_grad():
        got = head(f).to(F64)
    want = S.direct(f, w, b)
    assert (got - want).abs().max().item() < 1e-5 * want.abs().max().item()


def _kernel_like_fp32(f, w, b):
    """The kernel's arithmetic in fp32: Y by an fp32 matmul over D, then the stencil in fp32 (the bound's positive control)."""
    Y = torch.einsum("bchw,kct->btkhw", torch.relu(f).float(), w.float().flatten(2))
    return S.stencil(Y.double(), None).float().double() + b.double().view(1, -1, 1, 1)


@pytest.mark.parametrize("mutant", S.MUTANTS)
def test_bound_rejects_mutants(mutant):
    g = torch.Generator().manual_seed(5)
    D, K = 768, 17
    f = torch.randn(2, D, 16, 12, generator=g).bfloat16().to(F64)
    w = (torch.randn(K, D, 3, 3, generator=g) / np.sqrt(9 * D)).bfloat16().to(F64)
    b = (torch.randn(K, generator=g) * 0.01).to(F64)
    ref, bound = S.bound(f, w, b)
    assert ((_kernel_like_fp32(f, w, b) - ref).abs() / bound).max().item() <= 1.0
    assert ((S.mutant(mutant, f, w, b) - ref).abs() / bound).max().item() > 10.0


@pytest.mark.parametrize("size,name", [("b", "base"), ("l", "large"), ("h", "huge")])
def test_reference_simple_configs_are_accepted(size, name):
    from easy_vitpose_b200.configs import model_cfg
    from easy_vitpose_b200.model import ViTPose, head_decoder
    ours = model_cfg(size, 17, decoder="simple")
    assert head_decoder(ours["keypoint_head"]) == "simple"
    assert ViTPose(ours).decoder == "simple"
    if ref_import.available():
        from oracle.make_golden_simple import config_model
        cfg = config_model(name)
        assert ViTPose(cfg).decoder == "simple"
        theirs = {k: v for k, v in cfg["keypoint_head"].items() if k != "loss_keypoint"}
        assert {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in ours["keypoint_head"].items()} == \
            {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in theirs.items()}
    assert ViTPose(model_cfg(size, 17)).decoder == "classic"


@pytest.mark.parametrize("change", [dict(upsample=2), dict(upsample=0), dict(extra=dict(final_conv_kernel=1)),
                                    dict(extra=dict(final_conv_kernel=0)), dict(extra=dict(final_conv_kernel=3, num_conv_layers=1)),
                                    dict(extra=dict(final_conv_kernel=3, num_conv_layers=0)), dict(align_corners=True),
                                    dict(num_deconv_layers=1, num_deconv_filters=[256], num_deconv_kernels=[4]),
                                    dict(num_deconv_filters=[256])])
def test_other_heads_are_rejected(change):
    from easy_vitpose_b200.configs import model_cfg
    from easy_vitpose_b200.model import ViTPose
    cfg = model_cfg("b", 17, decoder="simple")
    cfg["keypoint_head"].update(change)
    with pytest.raises(ValueError):
        ViTPose(cfg)


def test_explicit_align_corners_false_is_accepted():
    from easy_vitpose_b200.configs import model_cfg
    from easy_vitpose_b200.model import ViTPose
    cfg = model_cfg("s", 17, decoder="simple")
    cfg["keypoint_head"]["align_corners"] = False
    assert ViTPose(cfg).decoder == "simple"


def test_strict_state_dict_contract():
    from easy_vitpose_b200.configs import model_cfg
    from easy_vitpose_b200.model import ViTPose, _expected_shapes
    D, depth, K = 384, 12, 17
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in S.make_state_dict(D, depth, K, 3).items()}
    assert set(sd) == set(_expected_shapes(D, depth, K, decoder="simple"))
    assert tuple(sd["keypoint_head.final_layer.weight"].shape) == (K, D, 3, 3)
    m = ViTPose(model_cfg("s", K, decoder="simple"))
    m.load_state_dict(sd)                                             # no device: nothing is uploaded yet
    classic = {k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(D, depth, K, 3).items()}
    with pytest.raises(RuntimeError, match="unexpected keys.*deconv_layers"):
        ViTPose(model_cfg("s", K, decoder="simple")).load_state_dict({**sd, **{k: v for k, v in classic.items() if "deconv" in k}})
    missing = {k: v for k, v in sd.items() if not k.startswith("keypoint_head.final_layer.weight")}
    with pytest.raises(RuntimeError, match="missing keys.*final_layer.weight"):
        ViTPose(model_cfg("s", K, decoder="simple")).load_state_dict(missing)
    with pytest.raises(RuntimeError, match="size mismatch"):
        ViTPose(model_cfg("s", K)).load_state_dict({**classic, "keypoint_head.final_layer.weight": sd["keypoint_head.final_layer.weight"]})
    with pytest.raises(RuntimeError):
        ViTPose(model_cfg("s", K)).load_state_dict(sd)               # a classic engine reports the missing deconvs


def test_decoder_detection_and_unwrap():
    from easy_vitpose_b200.model import state_dict_decoder
    simple = S.make_state_dict(384, 1, 17, 3)
    classic = O.make_state_dict(384, 1, 17, 3)
    assert state_dict_decoder(simple) == "simple" and state_dict_decoder({"state_dict": simple}) == "simple"
    assert state_dict_decoder(classic) == "classic" and state_dict_decoder({"state_dict": classic}) == "classic"


def test_multi_head_simple_keys_and_split():
    from easy_vitpose_b200.model import _expected_shapes, split_vitpose_plus
    s = _expected_shapes(384, 1, 17, head_keypoints=[17, 133], decoder="simple")
    heads = [k for k in s if "head" in k]
    assert heads == ["keypoint_head.final_layer.weight", "keypoint_head.final_layer.bias",
                     "associate_keypoint_heads.0.final_layer.weight", "associate_keypoint_heads.0.final_layer.bias"]
    assert s["associate_keypoint_heads.0.final_layer.weight"] == (133, 384, 3, 3)
    sd = {k: torch.zeros(v) for k, v in s.items()}
    parts = split_vitpose_plus(sd, names=["coco", "wholebody"], keypoints=[17, 133])
    assert tuple(parts["wholebody"]["keypoint_head.final_layer.weight"].shape) == (133, 384, 3, 3)
    assert not any("deconv" in k for p in parts.values() for k in p)


def test_model_cfg_and_dyn_model_import_pass_the_decoder():
    from easy_vitpose_b200.configs import dyn_model_import, model_cfg
    assert dyn_model_import("coco", "b", decoder="simple") == model_cfg("b", 17, decoder="simple")
    assert dyn_model_import("coco", "b") == model_cfg("b", 17)
    with pytest.raises(ValueError):
        model_cfg("b", 17, decoder="other")


def test_synthetic_simple_weights_have_the_contract_shapes():
    from easy_vitpose_b200.model import _expected_shapes
    from easy_vitpose_b200.synthetic import random_state_dict
    sd = random_state_dict("s", 17, decoder="simple")
    exp = {k: v for k, v in _expected_shapes(384, 12, 17, decoder="simple").items()}
    assert {k: tuple(v.shape) for k, v in sd.items()} == exp


def test_create_ex_is_exported():
    from easy_vitpose_b200 import _lib
    assert "vpb_create_ex" in _lib.EXPORTS and _lib.DECODERS == {"classic": 0, "simple": 1}
