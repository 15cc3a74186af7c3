"""CPU: the host side of the multi-head engine -- split_vitpose_plus / merge_split_state_dicts, the head grouping and its
inverse, the chunk planner on head groups, the ctypes mirror of vpb_segment and the Python argument checks."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import zlib

import numpy as np
import pytest
import torch

from easy_vitpose_b200 import VITPOSE_PLUS_HEADS, ViTPose, _lib, merge_split_state_dicts, model_cfg, split_vitpose_plus
from easy_vitpose_b200.model import _expected_shapes, _inverse, group_by_head, plan_frame_chunks
from oracle.multi_head import plus_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _plus(P=96):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict("s", [k for _, k in VITPOSE_PLUS_HEADS], P, 31).items()}


def test_plus_key_set_is_the_engine_contract():
    sd = _plus()
    exp = _expected_shapes(384, 12, 17, [k for _, k in VITPOSE_PLUS_HEADS], 96)
    assert set(sd) == set(exp)
    assert all(tuple(sd[k].shape) == exp[k] for k in sd)


def test_split_restates_model_split():
    sd = _plus()
    out = split_vitpose_plus(sd)
    assert list(out) == [n for n, _ in VITPOSE_PLUS_HEADS]
    for i, (name, K) in enumerate(VITPOSE_PLUS_HEADS):
        d = out[name]
        assert set(d) == set(_expected_shapes(384, 12, K))
        for b in range(12):
            p = f"backbone.blocks.{b}.mlp."
            assert torch.equal(d[p + "fc2.weight"], torch.cat([sd[p + "fc2.weight"], sd[p + f"experts.{i}.weight"]]))
            assert torch.equal(d[p + "fc2.bias"], torch.cat([sd[p + "fc2.bias"], sd[p + f"experts.{i}.bias"]]))
        src = "keypoint_head." if i == 0 else f"associate_keypoint_heads.{i - 1}."
        assert torch.equal(d["keypoint_head.deconv_layers.3.weight"], sd[src + "deconv_layers.3.weight"])
        assert torch.equal(d["keypoint_head.final_layer.weight"], sd[src + "final_layer.weight"][:K])
        assert torch.equal(d["backbone.blocks.4.attn.qkv.weight"], sd["backbone.blocks.4.attn.qkv.weight"])


def test_split_cuts_wider_final_layers():
    sd = _plus()
    sd["associate_keypoint_heads.4.final_layer.weight"] = torch.randn(140, 256, 1, 1)
    sd["associate_keypoint_heads.4.final_layer.bias"] = torch.randn(140)
    d = split_vitpose_plus(sd)["wholebody"]
    assert d["keypoint_head.final_layer.weight"].shape[0] == 133
    assert torch.equal(d["keypoint_head.final_layer.bias"], sd["associate_keypoint_heads.4.final_layer.bias"][:133])


@pytest.mark.parametrize("P", [96, 0])
def test_merge_round_trips(P):
    sd = _plus(P)
    merged = merge_split_state_dicts(split_vitpose_plus(sd), P)
    assert set(merged) == set(sd)
    assert all(torch.equal(merged[k], sd[k]) for k in sd)


def test_merge_names_the_first_differing_shared_key():
    parts = split_vitpose_plus(_plus())
    bad = {k: v.clone() for k, v in parts["mpii"].items()}
    bad["backbone.blocks.3.mlp.fc2.weight"][5, 7] += 1.0            # a shared row
    bad["backbone.blocks.9.attn.proj.bias"][0] += 1.0
    parts["mpii"] = bad
    with pytest.raises(ValueError, match=r"backbone\.blocks\.3\.mlp\.fc2\.weight.*'mpii'"):
        merge_split_state_dicts(parts, 96)
    ok = split_vitpose_plus(_plus())
    ok["aic"]["backbone.blocks.2.mlp.fc2.weight"][-1, 0] += 1.0     # an expert row may differ
    merge_split_state_dicts(ok, 96)


def test_grouping_is_stable_and_inverts():
    rs = np.random.RandomState(2)
    for _ in range(50):
        h = rs.randint(0, 6, size=rs.randint(0, 90))
        order, counts = group_by_head(h, 6)
        assert counts == [int((h == j).sum()) for j in range(6)]
        g = h[order]
        assert np.all(np.diff(g) >= 0)
        for j in range(6):                                           # stable inside a head
            assert np.all(np.diff(order[g == j]) > 0)
        assert np.array_equal(order[_inverse(order)], np.arange(h.size))
        for chunk in plan_frame_chunks(counts, 24):
            assert len(chunk) <= 6 and sum(e - s for _, s, e in chunk) <= 24
    for bad in ([0, 6], [-1], [0.5]):
        with pytest.raises(ValueError):
            group_by_head(np.array(bad), 6)


def test_vpb_segment_layout_matches_the_header():
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    if cc is None:
        pytest.skip("no host C compiler")
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "vitpose_b200.h"\n'
           'int main(void) { printf("%d %d %d %d %d\\n", (int)sizeof(vpb_segment), (int)offsetof(vpb_segment, head),'
           ' (int)offsetof(vpb_segment, count), VPB_MAX_SEGMENTS, VPB_MAX_HEADS); return 0; }\n')
    with tempfile.TemporaryDirectory() as d:
        c_file, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c_file, "w") as f:
            f.write(src)
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", exe, c_file], check=True, capture_output=True)
        got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    S = _lib.VpbSegment
    assert got == [C.sizeof(S), S.head.offset, S.count.offset, _lib.MAX_SEGMENTS, _lib.MAX_HEADS]


def test_python_argument_checks():
    cfg = model_cfg("s", 17)
    with pytest.raises(ValueError):
        ViTPose(cfg, heads=[17] * 9)
    with pytest.raises(ValueError):
        ViTPose(cfg, heads=[17, 0])
    with pytest.raises(ValueError):
        ViTPose(cfg, heads=[17, 14], expert_rows=100)
    with pytest.raises(ValueError):
        ViTPose(cfg, heads=[17, 14], expert_rows=384)
    with pytest.raises(ValueError):
        ViTPose(cfg, expert_rows=96)
    m = ViTPose(cfg, heads=VITPOSE_PLUS_HEADS, expert_rows=96)
    assert m.head_names == [n for n, _ in VITPOSE_PLUS_HEADS] and m.num_keypoints == 17 and m.num_keypoints_max == 133
    sd = _plus()
    sd.pop("backbone.blocks.0.mlp.experts.5.bias")
    with pytest.raises(RuntimeError, match="missing"):
        m.load_state_dict(sd)
    m.load_state_dict(_plus())                                        # strict key set accepted (no device needed)


@pytest.mark.parametrize("name", ["multi_head_s", "multi_head_b"])
def test_split_matches_model_split_fixture(golden_dir, name):
    """split_vitpose_plus against the checkpoints the unmodified model_split.py made from the same seeded ViTPose+ state_dict
    (oracle/make_golden_multi_head.py): same key set, same CRC-32 of every tensor, for all six datasets."""
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    D, depth, heads, P, n, wseed, xseed = (int(v) for v in g["meta"])
    size = {384: "s", 768: "b"}[D]
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in plus_state_dict(size, [k for _, k in VITPOSE_PLUS_HEADS], P, wseed).items()}
    keys = [str(k) for k in g["keys"]]
    for j, d in enumerate(split_vitpose_plus(sd).values()):
        assert sorted(d) == keys
        got = np.array([zlib.crc32(np.ascontiguousarray(d[k].numpy()).tobytes()) for k in keys], np.uint32)
        bad = [k for k, a, b in zip(keys, got, g["crc"][j]) if a != b]
        assert not bad, f"{VITPOSE_PLUS_HEADS[j][0]}: {len(bad)} tensors differ from model_split.py's, first {bad[0]}"
