"""-m gpu: simple-decoder engines (VPB_DECODER_SIMPLE, csrc/simple_head.cuh) against the reference's goldens, against the fp64
oracle within its per-element bound, for their invariances, and through the keypoint entry points and multi-head calls."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import simple_head_oracle as S
from oracle import vitpose_oracle as O

pytestmark = pytest.mark.gpu

HEATMAP_TOL = 0.01               # as tests/test_gpu_engine.py
KPT_MEAN_PX_TOL = 0.5


def _cfg(D, depth, K):
    from easy_vitpose_b200 import model_cfg
    size = {384: "s", 768: "b", 1024: "l", 1280: "h"}[D]
    cfg = model_cfg(size, K, decoder="simple")
    cfg["backbone"]["depth"] = depth
    return cfg


def _engine(D, depth, K, seed, max_batch=8, heads=None, peaky=0.1, bumps=True):
    from easy_vitpose_b200 import ViTPose
    m = ViTPose(_cfg(D, depth, K), max_batch=max_batch, heads=heads)
    ks = heads or [K]
    sd = S.make_state_dict(D, depth, ks[0], seed, peaky=peaky, bumps=bumps)
    for j, Kj in enumerate(ks[1:], 1):
        hsd = S.make_state_dict(D, 1, Kj, seed + j, peaky=peaky, bumps=bumps)
        for part in ("weight", "bias"):
            sd[f"associate_keypoint_heads.{j - 1}.final_layer.{part}"] = hsd[f"keypoint_head.final_layer.{part}"]
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    m.to("cuda:0")
    return m, sd


@pytest.mark.parametrize("size", ["b", "l", "h"])
def test_forward_vs_reference_goldens(golden_dir, size):
    g = np.load(os.path.join(golden_dir, f"simple_{size}_coco.npz"))
    D, depth, heads, K, B, wseed, xseed = (int(v) for v in g["meta"])
    m, _ = _engine(D, depth, K, wseed, peaky=float(g["peaky"]))
    assert m.decoder == "simple"
    x = torch.from_numpy(O.make_crops(B, xseed)).cuda()
    hm = m(x).cpu().numpy()
    ref = g["heatmaps"]
    rng = float(ref.max() - ref.min())
    linf = float(np.abs(hm - ref).max())
    print(size, f"heatmap Linf {linf:.5f} = {linf / rng:.3%} of range {rng:.4f}")
    assert linf < HEATMAP_TOL * rng
    kp, idx, hm2 = m.infer_crops(x, torch.from_numpy(g["org_wh"]), return_heatmaps=True)
    assert np.array_equal(hm2.cpu().numpy(), hm)
    assert np.array_equal(idx.cpu().numpy(), hm.reshape(B, K, -1).argmax(-1).astype(np.int32))
    kpn = kp.cpu().numpy()
    to_model_px = np.stack([256.0 / g["org_wh"][:, 1], 192.0 / g["org_wh"][:, 0]], -1)[:, None, :]
    dev = np.linalg.norm((kpn[..., :2] - g["kpts"][..., :2]) * to_model_px, axis=-1)
    vis = g["kpts"][..., 2] > 0.3
    print(size, "visible", int(vis.sum()), "/", vis.size, "deviation px mean", dev[vis].mean(), "max", dev[vis].max())
    assert vis.sum() >= 0.7 * vis.size
    assert dev[vis].mean() < KPT_MEAN_PX_TOL


def _head_call(m, feats, out):
    from easy_vitpose_b200 import _lib
    _lib.check(_lib.lib().vpb_head(m._handle, C.c_void_p(feats.data_ptr()), feats.shape[0], C.c_void_p(out.data_ptr()),
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)))


@pytest.mark.parametrize("D", [384, 768, 1280])
@pytest.mark.parametrize("K", [1, 16, 17, 133, 144])
def test_head_within_fp64_bound(D, K):
    m, sd = _engine(D, 1, K, 900 + K, max_batch=64, peaky=1.0, bumps=False)
    w = S.engine_weights(sd["keypoint_head.final_layer.weight"]).cuda()
    b = torch.from_numpy(sd["keypoint_head.final_layer.bias"]).to(torch.float64).cuda()
    g = torch.Generator(device="cuda").manual_seed(D + K)
    for B in (1, 3, 64):
        feats = torch.randn(B, D, 16, 12, generator=g, device="cuda").bfloat16().float()
        out = torch.full((B + 1, K, 64, 48), 12345.0, device="cuda")         # one crop of sentinel past the batch
        _head_call(m, feats, out)
        torch.cuda.synchronize()
        assert torch.all(out[B] == 12345.0), (D, K, B)
        ref, bound = S.bound(feats.double(), w, b)
        r = ((out[:B].double() - ref).abs() / bound)
        r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
        print(D, K, B, "worst |err| / bound", float(r.max()))
        assert float(r.max()) <= 1.0, (D, K, B)


def test_invariances():
    m, _ = _engine(768, 2, 17, 31, max_batch=64)
    x = torch.from_numpy(O.make_crops(64, 32)).cuda()
    hm = m(x)
    assert torch.equal(m.head_forward(m.forward_features(x)), hm)
    assert torch.equal(torch.cat([m(x[i:i + 1]) for i in range(64)]), hm)
    org = torch.tensor([[192, 256]] * 5, dtype=torch.int32)
    outs = [m.infer_crops(x[:5], org, return_heatmaps=True) for _ in range(3)]    # eager, capture, replay
    assert m.cached_graphs() == (1, 1)
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))
    assert torch.equal(outs[0][2], hm[:5])


def _decode_mode4(hm, cs):
    """keypoints_from_heatmaps(hm, c, s, use_udp=True) on the device (vpb_decode_modes mode 4), as infer_affine decodes."""
    from easy_vitpose_b200 import _lib
    n, K = hm.shape[:2]
    kp = torch.empty((n, K, 3), dtype=torch.float32, device=hm.device)
    idx = torch.empty((n, K), dtype=torch.int32, device=hm.device)
    _lib.check(_lib.lib().vpb_decode_modes(C.c_void_p(hm.data_ptr()), n, K, 4, C.c_void_p(cs.data_ptr()), None,
                                           C.c_void_p(kp.data_ptr()), C.c_void_p(idx.data_ptr()),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return kp, idx


def test_entry_points():
    from easy_vitpose_b200 import COCO_FLIP_PAIRS
    from easy_vitpose_b200.top_down_eval import decode_heatmaps
    m, _ = _engine(384, 2, 17, 41, max_batch=16)
    x = torch.from_numpy(O.make_crops(6, 42)).cuda()
    org = torch.tensor([[192, 256], [151, 211], [100, 300], [333, 222], [64, 64], [500, 400]], dtype=torch.int32)
    # infer_crops = forward + decode
    kp, idx = m.infer_crops(x, org)
    kw, iw = decode_heatmaps(m(x), org.cuda())
    assert torch.equal(kp, kw) and torch.equal(idx, iw)
    # host pipelined form = the device form
    crops = x.cpu().numpy()
    outs = [(np.empty((3, 17, 3), np.float32), np.empty((3, 17), np.int32)) for _ in range(2)]
    for s in range(2):
        m.submit_host(np.ascontiguousarray(crops[3 * s:3 * s + 3]), np.ascontiguousarray(org[3 * s:3 * s + 3].numpy()), *outs[s], s)
    for s in range(2):
        m.wait_host(s)
    assert np.array_equal(np.concatenate([o[0] for o in outs]), kp.cpu().numpy())
    # frames: the gathered crops through forward, argmax / score bit for bit, positions = crop decode + box offset
    rs = np.random.RandomState(43)
    frame = torch.from_numpy(rs.randint(0, 256, (480, 640, 3), dtype=np.uint8)).cuda()
    boxes = np.array([[10, 20, 200, 400], [300, 50, 600, 470], [100, 100, 180, 160]], np.float32)
    from oracle import preproc_oracle as P
    fk, fi = m.infer_frames([frame], [boxes])
    c, o, offs = m.preprocess(frame, boxes)
    hk, hi = decode_heatmaps(m(c), o)
    assert torch.equal(torch.cat(fi), hi)
    assert np.array_equal(torch.cat(fk).cpu().numpy(), P.to_frame_coords(hk.cpu().numpy(), offs.cpu().numpy()))
    # flip test: infer_crops and infer_affine = forward_flip_test + decode
    pairs = [tuple(p) for p in COCO_FLIP_PAIRS]
    m.set_flip_test(pairs, False)
    try:
        kp, idx = m.infer_crops(x, org)
        kw, iw = decode_heatmaps(m.forward_flip_test(x, pairs), org.cuda())
        assert torch.equal(kp, kw) and torch.equal(idx, iw)
        mats = [np.array([[[0.5, 0.0, 30.0], [0.0, 0.5, 40.0]], [[0.8, 0.1, 5.0], [-0.1, 0.8, 60.0]]], np.float64)]
        cs = [np.array([[120.0, 150.0], [300.0, 200.0]], np.float32)]
        ss = [np.array([[1.2, 1.6], [2.0, 2.6]], np.float32)]
        ak, ai = m.infer_affine([frame], mats, cs, ss)
        hm = m.forward_flip_test(m.preprocess_affine([frame], mats), pairs)
        dk, di = _decode_mode4(hm, torch.from_numpy(np.concatenate([cs[0], ss[0]], 1)).cuda())
        assert torch.equal(torch.cat(ak), dk) and torch.equal(torch.cat(ai), di)
    finally:
        m.set_flip_test(None)


def test_multi_head_equals_single_heads():
    from easy_vitpose_b200 import ViTPose
    from easy_vitpose_b200.model import split_vitpose_plus
    m, sd = _engine(384, 2, 17, 51, max_batch=16, heads=[17, 133])
    x = torch.from_numpy(O.make_crops(7, 52)).cuda()
    org = torch.tensor([[192, 256]] * 7, dtype=torch.int32)
    heads = [0, 1, 1, 0, 1, 0, 0]
    kp, idx, hm = m.infer_crops_heads(x, org, heads, return_heatmaps=True)
    parts = split_vitpose_plus({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, names=["a", "b"], keypoints=[17, 133])
    for j, (name, K) in enumerate((("a", 17), ("b", 133))):
        s = ViTPose(_cfg(384, 2, K), max_batch=16)
        s.load_state_dict(parts[name])
        s.to("cuda:0")
        sel = [i for i, h in enumerate(heads) if h == j]
        k1, i1, h1 = s.infer_crops(x[sel], org[sel], return_heatmaps=True)
        assert torch.equal(kp[sel, :K], k1) and torch.equal(idx[sel, :K], i1) and torch.equal(hm[sel, :K], h1)
        assert not torch.any(hm[sel, K:])                                   # nothing past a smaller head's K rows


def test_from_state_dict_detects_the_decoder_and_memory():
    from easy_vitpose_b200 import ViTPose, model_cfg
    from easy_vitpose_b200.inference import B200PoseBackend
    sd = S.make_state_dict(384, 12, 17, 61)
    be = B200PoseBackend.from_state_dict({"state_dict": {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}}, "s", 17, max_batch=8)
    assert be.model.decoder == "simple"
    classic = ViTPose(model_cfg("s", 17), max_batch=8)
    classic.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in O.make_state_dict(384, 12, 17, 61).items()})
    classic.to("cuda:0")
    # no deconv workspace: d1 + d2 are 8 * (768 + 3072) * 256 bf16
    assert classic.device_bytes() - be.model.device_bytes() >= 8 * (768 + 3072) * 256 * 2
    with pytest.raises(RuntimeError, match="not allocated"):
        be.model.read_buffer("d2", (8, 64, 48, 256), "bf16")
