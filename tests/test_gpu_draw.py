"""-m gpu: vpb_draw_poses (easy_vitpose_b200.draw) draws whole frames bit-exact with live cv2 and with oracle/draw_oracle.py:
untouched pixels included (the frames carry a seeded pattern), RGB and BGR, packed and padded pitch, 1 / 3 / 16 frames per call,
every fixture skeleton, graph capture, the error returns, and install(batched=True)'s draw()."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import draw_oracle as D

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "draw_poses.npz"))


def _cv_draw(frames, kp, counts, sk, ids, thr, pts, lms, order="rgb", radius=0):
    """draw()'s loop on live cv2, frame by frame: BGR copy, lines then circles per person, flip back."""
    out, p = [], 0
    for f, c in zip(frames, counts):
        img = np.ascontiguousarray(f[..., ::-1] if order == "rgb" else f)
        h, w = img.shape[:2]
        r = radius if radius > 0 else max(1, min(h, w) // 150)
        for q in range(c):
            k, idx = kp[p], (q if ids is None else int(ids[p]))
            for a, b in sk:
                if k[a, 2] > thr and k[b, 2] > thr:
                    cv2.line(img, (int(k[a, 1]), int(k[a, 0])), (int(k[b, 1]), int(k[b, 0])), tuple(int(v) for v in lms[idx % len(lms)]), 2)
            for i, pt in enumerate(k):
                if pt[2] > thr:
                    cv2.circle(img, (int(pt[1]), int(pt[0])), r, tuple(int(v) for v in pts[i % len(pts)]), -1)
            p += 1
        out.append(np.ascontiguousarray(img[..., ::-1] if order == "rgb" else img))
    return out


def _device_frames(frames, pad):
    """CUDA views of the frames, each inside a wider buffer when pad > 0 (row pitch 3 * (w + pad))."""
    out = []
    for f in frames:
        h, w = f.shape[:2]
        buf = torch.full((h, w + pad, 3), 77, dtype=torch.uint8, device="cuda")
        view = buf[:, :w]
        view.copy_(torch.from_numpy(f))
        out.append(view)
    return out


def _run(frames, kp, counts, sk, ids=None, thr=0.5, order="rgb", pad=0, radius=0):
    from easy_vitpose_b200.draw import draw_poses
    dev = _device_frames(frames, pad)
    draw_poses(dev, torch.from_numpy(kp).cuda(), counts, sk, None if ids is None else torch.tensor(ids, dtype=torch.int32).cuda(),
               confidence_threshold=thr, channel_order=order, radius=radius)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dev]


def _cases(sizes, n_per, k, seed):
    frames, kps = [], []
    for j, (h, w) in enumerate(sizes):
        f, kp = D.make_case(seed + j, h, w, n_per[j], k)
        frames.append(f)
        kps.append(kp)
    return frames, np.concatenate(kps, 0)


@pytest.mark.parametrize("sizes,n_per,order,pad,with_ids", [
    ([(1, 1)], [3], "rgb", 0, False),
    ([(7, 5), (33, 17), (1, 1)], [4, 6, 2], "bgr", 5, True),
    ([(1080, 1920)], [12], "rgb", 0, True),
    ([(1080, 1920)] * 3, [9, 0, 11], "bgr", 16, False),
    ([(1080, 1920) if j % 4 == 0 else (240 + 8 * j, 320 + 4 * j) for j in range(16)], [9, 8, 10, 0, 12, 9, 7, 9, 8, 10, 9, 9, 11, 8, 7, 10],
     "rgb", 3, True),
])
def test_frames_bit_exact_vs_cv2(golden_dir, sizes, n_per, order, pad, with_ids):
    from easy_vitpose_b200.draw import reference_palettes
    g = _golden(golden_dir)
    sk, k = g["skeleton_coco"], int(g["num_keypoints_coco"])
    frames, kp = _cases(sizes, n_per, k, seed=len(sizes) * 10 + pad)
    ids = (np.arange(len(kp)) * 7 + 3) % 23 if with_ids else None
    pts, lms = reference_palettes()
    got = _run(frames, kp, n_per, sk, ids, order=order, pad=pad)
    want = _cv_draw(frames, kp, n_per, sk, ids, np.float32(0.5), pts, lms, order)
    for j, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), (j, int((a != b).any(-1).sum()))
        if n_per[j] == 0:
            assert np.array_equal(a, frames[j])                       # a frame of the call without people is left as it was


def test_oracle_and_device_agree_on_every_fixture_skeleton(golden_dir):
    """Every dataset's skeleton (wholebody: K = 133, 65 limbs), overlapping people in small frames, scores at the threshold,
    explicit radii; the device against the oracle's draw loop."""
    from easy_vitpose_b200.draw import reference_palettes
    g = _golden(golden_dir)
    pts, lms = reference_palettes()
    for t, ds in enumerate(g["datasets"]):
        sk, k = g[f"skeleton_{ds}"], int(g[f"num_keypoints_{ds}"])
        frames, kp = _cases([(48, 64), (90, 70)], [7, 5], k, seed=300 + t)
        for radius in (0, 1 + t):
            got = _run(frames, kp, [7, 5], sk, radius=radius)
            want = D.draw_poses([f.copy() for f in frames], kp, [7, 5], sk, pts, lms, radius=radius)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (ds, radius)


def test_threshold_is_strict_and_painters_order_holds():
    """Scores exactly at the threshold are not drawn; a later person's limb overwrites an earlier person's point."""
    from easy_vitpose_b200.draw import reference_palettes
    pts, lms = reference_palettes()
    f = np.full((40, 40, 3), 9, np.uint8)
    kp = np.array([[[20, 20, 0.9], [20, 5, 0.5]], [[10, 20, 0.8], [30, 20, 0.8]]], np.float32)   # person 1's vertical limb crosses person 0's point
    got = _run([f], kp, [2], [[0, 1]], thr=0.5)[0]
    want = _cv_draw([f], kp, [2], [[0, 1]], None, np.float32(0.5), pts, lms)[0]
    assert np.array_equal(got, want)
    assert np.array_equal(got[20, 5], f[20, 5])                                          # score 0.5: neither point nor limb
    assert got[20, 20].tolist() == lms[1][::-1].tolist()                                 # RGB of person 1's limb colour


def test_keypoints_from_infer_frames(golden_dir):
    """The keypoints a real multi-frame engine call returns feed straight in (same [n, K, 3] rows, same frame order)."""
    from easy_vitpose_b200 import ViTPose, model_cfg
    from easy_vitpose_b200.draw import draw_poses, reference_palettes
    from oracle import preproc_oracle as P, vitpose_oracle as O
    sk = _golden(golden_dir)["skeleton_coco"]
    sd = O.make_state_dict(384, 12, 17, 5, peaky=0.1, bumps=True)
    m = ViTPose(model_cfg("s", 17), max_batch=8)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}).to("cuda:0")
    frames = [P.make_frame(240, 320, seed=1), P.make_frame(180, 200, seed=2)]
    boxes = [np.array([[20, 30, 150, 200], [100, 20, 300, 230]], np.int32), np.array([[10, 10, 120, 170]], np.int32)]
    kps, _ = m.infer_frames([torch.from_numpy(f).cuda() for f in frames], boxes)
    kp = torch.cat(kps, 0)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    draw_poses(dev, kp, [2, 1], sk, confidence_threshold=0.0)
    torch.cuda.synchronize()
    pts, lms = reference_palettes()
    want = _cv_draw(frames, kp.cpu().numpy(), [2, 1], sk, None, np.float32(0.0), pts, lms)
    for a, b in zip(dev, want):
        assert np.array_equal(a.cpu().numpy(), b)


def test_no_people_launches_nothing_and_graph_capture_replays(golden_dir):
    from easy_vitpose_b200.draw import draw_poses
    g = _golden(golden_dir)
    sk = g["skeleton_coco"]
    f = D.make_case(1, 64, 80, 1, 17)[0]
    dev = [torch.from_numpy(f).cuda()]
    draw_poses(dev, torch.zeros((0, 17, 3), device="cuda"), [0], sk)
    torch.cuda.synchronize()
    assert np.array_equal(dev[0].cpu().numpy(), f)
    frames, kp = _cases([(120, 160), (64, 80)], [5, 4], 17, seed=900)
    want = _run(frames, kp, [5, 4], sk, ids=[3, 1, 4, 1, 5, 9, 2, 6, 5])
    dev = [torch.from_numpy(x).cuda() for x in frames]
    kd, ids = torch.from_numpy(kp).cuda(), torch.tensor([3, 1, 4, 1, 5, 9, 2, 6, 5], dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        draw_poses(dev, kd, [5, 4], sk, ids)
    torch.cuda.synchronize()
    assert all(np.array_equal(d.cpu().numpy(), x) for d, x in zip(dev, frames))      # capture launched nothing
    graph.replay()
    torch.cuda.synchronize()
    assert all(np.array_equal(d.cpu().numpy(), w) for d, w in zip(dev, want))
    for d, x in zip(dev, frames):
        d.copy_(torch.from_numpy(x))
    graph.replay()
    torch.cuda.synchronize()
    assert all(np.array_equal(d.cpu().numpy(), w) for d, w in zip(dev, want))


def test_error_returns():
    from easy_vitpose_b200 import _lib
    lib = _lib.lib()
    f = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")
    kp = torch.zeros((1, 4, 3), device="cuda")
    ws = torch.empty(int(lib.vpb_draw_workspace_bytes(1, 4, 2)), dtype=torch.uint8, device="cuda")
    assert lib.vpb_draw_workspace_bytes(-1, 4, 2) == -1 and lib.vpb_draw_workspace_bytes(1, 0, 2) == -1
    col = np.zeros((4, 3), np.uint8)

    def call(h=8, w=8, pitch=24, data=True, people=1, order=0, limbs=((0, 1), (1, 2)), k=4, npc=4, nlc=4, radius=0, frames=1, wsp=True):
        canv = (_lib.VpbCanvas * frames)()
        for j in range(frames):
            canv[j].data, canv[j].height, canv[j].width, canv[j].pitch_bytes, canv[j].num_people = (
                f.data_ptr() if data else None, h, w, pitch, people if j == 0 else 1)
        lm = np.ascontiguousarray(np.array(limbs, np.int32).reshape(-1, 2))
        return lib.vpb_draw_poses(canv, frames, order, C.c_void_p(kp.data_ptr()), k, None, lm.ctypes.data_as(C.c_void_p), len(lm),
                                  col.ctypes.data_as(C.c_void_p), npc, col.ctypes.data_as(C.c_void_p), nlc, radius, 0.5,
                                  C.c_void_p(ws.data_ptr()) if wsp else None, None)
    assert call() == 0
    assert call(people=0, wsp=False) == 0                                           # n = 0: nothing to check the workspace for
    for kw in [dict(limbs=((0, 4),)), dict(limbs=((0, 1),) * 129), dict(npc=0), dict(nlc=0), dict(npc=65), dict(data=False), dict(h=0),
               dict(w=0), dict(pitch=23), dict(frames=65), dict(order=2), dict(radius=1024), dict(people=-1), dict(wsp=False), dict(k=0)]:
        assert call(**kw) == 1, kw                                                 # VPB_ERR_ARG
    torch.cuda.synchronize()


def test_install_batched_rebinds_draw(golden_dir, monkeypatch):
    """install(vi, batched=True): vi.draw() returns what the reference's draw() returns on the same state -- here draw()'s pose
    loop on live cv2 with the reference palettes and joints_dict()'s skeleton (a stand-in module carries the fixture's tables
    where the reference package is absent)."""
    from easy_vitpose_b200 import install
    from easy_vitpose_b200.draw import reference_palettes
    from oracle import vitpose_oracle as O
    g = _golden(golden_dir)
    try:
        import easy_ViTPose.vit_utils.visualization  # noqa: F401
    except Exception:
        joints = {str(ds): {"skeleton": g[f"skeleton_{ds}"].tolist(), "keypoints": {i: str(i) for i in range(int(g[f"num_keypoints_{ds}"]))}}
                  for ds in g["datasets"]}
        for name in ("easy_ViTPose", "easy_ViTPose.vit_utils"):
            monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
        vis = types.ModuleType("easy_ViTPose.vit_utils.visualization")
        vis.joints_dict = lambda: joints
        monkeypatch.setitem(sys.modules, "easy_ViTPose.vit_utils.visualization", vis)
    sd = O.make_state_dict(384, 12, 17, 3, peaky=0.1, bumps=True)

    class FakeRefModel(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for k, v in sd.items():
                self.register_buffer(k.replace(".", "__"), torch.from_numpy(np.asarray(v)))
            self.backbone = types.SimpleNamespace(blocks=[types.SimpleNamespace(attn=types.SimpleNamespace(num_heads=12))])

        def state_dict(self, *a, **kw):
            return {k.replace("__", "."): v for k, v in super().state_dict(*a, **kw).items()}

    frame, kp = D.make_case(11, 360, 480, 5, 17)
    ids = [4, 0, 9, 2, 13]
    vi = types.SimpleNamespace(_vit_pose=FakeRefModel(), _inference=None, postprocess=None, tracker=None, save_state=True, dataset="coco",
                               _img=frame, _yolo_res=None, _tracker_res=(np.zeros((5, 4), int), ids, [0.9] * 5),
                               _keypoints={i: kp[j] for j, i in enumerate(ids)})
    install(vi, max_batch=8, batched=True)
    pts, lms = reference_palettes()
    for thr in (0.5, 0.2):
        got = vi.draw(show_yolo=True, confidence_threshold=thr)
        want = _cv_draw([frame], kp, [5], g["skeleton_coco"], ids, np.float32(thr), pts, lms)[0]
        assert got.shape == frame.shape and np.array_equal(got, want), thr
    assert np.array_equal(vi._img, frame)                                            # draw() works on a copy
    vi._keypoints = {}
    assert np.array_equal(vi.draw(), frame)
