"""-m gpu: vpb_tracker_update (easy_vitpose_b200.track.DeviceSort) equals the unmodified sort.py's fixture and
oracle/sort_oracle.py as float64 values: 1 / 3 / 16 / 64 streams, three (max_age, min_hits) settings, up to 128 boxes per
stream; graph replays equal eager calls bit for bit; reset of one stream; the status bits and argument errors;
inference_frames_tracked; install(..., batched=True, device_tracker=True)."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from oracle import sort_oracle as SO
from oracle.make_golden_track import CASES, RAW_FRAMES, case_inputs, crc

pytestmark = pytest.mark.gpu


def _same(got, want):
    return len(got) == len(want) and all(g.shape == w.shape and np.array_equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_device_equals_reference_fixture(golden_dir, case):
    from easy_vitpose_b200.track import DeviceSort
    g = np.load(os.path.join(golden_dir, "track_sort.npz"))
    name, max_age, min_hits = case[:3]
    t = DeviceSort(len(case[5]), max_age, min_hits, 0.3)
    first = []
    for f, dl in enumerate(case_inputs(case)):
        outs = t.update(dl)
        assert [len(r) for r in outs] == g[f"{name}_counts"][f].tolist(), f
        assert [crc(r) for r in outs] == g[f"{name}_crc32"][f].tolist(), f
        if f < RAW_FRAMES:
            first.append(outs[0])
    assert np.array_equal(np.concatenate(first), g[f"{name}_stream0_rows"])
    assert t.next_id == int(g[f"{name}_next_id"]) and t.status() == 0


def _streams(S, frames, seed, max_age):
    """Seeded per-stream sequences with every kind, one stream of 128 sparse people and one of 128 crowded boxes."""
    kinds = ["walk", "crowd", "jump", "dup", "shrink", "occlude", "empty"]
    seqs = []
    for s in range(S):
        k = kinds[(s + seed) % len(kinds)]
        if s == 1:
            seqs.append(SO.make_sequence(seed * 1000 + s, frames, 128, "walk", 3840., 2160.))
        elif s == 2:
            seqs.append(SO.make_sequence(seed * 1000 + s, frames, 128, "crowd", 900., 700.))
        else:
            people = int(np.random.default_rng(seed * 7 + s).integers(1, 90 if k == "crowd" else 16))
            seqs.append(SO.make_sequence(seed * 1000 + s, frames, people, k, *((700., 500.) if k == "crowd" else (1920., 1080.))))
    step = max_age if max_age > 1 else 1                      # detector cadence yolo_step = max_age, as VitInference.reset() pairs them
    return [[sq[f] if (f < 3 or f % step == 0) else np.empty((0, 5)) for sq in seqs] for f in range(frames)]


@pytest.mark.parametrize("S", [1, 3, 16, 64])
@pytest.mark.parametrize("max_age,min_hits", [(1, 3), (3, 1), (5, 1)])
def test_device_equals_oracle(S, max_age, min_hits):
    from easy_vitpose_b200.track import DeviceSort
    frames = 24 if S == 64 else 40
    t = DeviceSort(S, max_age, min_hits, 0.3)
    o = SO.SortOracle(S, max_age, min_hits, 0.3, limit=SO.TRACK_MAX)
    rows = 0
    for f, dl in enumerate(_streams(S, frames, S + 10 * max_age, max_age)):
        got, want = t.update(dl), o.update(dl)
        assert _same(got, want), (f, [len(x) for x in got], [len(x) for x in want])
        rows += sum(len(w) for w in want)
    assert rows > 0 and t.next_id == o.next_id and t.status() == o.status


def test_float32_and_cuda_inputs_match_float64_host():
    from easy_vitpose_b200.track import DeviceSort
    dl0 = _streams(3, 12, 5, 1)
    a, b = DeviceSort(3), DeviceSort(3)
    for f, dl in enumerate(dl0):
        dl32 = [d.astype(np.float32) for d in dl]
        want = a.update([d.astype(np.float64) for d in dl32])
        got = b.update([torch.from_numpy(d).cuda() if s % 2 else d for s, d in enumerate(dl32)])
        assert _same(got, want), f


def test_graph_replay_equals_eager():
    from easy_vitpose_b200.track import DeviceSort
    S = 16
    eager, captured = DeviceSort(S, 3, 1), DeviceSort(S, 3, 1)
    dets = torch.zeros((S, SO.TRACK_MAX, 5), dtype=torch.float64, device="cuda")
    counts = torch.zeros(S, dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        g_rows, g_boxes, g_counts = captured.update_device(dets, counts)
    torch.cuda.synchronize()
    assert captured.next_id == 0
    for f, dl in enumerate(_streams(S, 30, 3, 3)):
        d, c = eager.pack(dl)
        dets.copy_(d)
        counts.copy_(c)
        graph.replay()
        e_rows, e_boxes, e_counts = eager.update_device(d, c)
        torch.cuda.synchronize()
        n = e_counts.cpu()
        assert torch.equal(n, g_counts.cpu()), f
        for s in range(S):
            m = int(n[s])
            assert torch.equal(e_rows[s, :m], g_rows[s, :m]) and torch.equal(e_boxes[s, :m], g_boxes[s, :m]), (f, s)
    assert eager.next_id == captured.next_id > 0


def test_boxes_are_rows_rounded_half_to_even():
    from easy_vitpose_b200.track import DeviceSort
    t = DeviceSort(2, 1, 0)
    dets = [np.array([[10.5, 11.5, 60.5, 91.5, 0.9], [100.25, 20.75, 140.5, 70.5, 0.8]]), np.empty((0, 5))]
    d, c = t.pack(dets)
    rows, boxes, counts = t.update_device(d, c)
    assert counts.tolist() == [2, 0]
    r = rows[0, :2].cpu().numpy()
    assert np.array_equal(boxes[0, :2].cpu().numpy(), np.round(r[:, :4]).astype(np.int32))
    assert r[:, 5].tolist() == [2.0, 1.0] and np.abs(r[:, :4] - dets[0][::-1, :4]).max() < 1e-9


def test_reset_one_stream_keeps_the_others_and_the_counter():
    from easy_vitpose_b200.track import DeviceSort
    S = 4
    t = DeviceSort(S, 1, 3)
    o = SO.SortOracle(S, 1, 3, limit=SO.TRACK_MAX)
    seq = _streams(S, 20, 8, 1)
    for f, dl in enumerate(seq):
        if f == 10:
            t.reset(2)
            o.reset(2)
        if f == 15:
            t.reset()
            o.reset()
        assert _same(t.update(dl), o.update(dl)), f
    assert t.next_id == o.next_id
    t.next_id = 1000
    o.next_id = 1000
    assert _same(t.update(seq[0]), o.update(seq[0])) and t.next_id == o.next_id > 1000


def test_status_bits_skip_only_the_bad_streams():
    """Bad rows and over-capacity streams are skipped (no rows, state kept) and raise their bits; the other streams carry on
    as the oracle with the device's limits says, and so do the skipped ones on later frames."""
    from easy_vitpose_b200.track import STATUS_BAD_ROW, STATUS_OVER_CAPACITY, DeviceSort
    S = 6
    t = DeviceSort(S, 1, 1)
    o = SO.SortOracle(S, 1, 1, limit=SO.TRACK_MAX)
    seqs = [SO.make_sequence(12 + s, 7, 6, "walk") for s in range(S)]
    base = [[sq[f] for sq in seqs] for f in range(7)]
    rng = np.random.default_rng(0)
    far = np.stack([rng.uniform(0, 5000, 128), rng.uniform(0, 5000, 128)], 1)
    spread = np.concatenate([far, far + [8.0, 8.0], np.full((128, 1), 0.9)], 1)   # 128 tiny boxes nobody overlaps
    expect = {2: STATUS_BAD_ROW | STATUS_OVER_CAPACITY, 3: STATUS_BAD_ROW, 4: STATUS_OVER_CAPACITY}
    for f, dl in enumerate(base):
        dl = [d.copy() for d in dl]
        dl[4] = np.empty((0, 5)) if f == 0 else spread + ([100.0, 100.0, 100.0, 100.0, 0.0] if f == 4 else 0.0)   # 128 tracks, then 128 more
        if f == 2:
            dl[0] = np.concatenate([dl[0], [[1.0, 2.0, np.nan, 4.0, 0.5]]])                          # non-finite
            dl[1] = np.concatenate([dl[1], [[5.0, 5.0, 5.0, 9.0, 0.5]]])                             # x2 <= x1
            dl[2] = np.tile(np.array([[1.0, 1.0, 9.0, 9.0, 0.9]]), (129, 1))                          # 129 > 128 rows
        if f == 3:
            dl[3] = np.concatenate([dl[3], [[1.0, 2.0, 3.0, 4.0, np.inf]]])
        got, want = t.update(dl), o.update(dl)
        assert _same(got, want), f
        assert o.status == expect.get(f, 0) and t.status() == o.status, f
        o.status = 0
        if f == 2:
            assert all(len(got[s]) == 0 for s in range(3))
    assert t.next_id == o.next_id
    t.update([np.array([[1.0, 1.0, 1.0, 2.0, 0.5]])] + [np.empty((0, 5))] * (S - 1))
    with pytest.raises(ValueError):
        t.check()
    t.check()                                                                # the query cleared the word


def test_argument_errors():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.track import DeviceSort
    lib = _lib.lib()
    h = C.c_void_p()
    for args in [(0, 1, 3, 0.3, 0), (70000, 1, 3, 0.3, 0), (2, -1, 3, 0.3, 0), (2, 1, -1, 0.3, 0), (2, 1, 3, float("nan"), 0),
                 (2, 1, 3, 0.3, 999), (2, 1, 3, 0.3, -1)]:
        assert lib.vpb_tracker_create(*args, C.byref(h)) == 1, args
    assert lib.vpb_tracker_create(2, 1, 3, 0.3, 0, None) == 1
    t = DeviceSort(2)
    x = torch.zeros(16, dtype=torch.float64, device="cuda")
    p = C.c_void_p(x.data_ptr())
    assert lib.vpb_tracker_update(t._handle, None, p, p, p, p, None) == 1
    assert lib.vpb_tracker_update(None, p, p, p, p, p, None) == 1
    assert lib.vpb_tracker_reset(t._handle, 2, None) == 1 and lib.vpb_tracker_reset(t._handle, -2, None) == 1
    assert lib.vpb_tracker_set_next_id(t._handle, -1) == 1
    with pytest.raises(ValueError):
        t.update([np.zeros((1, 5))])                                         # one array for two streams
    with pytest.raises(ValueError):
        t.update([np.zeros((1, 4)), np.zeros((0, 5))])
    with pytest.raises(ValueError):
        t.update_device(torch.zeros((2, 128, 5), device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda"))   # float32
    with pytest.raises(ValueError):
        DeviceSort(2, -1)
    torch.cuda.synchronize()


def _engine(max_batch=16, seed=5):
    from easy_vitpose_b200 import ViTPose, model_cfg
    from oracle import vitpose_oracle as O
    sd = O.make_state_dict(384, 12, 17, seed, peaky=0.1, bumps=True)
    m = ViTPose(model_cfg("s", 17), max_batch=max_batch)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}).to("cuda:0")
    return m, sd


def _in_frame_dets(seed, frames, people, h, w):
    """Boxes that stay inside an h x w frame (so every tracked box keeps pixels after padding and clipping)."""
    rng = np.random.default_rng(seed)
    x0, y0 = rng.uniform(10, w - 90, people), rng.uniform(10, h - 120, people)
    out = []
    for f in range(frames):
        j = rng.uniform(-2, 2, (people, 2))
        d = np.stack([x0 + j[:, 0], y0 + j[:, 1], x0 + 60 + j[:, 0], y0 + 100 + j[:, 1], rng.uniform(0.4, 1, people)], 1)
        out.append(d[rng.uniform(size=people) > 0.15])
    return out


def test_inference_frames_tracked_equals_oracle_boxes_through_infer_frames_host():
    from easy_vitpose_b200 import B200PoseBackend
    from easy_vitpose_b200.track import DeviceSort
    from oracle import preproc_oracle as P
    m, _ = _engine()
    backend = B200PoseBackend(m)
    sizes = [(240, 320), (180, 260), (300, 200)]
    imgs = [P.make_frame(h, w, seed=20 + j) for j, (h, w) in enumerate(sizes)]
    seqs = [_in_frame_dets(30 + j, 8, 5, h, w) for j, (h, w) in enumerate(sizes)]
    t = DeviceSort(3, 1, 3, device=0)
    o = SO.SortOracle(3, 1, 3)
    for f in range(8):
        dl = [sq[f] for sq in seqs]
        got = backend.inference_frames_tracked(imgs, dl, t)
        want_rows = o.update(dl)
        kps, _ = m.infer_frames_host(imgs, [r[:, :4] for r in want_rows])
        for s in range(3):
            assert list(got[s].keys()) == want_rows[s][:, 5].astype(int).tolist(), (f, s)
            assert all(np.array_equal(got[s][i], k) for i, k in zip(got[s], kps[s])), (f, s)
    assert t.next_id == o.next_id


def test_install_device_tracker_matches_cpu_tracker_path():
    """install(vi, batched=True, device_tracker=True) on a fake VitInference gives, frame by frame, the ids, keypoints and
    save_state fields of the same object with a CPU SORT (the oracle standing in for the reference Sort)."""
    from easy_vitpose_b200 import install
    from easy_vitpose_b200.inference import DeviceTracker
    from oracle import preproc_oracle as P
    _, sd = _engine()

    class FakeRefModel(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for k, v in sd.items():
                self.register_buffer(k.replace(".", "__"), torch.from_numpy(np.asarray(v)))
            self.backbone = types.SimpleNamespace(blocks=[types.SimpleNamespace(attn=types.SimpleNamespace(num_heads=12))])

        def state_dict(self, *a, **kw):
            return {k.replace("__", "."): v for k, v in super().state_dict(*a, **kw).items()}

    class CpuSort:
        def __init__(self, max_age, min_hits, iou_threshold):
            self.max_age, self.min_hits, self.iou_threshold = max_age, min_hits, iou_threshold
            self.o = SO.SortOracle(1, max_age, min_hits, iou_threshold)

        def update(self, dets=np.empty((0, 5))):
            return self.o.update([dets])[0]

    frame = P.make_frame(240, 320, seed=4)
    dets = _in_frame_dets(77, 9, 6, 240, 320)

    def make_vi(step):
        calls = []

        def yolo(img, **kw):
            rows = dets[len(calls)]
            calls.append(kw)
            data = np.concatenate([rows, np.zeros((len(rows), 1))], 1).astype(np.float32)
            return [types.SimpleNamespace(boxes=types.SimpleNamespace(data=types.SimpleNamespace(cpu=lambda: types.SimpleNamespace(numpy=lambda: data))))]
        return types.SimpleNamespace(_vit_pose=FakeRefModel(), _inference=None, postprocess=None, frame_counter=0, yolo_step=step, yolo=yolo,
                                     yolo_size=320, device="cuda", yolo_classes=[0], save_state=True, is_video=True, single_pose=False,
                                     tracker=CpuSort(step, 3 if step == 1 else 1, 0.3))

    for step in (1, 3):
        cpu, dev = make_vi(step), make_vi(step)
        install(cpu, max_batch=8, batched=True)
        install(dev, max_batch=8, batched=True, device_tracker=True)
        assert isinstance(dev.tracker, DeviceTracker) and isinstance(cpu.tracker, CpuSort)
        assert (dev.tracker.max_age, dev.tracker.min_hits) == (step, 3 if step == 1 else 1)
        for f in range(9):
            a, b = cpu.inference(frame), dev.inference(frame)
            assert list(a) == list(b) and all(np.array_equal(a[i], b[i]) for i in a), (step, f)
            assert np.array_equal(cpu._tracker_res[0], dev._tracker_res[0]) and cpu._tracker_res[1:] == dev._tracker_res[1:]
        old = dev.tracker
        dev.reset()
        assert isinstance(dev.tracker, DeviceTracker) and dev.tracker is not old and dev.frame_counter == 0
        dev.single_pose = True
        dev.reset()
        assert dev.tracker is None
