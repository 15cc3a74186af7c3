"""-m gpu: vpb_smoother_update (easy_vitpose_b200.smooth.DeviceOneEuro) equals the unmodified reference OneEuroFilter's
fixture and oracle/one_euro_oracle.py as float64 values: 1 / 16 / 64 streams, K = 1 / 17 / 133 / 144, up to 128 rows per
stream, fps and realtime modes; the in-place float32 keypoints; graph replays equal eager calls; the status bits leave their
stream unchanged and their neighbours exact; reset of one stream; argument errors; inference_frames_tracked(smoother=);
install(..., batched=True, smoothing=...) with draw()."""
import ctypes as C
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from oracle import make_golden_smooth as MG
from oracle import one_euro_oracle as OE
from oracle import sort_oracle as SO

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _quiet_numpy():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)          # the oracle's t_e = 0 and NaN inputs
        yield


def _same(got, want):
    """Device rows against oracle rows as float64 values (NaN equal to NaN); a stream the oracle skips comes back as NaN."""
    for g, w in zip(got, want):
        if w is None:
            if not np.isnan(g).all():
                return False
        elif g.shape != w.shape or not np.array_equal(g, w, equal_nan=True):
            return False
    return len(got) == len(want)


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_device_equals_reference_fixture(golden_dir, case):
    from easy_vitpose_b200.smooth import DeviceOneEuro
    g = np.load(os.path.join(golden_dir, "smooth_one_euro.npz"))
    name, _, K, params, max_gap = case
    inputs = MG.case_inputs(case)
    s = DeviceOneEuro(len(inputs[0][0]), K, max_gap=max_gap, **params)
    first = []
    for f, (kl, il, clock) in enumerate(inputs):
        outs = s.update(kl, il, clock)
        assert [len(x) for x in outs] == g[f"{name}_counts"][f].tolist(), f
        assert [MG.crc(x) for x in outs] == g[f"{name}_crc32"][f].tolist(), f
        if f < MG.RAW_FRAMES:
            first.append(outs[0])
    assert np.array_equal(np.concatenate(first), g[f"{name}_stream0_rows"])
    assert s.status() == 0


def _workload(S, K, steps, seed, full=True):
    """Per update (per-stream float32 [n, K, 3], per-stream ids, clock [S]).  Stream 0 holds 128 people with fixed ids (when
    `full`); the others churn through a pool of 125 ids with gaps, 0..110 rows, so no stream exceeds 128 live ids.  Coordinates at or below 0 and a few NaN included;
    the clocks repeat once (t_e = 0)."""
    rng = np.random.default_rng(seed)
    pools = [np.arange(1000 * s, 1000 * s + (128 if s == 0 else 125)) for s in range(S)]
    poses = {}
    clock = 50.0 + np.zeros(S)
    out = []
    for t in range(steps):
        kl, il = [], []
        for s in range(S):
            if s == 0 and full:
                ids = pools[0][:128]
            else:
                lo = int(rng.integers(0, 60))
                ids = pools[s][lo:lo + int(rng.integers(0, 111))]
                ids = ids[rng.uniform(size=len(ids)) > 0.2]
                ids = rng.permutation(ids)
            k = np.zeros((len(ids), K, 3), np.float32)
            for r, i in enumerate(ids):
                if i not in poses:
                    poses[i] = rng.uniform(1, 1000, (K, 2))
                yx = poses[i] + rng.normal(0, 1.5, (K, 2))
                yx[rng.uniform(size=(K, 2)) < 0.05] = rng.choice([0.0, -2.0])
                k[r, :, :2] = yx
                k[r, :, 2] = rng.uniform(0, 1, K)
            if t == 3 and len(ids):
                k[0, 0, 1] = np.nan
            kl.append(k)
            il.append([int(i) for i in ids])
        clock = clock + (0.0 if t == 5 else rng.uniform(0.02, 0.05, S))
        out.append((kl, il, clock.tolist()))
    return out


@pytest.mark.parametrize("S", [1, 16, 64])
@pytest.mark.parametrize("K", [1, 17, 133, 144])
def test_device_equals_oracle(S, K):
    """fps mode for K = 1 / 133 (the second with a caller clock), realtime mode for K = 17 / 144; max_gap 2, so ids that
    come back after a longer gap start again."""
    from easy_vitpose_b200.smooth import DeviceOneEuro
    realtime = K in (17, 144)
    params = dict(fps=None, min_cutoff=1.0, beta=0.1, d_cutoff=30.0) if realtime else dict(fps=30.0, dx0=0.5)
    steps = 6 if S * K > 2000 else 12
    s = DeviceOneEuro(S, K, max_gap=2, **params)
    o = OE.SmoothOracle(S, max_gap=2, limit=True, **params)
    use_clock = realtime or K == 133
    rows = 0
    for t, (kl, il, clock) in enumerate(_workload(S, K, steps, S * 1000 + K)):
        c = clock if use_clock else None
        got, want = s.update(kl, il, c), o.update(kl, il, c)
        assert _same(got, want), t
        rows += sum(len(x) for x in il)
    assert rows > 0 and s.status() == o.status == 0


def _pack(kl, il, dev="cuda"):
    kp = torch.from_numpy(np.concatenate(kl)).to(dev)
    ids = torch.tensor([i for x in il for i in x], dtype=torch.int32, device=dev)
    counts = torch.tensor([len(x) for x in il], dtype=torch.int32, device=dev)
    return kp, counts, ids


def test_in_place_keypoints_are_the_rounded_result():
    from easy_vitpose_b200.smooth import DeviceOneEuro
    S, K = 4, 17
    s = DeviceOneEuro(S, K, fps=30.0)
    for t, (kl, il, _) in enumerate(_workload(S, K, 6, 9)):
        kp, counts, ids = _pack(kl, il)
        before = kp.clone()
        out = torch.empty((kp.shape[0], K, 2), dtype=torch.float64, device="cuda")
        assert s.update_device(kp, counts, ids, out=out) is out
        assert torch.equal(kp[:, :, :2].nan_to_num(7.0), out.to(torch.float32).nan_to_num(7.0))
        assert torch.equal(kp[:, :, :2].isnan(), out.isnan())
        assert torch.equal(kp[:, :, 2], before[:, :, 2]), t            # scores untouched
        if t == 0:
            assert torch.equal(kp, before) and torch.equal(out, before[:, :, :2].double())   # new ids: unchanged
    s.check()


def test_graph_replay_equals_eager():
    from easy_vitpose_b200.smooth import DeviceOneEuro
    S, K, cap = 16, 17, 16 * 128
    eager, captured = DeviceOneEuro(S, K), DeviceOneEuro(S, K)
    kp = torch.zeros((cap, K, 3), dtype=torch.float32, device="cuda")
    ids = torch.zeros(cap, dtype=torch.int32, device="cuda")
    counts = torch.zeros(S, dtype=torch.int32, device="cuda")
    clock = torch.zeros(S, dtype=torch.float64, device="cuda")
    out = torch.zeros((cap, K, 2), dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        captured.update_device(kp, counts, ids, clock, out)
    torch.cuda.synchronize()
    for t, (kl, il, c) in enumerate(_workload(S, K, 12, 4)):
        k, n_s, i = _pack(kl, il)
        n = k.shape[0]
        kp[:n].copy_(k)
        ids[:n].copy_(i)
        counts.copy_(n_s)
        clock.copy_(torch.tensor(c, dtype=torch.float64))
        graph.replay()
        e_out = torch.empty((n, K, 2), dtype=torch.float64, device="cuda")
        eager.update_device(k, n_s, i, clock.clone(), e_out)
        torch.cuda.synchronize()
        assert torch.equal(out[:n].nan_to_num(7.0), e_out.nan_to_num(7.0)) and torch.equal(kp[:n].nan_to_num(7.0), k.nan_to_num(7.0)), t
    assert eager.status() == captured.status() == 0


def test_reset_one_stream():
    from easy_vitpose_b200.smooth import DeviceOneEuro
    S, K = 4, 5
    s = DeviceOneEuro(S, K, fps=25.0, max_gap=3)
    o = OE.SmoothOracle(S, fps=25.0, max_gap=3, limit=True)
    for t, (kl, il, _) in enumerate(_workload(S, K, 14, 21)):
        if t == 5:
            s.reset(2)
            o.reset(2)
        if t == 9:
            s.reset()
            o.reset()
        assert _same(s.update(kl, il), o.update(kl, il)), t


def test_status_bits_leave_their_stream_unchanged():
    """A duplicate id (stream 1), 129 rows (stream 2), 128 live ids + 1 new (stream 3) and, on the device call, rows past n
    (stream 4): each sets its bit, writes no rows and keeps its filters and update count; the neighbours stay exact, and so
    do the skipped streams on later updates."""
    from easy_vitpose_b200.smooth import STATUS_DUPLICATE_ID, STATUS_OVER_CAPACITY, DeviceOneEuro
    S, K = 5, 3
    s = DeviceOneEuro(S, K, fps=30.0, max_gap=5)
    o = OE.SmoothOracle(S, fps=30.0, max_gap=5, limit=True)
    rng = np.random.default_rng(2)
    kp = lambda n: rng.uniform(1, 100, (n, K, 3)).astype(np.float32)   # noqa: E731
    base = [list(range(10)), list(range(20, 30)), list(range(40, 50)), list(range(100, 228)), list(range(300, 305))]
    expect = {2: STATUS_DUPLICATE_ID | STATUS_OVER_CAPACITY}
    for t in range(6):
        il = [list(x) for x in base]
        if t == 2:
            il[1][3] = il[1][4]                                                    # duplicate
            il[2] = list(range(40, 169))                                           # 129 rows
            il[3] = list(range(101, 228)) + [999]                                  # 127 known + 1 new, 128 live -> 129
        kl = [kp(len(x)) for x in il]
        got, want = s.update(kl, il), o.update(kl, il)
        assert _same(got, want), t
        assert o.status == expect.get(t, 0) and s.status() == o.status, t
        o.status = 0
    # rows past n: counts claim 5 more rows than the keypoints hold for the last stream
    kl = [kp(len(x)) for x in base]
    k, counts, ids = _pack(kl, base)
    counts[4] += 5
    out = torch.full((k.shape[0], K, 2), float("nan"), dtype=torch.float64, device="cuda")
    s.update_device(k, counts, ids, out=out)
    saved = (o.streams[4].filters, o.streams[4].updates)
    want = o.update(kl[:4] + [kl[4][:0]], base[:4] + [[]])       # the oracle's stream 4 does not move either
    o.streams[4].filters, o.streams[4].updates = saved
    assert s.status() == STATUS_OVER_CAPACITY
    got = out.cpu().numpy()
    assert _same([got[:10], got[10:20], got[20:30], got[30:158]], want[:4]) and np.isnan(got[158:]).all()
    kl = [kp(len(x)) for x in base]
    assert _same(s.update(kl, base), o.update(kl, base))
    with pytest.raises(ValueError):
        s.update([kp(2)] + [kp(0)] * 4, [[1, 1]] + [[]] * 4)
        s.check()


def test_argument_errors():
    from easy_vitpose_b200 import _lib
    from easy_vitpose_b200.smooth import DeviceOneEuro
    lib = _lib.lib()
    h = C.c_void_p()
    nan = float("nan")
    for args in [(0, 17, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 0), (70000, 17, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 0),
                 (1, 0, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 0), (1, 145, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 0),
                 (1, 17, nan, 0.3, 30.0, 0.0, 0.0, 30, 0), (1, 17, 1.7, 0.3, 30.0, nan, 0.0, 30, 0),
                 (1, 17, 1.7, 0.3, 30.0, 0.0, float("inf"), 30, 0), (1, 17, 1.7, 0.3, 30.0, 0.0, 0.0, -1, 0),
                 (1, 17, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 999)]:
        assert lib.vpb_smoother_create(*args, C.byref(h)) == 1, args
    assert lib.vpb_smoother_create(1, 17, 1.7, 0.3, 30.0, 0.0, 0.0, 30, 0, None) == 1
    s = DeviceOneEuro(2, 17)                                                  # realtime
    x = torch.zeros(64, dtype=torch.float64, device="cuda")
    p = C.c_void_p(x.data_ptr())
    assert lib.vpb_smoother_update(s._handle, p, 1, p, p, None, None, None) == 1      # realtime without a clock
    assert lib.vpb_smoother_update(s._handle, p, -1, p, p, p, None, None) == 1
    assert lib.vpb_smoother_update(s._handle, None, 1, p, p, p, None, None) == 1
    assert lib.vpb_smoother_update(None, p, 1, p, p, p, None, None) == 1
    assert lib.vpb_smoother_reset(s._handle, 2, None) == 1 and lib.vpb_smoother_reset(s._handle, -2, None) == 1
    kp = torch.zeros((3, 17, 3), device="cuda")
    counts = torch.tensor([3, 0], dtype=torch.int32, device="cuda")
    ids = torch.arange(3, dtype=torch.int32, device="cuda")
    clock = torch.zeros(2, dtype=torch.float64, device="cuda")
    for bad in [dict(kpts=kp.double()), dict(kpts=kp[:, :16]), dict(counts=counts[:1]), dict(ids=ids.long()), dict(clock=None),
                dict(clock=clock.float()), dict(out=torch.zeros((3, 17, 2), device="cuda"))]:
        a = {**dict(kpts=kp, counts=counts, ids=ids, clock=clock, out=None), **bad}
        with pytest.raises(ValueError):
            s.update_device(a["kpts"], a["counts"], a["ids"], a["clock"], a["out"])
    with pytest.raises(ValueError):
        DeviceOneEuro(1, 145)
    with pytest.raises(ValueError):
        s.update([kp.cpu().numpy(), np.zeros((0, 17, 3), np.float32)], [[0, 1, 2], []])          # realtime without a clock
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ integration
def _engine(max_batch=16, seed=5):
    from easy_vitpose_b200 import ViTPose, model_cfg
    from oracle import vitpose_oracle as O
    sd = O.make_state_dict(384, 12, 17, seed, peaky=0.1, bumps=True)
    m = ViTPose(model_cfg("s", 17), max_batch=max_batch)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}).to("cuda:0")
    return m, sd


def _in_frame_dets(seed, frames, people, h, w):
    rng = np.random.default_rng(seed)
    x0, y0 = rng.uniform(10, w - 90, people), rng.uniform(10, h - 120, people)
    out = []
    for f in range(frames):
        j = rng.uniform(-4, 4, (people, 2))
        d = np.stack([x0 + j[:, 0], y0 + j[:, 1], x0 + 60 + j[:, 0], y0 + 100 + j[:, 1], rng.uniform(0.4, 1, people)], 1)
        out.append(d[rng.uniform(size=people) > 0.15])
    return out


def _oracle_on_dicts(o, dicts, clock=None):
    """The oracle applied to unsmoothed {id: [K, 3]} dicts -> the dicts with smoothed (y, x), rounded to float32."""
    res = o.update([np.stack(list(d.values())) if d else np.zeros((0, 17, 3), np.float32) for d in dicts],
                   [list(d.keys()) for d in dicts], clock)
    out = []
    for d, r in zip(dicts, res):
        e = {}
        for (i, k), yx in zip(d.items(), r):
            k = k.copy()
            k[:, :2] = yx
            e[i] = k
        out.append(e)
    return out


@pytest.mark.parametrize("fps", [30.0, None])
def test_inference_frames_tracked_with_smoother_equals_oracle(fps):
    from easy_vitpose_b200 import B200PoseBackend
    from easy_vitpose_b200.smooth import DeviceOneEuro
    from easy_vitpose_b200.track import DeviceSort
    from oracle import preproc_oracle as P
    m, _ = _engine()
    backend = B200PoseBackend(m)
    sizes = [(240, 320), (180, 260), (300, 200)]
    imgs = [P.make_frame(h, w, seed=20 + j) for j, (h, w) in enumerate(sizes)]
    seqs = [_in_frame_dets(30 + j, 8, 5, h, w) for j, (h, w) in enumerate(sizes)]
    plain, tracked = DeviceSort(3, 1, 1, device=0), DeviceSort(3, 1, 1, device=0)
    sm = DeviceOneEuro(3, 17, fps=fps, max_gap=1, device=0)
    o = OE.SmoothOracle(3, fps=fps, max_gap=1)
    for f in range(8):
        dl = [sq[f] for sq in seqs]
        clock = [100.0 + f / 30 + 0.001 * s for s in range(3)] if fps is None else None
        raw = backend.inference_frames_tracked(imgs, dl, plain)
        got = backend.inference_frames_tracked(imgs, dl, tracked, smoother=sm, clock=clock)
        want = _oracle_on_dicts(o, raw, clock)
        for s in range(3):
            assert list(got[s]) == list(want[s]), (f, s)
            assert all(np.array_equal(got[s][i], want[s][i], equal_nan=True) for i in got[s]), (f, s)
    sm.check()


def test_install_smoothing_equals_oracle_and_draws_smoothed(monkeypatch):
    """install(vi, batched=True, smoothing=...) on a fake VitInference with a stub detector: frame by frame the returned dict
    and `_keypoints` equal the oracle applied to an unsmoothed object's keypoints (CPU Sort and device tracker), draw()
    draws the smoothed ones, reset() forgets the filters, and a tracker-less object is left unsmoothed."""
    from easy_vitpose_b200 import inference as I
    from easy_vitpose_b200 import install
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

    skeleton = [[0, 1], [1, 2], [2, 3], [5, 6], [11, 12]]
    viz = types.ModuleType("easy_ViTPose.vit_utils.visualization")
    viz.joints_dict = lambda: {"coco": {"skeleton": skeleton}}
    monkeypatch.setitem(sys.modules, "easy_ViTPose.vit_utils.visualization", viz)
    clocks = []

    def tick():
        clocks.append(5.0 + len(clocks) / 30.0 + (0.02 if len(clocks) == 4 else 0.0))
        return clocks[-1]
    monkeypatch.setattr(I, "time", types.SimpleNamespace(time=tick))
    frame = P.make_frame(240, 320, seed=4)
    dets = _in_frame_dets(77, 12, 6, 240, 320)

    def make_vi(video=True):
        calls = []

        def yolo(img, **kw):
            rows = dets[len(calls) % len(dets)]
            calls.append(kw)
            data = np.concatenate([rows, np.zeros((len(rows), 1))], 1).astype(np.float32)
            return [types.SimpleNamespace(boxes=types.SimpleNamespace(data=types.SimpleNamespace(cpu=lambda: types.SimpleNamespace(numpy=lambda: data))))]
        vi = types.SimpleNamespace(_vit_pose=FakeRefModel(), _inference=None, postprocess=None, frame_counter=0, yolo_step=1, yolo=yolo,
                                   yolo_size=320, device="cuda", yolo_classes=[0], save_state=True, is_video=video, single_pose=False,
                                   tracker=CpuSort(1, 3, 0.3) if video else None, dataset="coco", resets=0)
        vi.reset = lambda: setattr(vi, "resets", vi.resets + 1)
        return vi

    for device_tracker, opts in ((False, dict(min_cutoff=0.9, beta=0.2, fps=None, max_gap=0)), (True, dict(fps=30.0, dx0=0.5))):
        raw, sm = make_vi(), make_vi()
        install(raw, max_batch=8, batched=True, device_tracker=device_tracker)
        install(sm, max_batch=8, batched=True, device_tracker=device_tracker, smoothing=opts)
        o = OE.SmoothOracle(1, **{**I.SMOOTHING_DEFAULTS, **opts})
        clocks.clear()
        for f in range(10):
            a, b = raw.inference(frame), sm.inference(frame)
            want = _oracle_on_dicts(o, [a], clocks[-1:] if o.realtime else None)[0]
            assert len(want) and list(b) == list(want) and all(np.array_equal(b[i], want[i]) for i in b), (device_tracker, f)
            assert sm._keypoints is b and list(sm._tracker_res[1]) == list(b)
            img = sm.draw(show_yolo=False)
            exp = sm._b200.draw_frames([frame], [np.stack(list(want.values()))], skeleton, person_index=[list(want)])[0]
            assert np.array_equal(img, exp), (device_tracker, f)
        assert len(clocks) == (10 if o.realtime else 0)
        if not device_tracker:
            sm.reset()                                          # the object's own reset, then the filters: every id is new again
            assert sm.resets == 1
            a, b = raw.inference(frame), sm.inference(frame)
            assert list(a) == list(b) and all(np.array_equal(a[i], b[i]) for i in a)
    raw, sm = make_vi(video=False), make_vi(video=False)       # no tracker: ids are positions, nothing is smoothed
    install(raw, max_batch=8, batched=True)
    install(sm, max_batch=8, batched=True, smoothing={})
    for f in range(3):
        a, b = raw.inference(frame), sm.inference(frame)
        assert list(a) == list(b) and all(np.array_equal(a[i], b[i]) for i in a)
