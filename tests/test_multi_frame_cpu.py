"""CPU: the host side of the multi-frame calls -- the chunk planner and the ctypes mirror of vpb_frame."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from easy_vitpose_b200 import _lib
from easy_vitpose_b200.model import plan_frame_chunks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_plan(counts, limit, max_frames):
    chunks = plan_frame_chunks(counts, limit, max_frames)
    seen = []
    for chunk in chunks:
        assert chunk, "no empty calls"
        assert sum(e - s for _, s, e in chunk) <= limit
        assert len(chunk) <= max_frames
        assert len({f for f, _, _ in chunk}) == len(chunk), "a frame appears once per call"
        for f, s, e in chunk:
            assert 0 <= s < e <= counts[f], "only frames with boxes, only ranges inside them"
            seen.extend((f, b) for b in range(s, e))
    assert seen == [(f, b) for f, c in enumerate(counts) for b in range(c)], "every box once, in order"
    return chunks


def test_plan_covers_every_box_once_in_order_within_both_limits():
    rs = np.random.RandomState(5)
    for _ in range(300):
        nf = rs.randint(0, 150)
        counts = [int(c) for c in rs.poisson(rs.choice([0.5, 3, 10, 40]), nf)]
        limit, max_frames = int(rs.choice([1, 3, 16, 32, 64])), int(rs.choice([1, 2, 7, 64]))
        chunks = _check_plan(counts, limit, max_frames)
        # greedy: a call is closed only when it is full in boxes or in frames
        for chunk in chunks[:-1]:
            assert sum(e - s for _, s, e in chunk) == limit or len(chunk) == max_frames


def test_plan_skips_empty_frames_and_splits_a_frame_over_two_calls():
    assert plan_frame_chunks([], 8) == []
    assert plan_frame_chunks([0, 0], 8) == []
    assert plan_frame_chunks([3, 0, 4], 8) == [[(0, 0, 3), (2, 0, 4)]]
    assert plan_frame_chunks([5, 0, 6], 8) == [[(0, 0, 5), (2, 0, 3)], [(2, 3, 6)]]
    assert plan_frame_chunks([1, 1, 1], 8, max_frames=2) == [[(0, 0, 1), (1, 0, 1)], [(2, 0, 1)]]
    assert plan_frame_chunks([20], 8) == [[(0, 0, 8)], [(0, 8, 16)], [(0, 16, 20)]]
    assert len(plan_frame_chunks([1] * 130, 64)) == 3                 # 64 frames per call at most
    with pytest.raises(ValueError):
        plan_frame_chunks([2, -1], 8)
    with pytest.raises(ValueError):
        plan_frame_chunks([2], 0)


def test_frame_array_names_the_callers_frame_indices():
    from easy_vitpose_b200.model import _frame_array
    table = [(0x1000 * (j + 1), 10 + j, 20 + j, 3 * (20 + j)) for j in range(4)]
    arr = _frame_array(table, [(1, 2, 5), (3, 0, 1)])
    assert len(arr) == 4
    assert [a.num_boxes for a in arr] == [0, 3, 0, 1]
    assert (arr[1].data, arr[1].height, arr[1].width, arr[1].pitch_bytes) == table[1]


def test_vpb_frame_layout_matches_the_header():
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    if cc is None:
        pytest.skip("no host C compiler")
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "vitpose_b200.h"\n'
           'int main(void) { printf("%d %d %d %d %d %d %d\\n", (int)sizeof(vpb_frame), (int)offsetof(vpb_frame, data),'
           ' (int)offsetof(vpb_frame, height), (int)offsetof(vpb_frame, width), (int)offsetof(vpb_frame, pitch_bytes),'
           ' (int)offsetof(vpb_frame, num_boxes), VPB_MAX_FRAMES); return 0; }\n')
    with tempfile.TemporaryDirectory() as d:
        c_file, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c_file, "w") as f:
            f.write(src)
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", exe, c_file], check=True, capture_output=True)
        got = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    F = _lib.VpbFrame
    want = [C.sizeof(F), F.data.offset, F.height.offset, F.width.offset, F.pitch_bytes.offset, F.num_boxes.offset, _lib.MAX_FRAMES]
    assert got == want
